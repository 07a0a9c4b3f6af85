"""GPU: every entry point at the zero edges, and every golden_v13 case (queries over zero rows,
tests/golden/make_golden_v13.py) through the Frame.

- The per-group functions over no group (ngroups = 0), over the one empty group of zero rows (offsets [0, 0], the
  reference's Groupby::single_group(0)), and over positions beyond a value column of zero rows (nrows_value = 0, read
  as NA by the reducers), with host, device and 0-element tensor buffers: bit for bit against
  tests/zero_rows_reference.py, output stypes included.  Every other empty group stays refused.
- The handle (dtb_groupby_create / _create_reduce, fused and piecewise), group / group64, gather, slice_groups,
  mask_rows, int_rows, join / join_gather, set_select, largest_group, lower_bound, dense_scatter and cut over zero
  rows.
- The Frame against every golden_v13 case, host and device frames.
"""
import ctypes
import json
import os

import numpy as np
import pytest

import zero_rows_reference as zr

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = json.load(open(os.path.join(G, "golden_v13.json")))["cases"]
ARR = dict(np.load(os.path.join(G, "golden_v13.npz")))
ALL_ST = (zr.BOOL, zr.INT8, zr.INT16, zr.INT32, zr.INT64, zr.FLOAT32, zr.FLOAT64)
ROW_OPS = {"cumsum": 1, "cumprod": 13, "cummin": 3, "cummax": 4}

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    torch.cuda.set_device(0)
    return torch


def _buf(torch, a, kind):
    """a as a host array, a device tensor, or (for 0 elements) a 0-element device tensor, whose data_ptr() may be 0."""
    if kind == "host":
        return np.ascontiguousarray(a)
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if kind == "device" else torch.empty(0, dtype=t.dtype, device="cuda")


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _same(got, want):
    got, want = _np(got), np.asarray(want)
    return got.dtype == want.dtype and got.shape == want.shape and \
        np.array_equal(got, want, equal_nan=got.dtype.kind == "f")


KINDS = ["host", "device", "empty_tensor"]


@pytest.mark.parametrize("kind", KINDS)
def test_reducers_over_the_one_empty_group(torch, kind):
    """offsets [0, 0], ngroups 1, no row: every reducer writes the empty group's value; reads nothing."""
    from datatable_b200 import engine
    for st in ALL_ST:
        v = _buf(torch, np.zeros(0, zr.NPT[st]), kind)
        offs = _buf(torch, np.zeros(2, np.int32), "host" if kind == "host" else "device")
        for nm, op in zr.OPS.items():
            if op in (zr.COV, zr.CORR):
                got = engine.reduce2(op, v, v, None, offs, stype_x=st, stype_y=st)
                want, _ = zr.empty_group(op, st, st)
            else:
                got = engine.reduce(op, None if op == zr.NROWS else v, None, offs, stype=st)
                want, _ = zr.empty_group(op, st)
            assert _same(got, want), (st, nm, _np(got), want)
            if op not in (zr.COV, zr.CORR, zr.NROWS):               # an empty RowIndex gives the same
                order = _buf(torch, np.zeros(0, np.int32), kind)
                assert _same(engine.reduce(op, v, order, offs, stype=st), want), nm


@pytest.mark.parametrize("kind", KINDS)
def test_per_position_functions_over_zero_positions(torch, kind):
    """ngroups 0 and the one empty group: the row functions, sort_grouped, cumcount / ngroup and qcut return no
    position, of their output stype."""
    from datatable_b200 import engine
    for st in ALL_ST:
        v = _buf(torch, np.zeros(0, zr.NPT[st]), kind)
        for offsets in ([0], [0, 0]):
            offs = _buf(torch, np.array(offsets, np.int32), "host" if kind == "host" else "device")
            for nm, op in ROW_OPS.items():
                got = engine.cumulative(op, v, None, offs, stype=st)
                assert len(got) == 0 and _np(got).dtype == zr.NPT[engine.cumulative_out_stype(op, st)], nm
            for got, dt_ in ((engine.shift(v, None, offs, 1, stype=st), zr.NPT[st]),
                             (engine.shift(v, None, offs, -2, stype=st), zr.NPT[st]),
                             (engine.fillna(v, None, offs, stype=st), zr.NPT[st]),
                             (engine.fillna(v, None, offs, reverse=True, stype=st), zr.NPT[st]),
                             (engine.group_index(1, offs), np.int64),
                             (engine.group_index(2, offs, reverse=True), np.int64),
                             (engine.qcut(v, None, offs, 5, stype=st), np.int32),
                             (engine.sort_grouped(v, None, offs, stype=st), np.int32)):
                assert len(got) == 0 and _np(got).dtype == dt_


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_positions_beyond_an_empty_value_column(torch, device):
    """nrows_value = 0 with n > 0 positions: the reducers read every position as NA; the row functions refuse it."""
    from datatable_b200 import engine, _lib
    offs = np.array([0, 2, 5], np.int32)
    offs = torch.from_numpy(offs).cuda() if device else offs
    for st in ALL_ST:
        v = torch.empty(0, dtype=engine._torch_dtype(st), device="cuda") if device else np.zeros(0, zr.NPT[st])
        for nm, op in zr.OPS.items():
            if op in (zr.COV, zr.CORR, zr.MEDIAN, zr.NUNIQUE):
                continue
            got = engine.reduce(op, None if op == zr.NROWS else v, None, offs, stype=st)
            want = np.concatenate([zr.reduce_rows(op, np.full(m, zr.na_of(st), zr.NPT[st]), st)[0] for m in (2, 3)])
            assert _same(got, want), (st, nm)
        with pytest.raises(_lib.DtbValueError, match="offsets cover more rows than the value column has"):
            engine.cumulative(1, v, None, offs, stype=st)


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_other_empty_groups_stay_refused(torch, device):
    """Only ngroups 1 with offsets [0, 0] may be empty: [0, 0, 0], [0, 0, 3], [0, 2, 2, 3] and [1, 0] are not a
    Groupby, for every per-group entry point."""
    from datatable_b200 import engine, _lib
    v = np.zeros(3)
    vd = torch.from_numpy(v).cuda() if device else v
    for offsets in ([0, 0, 0], [0, 0, 3], [0, 2, 2, 3], [1, 0], [-1, 0]):
        o = np.array(offsets, np.int32)
        o = torch.from_numpy(o).cuda() if device else o
        for call in (lambda: engine.reduce(zr.SUM, vd, None, o), lambda: engine.reduce(zr.FIRST, vd, None, o),
                     lambda: engine.reduce(zr.PROD, vd, None, o), lambda: engine.reduce2(zr.COV, vd, vd, None, o),
                     lambda: engine.cumulative(1, vd, None, o), lambda: engine.shift(vd, None, o),
                     lambda: engine.fillna(vd, None, o), lambda: engine.group_index(1, o),
                     lambda: engine.qcut(vd, None, o), lambda: engine.sort_grouped(vd, None, o)):
            # [0, 0, 0] in HBM: a per-position function's output of 0 elements has no data pointer, and out NULL
            # (check 7) comes before the offsets are read
            with pytest.raises(_lib.DtbValueError, match="not a Groupby" if offsets[-1] or not device
                               else "not a Groupby|out is NULL"):
                call()


@pytest.mark.parametrize("kind", KINDS)
def test_grouping_and_row_entry_points_over_zero_rows(torch, kind):
    from datatable_b200 import engine, _lib
    k = _buf(torch, np.zeros(0, np.int32), kind)
    v = _buf(torch, np.zeros(0, np.float64), kind)
    order, offsets, ng = engine.group([k], [0], _lib.NA_FIRST)
    assert len(order) == 0 and ng == 0 and _np(offsets).tolist() == [0]
    order, offsets, ng = engine.group([k], [_lib.FLAG_SORT_ONLY], _lib.NA_LAST)
    assert len(order) == 0 and offsets is None
    order, offsets, ng = engine.group64([k, v], [0, 0], _lib.NA_FIRST)
    assert len(order) == 0 and ng == 0 and _np(offsets).tolist() == [0]
    assert len(engine.gather(v, _buf(torch, np.zeros(0, np.int32), kind))) == 0
    assert len(engine.gather(_buf(torch, np.arange(4.0), kind if kind != "empty_tensor" else "device"),
                             _buf(torch, np.zeros(0, np.int64), kind))) == 0
    assert len(engine.mask_rows(_buf(torch, np.zeros(0, np.int8), kind))) == 0
    rows, lo, hi, nna = engine.int_rows(_buf(torch, np.zeros(0, np.int16), kind), zr.INT16)
    assert (len(rows), nna) == (0, 0)
    for offs in ([0], ):
        o = _buf(torch, np.array(offs, np.int32), "host" if kind == "host" else "device")
        sel, o2 = engine.slice_groups(o, 100, None, 1)
        assert len(sel) == 0 and _np(o2).tolist() == [0]
        assert engine.largest_group(o) == (-1, 0)
    o = _buf(torch, np.array([0, 2, 3], np.int32), "host" if kind == "host" else "device")
    sel, o2 = engine.slice_groups(o, 100, None, 1)                 # every group emptied: no group left
    assert len(sel) == 0 and _np(o2).tolist() == [0]
    assert len(engine.cut(v, None, 4, stype=zr.FLOAT64)) == 0
    assert len(engine.cut(v, None, edges=[-1.0, 0.0, 1.0], stype=zr.FLOAT64)) == 0
    jk = _buf(torch, np.arange(3, dtype=np.int32), "host" if kind == "host" else "device")
    jv = _buf(torch, np.array([1.5, 2.5, 3.5]), "host" if kind == "host" else "device")
    assert len(engine.join_index([k], [jk])) == 0                  # a 0-row X
    idx, vals = engine.join_gather([k], [jk], [jv], index=True)
    assert len(idx) == 0 and len(vals[0]) == 0
    xk = _buf(torch, np.array([0, 2, -2**31], np.int32), "host" if kind == "host" else "device")
    assert _np(engine.join_index([xk], [k])).tolist() == [-2**31] * 3      # a 0-row J: nothing matches
    got = engine.join_gather([xk], [k], [v])[0]
    assert _same(got, np.full(3, np.nan))


def test_set_select_over_zero_rows(torch):
    from datatable_b200 import engine, _lib
    for mode in (_lib.SET_UNION, _lib.SET_INTERSECT, _lib.SET_SETDIFF, _lib.SET_SYMDIFF):
        for dev in (False, True):
            o = torch.zeros(0, dtype=torch.int32, device="cuda") if dev else np.zeros(0, np.int32)
            f = torch.zeros(1, dtype=torch.int32, device="cuda") if dev else np.zeros(1, np.int32)
            assert len(engine.set_select(mode, o, f, [0, 0])) == 0


def test_lower_bound_and_dense_scatter_over_zero_rows(torch):
    from datatable_b200 import _lib
    L = _lib.lib
    s = torch.arange(5, dtype=torch.int32, device="cuda")
    e = torch.zeros(0, dtype=torch.int32, device="cuda")
    out = torch.full((3,), -7, dtype=torch.int64, device="cuda")
    col = lambda t: _lib.dtb_col(ctypes.c_void_p(t.data_ptr()), zr.INT32, 0)        # noqa: E731
    _lib.check(L.dtb_lower_bound(col(s), 5, col(e), 0, None, ctypes.c_void_p(out.data_ptr())))
    vals = torch.tensor([-1, 3, 9], dtype=torch.int32, device="cuda")
    _lib.check(L.dtb_lower_bound(col(e), 0, col(vals), 3, None, ctypes.c_void_p(out.data_ptr())))
    torch.cuda.synchronize()
    assert out.cpu().tolist() == [0, 0, 0]                         # nothing is smaller than any value
    table = torch.zeros(1024, dtype=torch.float64, device="cuda")
    present = torch.zeros(1024, dtype=torch.int32, device="cuda")
    _lib.check(L.dtb_dense_scatter(None, zr.INT32, None, 0, 0, 1024, ctypes.c_void_p(table.data_ptr()),
                                   ctypes.c_void_p(present.data_ptr()), None))
    ng = ctypes.c_int64(-1)
    ok = torch.zeros(1024, dtype=torch.int32, device="cuda")
    ov = torch.zeros(1024, dtype=torch.float64, device="cuda")
    _lib.check(L.dtb_dense_compact(ctypes.c_void_p(table.data_ptr()), ctypes.c_void_p(present.data_ptr()), 1024, 0,
                                   zr.INT32, ctypes.c_void_p(ok.data_ptr()), ctypes.c_void_p(ov.data_ptr()),
                                   ctypes.byref(ng), None))
    assert ng.value == 0


def test_handle_over_zero_rows(torch):
    """dtb_groupby_create(_reduce) over zero rows: no group; fused reducers (bucketed and direct key plans), the
    handle's reducers and reduce_begin / _end without a piece give no result."""
    from datatable_b200 import engine, _lib
    for st in ALL_ST:
        k = torch.zeros(0, dtype=torch.int32, device="cuda")
        v = torch.zeros(0, dtype=engine._torch_dtype(st), device="cuda")
        reds = [(op, None if op == zr.NROWS else v) for op in (zr.SUM, zr.MEAN, zr.MIN, zr.MAX, zr.COUNT, zr.COUNTNA,
                                                               zr.NROWS, zr.FIRST, zr.LAST, zr.SD, zr.PROD)]
        for keys in ([k], [k, torch.zeros(0, dtype=torch.int64, device="cuda")]):
            gb = engine.Groupby(keys, [0] * len(keys), _lib.NA_FIRST, reducers=reds)
            try:
                assert (gb.ngroups, gb.norder) == (0, 0)
                for i in range(len(reds)):
                    assert len(gb.reduced(i)) == 0
                assert len(gb.reduce(zr.SUM, v)) == 0 and len(gb.reduce2(zr.COV, v, v)) == 0
                assert len(gb.first_rows()) == 0 and len(gb.sort_grouped(v)) == 0
                got = gb.reduce_pieces(zr.SUM, st, [])
                assert got is None or len(got) == 0
            finally:
                gb.close()


# ---- the Frame against golden_v13 ------------------------------------------------------------------------------------
def A(case, key):
    return ARR[f"{case['name']}.{key}"]


def _env(case, device):
    import datatable_b200 as dtb

    def fr(cols, prefix):
        F = dtb.Frame({nm: A(case, f"{prefix}.{nm}") for nm in cols}, stypes=cols)
        return F.to_device() if device else F
    env = {"X": fr(case["x"], "x"), "S": {s: fr(cols, f"s.{s}") for s, cols in case["s"].items()}, "dt": dtb,
           "f": dtb.f, "g": dtb.g, "join": dtb.join, "by": dtb.by, "sort": dtb.sort, "np": np}
    if case["j"]:
        env["J"] = fr(case["j"], "j")
        env["J"].key = case["jkey"]
    return env


def _fault_result(case):
    """What the Frame returns where the reference dies (fillna over 0 rows) or raises KeyError('stype.void') (qcut
    under by() over 0 rows): no row, the by() key first, the function's output stype."""
    X = case["x"]
    fn = case["name"].split(".")[2]
    names = (["k"] if fn.endswith("_by") else []) + ["v"]
    stypes = ([X["k"]] if fn.endswith("_by") else []) + [zr.INT32 if fn.startswith("qcut") else X["v"]]
    return names, stypes


def _check_case(case, env):
    fault = "reference_crash" in case or case.get("error") == ["KeyError", "stype.void"]
    if "error" in case and not fault:
        etype, msg = case["error"]
        with pytest.raises(Exception) as e:
            eval(case["query"], env)
        assert etype in [t.__name__ for t in type(e.value).__mro__], (type(e.value), etype)
        assert e.value.args[0] == msg
        return
    R = eval(case["query"], env)
    if fault:
        names, stypes = _fault_result(case)
        assert list(R.names) == names and list(R.stypes) == stypes and R.nrows == 0
        return
    assert list(R.names) == case["names"] and R.nrows == case["nrows"], (list(R.names), R.nrows)
    for i, nm in enumerate(R.names):
        assert R.stypes[i] == case["stypes"][i], nm
        # a reference column may hold one stray NA row in a 0-row frame (tests/test_oracle_golden_v13.py)
        want = A(case, f"r{i}")[:case["nrows"]]
        assert _same(R.to_numpy(nm), want), (nm, R.to_numpy(nm), want)


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_frame_against_golden(torch, device):
    """Every case, one after the other in one test (each runs in well under a millisecond); the report names every
    case that differs."""
    failed = []
    for case in CASES:
        try:
            _check_case(case, _env(case, device))
        except AssertionError as e:
            failed.append(f"{case['name']}: {e}")
    assert not failed, "\n".join(failed)
