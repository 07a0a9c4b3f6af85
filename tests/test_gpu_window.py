"""GPU: shift, fillna, cumcount and ngroup (dtb_shift, dtb_fillna, dtb_group_index, engine.shift / fillna /
group_index, the Frame's dt.shift / fillna / cumcount / ngroup) against the reference's goldens (golden_v8) and, on
large seeded inputs, against the numpy restatement in tests/window_reference.py.  All four functions are exact, so
every comparison is bit for bit (-0.0 included; every NaN is NA).
"""
import numpy as np
import pytest

from oracle import oracle as orc
from window_reference import (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64, NA, NPT, FLOATS,
                              case_groups, j_columns, load_golden, query, row_fn_fast)

pytestmark = pytest.mark.gpu

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if "error" not in c]
STYPE_OF = {"stype.bool8": BOOL, "stype.int8": INT8, "stype.int16": INT16, "stype.int32": INT32,
            "stype.int64": INT64, "stype.float32": FLOAT32, "stype.float64": FLOAT64, "stype.date32": DATE32,
            "stype.time64": TIME64}
ROW_FNS = ("shift", "fillna", "cumcount", "ngroup")


@pytest.fixture(scope="module")
def eng():
    import torch
    torch.cuda.set_device(0)
    from datatable_b200 import engine, _lib
    return engine, _lib, torch


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _bits(a):
    a = np.where(np.isnan(a), np.nan, a).astype(a.dtype)             # every NaN is NA: one pattern
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _assert_same(got, want, label=""):
    got = _np(got)
    assert got.dtype == want.dtype, label
    if want.dtype.kind == "f":
        assert np.array_equal(_bits(got), _bits(want)), label
    else:
        assert np.array_equal(got, want), label


def _run(engine, _lib, kind, v, st, order, offsets, rev, n):
    if kind == "shift":
        return engine.shift(v, order, offsets, n, stype=st)
    if kind == "fillna":
        return engine.fillna(v, order, offsets, rev, stype=st)
    return engine.group_index(_lib.GROUP_CUMCOUNT if kind == "cumcount" else _lib.GROUP_NGROUP, offsets, rev)


def _failures(cases, check):
    bad = []
    for case in cases:
        try:
            check(case)
        except AssertionError as e:                                # noqa: PERF203
            bad.append(f"{case['name']}: {str(e).splitlines()[0] if str(e) else ''}")
    return bad


@pytest.mark.parametrize("fn", ROW_FNS)
def test_engine_golden(eng, fn):
    """Every golden output of `fn` through the engine, with host and device buffers and an int32 and an int64
    RowIndex.  Without by() the engine runs one group of the selected rows; the reference's Shift_ColumnImpl,
    Range_ColumnImpl and constant 0 agree with that wherever the goldens pin them."""
    engine, _lib, torch = eng

    def check(case):
        order, offsets = case_groups(case, ARR, orc)
        grouped = case["mode"] in ("by", "by2", "bysort")
        if not grouped:
            offsets = np.array([0, offsets[-1]] if len(offsets) > 1 and offsets[-1] else [0], np.int32)
        outs = [(nm, k) for nm, k in zip(case["names"][-len(j_columns(case)):], j_columns(case)) if k[0] == fn]
        for device in (False, True):
            put = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if device else (lambda a: a)
            for order64 in (False, True):
                ordr = order
                if ordr is None and order64:
                    ordr = np.arange(int(offsets[-1]) if len(offsets) > 1 else 0)
                o = None if ordr is None else put(np.asarray(ordr, np.int64 if order64 else np.int32))
                for nm, (kind, src, rev) in outs:
                    v = None if src is None else put(ARR[case["name"] + "." + src])
                    got = _run(engine, _lib, kind, v, case["stypes"].get(src), o, put(offsets), rev, case["n"])
                    label = f"{nm} {'device' if device else 'host'} {'ord64' if order64 else 'ord32'}"
                    assert engine.is_tensor(got) == device, label
                    _assert_same(got, ARR[case["name"] + ".out_" + nm], label)

    bad = _failures([c for c in CASES if fn in [k[0] for k in j_columns(c)]], check)
    assert not bad, bad


@pytest.mark.parametrize("fn", ROW_FNS + ("mix",))
def test_frame_golden(eng, fn):
    """Every golden case of `fn` through the Frame, on a host frame and on a device frame."""
    import datatable_b200 as dtb

    def check(case):
        for device in (False, True):
            fr = dtb.Frame({nm: ARR[case["name"] + "." + nm] for nm in case["stypes"]}, stypes=case["stypes"])
            if device:
                fr = fr.to_device()
            R = query(dtb, case, fr)
            where = "device" if device else "host"
            assert list(R.names) == case["names"], where
            assert R.nrows == case["nrows"], where
            assert list(R.stypes) == [STYPE_OF[st] for st in case["out_stypes"]], where
            for nm in case["names"]:
                want = ARR[case["name"] + ".out_" + nm]
                _assert_same(R.to_numpy(nm).astype(want.dtype), want, f"{nm} {where}")

    bad = _failures([c for c in CASES if c["fn"] == fn], check)
    assert not bad, bad


def test_frame_next_to_a_reducer(eng):
    import datatable_b200 as dtb
    f = dtb.f
    fr = dtb.Frame({"x": np.array([1.5, np.nan, -0.0, 0.0]), "g": np.array([1, 2, 1, 2], np.int32)})
    for fn in (lambda: dtb.shift(f.x), lambda: dtb.fillna(f.x), dtb.cumcount, dtb.ngroup):
        with pytest.raises(NotImplementedError):
            fr[:, [dtb.sum(f.x), fn()], dtb.by(f.g)]
        with pytest.raises(NotImplementedError):
            fr[:, [fn(), dtb.mean(f.x)]]


# ---- large seeded cases against the restatement --------------------------------------------------------------------
def _offsets(rng, n, kind):
    if kind == "one":                                              # one group over thousands of tiles
        return np.array([0, n], np.int32)
    if kind == "ones":                                             # runs of 1-row groups
        return np.arange(n + 1, dtype=np.int32)
    if kind == "tile":                                             # groups of 2047, 2048 and 2049 rows: heads on
        lens = np.array([2047, 2048, 2049, 2048, 1, 2048, 4096] * 200)   # tile boundaries and one past them
    elif kind == "random":                                         # lengths 1 .. ~5000
        lens = rng.integers(1, 5000, n // 2000 + 2)
    else:                                                          # C2-like: 1e6 groups
        lens = rng.multinomial(n - 1_000_000, np.full(1_000_000, 1e-6)) + 1
    ends = np.cumsum(lens)
    ends = ends[ends < n]
    return np.concatenate([[0], ends, [n]]).astype(np.int32)


def _values(rng, st, n, na):
    if st in FLOATS:
        v = rng.integers(-8, 9, n).astype(NPT[st])
        v[rng.random(n) < 0.05] = -0.0
        v[rng.random(n) < 0.01] = np.inf
    elif st == BOOL:
        v = rng.integers(0, 2, n).astype(np.int8)
    else:
        info = np.iinfo(NPT[st])
        v = rng.integers(info.min + 1, info.max, n, dtype=np.int64).astype(NPT[st])
    v[rng.random(n) < na] = np.nan if st in FLOATS else NA[st]
    return v


KINDS = [("one", 3_000_001), ("ones", 10_001), ("tile", 2_500_000), ("random", 4_000_000), ("c2", 20_000_000)]
SHIFTS = (1, -1, 2047, -2047, 2048, -2048, 2049, -2049, 10**6, -10**6, 2**31 - 1, -2**31)


@pytest.mark.parametrize("kind,n", KINDS, ids=[k for k, _ in KINDS])
def test_seeded_exact(eng, kind, n):
    """Every function bit for bit against the whole-array restatement, through a random permutation as the RowIndex:
    shift over SHIFTS, fillna forward and reverse at NA densities 0, 1 %, 99 % and 100 %, cumcount and ngroup both
    ways."""
    engine, _lib, torch = eng
    rng = np.random.default_rng(sum(map(ord, kind)))
    offsets = _offsets(rng, n, kind)
    order = rng.permutation(n).astype(np.int32)
    od, fd = torch.from_numpy(order).cuda(), torch.from_numpy(offsets).cuda()
    stypes = (INT32, FLOAT64) if kind == "c2" else (BOOL, INT8, INT16, INT32, INT64, DATE32, TIME64, FLOAT32, FLOAT64)
    for st in stypes:
        for na in ((0.01,) if kind == "c2" else (0.0, 0.01, 0.99, 1.0)):
            v = _values(rng, st, n, na)
            vd = torch.from_numpy(v).cuda()
            vals = v[order]
            for rev in (False, True):
                got = engine.fillna(vd, od, fd, rev, stype=st)
                _assert_same(got, row_fn_fast("fillna", vals, st, offsets, rev), (st, na, "fillna", rev))
            if na == 0.01:
                for s in SHIFTS:
                    got = engine.shift(vd, od, fd, s, stype=st)
                    _assert_same(got, row_fn_fast("shift", vals, st, offsets, n=s), (st, "shift", s))
            del vd
    for fn, kind_ in (("cumcount", _lib.GROUP_CUMCOUNT), ("ngroup", _lib.GROUP_NGROUP)):
        for rev in (False, True):
            _assert_same(engine.group_index(kind_, fd, rev), row_fn_fast(fn, None, INT64, offsets, rev), (fn, rev))


def test_int64_row_ids(eng):
    """A RowIndex of int64 row ids from engine.group64, every function against the restatement."""
    engine, _lib, torch = eng
    rng = np.random.default_rng(5)
    n = 3_000_000
    k = torch.from_numpy(rng.integers(0, 5000, n).astype(np.int32)).cuda()
    order, offsets, ng = engine.group64([k], [0], _lib.NA_FIRST)
    assert order.dtype == torch.int64
    offsets = offsets.to(torch.int32)                              # a Groupby of int32 offsets, as every row function takes
    o, f_ = _np(order), _np(offsets)
    for st in (INT16, FLOAT64):
        v = _values(rng, st, n, 0.3)
        vd = torch.from_numpy(v).cuda()
        vals = v[o]
        for s in (1, -3, 700):
            _assert_same(engine.shift(vd, order, offsets, s, stype=st), row_fn_fast("shift", vals, st, f_, n=s), s)
        for rev in (False, True):
            _assert_same(engine.fillna(vd, order, offsets, rev, stype=st), row_fn_fast("fillna", vals, st, f_, rev), rev)


def test_nan_payloads_come_out_as_the_na(eng):
    """A NaN with another payload, or negative, is NA: shift and fillna write the quiet NaN dtb_gather writes."""
    engine, _lib, torch = eng
    raw = np.array([0x7FF0000000000001, 0xFFF8000000000000, 0x3FF0000000000000, 0x8000000000000000], np.uint64)
    v = raw.view(np.float64)
    offsets = np.array([0, 4], np.int32)
    got = _np(engine.shift(v, None, offsets, 0)).view(np.uint64)
    assert list(got) == [0x7FF8000000000000, 0x7FF8000000000000, 0x3FF0000000000000, 0x8000000000000000]
    got = _np(engine.fillna(v, None, offsets)).view(np.uint64)
    assert list(got) == [0x7FF8000000000000, 0x7FF8000000000000, 0x3FF0000000000000, 0x8000000000000000]
    f32 = np.array([0x7F800001, 0xFFC00000, 0x80000000], np.uint32).view(np.float32)
    got = _np(engine.fillna(f32, None, np.array([0, 3], np.int32), True)).view(np.uint32)
    assert list(got) == [0x80000000, 0x80000000, 0x80000000]


def test_repeated_calls_are_byte_identical(eng):
    engine, _lib, torch = eng
    n = 20_000_000
    rng = np.random.default_rng(13)
    x = rng.standard_normal(n)
    x[rng.random(n) < 0.3] = np.nan
    xd = torch.from_numpy(x).cuda()
    offsets = torch.from_numpy(_offsets(rng, n, "random")).cuda()
    order = torch.from_numpy(rng.permutation(n).astype(np.int32)).cuda()
    for call in (lambda: engine.shift(xd, order, offsets, -3), lambda: engine.fillna(xd, order, offsets),
                 lambda: engine.fillna(xd, order, offsets, True),
                 lambda: engine.group_index(_lib.GROUP_CUMCOUNT, offsets, True),
                 lambda: engine.group_index(_lib.GROUP_NGROUP, offsets)):
        a, b = call(), call()
        assert torch.equal(a.view(torch.int64), b.view(torch.int64))


def test_window_query_on_host_and_device_frames(eng):
    """DT[:, {"lag": shift(f.v), "filled": fillna(f.v), "i": cumcount(), "g": ngroup()}, by(f.k)] at 1e6 rows,
    against the restatement."""
    import datatable_b200 as dtb
    f = dtb.f
    rng = np.random.default_rng(21)
    n = 1_000_000
    k = rng.integers(0, 1000, n).astype(np.int32)
    v = _values(rng, FLOAT64, n, 0.2)
    order, offsets, _ = orc.group([k], [0], orc.NA_FIRST)
    vals = v[np.asarray(order, np.int64)]
    want = {"k": k[np.asarray(order, np.int64)], "lag": row_fn_fast("shift", vals, FLOAT64, offsets, n=1),
            "filled": row_fn_fast("fillna", vals, FLOAT64, offsets),
            "i": row_fn_fast("cumcount", None, INT64, offsets), "g": row_fn_fast("ngroup", None, INT64, offsets)}
    for device in (False, True):
        fr = dtb.Frame({"k": k, "v": v})
        if device:
            fr = fr.to_device()
        R = fr[:, {"lag": dtb.shift(f.v), "filled": dtb.fillna(f.v), "i": dtb.cumcount(), "g": dtb.ngroup()}, dtb.by(f.k)]
        assert list(R.names) == ["k", "lag", "filled", "i", "g"]
        for nm, w in want.items():
            _assert_same(R.to_numpy(nm).astype(w.dtype), w, (nm, device))
