"""GPU: the per-group product (DTB_OP_PROD, dt.prod) and cov / corr (DTB_OP_COV / DTB_OP_CORR, dt.cov / dt.corr)
against the reference's goldens and against exact results.

cov / corr: the NA pattern must match the reference's exactly, and every value must lie within the bound derived in
tests/binary_reference.py (`result_ok`) of the exact rational result (corr's square root in `decimal`, 60 digits).

Integer products are compared bit for bit, with the reference (golden_v5) and with Python int products modulo 2^64.
Float products are compared with the exact product under the bound derived in tests/prod_reference.py (`prod_ok`);
the NA pattern must match the reference's, except in the cases golden_v5 tags as deviations, where the reference's
running product left the range part-way: there the engine must return the in-range value and differ from the
reference.  Every path that takes PROD is exercised and asserts from the profile records which path ran.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from prod_reference import (BOOL, FLOAT32, FLOAT64, INT32, INT64, NA, NPT, case_query, int_prod, load_golden,
                            out_dtype, prod_ok, valid_values)

pytestmark = pytest.mark.gpu

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if c["op"] == "prod"]
CASES2 = [c for c in ALL_CASES if c["op"] != "prod"]


@pytest.fixture(scope="module")
def eng():
    import torch
    torch.cuda.set_device(0)
    from datatable_b200 import engine, _lib
    return engine, _lib, torch


def ref_groups(case):
    v, keys, flags = case_query(case, ARR)
    if not keys:
        return None, np.array([0, len(v)], dtype=np.int32)
    order, offsets, _ = orc.group(keys, flags, orc.NA_FIRST)
    if case["i"] is not None:
        pos, offsets = orc.slice_groups(offsets, *case["i"])
        order = order[pos]
    return order, offsets


def check_against(got, groups, st, want=None, deviation=False, ctx=""):
    got = np.asarray(got)
    assert got.dtype == out_dtype(st), ctx
    assert len(got) == len(groups), ctx
    if st not in (FLOAT32, FLOAT64):
        exact = np.array([int_prod(g) for g in groups], dtype=np.int64)
        assert np.array_equal(got, exact), ctx
        if want is not None:
            assert np.array_equal(got, want), ctx
        return
    for i, g in enumerate(groups):
        assert prod_ok(got[i], g, got.dtype.type), f"{ctx}: group {i}: {got[i]!r} is not the product of {g.tolist()}"
    if want is not None:
        if deviation:
            same = (np.isnan(got) & np.isnan(want)) | (got == want)
            assert not np.any(same), f"{ctx}: the reference's out-of-range running product should differ"
        else:
            assert np.array_equal(np.isnan(got), np.isnan(want)), f"{ctx}: NA pattern differs from the reference"


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
@pytest.mark.parametrize("where", ["device", "host"])
@pytest.mark.parametrize("is64", [False, True])
def test_golden_parity_dtb_reduce(eng, case, where, is64):
    engine, _lib, torch = eng
    v, _, _ = case_query(case, ARR)
    st = INT32 if case["mode"] == "bykey" else case["stype"]
    want = ARR[case["name"] + ".out_p"]
    if len(v) == 0:
        return
    order, offsets = ref_groups(case)
    if order is None:
        order = np.arange(len(v), dtype=np.int32)
    order = order.astype(np.int64 if is64 else np.int32)
    offsets = np.asarray(offsets, dtype=np.int32)
    if where == "device":
        args = (torch.from_numpy(v).cuda(), torch.from_numpy(order).cuda(), torch.from_numpy(offsets).cuda())
    else:
        args = (v, order, offsets)
    got = engine.reduce(_lib.OP_PROD, args[0], args[1], args[2], stype=st)
    got = got.cpu().numpy() if hasattr(got, "cpu") else got
    check_against(got, valid_values(v, st, order, offsets), st, want, case["deviation"], case["name"])


def frame_query(dtb, case, device):
    name = case["name"]
    cols, stypes = {}, {}
    for nm in ("k1", "k2", "s"):
        if name + "." + nm in ARR:
            cols[nm] = ARR[name + "." + nm]
            stypes[nm] = INT32
    cols["v"] = ARR[name + ".v"]
    stypes["v"] = case["stype"]
    DT = dtb.Frame(cols, stypes=stypes)
    if device:
        DT = DT.to_device()
    f = dtb.f
    rows = slice(None) if case["i"] is None else slice(*case["i"])
    m = case["mode"]
    if m == "by":
        return DT[rows, {"p": dtb.prod(f.v)}, dtb.by(f.k1)]
    if m == "by2":
        return DT[rows, {"p": dtb.prod(f.v)}, dtb.by(f.k1, f.k2)]
    if m == "bysort":
        return DT[rows, {"p": dtb.prod(f.v)}, dtb.by(f.k1), dtb.sort(f.s)]
    if m == "none":
        return DT[rows, {"p": dtb.prod(f.v)}]
    return DT[rows, {"p": dtb.prod(f.k1)}, dtb.by(f.k1)]


@pytest.mark.parametrize("case", [c for c in CASES if c["nrows"] > 0], ids=[c["name"] for c in CASES if c["nrows"] > 0])
@pytest.mark.parametrize("device", [False, True], ids=["host_frame", "device_frame"])
def test_frame_queries(eng, case, device):
    import datatable_b200 as dtb
    R = frame_query(dtb, case, device)
    assert list(R.names) == case["names"]
    assert R.nrows == case["nrows"]
    st = INT32 if case["mode"] == "bykey" else case["stype"]
    assert R.stypes[-1] == {FLOAT32: FLOAT32, FLOAT64: FLOAT64}.get(st, INT64)
    for nm in case["names"][:-1]:                          # the group keys, bit for bit
        assert np.array_equal(np.asarray(R.to_numpy(nm)), ARR[case["name"] + ".out_" + nm])
    v, _, _ = case_query(case, ARR)
    order, offsets = ref_groups(case)
    check_against(np.asarray(R.to_numpy("p")), valid_values(v, st, order, offsets), st,
                  ARR[case["name"] + ".out_p"], case["deviation"], case["name"])


# ---------------------------------------------------------------------------------------------------------------
# exact checks on hard data
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("st", [BOOL, 2, 3, INT32, INT64])
@pytest.mark.parametrize("is64", [False, True])
def test_int_prod_exact_mod_2_64(eng, st, is64):
    engine, _lib, torch = eng
    rng = np.random.default_rng(100 + st)
    n = 200_000
    if st == BOOL:
        v = (rng.random(n) < 0.995).astype(np.int8)            # mostly 1: some groups keep 1, the others hold a 0
    else:
        info = np.iinfo(NPT[st])
        v = rng.integers(info.min + 1, info.max, n, dtype=NPT[st], endpoint=True)
        odd = rng.random(n) < 0.9                             # mostly odd: products that do not collapse to 0 mod 2^64
        v[odd] |= 1
        v[rng.random(n) < 0.01] = info.max
        v[rng.random(n) < 0.01] = info.min + 1
    v[rng.random(n) < 0.1] = NA[st]
    k = rng.integers(0, 3000, n).astype(np.int32)
    kd, vd = torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda()
    order, offsets, ng = engine.group([kd], [0], _lib.NA_FIRST)
    o = order.to(torch.int64) if is64 else order
    got = engine.reduce(_lib.OP_PROD, vd, o, offsets, stype=st).cpu().numpy()
    groups = valid_values(v, st, order.cpu().numpy(), offsets.cpu().numpy())
    exact = np.array([int_prod(g) for g in groups], dtype=np.int64)
    assert np.array_equal(got, exact)


@pytest.mark.parametrize("st", [FLOAT32, FLOAT64])
@pytest.mark.parametrize("is64", [False, True])
def test_float_prod_exact(eng, st, is64):
    engine, _lib, torch = eng
    rng = np.random.default_rng(7 + st)
    n = 120_000
    T = NPT[st]
    span = 6 if st == FLOAT32 else 60                       # group exponent sums spread by ~10 * span
    # signs at random; magnitudes over the whole exponent range, so running products leave the range both ways
    v = (rng.choice([-1.0, 1.0], n) * np.exp2(rng.uniform(-span, span, n)) * (1 + rng.random(n))).astype(T)
    v[rng.random(n) < 0.05] = np.nan
    v[rng.random(n) < 0.002] = 0.0
    v[rng.random(n) < 0.002] = -np.inf
    v[: n // 100] = (1.0 + rng.random(n // 100) * 2.0 ** -20).astype(T)     # near 1: offsets that barely move
    if st == FLOAT64:
        v[n // 100: n // 50] = np.finfo(np.float64).smallest_subnormal * rng.integers(1, 9, n // 100)
    k = rng.integers(0, 400, n).astype(np.int32)
    kd, vd = torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda()
    order, offsets, ng = engine.group([kd], [0], _lib.NA_FIRST)
    o = order.to(torch.int64) if is64 else order
    got = engine.reduce(_lib.OP_PROD, vd, o, offsets).cpu().numpy()
    groups = valid_values(v, st, order.cpu().numpy(), offsets.cpu().numpy())
    check_against(got, groups, st, ctx=f"st={st}")


# ---------------------------------------------------------------------------------------------------------------
# every path
# ---------------------------------------------------------------------------------------------------------------
def families(_lib):
    return {name for name, _ in _lib.profile_records()}


@pytest.mark.parametrize("st", [INT64, FLOAT64])
def test_every_path_takes_the_rowindex(eng, st):
    engine, _lib, torch = eng
    rng = np.random.default_rng(11)
    n = 300_000
    k = rng.integers(0, 1000, n).astype(np.int32)          # a small key domain: SUM would stream the rows
    v = rng.integers(-5, 6, n).astype(np.int64) if st == INT64 else rng.uniform(0.5, 2.0, n)
    kd, vd = torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda()
    order, offsets, ng = engine.group([kd], [0], _lib.NA_FIRST)
    want = engine.reduce(_lib.OP_PROD, vd, order, offsets).cpu().numpy()
    groups = valid_values(v, st, order.cpu().numpy(), offsets.cpu().numpy())
    check_against(want, groups, st, ctx="dtb_reduce")
    engine.set_option("profile", 1)
    try:
        _lib.profile_records()
        # the fused call: PROD next to SUM of the same column; the SUM streams unless PROD is in the call
        gb = engine.Groupby([kd], [0], _lib.NA_FIRST, reducers=[(_lib.OP_PROD, vd)])
        fam = families(_lib)
        assert "reduce" in fam and "reduce_direct" not in fam, fam
        check_against(gb.reduced(0).cpu().numpy(), groups, st, ctx="fused")
        # the handle: direct-eligible (device keys, small domain) and not (host keys)
        gb.reduce(_lib.OP_SUM, vd)                       # this handle streams SUM ...
        assert "reduce_direct" in families(_lib)
        got = gb.reduce(_lib.OP_PROD, vd).cpu().numpy()  # ... but PROD takes the RowIndex
        fam = families(_lib)
        assert "reduce" in fam and "reduce_direct" not in fam, fam
        check_against(got, groups, st, ctx="handle, direct-eligible")
        assert gb.reduce_pieces(_lib.OP_PROD, st, [(vd, 0, None)]) is None    # reduce_begin: DTB_ENOTIMPL
        gb2 = engine.Groupby([k], [0], _lib.NA_FIRST)
        got2 = gb2.reduce(_lib.OP_PROD, vd).cpu().numpy()
        assert "reduce" in families(_lib)
        check_against(got2, groups, st, ctx="handle, not direct-eligible")
        gb.close(); gb2.close()
    finally:
        engine.set_option("profile", 0)
        _lib.profile_records()
    if st == INT64:
        assert np.array_equal(got, want) and np.array_equal(got2, want)


def test_reduce_begin_prod_is_not_implemented(eng):
    engine, _lib, torch = eng
    import ctypes
    kd = torch.arange(1000, dtype=torch.int32, device="cuda") % 7
    gb = engine.Groupby([kd], [0], _lib.NA_FIRST)
    st = ctypes.c_void_p(0)
    rc = _lib.lib.dtb_groupby_reduce_begin(gb._h, _lib.OP_PROD, FLOAT64, engine._stream(), ctypes.byref(st))
    assert rc == _lib.ENOTIMPL and not st.value
    gb.close()


def test_out_stypes(eng):
    engine, _lib, torch = eng
    for st, want in ((BOOL, INT64), (2, INT64), (3, INT64), (INT32, INT64), (INT64, INT64), (FLOAT32, FLOAT32),
                     (FLOAT64, FLOAT64), (17, 0), (18, 0)):
        assert engine.reduce_out_stype(_lib.OP_PROD, st) == want


# ---------------------------------------------------------------------------------------------------------------
# one group of 2e7 rows whose first 60 % (in RowIndex order) are NA: every tile's slots fold into one result
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("st", [INT64, FLOAT64])
def test_one_large_group(eng, st):
    engine, _lib, torch = eng
    n = 20_000_000
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    order = torch.randperm(n, device="cuda", generator=g, dtype=torch.int64).to(torch.int32)
    offsets = torch.tensor([0, n], dtype=torch.int32, device="cuda")
    nna = n * 6 // 10
    if st == INT64:
        v = torch.randint(-2**62, 2**62, (n,), device="cuda", generator=g, dtype=torch.int64) | 1   # odd: no zero product
        v[order[:nna].long()] = -2**63
        vn = v.cpu().numpy()
        valid = vn[vn != -2**63]
        want = np.multiply.reduce(valid.view(np.uint64), dtype=np.uint64).view(np.int64)   # wraps modulo 2^64
    else:
        # +-2^e in pairs (2^e, 2^-e) along the RowIndex after the NA prefix, and one extra 2^37: every product is exact,
        # so the result is exactly +-2^37 although the running product wanders far from it
        m = n - nna
        e = torch.randint(-40, 41, (m // 2,), device="cuda", generator=g, dtype=torch.int64)
        ew = torch.stack([e, -e], 1).reshape(-1)
        ew[0] += 37
        sgn = torch.randint(0, 2, (m,), device="cuda", generator=g, dtype=torch.int64)
        w = torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")
        w[nna:] = torch.ldexp((1 - 2 * sgn).double(), ew)
        v = torch.empty_like(w)
        v[order.long()] = w                                  # position p of the RowIndex holds w[p]
        want = np.ldexp(-1.0 if int(sgn.sum().item()) % 2 else 1.0, 37)
    for o in (order, order.to(torch.int64)):
        got = engine.reduce(_lib.OP_PROD, v, o, offsets).cpu().numpy()
        assert got.shape == (1,)
        if st == INT64:
            assert got[0] == want
        else:
            assert got[0] == want and np.signbit(got[0]) == np.signbit(want), (got[0], want)


def test_fused_reducers_on_constant_keys(eng):
    """Every key column constant: one group, and the fused reducers still run (they were skipped before)."""
    engine, _lib, torch = eng
    k = torch.zeros(1000, dtype=torch.int32, device="cuda")
    v = torch.arange(1, 1001, dtype=torch.float64, device="cuda") / 500
    gb = engine.Groupby([k], [0], _lib.NA_FIRST, reducers=[(_lib.OP_SUM, v), (_lib.OP_PROD, v), (_lib.OP_NROWS, None)])
    assert gb.ngroups == 1
    vals = v.cpu().numpy()
    assert abs(gb.reduced(0).item() - vals.sum()) <= 1e-12 * vals.sum()
    check_against(gb.reduced(1).cpu().numpy(), [vals], FLOAT64, ctx="constant keys")
    assert gb.reduced(2).item() == 1000
    gb.close()


# ===============================================================================================================
# cov / corr
# ===============================================================================================================
import math  # noqa: E402
from fractions import Fraction  # noqa: E402

from binary_reference import out_dtype2, result_ok, valid_pairs  # noqa: E402
from test_oracle_golden_v5 import groups2, outputs2  # noqa: E402


def check2(got, groups, sx, sy, corr, want=None, ctx=""):
    got = np.asarray(got)
    assert got.dtype == out_dtype2(sx, sy), ctx
    assert len(got) == len(groups), ctx
    for i, (xs, ys) in enumerate(groups):
        assert result_ok(got[i], xs, ys, corr, got.dtype.type), f"{ctx}: group {i}: {got[i]!r} (m = {len(xs)})"
    if want is not None:
        assert np.array_equal(np.isnan(got), np.isnan(want)), f"{ctx}: NA pattern differs from the reference"


@pytest.mark.parametrize("case", [c for c in CASES2 if c["mode"] != "bykey"],
                         ids=[c["name"] for c in CASES2 if c["mode"] != "bykey"])
@pytest.mark.parametrize("where", ["device", "host"])
@pytest.mark.parametrize("is64", [False, True])
def test_golden_parity_dtb_reduce2(eng, case, where, is64):
    engine, _lib, torch = eng
    order, offsets = groups2(case)
    n = len(ARR[case["name"] + ".x"])
    order = (np.arange(n) if order is None else order).astype(np.int64 if is64 else np.int32)
    offsets = np.asarray(offsets, dtype=np.int32)
    op = _lib.OP_CORR if case["op"] == "corr" else _lib.OP_COV
    for x, sx, y, sy, col in outputs2(case):
        if where == "device":
            args = [torch.from_numpy(a).cuda() for a in (x, y, order, offsets)]
        else:
            args = [x, y, order, offsets]
        got = engine.reduce2(op, *args, stype_x=sx, stype_y=sy)
        got = got.cpu().numpy() if hasattr(got, "cpu") else got
        check2(got, valid_pairs(x, sx, y, sy, order, offsets), sx, sy, op == _lib.OP_CORR,
               ARR[case["name"] + ".out_" + col], case["name"])


def frame_query2(dtb, case, device):
    name = case["name"]
    cols, stypes = {}, {}
    for nm in ("k1", "k2", "s"):
        if name + "." + nm in ARR:
            cols[nm] = ARR[name + "." + nm]
            stypes[nm] = INT32
    cols["x"], cols["y"] = ARR[name + ".x"], ARR[name + ".y"]
    stypes["x"], stypes["y"] = case["stype"], case["stype2"]
    DT = dtb.Frame(cols, stypes=stypes)
    if device:
        DT = DT.to_device()
    f = dtb.f
    fn = dtb.corr if case["op"] == "corr" else dtb.cov
    rows = slice(None) if case["i"] is None else slice(*case["i"])
    j = [fn([f.x, f.y], f.y)] if case["bcast"] else {"r": fn(f.x, f.y)}
    m = case["mode"]
    if m == "by2":
        return DT[rows, j, dtb.by(f.k1, f.k2)]
    if m == "bysort":
        return DT[rows, j, dtb.by(f.k1), dtb.sort(f.s)]
    if m == "none":
        return DT[rows, j]
    if m == "bykey":
        return DT[rows, {"r": fn(f.k1, f.y)}, dtb.by(f.k1)]
    return DT[rows, j, dtb.by(f.k1)]


@pytest.mark.parametrize("case", CASES2, ids=[c["name"] for c in CASES2])
@pytest.mark.parametrize("device", [False, True], ids=["host_frame", "device_frame"])
def test_frame_queries2(eng, case, device):
    import datatable_b200 as dtb
    R = frame_query2(dtb, case, device)
    assert list(R.names) == case["names"]
    assert R.nrows == case["nrows"]
    for nm in case["names"]:
        if nm in ("k1", "k2"):
            assert np.array_equal(np.asarray(R.to_numpy(nm)), ARR[case["name"] + ".out_" + nm])
    want_st = FLOAT32 if case["out_stype"] == "stype.float32" else FLOAT64
    assert R.stypes[-1] == want_st
    if case["mode"] == "bykey":
        assert np.all(np.isnan(np.asarray(R.to_numpy("r"))))
        return
    order, offsets = groups2(case)
    for x, sx, y, sy, col in outputs2(case):
        check2(np.asarray(R.to_numpy(col)), valid_pairs(x, sx, y, sy, order, offsets), sx, sy, case["op"] == "corr",
               ARR[case["name"] + ".out_" + col], case["name"])


def hard_pairs(rng, n):
    """Cancelling values, offsets of 1e8 plus small noise, constant columns, one-valid-pair groups."""
    k = rng.integers(0, 300, n).astype(np.int32)
    x = 1e8 + np.round(rng.standard_normal(n), 6)
    y = -2e8 + 0.7 * (x - 1e8) + np.round(rng.standard_normal(n) * 1e-3, 9)
    big = rng.random(n) < 0.2
    x[big] = rng.choice([1e15, -1e15, 3.0, -3.0], big.sum())                # cancelling magnitudes
    x[k == 7] = 0.1                                                        # constant x: cov 0, corr NA
    y[k == 8] = -2.5                                                       # constant y
    one = np.nonzero(k == 9)[0]
    x[one[1:]] = np.nan                                                    # one valid pair
    x[rng.random(n) < 0.05] = np.nan
    y[rng.random(n) < 0.05] = np.nan
    return k, x, y


@pytest.mark.parametrize("op", ["cov", "corr"])
@pytest.mark.parametrize("is64", [False, True])
def test_cov_corr_exact_on_hard_data(eng, op, is64):
    engine, _lib, torch = eng
    rng = np.random.default_rng(21 if op == "cov" else 22)
    k, x, y = hard_pairs(rng, 60_000)
    kd = torch.from_numpy(k).cuda()
    order, offsets, ng = engine.group([kd], [0], _lib.NA_FIRST)
    o = order.to(torch.int64) if is64 else order
    code = _lib.OP_CORR if op == "corr" else _lib.OP_COV
    got = engine.reduce2(code, torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), o, offsets).cpu().numpy()
    groups = valid_pairs(x, FLOAT64, y, FLOAT64, order.cpu().numpy(), offsets.cpu().numpy())
    check2(got, groups, FLOAT64, FLOAT64, op == "corr", ctx=op)
    g7 = int(np.searchsorted(np.unique(k), 7))
    if op == "cov":
        assert got[g7] == 0.0                                   # constant x: exactly zero
    else:
        assert np.isnan(got[g7]) and np.isnan(got[int(np.searchsorted(np.unique(k), 8))])
    assert np.isnan(got[int(np.searchsorted(np.unique(k), 9))])  # one valid pair: NA


def test_cov_corr_paths_and_refusals(eng):
    engine, _lib, torch = eng
    import ctypes
    rng = np.random.default_rng(5)
    n = 200_000
    k = rng.integers(0, 1000, n).astype(np.int32)
    x, y = rng.standard_normal(n), rng.standard_normal(n)
    kd, xd, yd = (torch.from_numpy(a).cuda() for a in (k, x, y))
    order, offsets, ng = engine.group([kd], [0], _lib.NA_FIRST)
    want = engine.reduce2(_lib.OP_CORR, xd, yd, order, offsets).cpu().numpy()
    groups = valid_pairs(x, FLOAT64, y, FLOAT64, order.cpu().numpy(), offsets.cpu().numpy())
    check2(want, groups, FLOAT64, FLOAT64, True, ctx="dtb_reduce2")
    for keys in ([kd], [k]):                                    # direct-eligible handle, and not (host keys)
        gb = engine.Groupby(keys, [0], _lib.NA_FIRST)
        engine.set_option("profile", 1)
        try:
            _lib.profile_records()
            got = gb.reduce2(_lib.OP_CORR, xd, yd).cpu().numpy()
            fam = {nm for nm, _ in _lib.profile_records()}
        finally:
            engine.set_option("profile", 0)
            _lib.profile_records()
        assert "reduce2" in fam and "reduce_direct" not in fam, fam
        assert np.allclose(got, want, rtol=1e-12, atol=1e-15, equal_nan=True)
        gb.reduce(_lib.OP_SUM, xd)
        # one-column entry points refuse the two-column reducers with DTB_EINVAL
        out = torch.empty(gb.ngroups, dtype=torch.float64, device="cuda")
        rc = _lib.lib.dtb_groupby_reduce(gb._h, _lib.OP_COV, engine.Col(xd).c(), n, engine._stream(),
                                         ctypes.c_void_p(out.data_ptr()))
        assert rc == _lib.EINVAL
        st = ctypes.c_void_p(0)
        assert _lib.lib.dtb_groupby_reduce_begin(gb._h, _lib.OP_CORR, FLOAT64, engine._stream(), ctypes.byref(st)) == _lib.EINVAL
        gb.close()
    with pytest.raises(ValueError):
        engine.reduce(_lib.OP_CORR, xd, order, offsets)
    with pytest.raises(ValueError):
        engine.Groupby([kd], [0], _lib.NA_FIRST, reducers=[(_lib.OP_COV, xd)])
    with pytest.raises(ValueError):                             # caller offsets are checked as dtb_reduce checks them
        engine.reduce2(_lib.OP_COV, xd, yd, order, torch.tensor([0, 5, 5, n], dtype=torch.int32, device="cuda"))
    assert engine.reduce2_out_stype(_lib.OP_COV, FLOAT32, FLOAT32) == FLOAT32
    assert engine.reduce2_out_stype(_lib.OP_CORR, FLOAT32, INT64) == FLOAT64
    assert engine.reduce2_out_stype(_lib.OP_CORR, BOOL, BOOL) == FLOAT64
    assert engine.reduce2_out_stype(_lib.OP_CORR, 17, FLOAT64) == 0
    assert engine.reduce2_out_stype(_lib.OP_SUM, FLOAT64, FLOAT64) == 0


@pytest.mark.parametrize("op", ["cov", "corr"])
def test_one_large_group_corr(eng, op):
    """One group of 2e7 rows whose first 60 % in RowIndex order are NA pairs: the pivot lookup crosses the NA prefix
    and every thread's flush lands on the same words."""
    engine, _lib, torch = eng
    n = 20_000_000
    g = torch.Generator(device="cuda"); g.manual_seed(4)
    order = torch.randperm(n, device="cuda", generator=g, dtype=torch.int64).to(torch.int32)
    offsets = torch.tensor([0, n], dtype=torch.int32, device="cuda")
    nna = n * 6 // 10
    # small integers: every shifted sum is exact in float64, so the result is known exactly
    xw = torch.randint(-1000, 1001, (n,), device="cuda", generator=g, dtype=torch.int64).double() + 1e8
    yw = 3 * (xw - 1e8) + torch.randint(-5, 6, (n,), device="cuda", generator=g, dtype=torch.int64).double()
    xw[:nna] = float("nan")
    yw[: nna // 2] = float("nan")
    x, y = torch.empty_like(xw), torch.empty_like(yw)
    x[order.long()] = xw; y[order.long()] = yw                 # position p of the RowIndex holds (xw[p], yw[p])
    code = _lib.OP_CORR if op == "corr" else _lib.OP_COV
    ok = ~(torch.isnan(xw) | torch.isnan(yw))
    a = (xw[ok] - 1e8).to(torch.int64).cpu().numpy()           # exact small integers (the shift changes nothing)
    b = yw[ok].to(torch.int64).cpu().numpy()
    m = len(a)
    sa, sb = int(a.sum()), int(b.sum())
    Sxy = Fraction(m * int((a * b).sum()) - sa * sb, m)
    Sxx = Fraction(m * int((a * a).sum()) - sa * sa, m)
    Syy = Fraction(m * int((b * b).sum()) - sb * sb, m)
    want = Sxy / (m - 1) if op == "cov" else Sxy / Fraction(math.sqrt(Sxx)) / Fraction(math.sqrt(Syy))
    for o in (order, order.to(torch.int64)):
        got = engine.reduce2(code, x, y, o, offsets).cpu().numpy()
        assert got.shape == (1,)
        rel = abs(float(got[0]) - float(want)) / abs(float(want))
        assert rel <= 1e-9, (got[0], float(want))
