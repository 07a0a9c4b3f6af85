"""GPU: cumsum / cumprod / cummin / cummax (dtb_cumulative, engine.cumulative, the Frame's dt.cumsum ...) against the
reference's goldens (golden_v7) and, on large seeded inputs, against the numpy restatement in
tests/cumulative_reference.py: bit for bit wherever the result does not depend on the order of float operations,
within the documented bounds where it does.
"""
from fractions import Fraction

import numpy as np
import pytest

from oracle import oracle as orc
from cumulative_reference import (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64, NA, NPT,
                                  case_groups, cum_groups, j_columns, load_golden)

pytestmark = pytest.mark.gpu

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if "error" not in c]
OPS = {"cumsum": 1, "cumprod": 13, "cummin": 3, "cummax": 4}
STYPE_OF = {"stype.bool8": BOOL, "stype.int8": INT8, "stype.int16": INT16, "stype.int32": INT32,
            "stype.int64": INT64, "stype.float32": FLOAT32, "stype.float64": FLOAT64, "stype.date32": DATE32,
            "stype.time64": TIME64}


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


def _assert_same(got, want, label="", float_prod=False):
    """Bit for bit (-0.0 included).  float_prod: a float cumprod, which rounds the exact product once where the
    reference rounds after every row -- within (k + 1) units in the last place at prefix k."""
    got = _np(got)
    assert got.dtype == want.dtype, label
    if want.dtype.kind != "f":
        assert np.array_equal(got, want), label
        return
    assert np.array_equal(np.isnan(got), np.isnan(want)), label
    if not float_prod:
        assert np.array_equal(_bits(got), _bits(want)), label
        return
    ok = ~np.isnan(want)
    eps = np.finfo(want.dtype).eps
    g, w = got[ok].astype(np.float64), want[ok].astype(np.float64)
    with np.errstate(invalid="ignore"):                                # inf - inf: those are compared by ==
        assert np.all((g == w) | (np.abs(g - w) <= (len(want) + 1) * eps * np.abs(w))), label
    assert np.array_equal(np.signbit(got[ok]), np.signbit(want[ok])), label


def _cum_outputs(case):
    return [(nm, src) for nm, (kind, src) in zip(case["names"][-len(j_columns(case)):], j_columns(case)) if kind == "cum"]


FNREV = [(fn, rev) for fn in OPS for rev in (False, True)]
FNREV_IDS = [f"{fn}{'-rev' if rev else ''}" for fn, rev in FNREV]


def _cases(fn, rev):
    return [c for c in CASES if c["fn"] == fn and c["rev"] == rev]


def _failures(cases, check):
    """Runs check(case) on every case; returns the names of the cases that fail, with the first line of the error."""
    bad = []
    for case in cases:
        try:
            check(case)
        except AssertionError as e:                                # noqa: PERF203
            bad.append(f"{case['name']}: {str(e).splitlines()[0] if str(e) else ''}")
    return bad


@pytest.mark.parametrize("fn,rev", FNREV, ids=FNREV_IDS)
def test_engine_cumulative_golden(eng, fn, rev):
    """Every golden case of (fn, reverse) through engine.cumulative, with host and device buffers and an int32 and an
    int64 RowIndex (the identity too, materialised as int64)."""
    engine, _lib, torch = eng

    def check(case):
        order, offsets = case_groups(case, ARR, orc)
        for device in (False, True):
            for order64 in (False, True):
                put = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if device else (lambda a: a)
                ordr = order
                if ordr is None and order64:
                    ordr = np.arange(int(offsets[-1]) if len(offsets) > 1 else 0)
                o = None if ordr is None else put(np.asarray(ordr, np.int64 if order64 else np.int32))
                for nm, src in _cum_outputs(case):
                    st = case["stypes"][src]
                    got = engine.cumulative(OPS[fn], put(ARR[case["name"] + "." + src]), o, put(offsets), rev, stype=st)
                    label = f"{nm} {'device' if device else 'host'} {'ord64' if order64 else 'ord32'}"
                    assert engine.is_tensor(got) == device, label
                    _assert_same(got, ARR[case["name"] + ".out_" + nm], label, fn == "cumprod" and st in (FLOAT32, FLOAT64))

    bad = _failures(_cases(fn, rev), check)
    assert not bad, bad


def _frame_query(dtb, case, fr):
    f, j = dtb.f, case["j"]
    F = {"cumsum": dtb.cumsum, "cumprod": dtb.cumprod, "cummin": dtb.cummin, "cummax": dtb.cummax}[case["fn"]]
    rev = case["rev"]
    J = {"one": lambda: F(f.x, reverse=rev),
         "list": lambda: F([f.x, f.y], reverse=rev),
         "tuple": lambda: F((f.x, f.y), reverse=rev),
         "all": lambda: F(f[:], reverse=rev),
         "dict": lambda: {"c": F(f.x, reverse=rev)},
         "dictlist": lambda: {"c": F([f.x, f.y], reverse=rev)},
         "plain": lambda: [f.x, F(f.x, reverse=rev)],
         "withqcut": lambda: [F(f.x, reverse=rev), dtb.qcut(f.y)],
         "bykey": lambda: F(f.ka, reverse=rev)}[j]()
    i = case["i"]
    rows = slice(None) if i is None else (i if isinstance(i, int) else slice(*i))
    mods = {"none": (), "by": (dtb.by(f.ka),), "by2": (dtb.by(f.ka, f.kb),), "bysort": (dtb.by(f.ka), dtb.sort(f.s)),
            "sort": (dtb.sort(f.s),), "sortdesc": (dtb.sort(-f.s),)}[case["mode"]]
    return fr[(rows, J) + mods]


@pytest.mark.parametrize("fn,rev", FNREV, ids=FNREV_IDS)
def test_frame_cumulative_golden(eng, fn, rev):
    """Every golden case of (fn, reverse) through the Frame, on a host frame and on a device frame."""
    import datatable_b200 as dtb

    def check(case):
        for device in (False, True):
            fr = dtb.Frame({nm: ARR[case["name"] + "." + nm] for nm in case["stypes"]}, stypes=case["stypes"])
            if device:
                fr = fr.to_device()
            R = _frame_query(dtb, case, fr)
            where = "device" if device else "host"
            assert list(R.names) == case["names"], where
            assert R.nrows == case["nrows"], where
            assert list(R.stypes) == [STYPE_OF[st] for st in case["out_stypes"]], where
            cum = {nm for nm, _ in _cum_outputs(case)}
            for nm, st in zip(case["names"], R.stypes):
                want = ARR[case["name"] + ".out_" + nm]
                _assert_same(R.to_numpy(nm).astype(want.dtype), want, f"{nm} {where}",
                             nm in cum and fn == "cumprod" and st in (FLOAT32, FLOAT64))

    bad = _failures(_cases(fn, rev), check)
    assert not bad, bad


def test_frame_cumulative_next_to_a_reducer(eng):
    import datatable_b200 as dtb
    fr = dtb.Frame({"x": np.array([1.5, np.nan, -0.0, 0.0]), "g": np.array([1, 2, 1, 2], np.int32)})
    with pytest.raises(NotImplementedError):
        fr[:, [dtb.sum(dtb.f.x), dtb.cumsum(dtb.f.x)], dtb.by(dtb.f.g)]
    with pytest.raises(NotImplementedError):
        fr[:, [dtb.cummax(dtb.f.x), dtb.mean(dtb.f.x)]]


# ---- large seeded cases against the restatement --------------------------------------------------------------------
def _offsets(rng, n, kind):
    if kind == "one":
        return np.array([0, n], np.int32)
    if kind == "ones":
        return np.arange(n + 1, dtype=np.int32)
    if kind == "random":                                           # lengths 1 .. ~5000
        lens = rng.integers(1, 5000, n // 2000 + 2)
    elif kind == "pow2":                                           # 2^k - 1, 2^k, 2^k + 1 around the tile size
        lens = np.array([2**k + d for k in range(1, 15) for d in (-1, 0, 1)] * 40)
    else:                                                          # 1e5 groups
        lens = rng.multinomial(n - 100_000, np.full(100_000, 1e-5)) + 1
    ends = np.cumsum(lens)
    ends = ends[ends < n]
    return np.concatenate([[0], ends, [n]]).astype(np.int32)


def _values(rng, st, n, na=0.1):
    if st in (FLOAT32, FLOAT64):
        v = rng.integers(-8, 9, n).astype(NPT[st])
        v[rng.random(n) < 0.05] = -0.0
        v[rng.random(n) < na] = np.nan
        return v
    if st == BOOL:
        v = rng.integers(0, 2, n).astype(np.int8)
    else:
        info = np.iinfo(NPT[st])
        v = rng.integers(info.min + 1, info.max, n, dtype=np.int64).astype(NPT[st])
    v[rng.random(n) < na] = NA[st]
    return v


KINDS = [("one", 2_000_003), ("ones", 5_001), ("random", 3_000_000), ("pow2", 1_500_000), ("groups1e5", 20_000_000)]


@pytest.mark.parametrize("kind,n", KINDS, ids=[k for k, _ in KINDS])
def test_seeded_exact(eng, kind, n):
    """Every integer, bool, date and time op, and cummin / cummax on floats, bit for bit; float cumsum of
    integer-valued data (exact in any order) bit for bit.  Through a random permutation as the RowIndex."""
    engine, _lib, torch = eng
    # the restatement loops over the groups in Python: 1e5 groups take two stypes, forward only
    stypes = (INT32, FLOAT64) if kind == "groups1e5" else (BOOL, INT8, INT16, INT32, INT64, DATE32, TIME64, FLOAT32, FLOAT64)
    for st in stypes:
        rng = np.random.default_rng(sum(map(ord, kind)) * 100 + st)
        v = _values(rng, st, n)
        offsets = _offsets(rng, n, kind)
        order = rng.permutation(n).astype(np.int32)
        vd, od, fd = (torch.from_numpy(a).cuda() for a in (v, order, offsets))
        fns = (["cummin", "cummax"] if st in (DATE32, TIME64) else
               ["cumsum", "cummin", "cummax"] if st in (FLOAT32, FLOAT64) else list(OPS))
        for fn in fns:
            for rev in (False, True):
                if kind == "groups1e5" and (rev or fn == "cumprod"):
                    continue
                got = _np(engine.cumulative(OPS[fn], vd, od, fd, rev, stype=st))
                want = cum_groups(fn, v, st, order, offsets, rev)
                if want.dtype.kind == "f":
                    assert np.array_equal(_bits(got), _bits(want)), (st, fn, rev)
                else:
                    assert np.array_equal(got, want), (st, fn, rev)
        del vd, od, fd


def test_single_group_behind_na_prefix(eng):
    """One group of 2e7 rows whose first 60 % are NA: every op bit for bit (float cumsum of integers)."""
    engine, _lib, torch = eng
    n = 20_000_000
    rng = np.random.default_rng(7)
    for st in (INT32, INT64, FLOAT64):
        v = _values(rng, st, n, na=0.0)
        v[: int(0.6 * n)] = np.nan if st == FLOAT64 else NA[st]
        offsets = np.array([0, n], np.int32)
        vd, fd = torch.from_numpy(v).cuda(), torch.from_numpy(offsets).cuda()
        for fn in OPS:
            if fn == "cumprod" and st == FLOAT64:
                continue
            for rev in (False, True):
                got = _np(engine.cumulative(OPS[fn], vd, None, fd, rev, stype=st))
                want = cum_groups(fn, v, st, None, offsets, rev)
                if want.dtype.kind == "f":
                    assert np.array_equal(_bits(got), _bits(want)), (st, fn, rev)
                else:
                    assert np.array_equal(got, want), (st, fn, rev)


def _gamma(k, u=2.0**-53):
    return k * u / (1 - k * u)


def test_float_cumsum_within_bound(eng):
    """General float64 data: every prefix within gamma(k-1) * sum|x| of the exact prefix sum, plus its rounding."""
    engine, _lib, torch = eng
    rng = np.random.default_rng(11)
    n = 60_000
    m = rng.integers(-2**52, 2**52, n)
    e = rng.integers(-40, 1, n)
    x = np.ldexp(m.astype(np.float64), e)                          # exact: |m| < 2^53
    offsets = np.array([0, 3, 2050, 2051, 9000, 30000, n], np.int32)
    order = rng.permutation(n).astype(np.int32)
    for rev in (False, True):
        got = _np(engine.cumulative(1, torch.from_numpy(x).cuda(), torch.from_numpy(order).cuda(),
                                    torch.from_numpy(offsets).cuda(), rev))
        xs = x[order]
        for g in range(len(offsets) - 1):
            a, b = offsets[g], offsets[g + 1]
            idx = range(b - 1, a - 1, -1) if rev else range(a, b)
            s, sabs, k = Fraction(0), 0.0, 0
            for p in idx:
                s += Fraction(float(xs[p]))
                sabs += abs(float(xs[p]))
                k += 1
                err = abs(Fraction(float(got[p])) - s)
                assert err <= Fraction(_gamma(k - 1) * sabs * (1 + 2**-50)) + abs(s) * Fraction(2.0**-53), (g, p)


def test_float_cumprod_within_bound(eng):
    """Float cumprod: every prefix within gamma(k-1) of the exact product, rounded once; float32 too."""
    engine, _lib, torch = eng
    rng = np.random.default_rng(12)
    n = 3000
    offsets = np.array([0, 1, 300, 2047, 2049, 2300, n], np.int32)
    for T, st in ((np.float64, FLOAT64), (np.float32, FLOAT32)):
        x = (rng.choice([0.5, 0.625, 0.75, 0.875, 1.125, 1.25, 1.5, 1.75, 2.0], n)          # few bits: small Fractions
             * rng.choice([-1, 1], n)).astype(T)
        x[rng.random(n) < 0.05] = np.nan
        u = 2.0**-53 if T == np.float64 else 2.0**-24
        for rev in (False, True):
            got = _np(engine.cumulative(13, torch.from_numpy(x).cuda(), None, torch.from_numpy(offsets).cuda(), rev))
            for g in range(len(offsets) - 1):
                a, b = offsets[g], offsets[g + 1]
                idx = range(b - 1, a - 1, -1) if rev else range(a, b)
                p_exact, k = Fraction(1), 0
                for p in idx:
                    if not np.isnan(x[p]):
                        p_exact *= Fraction(float(x[p]))
                        k += 1
                    bound = Fraction(_gamma(max(k - 1, 0)) + u * (1 + _gamma(max(k - 1, 0))))
                    gp = float(got[p])
                    if np.isinf(gp):                                  # the exact product is beyond the type's range
                        assert abs(p_exact) * (1 + bound) >= Fraction(float(np.finfo(T).max)), (st, g, p)
                        assert (gp < 0) == (p_exact < 0), (st, g, p)
                    else:
                        tiny = Fraction(float(np.finfo(T).smallest_subnormal))
                        assert abs(Fraction(gp) - p_exact) <= abs(p_exact) * bound + tiny, (st, g, p)


def test_repeated_calls_are_byte_identical(eng):
    engine, _lib, torch = eng
    n = 20_000_000
    rng = np.random.default_rng(13)
    x = torch.from_numpy(rng.standard_normal(n)).cuda()
    y = torch.from_numpy(rng.uniform(0.9, 1.1, n)).cuda()
    offsets = torch.tensor([0, n], dtype=torch.int32, device="cuda")
    for op, v in ((1, x), (13, y)):
        a = engine.cumulative(op, v, None, offsets)
        b = engine.cumulative(op, v, None, offsets)
        assert torch.equal(a.view(torch.int64), b.view(torch.int64))
