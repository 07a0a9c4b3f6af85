"""Every reducer path against exact per-group results, on value columns chosen to expose a wrong kernel.

The oracle restates the reference's sequential loops, and a parallel float sum can never reproduce a sequential
one bit for bit once a group cancels.  So float sums and means are checked here against the EXACT sum under one
error bound that holds for float64 accumulation in any order (`sum_bound`).  Integer sums are exact modulo 2^64.
min / max / first / last / median / nunique / count come from the oracle and are compared bit for bit (the sign
of a zero included), sd against an exact rational computation.

The value columns (`hard_values`) hold cancelling groups from 1e-300 to 1e300, subnormals, infinities, groups
whose min or max is a zero of either sign, constant groups of non-dyadic values, groups with one valid row and
all-NA groups; integer columns hold the extremes next to the NA sentinels, and int64 sums wrap.

Paths: engine.reduce (int32 and int64 RowIndex, host and device buffers), the handle's four streaming modes, the
bucketed multi-reducer in each of its shapes (against bucketed_reducers = 0 as well), piecewise reduction,
sd / median / first / last / nunique, and the Frame query by() + sort() on a device frame.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

from helpers import BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, SORT_ONLY

U = 2.0 ** -53
NP = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
      FLOAT32: np.float32, FLOAT64: np.float64}
NA_INT = {BOOL: -128, INT8: -128, INT16: -2**15, INT32: -2**31, INT64: -2**63}
BASIC = ("sum", "mean", "min", "max", "count", "countna")


# ---------------------------------------------------------------------------------------------------------------
# exact references
# ---------------------------------------------------------------------------------------------------------------
def gamma(k):
    k = np.asarray(k, dtype=np.float64)
    return k * U / (1 - k * U)


def sum_bound(m, abs_sum):
    """Float64 accumulation of m values in any order is within gamma_{m-1} * sum|x| of the exact sum."""
    return gamma(np.maximum(np.asarray(m) - 1, 0)) * abs_sum


def _valid(v, st):
    return ~np.isnan(v) if st in (FLOAT32, FLOAT64) else v != NA_INT[st]


def group_values(v, st, order, offsets):
    """[(valid values of group g in RowIndex order)] and per-group row counts."""
    order = np.asarray(order, dtype=np.int64)
    offsets = np.asarray(offsets, dtype=np.int64)
    vo = v[order]
    ok = _valid(vo, st)
    return [vo[a:b][ok[a:b]] for a, b in zip(offsets[:-1], offsets[1:])]


def exact_float_sum(vals):
    """(exact sum rounded once, sum |x|, valid count) of one group; +-inf handled apart from the finite rows."""
    x = vals.astype(np.float64)
    fin = np.isfinite(x)
    pinf, ninf = bool(np.any(x == np.inf)), bool(np.any(x == -np.inf))
    if pinf and ninf:
        s = math.nan
    elif pinf or ninf:
        s = math.inf if pinf else -math.inf
    else:
        s = math.fsum(x[fin].tolist())
    return s, math.fsum(np.abs(x[fin]).tolist()), len(x)


def exact_int_sum(vals):
    return np.int64(((sum(int(t) for t in vals) + 2**63) % 2**64) - 2**63)


def exact_sd(vals):
    """Sample sd with an exact rational mean and sum of squared deviations, rounded once at the end."""
    m = len(vals)
    if m <= 1:
        return math.nan
    x = vals.astype(np.float64)
    if not np.all(np.isfinite(x)):
        return math.nan
    fr = [Fraction(float(t)) for t in x]
    mean = sum(fr) / m
    ss = sum((t - mean) ** 2 for t in fr)
    return math.sqrt(float(ss / (m - 1)))


_STATS = {}        # per-group exact results of one (value column, RowIndex, offsets); cleared after every test


@pytest.fixture(autouse=True)
def _clear_stats():
    yield
    _STATS.clear()


def group_stats(v, st, order, offsets):
    """Per group: valid rows m, the exact sum (floats: rounded once, +-inf / NaN apart; ints: Python int, not
    wrapped), sum |x|.  Kept with references to its inputs, so that the ids stay theirs for the cache's life."""
    key = (id(v), id(order), id(offsets))
    if key in _STATS:
        return _STATS[key][0]
    groups = group_values(v, st, order, offsets)
    m = np.array([len(g) for g in groups], dtype=np.int64)
    if st in (FLOAT32, FLOAT64):
        ex = [exact_float_sum(g) for g in groups]
        exact = [e[0] for e in ex]
        absum = np.array([e[1] for e in ex])
    else:
        # exact integer sums from exact int64 sums of the high and low 32-bit halves
        exact, absum = [], np.zeros(len(groups))
        for i, g in enumerate(groups):
            g = g.astype(np.int64)
            hi, lo = g >> 32, g & 0xFFFFFFFF
            exact.append(int(hi.sum()) * 2**32 + int(lo.sum()))
            absum[i] = float(np.abs(g.astype(np.float64)).sum()) * (1 + 1e-12)
    s = {"groups": groups, "m": m, "exact": exact, "abs": absum}
    _STATS[key] = (s, (v, order, offsets))
    return s


def check_float_sum_mean(got, stats, op, out_f32, ctx, int_input=False):
    got = np.asarray(got).astype(np.float64)
    assert len(got) == len(stats["m"]), ctx
    for g, (m, exact, a) in enumerate(zip(stats["m"], stats["exact"], stats["abs"])):
        if op == "mean" and m == 0:
            assert np.isnan(got[g]), f"{ctx}: group {g} has no valid row, mean must be NA"
            continue
        tol = sum_bound(m, a)
        if int_input:
            tol += U * a                             # every value is first rounded to a double: u * |x| per row
            exact_res = float(Fraction(exact, int(m))) if op == "mean" else float(exact)
        else:
            exact_res = exact / m if op == "mean" else exact
        if np.isnan(exact_res) or np.isinf(exact_res):
            assert (np.isnan(got[g]) and np.isnan(exact_res)) or got[g] == exact_res, \
                f"{ctx}: group {g}: {got[g]!r} != {exact_res!r}"
            continue
        if op == "mean":
            tol = tol / m + U * abs(exact_res) + 2.0 ** -1075   # the sum's bound over the count, the division's rounding
        if out_f32:
            tol += 2.0 ** -24 * abs(exact_res) + 2.0 ** -150    # the final rounding to float32 (subnormal results too)
        err = abs(got[g] - exact_res)
        assert err <= tol, f"{ctx}: group {g} {op}: got {got[g]!r}, exact {exact_res!r}, err {err:.3e} > bound {tol:.3e}"


def bits(a):
    a = np.ascontiguousarray(np.asarray(a))
    return a.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def canon_nan(a):
    """NA floats as one bit pattern (NaN payloads are not part of a result)."""
    a = np.array(a, copy=True)
    if a.dtype.kind == "f":
        a[np.isnan(a)] = np.nan
    return a


def assert_bits_equal(got, want, ctx):
    got, want = canon_nan(np.asarray(got)), canon_nan(np.asarray(want))
    assert got.dtype == want.dtype, f"{ctx}: dtype {got.dtype} != {want.dtype}"
    bad = np.nonzero(bits(got) != bits(want))[0]
    assert len(bad) == 0, f"{ctx}: {len(bad)} groups differ bitwise, first {bad[:5]}: got {got[bad[:5]]!r} want {want[bad[:5]]!r}"


def check_reducer(name, got, v, st, order, offsets, ctx):
    """One reducer result against the exact reference (sum / mean / sd) or the oracle, bitwise (the rest)."""
    from oracle import oracle as orc
    got = got.cpu().numpy() if hasattr(got, "cpu") else np.asarray(got)
    ctx = f"{ctx} {name} st={st}"
    if name in ("sum", "mean") and (st in (FLOAT32, FLOAT64) or name == "mean"):
        check_float_sum_mean(got, group_stats(v, st, order, offsets), name, got.dtype == np.float32, ctx,
                             int_input=st not in (FLOAT32, FLOAT64))
        return
    if name == "sum":
        want = np.array([exact_int_sum([e]) for e in group_stats(v, st, order, offsets)["exact"]], dtype=np.int64)
        assert_bits_equal(got, want, ctx)
        return
    if name == "sd":
        groups = group_stats(v, st, order, offsets)["groups"]
        atol = 2.0 ** -150 if got.dtype == np.float32 else 0.0         # a float32 sd in the subnormal range
        got = got.astype(np.float64)
        for g, vals in enumerate(groups):
            want = exact_sd(vals)
            if np.isnan(want):
                assert np.isnan(got[g]), f"{ctx}: group {g}: {got[g]!r}, want NA"
            elif len(vals) and np.all(vals == vals[0]):
                assert got[g] == 0.0, f"{ctx}: group {g} of {len(vals)} equal values {vals[0]!r}: sd {got[g]!r} != 0"
            else:
                assert abs(got[g] - want) <= 1e-6 * want + atol, f"{ctx}: group {g}: sd {got[g]!r}, exact {want!r}"
        return
    op = {"min": orc.MIN, "max": orc.MAX, "count": orc.COUNT, "countna": orc.COUNTNA, "first": orc.FIRST,
          "last": orc.LAST, "median": orc.MEDIAN, "nunique": orc.NUNIQUE}[name]
    want = orc.reduce(op, v, np.asarray(order, dtype=np.int32), np.asarray(offsets, dtype=np.int32), stype=st)
    assert_bits_equal(got, want, ctx)


# ---------------------------------------------------------------------------------------------------------------
# hard value columns
# ---------------------------------------------------------------------------------------------------------------
NKINDS = 8


def hard_values(rng, st, key):
    """A value column whose groups (rows with equal `key`) each get one kind of hard data, by key % NKINDS."""
    n = len(key)
    kind = np.asarray(key, dtype=np.int64) % NKINDS
    if st in (FLOAT32, FLOAT64):
        f32 = st == FLOAT32
        emax = 30 if f32 else 300
        # per-key scale: magnitudes from 10^-emax to 10^emax
        kk = np.asarray(key, dtype=np.int64)
        scale = 10.0 ** ((kk * 7919 % (2 * emax + 1)) - emax)
        v = rng.standard_normal(n) * scale
        # 0: cancelling groups: +-x pairs inside the group, and a small remainder on the unpaired rows
        idx = np.nonzero(kind == 0)[0]
        idx = idx[np.argsort(kk[idx], kind="stable")]
        x = (1.0 + rng.random(len(idx))) * scale[idx]
        same = np.zeros(len(idx), bool)
        same[1:] = kk[idx[1:]] == kk[idx[:-1]]
        pair = np.zeros(len(idx), bool)                       # idx[i] is the second row of a pair with idx[i-1]
        for i in range(1, len(idx)):
            pair[i] = same[i] and not pair[i - 1]
        x[pair] = -x[np.nonzero(pair)[0] - 1]
        lone = ~pair & ~np.append(pair[1:], False)
        x[lone] *= 1e-9
        if f32:
            x = x.astype(np.float32).astype(np.float64)
            x[pair] = -x[np.nonzero(pair)[0] - 1]
        v[idx] = x
        # 1: subnormals of both signs
        sub = kind == 1
        tiny = np.float32(1.4e-45) if f32 else 5e-324
        v[sub] = rng.integers(-1000, 1000, int(sub.sum())) * float(tiny)
        # 2: infinities among finite values (keys with bit 3 set also get -inf: inf - inf = NaN sum)
        inf = kind == 2
        r = rng.random(n)
        v[inf & (r < 0.1)] = np.inf
        v[inf & (r > 0.9) & ((kk & 8) != 0)] = -np.inf
        # 3: zeros of both signs that are the group's min (keys with bit 3 clear) or max (set), in random row order
        z = kind == 3
        sgn = np.where((kk & 8) != 0, -1.0, 1.0)
        v[z] = sgn[z] * (1.0 + rng.random(int(z.sum())))
        zz = z & (rng.random(n) < 0.5)
        v[zz] = np.where(rng.random(int(zz.sum())) < 0.5, 0.0, -0.0)
        # 4: constant groups of non-dyadic values
        c = kind == 4
        v[c] = np.where((kk[c] & 8) != 0, 0.1, 1.0 / 3.0)
        # 5: a single valid row; 6: all NA
        v[kind == 6] = np.nan
        k5 = np.nonzero(kind == 5)[0]
        if len(k5):
            _, first = np.unique(kk[k5], return_index=True)
            keep = np.zeros(len(k5), bool); keep[first] = True
            v[k5[~keep]] = np.nan
        # 7: plain normal values, and a few NA rows everywhere
        v[rng.random(n) < 0.02] = np.nan
        return v.astype(NP[st])
    info = {BOOL: (0, 1), INT8: (-127, 127), INT16: (-2**15 + 1, 2**15 - 1), INT32: (-2**31 + 1, 2**31 - 1),
            INT64: (-2**63 + 1, 2**63 - 1)}[st]
    lo, hi = info
    na = NA_INT[st]
    kk = np.asarray(key, dtype=np.int64)
    if st == BOOL:
        v = rng.integers(0, 2, n)
    elif st == INT64:
        # values near +-2^63 so that sums wrap, and the extremes next to the NA sentinel
        v = rng.integers(2**62, 2**63 - 1, n, dtype=np.int64) * np.where(rng.random(n) < 0.5, 1, -1)
        v[rng.random(n) < 0.1] = hi
        v[rng.random(n) < 0.1] = lo
    else:
        v = rng.integers(lo, hi, n, endpoint=True)
        v[rng.random(n) < 0.2] = hi
        v[rng.random(n) < 0.2] = lo
    v = np.asarray(v, dtype=np.int64)
    v[kind == 4] = np.where(st == BOOL, 1, hi)                 # constant groups
    v[kind == 6] = na                                           # all NA
    k5 = np.nonzero(kind == 5)[0]
    if len(k5):
        _, first = np.unique(kk[k5], return_index=True)
        keep = np.zeros(len(k5), bool); keep[first] = True
        v[k5[~keep]] = na
    v[rng.random(n) < 0.02] = na
    return v.astype(NP[st])


# ---------------------------------------------------------------------------------------------------------------
# CPU self-test of the bound (no GPU)
# ---------------------------------------------------------------------------------------------------------------
def test_sum_bound_tells_right_sums_from_wrong_ones():
    rng = np.random.default_rng(7)
    for trial in range(20):
        m = int(rng.integers(200, 3000))
        scale = 10.0 ** rng.integers(-300, 300)
        x = (1 + rng.random(m // 2)) * scale
        vals = np.concatenate([x, -x, (1 + rng.random(m - 2 * (m // 2))) * scale * 1e-3])
        vals = vals * (1 + 1e-3 * rng.standard_normal(len(vals)))       # cancels, but not exactly
        s, a, cnt = exact_float_sum(vals)
        tol = sum_bound(cnt, a)

        def ok(got):
            return abs(got - s) <= tol

        # float64 in a shuffled order and pairwise: accepted
        sh = vals[rng.permutation(len(vals))]
        acc = 0.0
        for t in sh:
            acc += t
        assert ok(acc), (trial, acc, s, tol)

        def pairwise(a_):
            if len(a_) <= 2:
                return float(np.sum(a_))
            h = len(a_) // 2
            return pairwise(a_[:h]) + pairwise(a_[h:])
        assert ok(pairwise(sh))
        # float32 accumulation: rejected
        acc32 = np.float32(0)
        for t in sh.astype(np.float32) if scale < 1e30 and scale > 1e-30 else (sh / scale).astype(np.float32):
            acc32 = np.float32(acc32 + t)
        acc32 = float(acc32) if scale < 1e30 and scale > 1e-30 else float(acc32) * scale
        assert not ok(acc32), (trial, acc32, s, tol)
        # one row left out: rejected
        drop = int(np.argmax(np.abs(vals[len(vals) - 5:]))) + len(vals) - 5
        assert not ok(math.fsum(np.delete(vals, drop).tolist())), trial
    # integer mean bound: exact sums of wrapped int64 values
    assert exact_int_sum([2**63 - 1, 1]) == -2**63
    assert exact_int_sum([-2**63 + 1, -2]) == 2**63 - 1


def test_hard_values_have_what_they_promise():
    rng = np.random.default_rng(3)
    key = rng.integers(0, 400, 50_000)
    for st in (FLOAT32, FLOAT64):
        v = hard_values(rng, st, key).astype(np.float64)
        kind = key % NKINDS
        assert np.any((v == 0) & np.signbit(v)) and np.any((v == 0) & ~np.signbit(v))
        assert np.any(np.isinf(v)) and np.any((v != 0) & (np.abs(v) < np.finfo(NP[st]).tiny))
        s, a, _ = exact_float_sum(v[(kind == 0) & (key == key[kind == 0][0])])
        assert abs(s) < 1e-2 * a                                  # cancels (NA rows break a few pairs)
    v = hard_values(rng, INT64, key)
    assert v.max() == 2**63 - 1 and v.min() == -2**63 and np.any(v == -2**63 + 1)


# ---------------------------------------------------------------------------------------------------------------
# GPU paths
# ---------------------------------------------------------------------------------------------------------------
ALL_ST = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)


def _ops():
    from datatable_b200 import _lib
    return {"sum": _lib.OP_SUM, "mean": _lib.OP_MEAN, "min": _lib.OP_MIN, "max": _lib.OP_MAX, "count": _lib.OP_COUNT,
            "countna": _lib.OP_COUNTNA, "first": _lib.OP_FIRST, "last": _lib.OP_LAST, "sd": _lib.OP_SD,
            "median": _lib.OP_MEDIAN, "nunique": _lib.OP_NUNIQUE}


def _families(fn):
    """Run fn with option "profile" on: (its result, the kernel families it launched)."""
    from datatable_b200 import engine, _lib
    _lib.profile_records()
    engine.set_option("profile", 1)
    try:
        out = fn()
    finally:
        engine.set_option("profile", 0)
    return out, {name for name, _ in _lib.profile_records()}


@pytest.mark.gpu
@pytest.mark.parametrize("st", ALL_ST)
def test_rowindex_reduce_int32_and_int64_host_and_device(st):
    import torch
    from datatable_b200 import engine, _lib
    from oracle import oracle as orc
    rng = np.random.default_rng(100 + st)
    n = 200_003
    k = rng.integers(0, 3000, n).astype(np.int32)
    k[::101] = -2**31
    v = hard_values(rng, st, k)
    order, offsets, _ = orc.group([k], [0], orc.NA_FIRST)
    kd, vd = torch.from_numpy(k).cuda(), engine.Col(torch.from_numpy(v).cuda(), st)
    ops = _ops()
    for where in ("device", "host"):
        o32, f, _ = engine.group([kd] if where == "device" else [k], [0], _lib.NA_FIRST)
        o64, _, _ = engine.group64([kd] if where == "device" else [k], [0], _lib.NA_FIRST)
        val = vd if where == "device" else engine.Col(v, st)
        for layout, o in (("int32", o32), ("int64", o64)):     # the offsets are int32 either way
            for name in BASIC:
                got, fams = _families(lambda: engine.reduce(ops[name], val, o, f))
                assert "reduce" in fams, fams
                check_reducer(name, got, v, st, order, offsets, f"reduce {layout} {where}")


@pytest.mark.gpu
@pytest.mark.parametrize("st", ALL_ST)
def test_ordered_reducers_sd_median_first_last_nunique(st):
    import torch
    from datatable_b200 import engine, _lib
    from oracle import oracle as orc
    rng = np.random.default_rng(200 + st)
    n = 30_001
    k = rng.integers(0, 2000, n).astype(np.int32)
    v = hard_values(rng, st, k)
    if st == FLOAT64:
        # squared deviations of +-1e300 overflow, and those of 1e-200 underflow, in any method: keep the squares
        # normal doubles, the rest of the column as it is
        a = np.abs(v)
        v[a > 1e100] *= 1e-200
        v[(a > 0) & (a < 1e-100)] *= 1e200
    order, offsets, _ = orc.group([k], [0], orc.NA_FIRST)
    kd, vd = torch.from_numpy(k).cuda(), torch.from_numpy(v).cuda()
    o, f, _ = engine.group([kd], [0], _lib.NA_FIRST)
    ops = _ops()
    col = engine.Col(vd, st)
    for name in ("sd", "first", "last", "min", "max"):
        check_reducer(name, engine.reduce(ops[name], col, o, f), v, st, order, offsets, "ordered")
    so = engine.sort_grouped(col, o, f)
    sorder = orc.sort_grouped(v, order, offsets, stype=st)
    assert np.array_equal(so.cpu().numpy(), sorder)
    for name in ("median", "nunique"):
        check_reducer(name, engine.reduce(ops[name], col, so, f), v, st, sorder, offsets, "ordered")


# The handle's streaming modes (plan_direct): table = 2^dbits accumulators, ng groups, gmax rows in the largest.
#   small : table <= 2048                                   (keys in [0, 1000))
#   dense : table > 2048 and ng <= 2048                     (1500 keys spread over [0, 2^20))
#   hot   : table > 2048, ng > 2048, gmax > max(n/1024, 8192)   (one key owns 30 000 rows)
#   plain : everything else                                 (keys in [0, 50 000))
def _mode_keys(rng, mode, n):
    if mode == "small":
        return rng.integers(0, 1000, n).astype(np.int32)
    if mode == "dense":
        return (rng.integers(0, 1500, n) * 699).astype(np.int32)
    k = rng.integers(0, 50_000, n).astype(np.int32)
    if mode == "hot":
        k[rng.permutation(n)[:30_000]] = 12_347
    return k


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["plain", "small", "dense", "hot"])
@pytest.mark.parametrize("st", ALL_ST)
def test_handle_streaming_modes(mode, st):
    import torch
    from datatable_b200 import engine, _lib
    from oracle import oracle as orc
    rng = np.random.default_rng(300 + st)
    n = 400_009
    k = _mode_keys(rng, mode, n)
    v = hard_values(rng, st, k)
    order, offsets, ng = orc.group([k], [0], orc.NA_FIRST)
    if mode == "hot":
        assert np.diff(offsets).max() > max(n // 1024, 8192) and ng > 2048
    kd, vd = torch.from_numpy(k).cuda(), engine.Col(torch.from_numpy(v).cuda(), st)
    gb = engine.Groupby([kd], [0], _lib.NA_FIRST)
    try:
        assert gb.ngroups == ng
        ops = _ops()
        for name in BASIC:
            got, fams = _families(lambda: gb.reduce(ops[name], vd))
            assert "reduce_direct" in fams and "reduce" not in fams, fams
            check_reducer(name, got, v, st, order, offsets, f"handle {mode}")
        if st in (FLOAT32, FLOAT64):
            for name in BASIC:
                pcs = [(vd.data[a:b], a, None) for a, b in ((0, 1), (1, n // 3), (n // 3, n - 7), (n - 7, n))]
                got = gb.reduce_pieces(ops[name], st, pcs)
                assert got is not None
                check_reducer(name, got, v, st, order, offsets, f"pieces {mode}")
    finally:
        gb.close()


def _fused(keys, flags, reducers, bucketed):
    """Groupby(..., reducers=...) with option bucketed_reducers; (results, whether the bucket sweep ran)."""
    from datatable_b200 import engine, _lib
    engine.set_option("bucketed_reducers", bucketed)
    try:
        gb, fams = _families(lambda: engine.Groupby(keys, flags, _lib.NA_FIRST, reducers=reducers))
    finally:
        engine.set_option("bucketed_reducers", 1)
    try:
        return [gb.reduced(i).cpu().numpy() for i in range(len(reducers))], "bucket_scatter" in fams
    finally:
        gb.close()


# Bucketed multi-reducer shapes.  Each needs a group-key domain of 2^12 .. 2^20 (dbits), more than 2048 groups
# and no hot key (so that plan_direct picks DIRECT_PLAIN), and a value column with >= 2 L2 atomics per row.
def _bucket_case(name, rng):
    if name == "raw_key":                               # one raw key column, dbits 15, n not a multiple of 4096
        n = 1_000_003
        keys = [rng.integers(0, 20_000, n).astype(np.int32)]
        return keys, [0], keys[0]
    if name == "composite_le32":                        # by(a, b): 8 + 9 = 17 bits, kept as a 32-bit composite
        n = 700_001
        a, b = rng.integers(0, 200, n).astype(np.int16), rng.integers(0, 300, n).astype(np.int32)
        return [a, b], [0, 0], a.astype(np.int64) * 300 + b
    if name == "by_sort_wide":                          # by(k) + sort(x): 14 + 20 = 34 bits, group_shift 20
        n = 600_007
        k = rng.integers(0, 10_000, n).astype(np.int32)
        k[:10_000] = np.arange(10_000)
        x = rng.integers(0, 2**20, n).astype(np.int32)
        x[:2] = (0, 2**20 - 1)
        return [k, x], [0, SORT_ONLY], k
    if name == "dbits12":                               # keys 0..4095 exactly: 12 bits
        n = 300_001
        k = rng.integers(0, 4096, n).astype(np.int32)
        k[:2] = (0, 4095)
        return [k], [0], k
    if name == "dbits20":                               # 5000 keys spread over 0..2^20-1: 20 bits, n not a multiple of 262144
        n = 1_600_007
        k = (rng.integers(0, 5000, n) * 209).astype(np.int32)
        k[:2] = (0, 2**20 - 1)
        return [k], [0], k
    raise AssertionError(name)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["raw_key", "composite_le32", "by_sort_wide", "dbits12", "dbits20"])
def test_bucketed_shapes_vs_exact_and_plain(shape):
    import torch
    from datatable_b200 import engine, _lib
    from oracle import oracle as orc
    rng = np.random.default_rng(len(shape) * 1000 + ord(shape[-1]))
    keys, flags, gkey = _bucket_case(shape, rng)
    sts = (FLOAT64, INT64, FLOAT32) if shape in ("raw_key", "by_sort_wide") else (FLOAT64, INT32)
    vals = {st: hard_values(rng, st, gkey) for st in sts}
    order, offsets, ng = orc.group(keys, flags, orc.NA_FIRST)
    assert ng > 2048
    kd = [torch.from_numpy(c).cuda() for c in keys]
    ops = _ops()
    reducers, names = [], []
    for st in sts:
        vd = engine.Col(torch.from_numpy(vals[st]).cuda(), st)
        for name in BASIC:
            reducers.append((ops[name], vd)); names.append((name, st))
    got1, ran1 = _fused(kd, flags, reducers, 1)
    got0, ran0 = _fused(kd, flags, reducers, 0)
    assert ran1 and not ran0, (ran1, ran0)
    for i, (name, st) in enumerate(names):
        check_reducer(name, got1[i], vals[st], st, order, offsets, f"bucketed {shape}")
        check_reducer(name, got0[i], vals[st], st, order, offsets, f"plain {shape}")


@pytest.mark.gpu
def test_bucketed_several_sweeps():
    """More than BK_MAXCOLS (4) value columns and more than 32 value bytes per row: several sweeps of the bucket
    partition over one key, every column against the exact results."""
    import torch
    from datatable_b200 import engine, _lib
    from oracle import oracle as orc
    rng = np.random.default_rng(77)
    n = 500_009
    k = rng.integers(0, 30_000, n).astype(np.int32)
    sts = (FLOAT64, FLOAT64, INT64, FLOAT64, INT32, FLOAT32, INT8)        # 8 + 8 + 8 + 8 | 4 + 4 + 1 bytes
    vals = [hard_values(rng, st, k) for st in sts]
    order, offsets, _ = orc.group([k], [0], orc.NA_FIRST)
    ops = _ops()
    reducers, names = [], []
    for st, v in zip(sts, vals):
        vd = engine.Col(torch.from_numpy(v).cuda(), st)
        for name in ("mean", "min", "max"):
            reducers.append((ops[name], vd)); names.append((name, st, v))
    kd = torch.from_numpy(k).cuda()
    got1, ran1 = _fused([kd], [0], reducers, 1)
    got0, _ = _fused([kd], [0], reducers, 0)
    assert ran1
    for i, (name, st, v) in enumerate(names):
        check_reducer(name, got1[i], v, st, order, offsets, f"sweeps col {i // 3}")
        check_reducer(name, got0[i], v, st, order, offsets, f"plain col {i // 3}")


@pytest.mark.gpu
def test_frame_by_sort_on_device_frame():
    """DT[:, {mean, min, max, sum}, by(f.k), sort(f.x)] on a device frame: a 34-bit (k, x) composite whose group key
    is k, reduced by the bucketed multi-reducer."""
    import torch
    import datatable_b200 as dt
    from oracle import oracle as orc
    f, by, sort = dt.f, dt.by, dt.sort
    rng = np.random.default_rng(5)
    n = 400_003
    k = rng.integers(0, 10_000, n).astype(np.int32)
    k[:10_000] = np.arange(10_000)
    x = rng.integers(0, 2**20, n).astype(np.int32)
    x[:2] = (0, 2**20 - 1)
    v = hard_values(rng, FLOAT64, k)
    DT = dt.Frame(k=torch.from_numpy(k).cuda(), x=torch.from_numpy(x).cuda(), v=torch.from_numpy(v).cuda())
    R = DT[:, {"m": dt.mean(f.v), "lo": dt.min(f.v), "hi": dt.max(f.v), "s": dt.sum(f.v)}, by(f.k), sort(f.x)]
    order, offsets, ng = orc.group([k, x], [0, SORT_ONLY], orc.NA_FIRST)
    assert R.nrows == ng == 10_000
    assert np.array_equal(R.column("k").cpu().numpy(), np.arange(10_000, dtype=np.int32))
    for col, name in (("m", "mean"), ("lo", "min"), ("hi", "max"), ("s", "sum")):
        check_reducer(name, R.column(col), v, FLOAT64, order, offsets, "frame by+sort")


@pytest.mark.gpu
def test_signed_zero_min_max_every_path():
    """min([+0.0, -0.0]) = +0.0 and max([-0.0, +0.0]) = -0.0: the first valid zero in RowIndex order, on the RowIndex
    gather, the handle's streaming path, piecewise reduction and the bucketed multi-reducer."""
    import torch
    from datatable_b200 import engine, _lib
    from oracle import oracle as orc
    rng = np.random.default_rng(11)
    n = 200_000
    k = rng.integers(0, 5000, n).astype(np.int32)
    for st in (FLOAT32, FLOAT64):
        v = np.where(rng.random(n) < 0.5, 0.0, -0.0)
        v[rng.random(n) < 0.3] = np.nan
        v[(k % 3 == 1) & (rng.random(n) < 0.5)] = 1.0      # zero is the min
        v[(k % 3 == 2) & (rng.random(n) < 0.5)] = -1.0     # zero is the max
        v = v.astype(NP[st])
        order, offsets, _ = orc.group([k], [0], orc.NA_FIRST)
        kd, vd = torch.from_numpy(k).cuda(), engine.Col(torch.from_numpy(v).cuda(), st)
        o, f, _ = engine.group([kd], [0], _lib.NA_FIRST)
        gb = engine.Groupby([kd], [0], _lib.NA_FIRST)
        try:
            for op, name in ((_lib.OP_MIN, "min"), (_lib.OP_MAX, "max")):
                check_reducer(name, engine.reduce(op, vd, o, f), v, st, order, offsets, "rowindex")
                check_reducer(name, gb.reduce(op, vd), v, st, order, offsets, "handle")
                pcs = [(vd.data[a:b], a, None) for a, b in ((0, 5), (5, n // 2), (n // 2, n))]
                check_reducer(name, gb.reduce_pieces(op, st, pcs), v, st, order, offsets, "pieces")
        finally:
            gb.close()
        got, ran = _fused([kd], [0], [(_lib.OP_MIN, vd), (_lib.OP_MAX, vd), (_lib.OP_MEAN, vd)], 1)
        assert ran
        check_reducer("min", got[0], v, st, order, offsets, "bucketed")
        check_reducer("max", got[1], v, st, order, offsets, "bucketed")


@pytest.mark.gpu
def test_first_valid_lookups_of_one_large_group_are_row_parallel():
    """sd's pivot and the sign of a zero min / max look up a group's first valid row (first valid zero).  One group of
    2e7 rows whose first 60 % are NA, with its first zero near the end: the results are exact, and the lookups do
    not walk the group row by row on one thread (that took seconds; a row-parallel pass takes about a millisecond)."""
    import time
    import torch
    from datatable_b200 import engine, _lib
    n = 20_000_000
    head = int(n * 0.6)
    offsets = torch.tensor([0, n], dtype=torch.int32, device="cuda")
    order = torch.arange(n, dtype=torch.int32, device="cuda")
    ident = np.array([0, n], dtype=np.int32)
    cases = []
    v = np.full(n, np.nan); v[head:] = 0.1                          # constant: sd exactly 0
    cases.append(("sd", v, 0.0))
    v = np.full(n, np.nan); v[head::2] = 1.0; v[head + 1::2] = 3.0   # m rows of 1, 3, 1, 3 ...: sd = sqrt(m / (m - 1))
    m = n - head
    cases.append(("sd", v, math.sqrt(m / (m - 1))))
    for first in (0.0, -0.0):
        v = np.full(n, np.nan); v[head:] = 2.0; v[n - 100] = first; v[n - 50] = -first   # first zero 100 rows from the end
        cases.append(("min", v, first))
        w = -v
        cases.append(("max", w, -first))
    ops = _ops()
    for name, v, want in cases:
        vd = torch.from_numpy(v).cuda()
        engine.reduce(ops[name], vd, order, offsets)                  # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got = engine.reduce(ops[name], vd, order, offsets)
        torch.cuda.synchronize()
        dt_s = time.perf_counter() - t0
        g = float(got.cpu().numpy()[0])
        if name == "sd" and want != 0.0:
            assert abs(g - want) <= 1e-12 * want, (name, g, want)
        else:
            assert np.array([g]).view(np.uint64)[0] == np.array([want]).view(np.uint64)[0], (name, g, want)
        if name != "sd":
            check_reducer(name, got, v, FLOAT64, np.arange(n, dtype=np.int32), ident, "one large group")
        assert dt_s < 0.5, f"{name}: {dt_s:.3f} s for one group of {n} rows"
