"""GPU: the keyed join (dtb_join), the set operations (dtb_set_select behind union / intersect / setdiff / symdiff /
unique), the column statistics (dtb_largest_group behind mode / nmodal, and Frame.nunique) and dtb_lower_bound, at
the edges of their types and at scale.

- golden_v9 (tests/golden/make_golden_v9.py, from the unmodified reference): through the C-ABI and the Frame mirror,
  with host and device buffers, bit for bit, stypes included.
- join at 1e7 X rows and every stype pair on wide random keys: against tests/join_reference.py.
- set selection at 1e6 .. 5e6 rows, the largest group over up to 1e7 groups and lower_bound: against numpy.
"""
import ctypes
import json
import os

import numpy as np
import pytest

from join_reference import (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64, NA, NPT, na_mask,
                            join_index)

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = json.load(open(os.path.join(G, "golden_v9.json")))["cases"]
ARR = dict(np.load(os.path.join(G, "golden_v9.npz")))
NUMERIC = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
FLOATS = (FLOAT32, FLOAT64)
OPS = ("union", "intersect", "setdiff", "symdiff")


def A(case, key):
    return ARR[f"{case['name']}.{key}"]


def of(kind):
    return [c for c in CASES if c["kind"] == kind]


def same(got, want):
    """dtype, shape and bits equal (-0.0 is not +0.0); any NaN is NA"""
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    if got.dtype.kind != "f":
        return np.array_equal(got, want)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint8), want[~nan].view(np.uint8))


def dev(a, device):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda() if device else a


def host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)


def na_of(st):
    return np.array([np.nan if st in FLOATS else NA[st]], NPT[st])


def promote(ins, sts):
    """rbind under Type::common (the highest numeric stype), every value cast once, NA to NA"""
    st = max(sts, key=list(NUMERIC).index)
    out = []
    for a, s in zip(ins, sts):
        b = a.astype(NPT[st])
        b[na_mask(a, s)] = np.nan if st in FLOATS else NA[st]
        out.append(b)
    return np.concatenate(out), st


# ---------------------------------------------------------------------------------------------------------------
# golden_v9 through the C-ABI and the Frame mirror
# ---------------------------------------------------------------------------------------------------------------
def join_groups():
    return sorted({c["name"].split(".")[0] for c in of("join")})


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("group", join_groups())
def test_join_golden_abi(group, device):
    from datatable_b200 import engine
    bad = []
    for case in of("join"):
        if case["name"].split(".")[0] != group:
            continue
        nk = len(case["xst"])
        xs = [engine.Col(dev(A(case, f"x{i}"), device), case["xst"][i]) for i in range(nk)]
        js = [engine.Col(dev(A(case, f"jsorted{i}"), device), case["jst"][i]) for i in range(nk)]
        got = host(engine.join_index(xs, js))
        if not same(got, A(case, "index")):
            bad.append(case["name"])
    assert not bad, bad


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("group", join_groups())
def test_join_golden_frame(group, device):
    import datatable_b200 as dtb
    bad = []
    for case in of("join"):
        if case["name"].split(".")[0] != group:
            continue
        names = [f"k{i}" for i in range(len(case["xst"]))]
        J = dtb.Frame({nm: A(case, f"jraw{i}") for i, nm in enumerate(names)}, stypes=dict(zip(names, case["jst"])))
        J = J.to_device() if device else J
        J.key = names                                           # sorts J, checks that the keys are unique
        if not all(same(host(J.column(nm)), A(case, f"jsorted{i}")) for i, nm in enumerate(names)):
            bad.append(case["name"] + " key")
            continue
        J = dtb.Frame({**{nm: J.column(nm) for nm in names}, "jrow": dev(np.arange(J.nrows, dtype=np.int32), device)},
                      stypes=dict(zip(names, case["jst"])))
        J.key = names
        X = dtb.Frame({nm: A(case, f"x{i}") for i, nm in enumerate(names)}, stypes=dict(zip(names, case["xst"])))
        X = X.to_device() if device else X
        R = X[:, :, dtb.join(J)]
        if R.names != tuple(names) + ("jrow",) or not same(host(R.column("jrow")), A(case, "index")):
            bad.append(case["name"])
    assert not bad, bad


def set_modes():
    from datatable_b200 import _lib
    return {"union": _lib.SET_UNION, "intersect": _lib.SET_INTERSECT, "setdiff": _lib.SET_SETDIFF,
            "symdiff": _lib.SET_SYMDIFF}


@pytest.mark.parametrize("device", [False, True])
def test_set_operations_golden_abi(device):
    """The caller concatenates the inputs under the common stype, groups them and selects."""
    from datatable_b200 import engine, _lib
    bad = []
    for case in of("sets"):
        ins = [A(case, f"in{i}") for i in range(case["K"])]
        cat, st = promote(ins, case["sts"])
        cs = np.cumsum([len(a) for a in ins])
        if not len(cat):
            continue
        c = engine.Col(dev(cat, device), st)
        order, offsets, _ = engine.group([c], [0], _lib.NA_FIRST)
        for op, mode in set_modes().items():
            rows = host(engine.set_select(mode, order, offsets, cs))
            if st != case["out_st"][op] or not same(cat[rows], A(case, op)):
                bad.append(f"{case['name']} {op}")
    assert not bad, bad


@pytest.mark.parametrize("device", [False, True])
def test_set_operations_golden_frame(device):
    import datatable_b200 as dtb
    fns = {"union": dtb.union, "intersect": dtb.intersect, "setdiff": dtb.setdiff, "symdiff": dtb.symdiff}
    bad = []
    for case in of("sets"):
        frames = []
        for i, st in enumerate(case["sts"]):
            fr = dtb.Frame({"A": A(case, f"in{i}")}, stypes={"A": st})
            frames.append(fr.to_device() if device else fr)
        for op in OPS:
            R = fns[op](*frames)
            if R.names != ("A",) or R.stypes != (case["out_st"][op],) or not same(host(R.column("A")), A(case, op)):
                bad.append(f"{case['name']} {op}: {R.stypes} vs {case['out_st'][op]}")
    assert not bad, bad


@pytest.mark.parametrize("device", [False, True])
def test_unique_of_mixed_columns_golden(device):
    import datatable_b200 as dtb
    for case in of("unique"):
        names = [f"c{i}" for i in range(len(case["sts"]))]
        F = dtb.Frame({nm: A(case, nm) for nm in names}, stypes=dict(zip(names, case["sts"])))
        R = dtb.unique(F.to_device() if device else F)
        assert R.names == (case["out_name"],) and R.stypes == (case["out_st"],), case["name"]
        assert same(host(R.column(case["out_name"])), A(case, "out")), case["name"]


@pytest.mark.parametrize("device", [False, True])
def test_column_stats_golden(device):
    """Frame.nunique / mode / nmodal, and the same from group() and dtb_largest_group through the C-ABI."""
    import datatable_b200 as dtb
    from datatable_b200 import engine, _lib
    bad = []
    for case in of("stats"):
        names = [f"c{i}" for i in range(len(case["sts"]))]
        F = dtb.Frame({nm: A(case, nm) for nm in names}, stypes=dict(zip(names, case["sts"])))
        F = F.to_device() if device else F
        M, NM, NU = F.mode(), F.nmodal(), F.nunique()
        for i, (nm, st) in enumerate(zip(names, case["sts"])):
            ok = M.stypes[i] == st and same(host(M.column(nm)), A(case, f"mode{i}")) and \
                int(host(NM.column(nm))[0]) == A(case, "nmodal")[i] and int(host(NU.column(nm))[0]) == A(case, "nunique")[i]
            a = A(case, nm)
            if len(a):
                order, offsets, ng = engine.group([engine.Col(dev(a, device), st)], [0], _lib.NA_FIRST)
                skip = int(na_mask(a[host(order)[:1]], st)[0])
                idx, size = engine.largest_group(offsets, skip)
                ok &= size == A(case, "nmodal")[i] and ng - skip == A(case, "nunique")[i]
                if size:
                    ok &= same(a[host(order)[host(offsets)[idx]]][None], A(case, f"mode{i}"))
            if not ok:
                bad.append(f"{case['name']} {nm}")
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------
# join at scale, against tests/join_reference.py
# ---------------------------------------------------------------------------------------------------------------
def wide_values(st, n, rng):
    """random values over the whole type: NA, the edges, and (int64 / float32) values beyond 2^24 / 2^53"""
    if st == BOOL:
        v = rng.integers(0, 2, n).astype(np.int8)
    elif st in (INT8, INT16, INT32):
        info = np.iinfo(NPT[st])
        v = rng.integers(info.min + 1, info.max, n, endpoint=True).astype(NPT[st])
    elif st == INT64:
        v = rng.integers(-2**63 + 1, 2**63 - 1, n, dtype=np.int64)
        v[: n // 2] >>= rng.integers(0, 63, n // 2)               # every magnitude
    else:
        v = (rng.standard_normal(n) * 2.0 ** rng.integers(-10, 70, n)).astype(NPT[st])
        v[: n // 8] = np.trunc(v[: n // 8])
        v[rng.random(n) < 0.01] = np.inf
        v[rng.random(n) < 0.01] = -np.inf
        v[rng.random(n) < 0.01] = -0.0
    return v


def planted_x(j, jst, xst, n, rng):
    """X of stype xst: exact hits of J's values, near misses (+-1, +-1 ulp), int64 values that round onto J's float32
    keys, and random wide values, with NA"""
    jv = j[~na_mask(j, jst)] if len(j) else j
    parts = [wide_values(xst, n // 4, rng)]
    if len(jv):
        pick = jv[rng.integers(0, len(jv), n)]
        if xst in FLOATS:
            hit = pick.astype(NPT[xst])
            parts += [hit[: n // 4], np.nextafter(hit[n // 4: n // 2], np.inf).astype(NPT[xst])]
        else:
            info = np.iinfo(NPT[xst])
            p = pick.astype(np.float64) if jst in FLOATS else pick.astype(np.int64)
            if jst in FLOATS:
                p = p[np.isfinite(p) & (p > float(info.min)) & (p < float(info.max))].astype(np.int64)
            lo, hi = (0, 1) if xst == BOOL else (info.min + 1, info.max)
            p = p[(p >= lo) & (p <= hi)]
            step = rng.integers(-2**20, 2**20, len(p)) if (xst == INT64 and jst == FLOAT32) else rng.integers(-1, 2, len(p))
            near = np.clip(p + step, lo, hi) if xst != INT64 else p + np.where((p > -2**62) & (p < 2**62), step, 0)
            parts += [p.astype(NPT[xst]), near.astype(NPT[xst])]
    x = np.concatenate(parts)
    x = x[rng.integers(0, len(x), n)]
    x[rng.random(n) < 0.03] = np.nan if xst in FLOATS else NA[xst]
    return x


def sorted_unique_keys(cols, sts):
    """J's key columns as setting the key leaves them: sorted ascending, NA first, rows unique"""
    from oracle import oracle as orc
    o, offs, _ = orc.group(cols, [0] * len(cols), orc.NA_FIRST, stypes=list(sts))
    first = o[offs[:-1]]
    return [c[first] for c in cols]


def check_join(xs, xst, js, jst, ctx):
    import torch
    from datatable_b200 import engine
    want = join_index(xs, xst, js, jst)
    got = engine.join_index([engine.Col(torch.from_numpy(a).cuda(), s) for a, s in zip(xs, xst)],
                            [engine.Col(torch.from_numpy(a).cuda(), s) for a, s in zip(js, jst)]).cpu().numpy()
    bad = np.flatnonzero(got != want)
    assert not len(bad), f"{ctx}: {len(bad)} rows differ, first X row {bad[0]}: " \
        f"x = {[a[bad[0]] for a in xs]}, got J row {got[bad[0]]}, want {want[bad[0]]}"
    return (want >= 0).mean()


@pytest.mark.parametrize("xst", NUMERIC)
def test_join_every_stype_pair_on_wide_keys(xst):
    rng = np.random.default_rng(xst)
    for jst in NUMERIC:
        small = rng.integers(0, 2, 100) if jst == BOOL else rng.integers(-100, 100, 100)
        j = np.concatenate([wide_values(jst, 4000, rng), small.astype(NPT[jst]), na_of(jst)])
        j = sorted_unique_keys([j], [jst])[0]
        x = planted_x(j, jst, xst, 200_000, rng)
        hit = check_join([x], [xst], [j], [jst], f"{xst} x {jst}")
        assert hit > 0.01, (xst, jst, hit)


def test_join_int64_against_float32_collisions_at_1e7():
    """1e7 X rows (the grid-stride loop wraps many times) against 2^20 + 1 float32 keys: NA and every float32 of
    +-[2^60, 2^60 + 2^56), spaced 2^37 apart.  The X values are the keys, keys + -1, and the points one either side of
    the midpoint between two keys (k + 2^36 +- 1), which one rounding sends to the nearer key and a rounding through
    float64 sends to the midpoint and then to the even key."""
    rng = np.random.default_rng(1)
    run = 2**60 + np.arange(2**19, dtype=np.int64) * 2**37
    j = np.concatenate([[np.nan], (-run[::-1]).astype(np.float32), run.astype(np.float32)]).astype(np.float32)
    assert len(np.unique(j[1:])) == 2**20
    n = 10_000_000
    k = j[rng.integers(1, len(j), n)].astype(np.int64)
    x = k + rng.choice(np.array([0, 1, -1, 2**36 + 1, 2**36 - 1, -2**36 + 1, -2**36 - 1]), n)
    x[::101] = NA[INT64]
    hit = check_join([x], [INT64], [j], [FLOAT32], "int64 x float32, 1e7 rows")
    assert hit > 0.9


@pytest.mark.parametrize("nk", [2, 3, 4])
def test_join_multi_key_at_1e7(nk):
    """Up to 1e7 X rows, nk key columns of different stypes, NA in any column, J of up to 2^18 rows."""
    rng = np.random.default_rng(nk)
    jst = [INT64, FLOAT32, INT8, FLOAT64][:nk]
    xst = [FLOAT64, INT64, INT32, INT16][:nk]
    nj = 2**18
    small = {INT8: np.array([0, 1, 2, NA[INT8]], np.int8)}
    jc = []
    for s in jst:
        if s in small:
            jc.append(small[s][rng.integers(0, 4, nj)])
        else:
            scale = 2**40 if s in (INT64, FLOAT32) else 300            # float32 holds multiples of 2^16 below 2^40
            v = (rng.integers(-scale, scale, nj) // 2**16 * 2**16 if scale > 300 else
                 rng.integers(-scale, scale, nj)).astype(NPT[s])
            v[rng.random(nj) < 0.02] = np.nan if s in FLOATS else NA[s]
            jc.append(v)
    js = sorted_unique_keys(jc, jst)
    n = 10_000_000 if nk == 4 else 2_000_000
    pick = rng.integers(0, len(js[0]), n)
    xs = []
    for c, (jcol, sj, sx) in enumerate(zip(js, jst, xst)):
        v = jcol[pick]
        xv = np.where(na_mask(v, sj), np.nan, v.astype(np.float64)) if sx in FLOATS else \
            np.where(na_mask(v, sj), NA[sx], np.nan_to_num(v.astype(np.float64)).astype(np.int64))
        xv = xv.astype(NPT[sx])
        miss = rng.random(n) < 0.1
        if sx in FLOATS:
            xv[miss] += 0.5
        else:
            xv[miss & (xv != NA[sx])] += 1
        xs.append(xv)
    hit = check_join(xs, xst, js, jst, f"{nk} keys, {n} rows")
    assert hit > 0.3


# ---------------------------------------------------------------------------------------------------------------
# dtb_set_select at scale, against a vectorised reference
# ---------------------------------------------------------------------------------------------------------------
def set_select_reference(mode, order, offsets, cum_sizes):
    """The first row of every kept group, from the unique (group, input) pairs: the inputs present in each group."""
    from datatable_b200 import _lib
    K = len(cum_sizes)
    ng = len(offsets) - 1
    gid = np.repeat(np.arange(ng, dtype=np.int64), np.diff(offsets))
    inp = np.searchsorted(np.asarray(cum_sizes), order, side="right")
    pairs = np.unique(gid * K + inp)
    pg, pk = pairs // K, pairs % K
    count = np.bincount(pg, minlength=ng)
    only0 = (count == 1) & (np.bincount(pg, weights=(pk == 0), minlength=ng) == 1)
    keep = {_lib.SET_UNION: np.ones(ng, bool), _lib.SET_INTERSECT: count == K, _lib.SET_SETDIFF: only0,
            _lib.SET_SYMDIFF: (count == 1) if K == 2 else (count % 2 == 1)}[mode]
    if K < 2:
        keep = np.ones(ng, bool)
    return order[offsets[:-1][keep]].astype(np.int32)


@pytest.mark.parametrize("K", [2, 3, 5, 17, 64])
def test_set_select_at_scale(K):
    import torch
    from datatable_b200 import engine, _lib
    rng = np.random.default_rng(K)
    total = 5_000_000 if K in (3, 17) else 1_000_000
    w = rng.pareto(1.0, K) + 0.05                                    # uneven inputs, some empty
    sizes = (w / w.sum() * total).astype(np.int64)
    sizes[rng.random(K) < 0.2] = 0
    sizes[K // 2] = 0
    cs = np.cumsum(sizes)
    for nvals in (1000, 10**6):                                      # large groups (bisection inside), small groups
        parts = [rng.integers(k, nvals + k, s).astype(np.int32) for k, s in enumerate(sizes)]
        for p in parts:
            p[:3] = NA[INT32]                                        # the NA group spans the inputs too
        cat = np.concatenate(parts)
        order, offsets, ng = engine.group([torch.from_numpy(cat).cuda()], [0], _lib.NA_FIRST)
        o, f = order.cpu().numpy(), offsets.cpu().numpy()
        assert np.array_equal(o, np.argsort(cat, kind="stable")), "group() order"
        for mode in (_lib.SET_UNION, _lib.SET_INTERSECT, _lib.SET_SETDIFF, _lib.SET_SYMDIFF):
            want = set_select_reference(mode, o, f, cs)
            got = engine.set_select(mode, order, offsets, cs).cpu().numpy()
            assert np.array_equal(got, want), (K, nvals, mode, len(got), len(want))


# ---------------------------------------------------------------------------------------------------------------
# dtb_largest_group
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ng", [1, 2, 33, 257, 100_003, 10_000_000])
def test_largest_group_ties(ng):
    import torch
    from datatable_b200 import engine
    rng = np.random.default_rng(ng)
    base = rng.integers(1, 9, ng)
    M = 12
    spots = [0, ng - 1, 31, 32, 255, 256, 1023, 1024, ng // 2, ng - 33]
    for plant in ([0, ng - 1], [ng - 1], spots[2:], [1, ng - 1], spots[4:8], []):
        sizes = base.copy()
        for s in plant:
            if 0 <= s < ng:
                sizes[s] = M
        for skip in (0, 1):
            for bump0 in (False, True):                              # the skipped group is larger than any other
                sz = sizes.copy()
                if bump0:
                    sz[0] = M + 5
                offsets = np.concatenate([[0], np.cumsum(sz)]).astype(np.int32)
                if ng <= skip:
                    want = (-1, 0)
                else:
                    i = int(np.argmax(sz[skip:]))
                    want = (i + skip, int(sz[skip + i]))
                for d in (False, True):
                    got = engine.largest_group(torch.from_numpy(offsets).cuda() if d else offsets, skip)
                    assert got == want, (ng, plant, skip, bump0, d)


# ---------------------------------------------------------------------------------------------------------------
# dtb_lower_bound: the cut points dist.py takes between GPUs
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("st", [BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64])
def test_lower_bound(st):
    import torch
    from datatable_b200 import engine, _lib
    rng = np.random.default_rng(st)
    for n in (0, 1, 2, 7, 1000, 3_000_001):
        if st == BOOL:
            s = np.sort(rng.integers(0, 2, n)).astype(np.int8)
            v = np.array([0, 1, -1, 2, 0, 1], np.int8)
        else:
            lo = -1000 if n < 10**6 else -10**5
            s = np.sort(rng.integers(lo, -lo, n).astype(NPT[st]))
            if st in FLOATS and n:
                s[s == 0] = -0.0
            v = np.concatenate([rng.integers(2 * lo, -2 * lo, 2000).astype(NPT[st]), s[:: max(1, n // 50)],
                                np.array([np.iinfo(np.int8).min + 1, 127], NPT[st])])
            if st in FLOATS:
                v = np.concatenate([v, np.array([-np.inf, np.inf, 0.0, -0.0, 0.5, -0.5], NPT[st])])
            elif st in (INT64, TIME64):
                v = np.concatenate([v, np.array([-2**63 + 1, 2**63 - 1], np.int64)])
        want = np.searchsorted(s, v, side="left").astype(np.int64)
        for d in (False, True):
            sc = engine.Col(torch.from_numpy(s).cuda() if d else s, st)
            vc = engine.Col(torch.from_numpy(v).cuda() if d else v, st)
            out = torch.empty(len(v), dtype=torch.int64, device="cuda") if d else np.empty(len(v), np.int64)
            ptr = out.data_ptr() if d else out.ctypes.data
            _lib.check(_lib.lib.dtb_lower_bound(sc.c(), sc.nrows, vc.c(), vc.nrows, engine._stream(),
                                                ctypes.c_void_p(ptr)))
            got = out.cpu().numpy() if d else out
            assert np.array_equal(got, want), (st, n, d)
