#!/usr/bin/env python
"""
Generates tests/golden/golden_v9.{npz,json} by running the *reference itself* (the unmodified build staged by
oracle/build_ref.sh) on the callers of group() beyond DT[i, j, by] at the edges of their types:

    PYTHONPATH=oracle/_ref python tests/golden/make_golden_v9.py

    keyed join        X[:, :, join(J)] with J.key set      (frame/key.cc:118-180, frame/join.cc:199-470)
    set operations    dt.union / intersect / setdiff / symdiff / unique        (set_funcs.cc:126-456)
    column stats      Frame.nunique(), Frame.mode(), Frame.nmodal()            (stats.cc:955-1003)

join: every (X stype, J stype) pair of the reference's comparator table (join.cc:322-377: the 7 x 7 of bool,
int8 .. int64, float32, float64, plus date32 / date32 and time64 / time64).  X holds every type's min + 1, max and
NA, J's NA sentinel as a value, int64 values beyond 2^53 next to their float neighbours (2^60 + 2^36 +- 1,
2^60 + 2^37, 2^53 + 1, 2^24 + 1), fractions, +-inf, -0.0 and +0.0, and values one past J's range (2^15, 2^31,
2^63 as floats), next to exact hits and near misses of J's values.  J sizes 0, 1, 2, 3, 2^k - 1, 2^k, 2^k + 1 up
to 4097 walk every exit of the binary search; multi-key joins put an NA in any one column; float J keys that hold
both -0.0 and +0.0 pin which row the search path lands on.
sets: inputs of mixed stypes (the output stype is recorded), K = 1 .. 10 with empty inputs first, in the middle and
last, groups that span every input, wide values, +-inf, -0.0 / +0.0 and NA, and unique() of a frame whose columns
have different stypes.
stats: ties for the largest group (at the first, a middle and the last valid group), an NA group larger than every
valid group, all-NA columns, one row, no rows, bool columns and float columns with -0.0 and +0.0.

The reference cannot travel to the GPU box, so the vectors are committed.
"""
import json
import math
import os
import warnings

import numpy as np

import datatable as dt
from datatable import f, join

HERE = os.path.dirname(os.path.abspath(__file__))
BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64 = 1, 2, 3, 4, 5, 6, 7, 17, 18
NUMERIC = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
NPT = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
       FLOAT32: np.float32, FLOAT64: np.float64, DATE32: np.int32, TIME64: np.int64}
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
RANGE = {BOOL: (0, 1), INT8: (-127, 127), INT16: (-2**15 + 1, 2**15 - 1), INT32: (-2**31 + 1, 2**31 - 1),
         INT64: (-2**63 + 1, 2**63 - 1), DATE32: (-10**6, 10**6), TIME64: (-10**15, 10**15)}
DTST = {BOOL: dt.bool8, INT8: dt.int8, INT16: dt.int16, INT32: dt.int32, INT64: dt.int64,
        FLOAT32: dt.float32, FLOAT64: dt.float64, DATE32: dt.int32, TIME64: dt.int64}
ST_OF = {dt.bool8: BOOL, dt.int8: INT8, dt.int16: INT16, dt.int32: INT32, dt.int64: INT64, dt.float32: FLOAT32,
         dt.float64: FLOAT64, dt.stype.date32: DATE32, dt.stype.time64: TIME64}
TAG = {BOOL: "bool", INT8: "i8", INT16: "i16", INT32: "i32", INT64: "i64", FLOAT32: "f32", FLOAT64: "f64",
       DATE32: "date32", TIME64: "time64"}
arrays, manifest = {}, []
rng = np.random.default_rng(20261016)
warnings.simplefilter("ignore", RuntimeWarning)             # float32 overflow of 1e300 is meant

# the values every typed pool is drawn from: integers as Python ints, floats as Python floats
INTS = [0, 1, -1, 2, -2, 5, -5, 100, -100, 126, -126, 127, -127, 128, -128, 255, 2**15 - 1, -(2**15 - 1), 2**15,
        -2**15, 2**24, 2**24 + 1, 2**24 + 2, 2**31 - 1, -(2**31 - 1), 2**31, -2**31, 2**53, 2**53 + 1, 2**53 + 2,
        2**60, 2**60 + 2**36 - 1, 2**60 + 2**36, 2**60 + 2**36 + 1, 2**60 + 2**37, -(2**60 + 2**36 + 1),
        2**63 - 1, -(2**63 - 1)]
FLOATS = [0.5, -0.5, 1.5, -2.25, 127.5, -0.0, 0.0, math.inf, -math.inf, 2.0**15, -2.0**15, 2.0**31, -2.0**31,
          2.0**63, -2.0**63, 2.0**64, 1e300, -1e300, 3.0e38, 1e-40, 2.0**60, 2.0**60 + 2.0**37, 2.0**53 + 2.0]


def typed(vals, st):
    """The members of `vals` a column of stype st holds, converted once (int64 -> float32 is one rounding, as
    numpy's astype and the reference's static_cast do); NA sentinels and values out of range are dropped."""
    if st in (FLOAT32, FLOAT64):
        ints = [v for v in vals if isinstance(v, int) and -2**63 <= v < 2**63]
        flts = [v for v in vals if isinstance(v, float)]
        return np.concatenate([np.array(ints, np.int64).astype(NPT[st]), np.array(flts, np.float64).astype(NPT[st])])
    lo, hi = RANGE[st]
    out = [int(v) for v in vals if (isinstance(v, int) or (math.isfinite(v) and v == int(v))) and lo <= int(v) <= hi]
    return np.array(out, dtype=NPT[st])


def na_of(st):
    return np.array([np.nan if st in (FLOAT32, FLOAT64) else NA[st]], NPT[st])


def pool(st):
    """every edge of the type: min + 1, max, and the shared pool"""
    if st in (DATE32, TIME64):
        lo, hi = RANGE[st]
        return np.concatenate([np.array([lo, hi, 0, 1, -1], NPT[st]), rng.integers(lo, hi, 20).astype(NPT[st])])
    extra = [] if st in (FLOAT32, FLOAT64) else list(RANGE[st])
    if st == FLOAT32:
        extra = [float(np.finfo(np.float32).max), -float(np.finfo(np.float32).max)]
    return typed(INTS + FLOATS + extra, st)


def pylist(a, st):
    if st in (FLOAT32, FLOAT64):
        return [None if np.isnan(x) else float(x) for x in a.tolist()]
    return [None if x == NA[st] else (bool(x) if st == BOOL else int(x)) for x in a.tolist()]


def column(a, st, name):
    """single-column reference Frame; floats keep their bit patterns (-0.0), integer NA sentinels become None"""
    a = np.ascontiguousarray(a, dtype=NPT[st])
    if st in (FLOAT32, FLOAT64):
        fr = dt.Frame({name: a})
    else:
        fr = dt.Frame({name: pylist(a, st)}, stypes={name: DTST[st]})
        if st == DATE32:
            fr[name] = fr[:, dt.as_type(f[name], dt.Type.date32)]
        elif st == TIME64:
            fr[name] = fr[:, dt.as_type(f[name], dt.Type.time64)]
    return fr


def frame(cols):
    fr = None
    for name, (a, st) in cols.items():
        c = column(a, st, name)
        fr = c if fr is None else dt.cbind(fr, c)
    return fr


def to_np(fr, i=0):
    """column i of a reference Frame as its stype's storage (float bits kept, NA as the sentinel) and its stype"""
    col = fr[:, i]
    st = ST_OF[col.stypes[0]]
    if st in (FLOAT32, FLOAT64):
        if col.nrows == 0:                                      # the reference's to_numpy() crashes on 0 rows
            return np.zeros(0, NPT[st]), st
        return col.to_numpy().reshape(-1).astype(NPT[st]), st
    if st in (DATE32, TIME64):
        col = col[:, dt.as_type(f[0], DTST[st])]
    return np.array([NA[st] if x is None else int(x) for x in col.to_list()[0]], dtype=NPT[st]), st


def put(name, key, a):
    arrays[f"{name}.{key}"] = np.ascontiguousarray(a)


# ---------------------------------------------------------------------------
# keyed join
# ---------------------------------------------------------------------------
def join_case(name, xcols, xst, jcols, jst, **meta):
    """J (given unsorted) gets its key set, X is joined; the golden is J's row (after the key sort) matched by
    every X row, read back from a payload column holding J's row numbers."""
    names = [f"k{i}" for i in range(len(xcols))]
    case = {"name": name, "kind": "join", "xst": list(xst), "jst": list(jst), **meta}
    for i in range(len(xcols)):
        put(name, f"x{i}", xcols[i].astype(NPT[xst[i]]))
        put(name, f"jraw{i}", jcols[i].astype(NPT[jst[i]]))
    J = frame({nm: (a, st) for nm, a, st in zip(names, jcols, jst)})
    try:
        J.key = names
    except Exception as e:                                      # noqa: BLE001
        case["key_error"] = f"{type(e).__name__}: {e}"
        manifest.append(case)
        return
    for i, st in enumerate(jst):
        put(name, f"jsorted{i}", to_np(J, i)[0])
    J = dt.cbind(J, dt.Frame(jrow=np.arange(J.nrows, dtype=np.int32)))
    J.key = names
    X = frame({nm: (a, st) for nm, a, st in zip(names, xcols, xst)})
    R = X[:, :, join(J)]
    put(name, "index", to_np(R[:, "jrow"])[0])
    case["nx"], case["nj"] = int(X.nrows), int(J.nrows)
    manifest.append(case)


def hits_and_misses(jv, jst, xst):
    """J's valid values as X values where X's type holds them, and their neighbours"""
    if jst in (FLOAT32, FLOAT64):
        v = [float(x) for x in jv if not np.isnan(x)]
        near = [float(np.nextafter(x, np.inf)) for x in v] + [x + 1.0 for x in v if math.isfinite(x)]
    else:
        v = [int(x) for x in jv if x != NA[jst]]
        near = [x + 1 for x in v] + [x - 1 for x in v]
    if xst in (DATE32, TIME64):
        lo, hi = RANGE[xst]
        return np.array([x for x in v + near if isinstance(x, int) and lo <= x <= hi], NPT[xst])
    return typed(v + near, xst)


# every pair of the comparator table, J = the typed pool of J's stype (unique, NA included, shuffled)
PAIRS = [(x, j) for x in NUMERIC for j in NUMERIC] + [(DATE32, DATE32), (TIME64, TIME64)]
for xst, jst in PAIRS:
    j = np.unique(np.concatenate([pool(jst), na_of(jst)]))     # np.unique keeps one NaN and one of -0.0 / +0.0
    j = j[rng.permutation(len(j))]
    base = np.concatenate([pool(xst), na_of(xst), hits_and_misses(j, jst, xst)])
    x = np.concatenate([base, rng.choice(base, 40)])
    join_case(f"join.{TAG[xst]}.{TAG[jst]}", [x], [xst], [j], [jst])


# J sizes around powers of two: every exit of the binary search (start == end after 0 .. 12 halvings)
def sized_j(jst, n):
    if jst == FLOAT32:          # int64 X against float32 J: the keys are float32 values of 2^40 + k 2^17
        return (np.arange(n, dtype=np.int64) * 2**17 + 2**40).astype(np.float32)
    if jst == FLOAT64:
        return (np.arange(n) - n // 2).astype(np.float64) * 0.5
    return (np.arange(n, dtype=np.int64) * 2 - n).astype(NPT[jst])


def sized_x(j, jst, xst):
    if jst == FLOAT32:          # exact hits, +-1 (one float32 rounding: still a hit), the halfway point 2^16
        base = j.astype(np.int64)
        x = np.concatenate([base, base + 1, base - 1, base + 2**16, base + 2**17 - 1, [2**40 - 2**17, 2**62]])
    elif jst == FLOAT64:
        x = np.concatenate([j, j + 0.25, [-1e9, 1e9, -0.0]]) if xst == FLOAT64 else \
            np.concatenate([np.trunc(j), np.trunc(j) + 1, [-10**6, 10**6]]).astype(np.int64)
    else:
        x = np.concatenate([j, j + 1, [-10**6, 10**6]]).astype(np.int64)
    return np.concatenate([x.astype(NPT[xst]), na_of(xst)])


SIZES = [0, 1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, 33, 255, 256, 257, 1023, 1024, 1025]
for xst, jst, big in ((INT32, INT32, True), (INT64, FLOAT32, True), (FLOAT64, FLOAT64, False),
                      (INT32, FLOAT64, False)):
    for n in SIZES + ([4095, 4096, 4097] if big else []):
        for with_na in ((False, True) if n in (1, 2, 3, 8, 257) else (False,)):
            j = sized_j(jst, n)
            if with_na:
                j = np.concatenate([j[: n - 1], na_of(jst)])     # NA sorts first: the search starts one row on
            x = sized_x(j[~np.isnan(j)] if jst in (FLOAT32, FLOAT64) else j[j != NA[jst]], jst, xst)
            join_case(f"jsize.{TAG[xst]}.{TAG[jst]}.{n}{'.na' if with_na else ''}", [x], [xst], [j[::-1].copy()],
                      [jst], size=n)


# multi-key joins: J is a product of small value sets with NA in every column; X adds misses in every column
def product(*sets):
    grids = np.meshgrid(*[np.arange(len(s)) for s in sets], indexing="ij")
    return [s[g.reshape(-1)] for s, g in zip(sets, grids)]


MULTI = [((INT32, FLOAT64), (INT64, FLOAT32)),
         ((INT8, INT16, FLOAT32), (INT16, INT8, FLOAT64)),
         ((BOOL, INT64), (BOOL, FLOAT64)),
         ((FLOAT64, INT32, INT64, INT16), (INT32, INT64, FLOAT32, INT16)),
         ((DATE32, INT32), (DATE32, INT32))]
for xst, jst in MULTI:
    jsets = [np.concatenate([typed([0, 1, 2**31 - 1, 2**60 + 2**37, 2.0**53 + 2.0, -0.5, 100], s)
                             if s not in (BOOL, DATE32) else np.array([0, 1], NPT[s]), na_of(s)]) for s in jst]
    jsets = [np.unique(s) for s in jsets]
    jk = product(*jsets)
    keep = rng.random(len(jk[0])) < 0.7
    jk = [a[keep] for a in jk]
    perm = rng.permutation(len(jk[0]))
    jk = [a[perm] for a in jk]
    xsets = [np.concatenate([hits_and_misses(jsets[c], jst[c], xst[c]), na_of(xst[c])]) for c in range(len(xst))]
    xsets = [np.unique(s)[: 12] if len(np.unique(s)) > 12 else np.unique(s) for s in xsets]
    xk = product(*xsets)
    if len(xk[0]) > 3000:
        pick = rng.choice(len(xk[0]), 3000, replace=False)
        xk = [a[pick] for a in xk]
    join_case(f"jmulti.{'_'.join(TAG[s] for s in xst)}", xk, xst, jk, jst)

# float keys holding both -0.0 and +0.0 (distinct keys to group()): the search path picks the row
for jst in (FLOAT64, FLOAT32):
    for pad_lo, pad_hi in ((0, 0), (1, 0), (0, 1), (1, 1), (2, 0), (0, 2), (3, 4), (5, 2)):
        j = np.concatenate([-1.0 - np.arange(pad_lo), [-0.0, 0.0], 1.0 + np.arange(pad_hi)]).astype(NPT[jst])
        for xst in (FLOAT64, FLOAT32, INT32):
            x = np.concatenate([typed([-0.0, 0.0, 0, 1, -1, 0.5], xst), na_of(xst)])
            join_case(f"jzero.{TAG[xst]}.{TAG[jst]}.{pad_lo}_{pad_hi}", [x], [xst], [j[::-1].copy()], [jst])


# ---------------------------------------------------------------------------
# set operations
# ---------------------------------------------------------------------------
SETS = {"union": dt.union, "intersect": dt.intersect, "setdiff": dt.setdiff, "symdiff": dt.symdiff}


def set_case(name, ins, sts, **meta):
    case = {"name": name, "kind": "sets", "sts": list(sts), "K": len(ins), "ops": list(SETS), **meta}
    frames = [column(a, st, "A") for a, st in zip(ins, sts)]
    for i, (a, st) in enumerate(zip(ins, sts)):
        put(name, f"in{i}", a.astype(NPT[st]))
    case["out_st"] = {}
    for op, fn in SETS.items():
        v, st = to_np(fn(*frames))
        put(name, op, v)
        case["out_st"][op] = st
    manifest.append(case)


def wide(st, n, extra=()):
    p = np.concatenate([pool(st), na_of(st), typed(list(extra), st)])
    return rng.choice(p, n)


MIXED = [(INT32, FLOAT32), (FLOAT32, INT32), (INT64, FLOAT32), (BOOL, INT8), (INT8, FLOAT64), (FLOAT32, FLOAT64),
         (FLOAT64, FLOAT32), (INT16, INT64), (BOOL, FLOAT32), (INT16, INT32, FLOAT32), (INT64, FLOAT32, INT8),
         (BOOL, INT8, INT16, INT32, INT64, FLOAT32)]
for sts in MIXED:
    for rep in range(2):
        ins = [wide(st, int(rng.integers(20, 60))) for st in sts]
        set_case(f"smix.{'_'.join(TAG[s] for s in sts)}.{rep}", ins, sts)
# int64 values that collide in float32 next to the float32 values they round to
coll = [2**60, 2**60 + 2**36 - 1, 2**60 + 2**36, 2**60 + 2**36 + 1, 2**60 + 2**37, 2**24, 2**24 + 1, 2**24 + 2,
        2**53 + 1, 0, 7]
set_case("scollide.i64_f32", [np.array(coll + [NA[INT64]], np.int64),
                              np.concatenate([typed(coll, FLOAT32)[::2], na_of(FLOAT32), [-0.0]]).astype(np.float32)],
         (INT64, FLOAT32))
set_case("scollide.i64_f32_i64", [np.array(coll, np.int64), typed([2**60 + 2**37, 2**24, 7], FLOAT32),
                                  np.array(coll[::-1], np.int64)], (INT64, FLOAT32, INT64))

# K = 1 .. 10: no empty input, empty first / in the middle / last / all; every input holds 7 and NA
for st in (INT32, FLOAT64):
    for K in range(1, 11):
        for empty in ("none", "first", "middle", "last", "all"):
            if K == 1 and empty in ("first", "middle", "last"):
                continue
            if K == 2 and empty == "middle":
                continue
            ins = []
            for k in range(K):
                a = np.concatenate([typed([7, k, k + 1, 2 * k, -3, 2**31 - 1, -0.0, math.inf], st), na_of(st),
                                    rng.integers(-4, 12, int(rng.integers(0, 30))).astype(NPT[st])])
                ins.append(a[rng.permutation(len(a))])
            drop = {"none": (), "first": (0,), "middle": (K // 2,), "last": (K - 1,), "all": tuple(range(K))}[empty]
            ins = [np.zeros(0, NPT[st]) if k in drop else a for k, a in enumerate(ins)]
            set_case(f"sk.{TAG[st]}.{K}.{empty}", ins, [st] * K)
# wide values, +-inf, -0.0 / +0.0 and NA, one stype
for st in (INT64, FLOAT32, FLOAT64, INT8, BOOL):
    for K in (2, 3, 5):
        set_case(f"swide.{TAG[st]}.{K}", [wide(st, int(rng.integers(5, 80))) for _ in range(K)], [st] * K)
for st in (FLOAT32, FLOAT64):
    z = np.array([-0.0, 0.0, np.nan, -np.inf, np.inf], NPT[st])
    set_case(f"szero.{TAG[st]}", [z[[0, 2]], z[[1, 3]], z[[0, 1, 4]]], [st] * 3)
    set_case(f"szero2.{TAG[st]}", [z[[0]], z[[1]]], [st] * 2)


# unique() of a frame whose columns have different stypes
def unique_case(name, cols):
    case = {"name": name, "kind": "unique", "sts": [st for _, st in cols]}
    for i, (a, st) in enumerate(cols):
        put(name, f"c{i}", a.astype(NPT[st]))
    U = dt.unique(frame({f"c{i}": (a, st) for i, (a, st) in enumerate(cols)}))
    v, st = to_np(U)
    put(name, "out", v)
    case["out_st"], case["out_name"] = st, U.names[0]
    manifest.append(case)


for sts in ((INT32, FLOAT32), (INT64, FLOAT32, INT8), (BOOL, INT8, FLOAT64), (INT16, INT32, INT64),
            (FLOAT32, FLOAT64, INT64, BOOL)):
    n = int(rng.integers(10, 50))
    unique_case(f"unique.{'_'.join(TAG[s] for s in sts)}", [(wide(st, n, coll), st) for st in sts])


# ---------------------------------------------------------------------------
# nunique / mode / nmodal
# ---------------------------------------------------------------------------
def stats_case(name, cols):
    case = {"name": name, "kind": "stats", "sts": [st for _, st in cols]}
    for i, (a, st) in enumerate(cols):
        put(name, f"c{i}", np.asarray(a).astype(NPT[st]))
    F = frame({f"c{i}": (np.asarray(a), st) for i, (a, st) in enumerate(cols)})
    M = F.mode()
    for i in range(len(cols)):
        v, st = to_np(M, i)
        put(name, f"mode{i}", v)
        assert st == cols[i][1], (name, st)
    put(name, "nunique", np.array(F.nunique().to_list(), np.int64).reshape(-1))
    put(name, "nmodal", np.array(F.nmodal().to_list(), np.int64).reshape(-1))
    manifest.append(case)


N_ = None
SHAPES = {                      # value layouts as small integers; N_ = NA
    "tie_first": [1, 1, 2, 2, 3],
    "tie_first_last": [3, 1, 1, 2, 3],
    "tie_middle": [1, 2, 2, 3, 3, 4],
    "last_only": [1, 2, 3, 3],
    "first_only": [0, 0, 0, 1, 2],
    "na_largest": [N_, N_, N_, N_, 1, 1, 2, 2, 0],
    "na_tie": [N_, N_, 1, 1, 2],
    "na_then_first": [2, N_, 1, 2, N_, 1],
    "all_na": [N_, N_, N_],
    "one_row": [5],
    "one_na": [N_],
    "empty": [],
    "all_same": [4, 4, 4, 4],
    "distinct": [5, 1, 4, 2, 3],
}
for st in (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64):
    for nm, shape in SHAPES.items():
        vals = [NA[st] if v is None and st not in (FLOAT32, FLOAT64) else (np.nan if v is None else
                (v % 2 if st == BOOL else v)) for v in shape]
        if st == INT64:
            vals = [v if v == NA[st] else v * 2**40 + 2**60 for v in vals]
        stats_case(f"stats.{TAG[st]}.{nm}", [(np.array(vals, NPT[st]), st)])
for st in (FLOAT32, FLOAT64):
    for nm, v in (("zeros", [-0.0, 0.0, 0.0, np.nan]), ("negzeros", [0.0, -0.0, -0.0, 1.0, 1.0]),
                  ("inf", [np.inf, -np.inf, np.inf, -0.0, np.nan, np.nan, np.nan])):
        stats_case(f"stats.{TAG[st]}.{nm}", [(np.array(v, NPT[st]), st)])
n = 200
stats_case("stats.multi", [(wide(st, n), st) for st in (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)])
stats_case("stats.multi_few", [(rng.choice(np.array([0, 1, NA[BOOL]], np.int8), 300), BOOL),
                               (rng.choice(np.array([-0.0, 0.0, np.nan, 1.0]), 300), FLOAT64),
                               (rng.choice(np.array([NA[INT32], 1, 2, 3], np.int32), 300), INT32)])

np.savez_compressed(os.path.join(HERE, "golden_v9.npz"), **arrays)
with open(os.path.join(HERE, "golden_v9.json"), "w") as fh:
    json.dump({"generator": "tests/golden/make_golden_v9.py",            # the version without its build stamp
               "datatable_version": dt.__version__.split("+")[0],
               "cases": manifest}, fh, indent=0)
print(f"{len(manifest)} cases, {sum(a.nbytes for a in arrays.values()) / 1e6:.2f} MB raw")
