#!/usr/bin/env python
"""
Generates tests/golden/golden_v14.{npz,json} by running the *reference itself* (the unmodified build staged by
oracle/build_ref.sh) on the time functions:

    PYTHONPATH=oracle/_ref:tests python tests/golden/make_golden_v14.py

    dt.time.year / month / day / day_of_week / hour / minute / second / nanosecond (src/core/expr/time/)

Every case stores the frame's columns, the query and what the reference returns (output names, stypes, columns), or
the error it raises.  The query shapes are tests/time_reference.py's query_args:
    part   the time function of j (and of the key with kpart)
    mode   none, sort (sort(f.s)), sortdesc (sort(-f.s)), by (by(f.s)), bysort (by(f.s), sort(f.v)), join (join(J),
           J's columns stored as J.<name>), bypart (by(kpart(f.d))), bypartneg (by(-kpart(f.d))), bykpart (by(f.s,
           kpart(f.d))), sortpart (sort(kpart(f.t), f.s)), sortpartneg (sort(-kpart(f.t), f.s)), bypart_t
           (by(kpart(f.t))), bypartjoin (by(kpart(g.d)), join(J)), bypartsort (by(kpart(f.d)), sort(f.s))
    i      None, ["slice", [a, b, c]], ["int", k], ["bool", "b"] (f.b), ["frame", "isel"] (an int32 Frame with NA),
           ["list", [...]], ["range", [a, b, c]]
    j      one = part(f.d), list = part([f.d, f.t]), tuple, all = part(f[:]), dict = {"y": part(f.d)}, plain = [f.d,
           part(f.d)], cut / qcut / cumsum / shift / fillna / cumcount / ngroup = [part(f.d), that function], joincol
           = part(g.d), joinlist = [part(f.d), part(g.d)], parts = every part of f.t, bysum = sum(f.v), bycount =
           count(), byall = :, bykeys = [f.v, part(f.t)]
    call   the argument errors of the functions themselves: noargs, twoargs, kwarg (the argument by keyword), badkw,
           dupkw
The reference cannot travel to the GPU box, so the vectors are committed.
"""
import json
import os
import sys

# datatable before numpy (see make_golden_v12.py)
import datatable as dt
from datatable import f

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from time_reference import PARTS, query_args  # noqa: E402

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64 = 1, 2, 3, 4, 5, 6, 7, 17, 18
NPT = {BOOL: np.int8, INT32: np.int32, INT64: np.int64, FLOAT64: np.float64, DATE32: np.int32, TIME64: np.int64}
NA = {BOOL: -128, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
DTST = {BOOL: dt.bool8, INT32: dt.int32, INT64: dt.int64, FLOAT64: dt.float64, DATE32: dt.int32, TIME64: dt.int64}
OUT_NP = {dt.bool8: np.int8, dt.int32: np.int32, dt.int64: np.int64}
DAY = 86400 * 10**9
arrays, manifest = {}, []
rng = np.random.default_rng(20261019)


def pylist(a, st):
    if st == FLOAT64:
        return [None if np.isnan(x) else float(x) for x in a.tolist()]
    return [None if x == NA[st] else (bool(x) if st == BOOL else int(x)) for x in a.tolist()]


def to_np(fr, name):
    col = fr[:, name]
    st = col.stypes[0]
    if st in (dt.stype.date32, dt.stype.time64):
        col = col[:, dt.as_type(f[0], dt.int32 if st == dt.stype.date32 else dt.int64)]
        st = col.stypes[0]
    lst = col.to_list()[0]
    if st == dt.float64:
        return np.array([np.nan if x is None else x for x in lst], dtype=np.float64)
    npdt = OUT_NP[st]
    na = -128 if st == dt.bool8 else np.iinfo(npdt).min
    return np.array([na if x is None else int(x) for x in lst], dtype=npdt)


def frame(cols):
    DT = dt.Frame({nm: (a if st == FLOAT64 else pylist(a, st)) for nm, (st, a) in cols.items()},
                  stypes={nm: DTST[st] for nm, (st, _) in cols.items()})
    for nm, (st, _) in cols.items():
        if st == DATE32:
            DT[nm] = DT[:, dt.as_type(f[nm], dt.Type.date32)]
        elif st == TIME64:
            DT[nm] = DT[:, dt.as_type(f[nm], dt.Type.time64)]
    return DT


CALLS = {"noargs": lambda P: P(), "twoargs": lambda P: P(f.d, f.t), "kwarg": lambda P: P(**{"date": f.d}),
         "badkw": lambda P: P(foo=f.d), "dupkw": lambda P: P(f.d, **{"date": f.t})}


def add(name, cols, part="year", mode="none", i=None, j="one", kpart=None, jcols=None, call=None):
    case = {"name": name, "part": part, "mode": mode, "i": i, "j": j, "kpart": kpart, "call": call,
            "stypes": {nm: st for nm, (st, _) in cols.items()}}
    for nm, (st, a) in cols.items():
        arrays[name + "." + nm] = np.ascontiguousarray(a, dtype=NPT[st])
    if i is not None and i[0] == "frame":
        arrays[name + ".isel"] = np.ascontiguousarray(i[2], dtype=np.int32)
        case["i"] = ["frame", "isel"]
    J = None
    if jcols is not None:
        case["jstypes"] = {nm: st for nm, (st, _) in jcols.items()}
        for nm, (st, a) in jcols.items():
            arrays[name + ".J." + nm] = np.ascontiguousarray(a, dtype=NPT[st])
        J = frame(jcols)
        J.key = "k"
    DT = frame(cols)
    try:
        if call is not None:
            CALLS[call](getattr(dt.time, part))
            raise AssertionError("no error")
        R = DT[query_args(dt, case, arrays, J, lambda p: dt.Frame(pylist(arrays[name + ".isel"], INT32),
                                                                  stype=dt.int32))]
    except Exception as e:                                      # noqa: BLE001
        case.update(error=type(e).__name__, message=str(e))
    else:
        case.update(nrows=int(R.nrows), names=list(R.names), out_stypes=[str(s) for s in R.stypes])
        for nm in R.names:
            arrays[name + ".out_" + nm] = to_np(R, nm)
    manifest.append(case)


def dates(n, na=0.1, lo=-10**5, hi=10**5):
    v = rng.integers(lo, hi, n).astype(np.int32)
    v[rng.random(n) < na] = NA[DATE32]
    return v


def times(n, na=0.1, lo=-10**18, hi=10**18):
    v = rng.integers(lo, hi, n, dtype=np.int64)
    v[rng.random(n) < na] = NA[TIME64]
    return v


# ---- every part at the type edges ----------------------------------------------------------------------------------
I32MIN, I32MAX = -2**31, 2**31 - 1
d_edges = np.array([I32MIN + 1, I32MIN + 2, I32MIN + 146096, I32MIN + 146097, I32MIN + 146098, I32MAX, I32MAX - 1,
                    I32MAX - 2, I32MAX - 3, I32MAX - 4, I32MAX - 719468, I32MAX - 719467, I32MAX - 719469,
                    I32MAX - 719468 - 146097, -719468, -719469, -719468 - 365, -719468 - 366, -719468 - 367,
                    -4, -3, -2, -1, 0, 1, 2, 59, 60, -25567, -25509, -25508, 11016, 11017, 47540, 47541, 47482,
                    -25203, -24837, NA[DATE32], -10**6, 10**6, -146097, 146097, 2932896, -2932897], np.int64)
d_edges = np.concatenate([d_edges, rng.integers(I32MIN + 1, I32MAX, 200), rng.integers(-800000, 800000, 200)])
t_edges = np.array([-2**63 + 1, -2**63 + 2, -2**63 + DAY - 2, -2**63 + DAY - 1, -2**63 + DAY, 2**63 - 1, 2**63 - 2,
                    -DAY, -2 * DAY, -DAY - 1, -DAY + 1, -1, 0, 1, DAY - 1, DAY, DAY + 1, -3600 * 10**9,
                    -3600 * 10**9 - 1, -60 * 10**9, -10**9, -10**9 - 1, -999999999, NA[TIME64],
                    11016 * DAY + 1, -25509 * DAY - 1, 47540 * DAY + DAY - 1,
                    -106751 * DAY, 106751 * DAY], dtype=object)
t_edges = np.concatenate([t_edges.astype(np.int64), rng.integers(-2**63 + 1, 2**63 - 1, 200, dtype=np.int64),
                          rng.integers(-10**18, 10**18, 200, dtype=np.int64)])
for p in PARTS:
    if PARTS.index(p) < 4:
        add(f"edge.date32.{p}", {"d": (DATE32, d_edges.astype(np.int32))}, part=p)
    add(f"edge.time64.{p}", {"d": (TIME64, t_edges)}, part=p)
add("edge.time64.parts", {"t": (TIME64, t_edges)}, j="parts")
add("empty.date32", {"d": (DATE32, np.zeros(0, np.int32))})
add("empty.time64", {"t": (TIME64, np.zeros(0, np.int64))}, j="parts")
add("allna.date32", {"d": (DATE32, np.full(5, NA[DATE32], np.int32))}, part="day_of_week")

# ---- query shapes ----------------------------------------------------------------------------------------------------
n = 60
base = {"d": (DATE32, dates(n)), "t": (TIME64, times(n)), "v": (FLOAT64, rng.standard_normal(n) * 10),
        "s": (INT32, rng.integers(0, 7, n).astype(np.int32))}
base["v"][1][::13] = np.nan
b = rng.integers(0, 2, n).astype(np.int8)
b[::11] = NA[BOOL]
based = dict(base, b=(BOOL, b))
for p in ("year", "month", "day_of_week"):
    for mode in ("none", "sort", "sortdesc", "by", "bysort"):
        add(f"{mode}.{p}", base, part=p, mode=mode)
for p in ("hour", "nanosecond"):
    for mode in ("none", "sortdesc", "by"):
        add(f"{mode}.{p}", base, part=p, mode=mode, j="list" if p == "hour" else "tuple")
add("sort_islice", base, mode="sort", i=["slice", [3, 50, 2]])
add("sort_int", base, mode="sort", i=["int", 4])
add("by_islice", base, mode="by", i=["slice", [1, None]], part="month")
add("by_int", base, mode="by", i=["int", -1], part="day")
for nm, i in (("islice", ["slice", [5, 45, 3]]), ("islice_neg", ["slice", [None, None, -2]]), ("iint", ["int", 7]),
              ("iint_neg", ["int", -3]), ("ibool", ["bool", "b"]),
              ("iframe", ["frame", None, np.array([3, NA[INT32], 0, 59, 17, 17, NA[INT32], 8], np.int32)]),
              ("ilist", ["list", [5, 0, 9, 9, 33]]), ("irange", ["range", [2, 58, 5]]),
              ("irange_neg", ["range", [50, 3, -4]])):
    add(f"{nm}.year", based, i=i)
    add(f"{nm}.list", based, i=i, j="list", part="day")
add("ibool_allfalse", dict(base, b=(BOOL, np.zeros(n, np.int8))), i=["bool", "b"])
for j in ("one", "list", "tuple", "dict", "plain", "cut", "qcut", "cumsum", "shift", "fillna", "cumcount", "ngroup"):
    add(f"j.{j}", base, part="month", j=j)
    if j not in ("cut",):
        add(f"j.{j}.by", base, part="day_of_week", j=j, mode="by")
add("j.all_dates", {"d": (DATE32, dates(20)), "t": (TIME64, times(20))}, j="all", part="day")
add("j.all_dates.bysort", {"d": (DATE32, dates(20)), "t": (TIME64, times(20)),
                           "s": (INT32, rng.integers(0, 3, 20).astype(np.int32))}, j="all", mode="by")
add("j.parts", base, j="parts")
add("j.parts.sort", base, j="parts", mode="sortdesc")
add("j.parts.by", base, j="parts", mode="by")

# join(J): the joined frame's columns
kx = rng.integers(0, 12, 80).astype(np.int32)
kx[::9] = NA[INT32]
jc = {"k": (INT32, np.arange(10, dtype=np.int32)), "d": (DATE32, dates(10))}
xj = {"d": (DATE32, dates(80)), "k": (INT32, kx), "v": (FLOAT64, rng.standard_normal(80))}
add("join.joincol", xj, mode="join", j="joincol", jcols=jc)
add("join.joinlist", xj, mode="join", j="joinlist", jcols=jc, part="day_of_week")
add("join.bypart", xj, mode="bypartjoin", j="bysum", jcols=jc, kpart="month")

# ---- time parts as by() / sort() keys -------------------------------------------------------------------------------
for kp in ("year", "month", "day_of_week"):
    for j in ("bysum", "bycount", "byall", "bykeys"):
        add(f"key.bypart.{kp}.{j}", base, mode="bypart", kpart=kp, j=j, part="hour")
    add(f"key.bypartneg.{kp}", base, mode="bypartneg", kpart=kp, j="bysum")
    add(f"key.bykpart.{kp}", base, mode="bykpart", kpart=kp, j="bysum")
    add(f"key.bypart_t.{kp}", base, mode="bypart_t", kpart=kp, j="bysum")
    add(f"key.bypartsort.{kp}", base, mode="bypartsort", kpart=kp, j="bykeys", part="minute")
for kp in ("year", "day_of_week", "hour", "second"):
    add(f"key.sortpart.{kp}", base, mode="sortpart", kpart=kp, j="bykeys", part="minute")
    add(f"key.sortpartneg.{kp}", base, mode="sortpartneg", kpart=kp, j="bykeys", part="nanosecond")
add("key.bypart.rowfn", base, mode="bypart", kpart="year", j="cumsum", part="day")
add("key.bypart.islice", base, mode="bypart", kpart="month", j="bysum", i=["slice", [0, 2]])
add("key.sortpart.iint", base, mode="sortpart", kpart="hour", j="bykeys", i=["int", 3], part="second")
ne = min(len(d_edges), len(t_edges))
add("key.bypart.edges", {"d": (DATE32, d_edges[:ne].astype(np.int32)), "t": (TIME64, t_edges[:ne]),
                         "v": (FLOAT64, rng.standard_normal(ne)), "s": (INT32, rng.integers(0, 3, ne).astype(np.int32))},
    mode="bypart", kpart="year", j="bysum")

# ---- errors ----------------------------------------------------------------------------------------------------------
for p in PARTS:
    add(f"err.stype.{p}", base, part=p, j="plain" if PARTS.index(p) < 4 else "one")   # clock parts of date32
    add(f"err.all.{p}", base, part=p, j="all")                                         # f[:] reaches v and s
for call in CALLS:
    for p in ("year", "day_of_week", "hour"):
        add(f"err.call.{call}.{p}", base, part=p, call=call)
add("err.key.bypart_clock", base, mode="bypart", kpart="hour", j="bysum")         # hour(f.d): date32
add("err.key.sortpart_clock", dict(base, t=(INT64, times(n))), mode="sortpart", kpart="hour", j="bykeys")

np.savez_compressed(os.path.join(HERE, "golden_v14.npz"), **arrays)
json.dump({"generator": "tests/golden/make_golden_v14.py", "datatable_version": dt.__version__, "cases": manifest},
          open(os.path.join(HERE, "golden_v14.json"), "w"), indent=0)
print(len(manifest), "cases,", sum(1 for c in manifest if "error" in c), "errors")
