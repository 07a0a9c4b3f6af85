#!/usr/bin/env python
"""
Generates tests/golden/golden_v5.{npz,json} by running the *reference itself* (the unmodified build staged by
oracle/build_ref.sh) on the per-group product:

    PYTHONPATH=oracle/_ref python tests/golden/make_golden_v5.py

    dt.prod   SumProd_ColumnImpl<T, false, ..>   (column/sumprod.h:34-59, expr/fexpr_sumprod.cc:47-67)
    dt.cov / dt.corr                             (expr/head_reduce_binary.cc:114-259)

cov / corr cases ("op": "cov" | "corr") store the columns x, y and the keys, and what the reference returns for
DT[i, {"r": dt.cov(f.x, f.y)}, by(...), sort(...)]: every stype pair, NA in x only / y only / both, groups with 0, 1
and 2 valid pairs, constant x and constant y, offsets of 1e8 plus small noise, one and two by() columns, by() +
sort(), no by(), an `i` slice, a by() column as an argument (an all-NA result), list broadcasting (unnamed columns
C0, C1, ...) and the error text of lists that do not broadcast.

Every case stores its columns and what the reference returns for DT[i, {"p": dt.prod(f.v)}, by(...), sort(...)]:
the output names, the key columns and the product.  The cases cover every input stype, NA rows, groups with 0, 1 and
2 valid rows, all-NA groups, int64 wrap-around, +-inf, +-0.0 and subnormals, zeros times infinities, one and two
by() columns, by() + sort(), no by(), a slice for i, and a by() column as the argument.  Cases tagged `deviation`
are those where the reference's sequential product overflows or underflows part-way although the exact product is
in range (the engine returns the in-range value, include/dtb200.h at dtb_reduce).  The reference cannot travel to
the GPU box, so the vectors are committed.
"""
import json
import os

import numpy as np

import datatable as dt
from datatable import f, by, sort

HERE = os.path.dirname(os.path.abspath(__file__))
BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64 = 1, 2, 3, 4, 5, 6, 7
NPT = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
       FLOAT32: np.float32, FLOAT64: np.float64}
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63}
DTST = {BOOL: dt.bool8, INT8: dt.int8, INT16: dt.int16, INT32: dt.int32, INT64: dt.int64,
        FLOAT32: dt.float32, FLOAT64: dt.float64}
arrays, manifest = {}, []
rng = np.random.default_rng(20261015)


def pylist(a, st):
    if st in (FLOAT32, FLOAT64):
        return [None if np.isnan(x) else float(x) for x in a.tolist()]
    return [None if x == NA[st] else (bool(x) if st == BOOL else int(x)) for x in a.tolist()]


def to_np(fr, name):
    lst = fr[:, name].to_list()[0]
    st = fr[:, name].stypes[0]
    if st in (dt.float32, dt.float64):
        return np.array([np.nan if x is None else x for x in lst], dtype=np.float32 if st == dt.float32 else np.float64)
    npdt = {dt.bool8: np.int8, dt.int8: np.int8, dt.int16: np.int16, dt.int32: np.int32, dt.int64: np.int64}[st]
    na = -128 if st == dt.bool8 else np.iinfo(npdt).min
    return np.array([na if x is None else int(x) for x in lst], dtype=npdt)


def add(name, st, v, k1=None, k2=None, s=None, mode="by", i=None, deviation=False):
    """mode: by = by(k1); by2 = by(k1, k2); bysort = by(k1), sort(s); none = no by(); bykey = prod(k1) by(k1)"""
    n = len(v)
    if st == BOOL:
        v = np.where(v == NA[BOOL], NA[BOOL], v != 0).astype(np.int8)
    cols = {"v": pylist(v, st)}
    stypes = {"v": DTST[st]}
    for nm, c in (("k1", k1), ("k2", k2), ("s", s)):
        if c is not None:
            cols[nm] = pylist(c, INT32)
            stypes[nm] = dt.int32
    DT = dt.Frame(cols, stypes=stypes) if n else dt.Frame({nm: [] for nm in cols}, stypes=stypes)
    rows = slice(None) if i is None else slice(*i)
    if mode == "by":
        R = DT[rows, {"p": dt.prod(f.v)}, by(f.k1)]
    elif mode == "by2":
        R = DT[rows, {"p": dt.prod(f.v)}, by(f.k1, f.k2)]
    elif mode == "bysort":
        R = DT[rows, {"p": dt.prod(f.v)}, by(f.k1), sort(f.s)]
    elif mode == "none":
        R = DT[rows, {"p": dt.prod(f.v)}]
    else:
        R = DT[rows, {"p": dt.prod(f.k1)}, by(f.k1)]
    case = {"name": name, "op": "prod", "stype": st, "mode": mode, "i": i, "deviation": deviation, "nrows": int(R.nrows),
            "names": list(R.names), "out_stype": str(R.stypes[-1])}
    arrays[name + ".v"] = np.ascontiguousarray(v, dtype=NPT[st])
    for nm, c in (("k1", k1), ("k2", k2), ("s", s)):
        if c is not None:
            arrays[name + "." + nm] = np.ascontiguousarray(c, dtype=np.int32)
    for nm in R.names:
        arrays[name + ".out_" + nm] = to_np(R, nm)
    manifest.append(case)


def keys(n, ng, na=0.05):
    k = rng.integers(0, ng, n).astype(np.int32)
    k[rng.random(n) < na] = NA[INT32]
    return k


def values(st, n, na=0.1):
    if st == BOOL:
        v = rng.integers(0, 2, n).astype(np.int8)
    elif st in (INT8, INT16):
        v = rng.integers(-3, 4, n).astype(NPT[st])
    elif st == INT32:
        v = rng.integers(-50, 51, n).astype(np.int32)
    elif st == INT64:
        v = rng.integers(-2**40, 2**40, n, dtype=np.int64)              # products wrap modulo 2^64
    else:
        v = (rng.choice([-1.0, 1.0], n) * np.exp2(rng.uniform(-4, 4, n))).astype(NPT[st])
    mask = rng.random(n) < na
    if st in (FLOAT32, FLOAT64):
        v[mask] = np.nan
    else:
        v[mask] = NA[st]
    return v


ALL = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
for st in ALL:
    tag = {BOOL: "bool", INT8: "i8", INT16: "i16", INT32: "i32", INT64: "i64", FLOAT32: "f32", FLOAT64: "f64"}[st]
    n = 300
    add(f"rand.{tag}", st, values(st, n), keys(n, 12))
    add(f"by2.{tag}", st, values(st, n), keys(n, 4), keys(n, 5), mode="by2")
    add(f"bysort.{tag}", st, values(st, n), keys(n, 6), s=rng.integers(-9, 10, n).astype(np.int32), mode="bysort")
    add(f"none.{tag}", st, values(st, n), mode="none")
    add(f"islice.{tag}", st, values(st, n), keys(n, 7), i=[1, None, 2])
    # groups with 0, 1 and 2 valid rows, and an all-NA group: k = 0 .. 3
    na = np.nan if st in (FLOAT32, FLOAT64) else NA[st]
    v = np.array([na, na, 3, na, 1, 1, na, na], dtype=NPT[st])
    add(f"fewvalid.{tag}", st, v, np.array([0, 0, 1, 1, 2, 2, 3, 3], np.int32))
    add(f"allna.{tag}", st, np.full(5, na, dtype=NPT[st]), np.zeros(5, np.int32))
    add(f"bykey.{tag}", st, values(st, 40), keys(40, 4), mode="bykey")
    add(f"empty.{tag}", st, np.zeros(0, NPT[st]), np.zeros(0, np.int32))

# int64 wrap-around: products far beyond 2^64, including INT64_MAX and -INT64_MAX
v = np.array([2**62, 4, -3, 2**63 - 1, 2**63 - 1, -(2**63 - 1), 3**39, 3**39, 7, NA[INT64]], dtype=np.int64)
add("wrap.i64", INT64, v, np.array([0, 0, 0, 1, 1, 1, 2, 2, 2, 2], np.int32))
add("wrap.i32", INT32, np.array([2**31 - 1] * 6 + [-2**31 + 1] * 5, np.int32), np.array([0] * 6 + [1] * 5, np.int32))

# +-inf, +-0.0, subnormals, zeros times infinities (NA), in float32 and float64
for st, tag in ((FLOAT32, "f32"), (FLOAT64, "f64")):
    T = NPT[st]
    tiny = np.finfo(T).smallest_subnormal
    groups = [
        [0.0, 2.0, 3.0], [-0.0, 2.0], [-0.0, -1.0], [np.inf, 2.0], [-np.inf, 0.5], [np.inf, -np.inf],
        [0.0, np.inf], [np.inf, 1.0, -0.0], [tiny, 2.0], [tiny, tiny], [tiny, 2.0**1000 if st == FLOAT64 else 2.0**100],
        [np.nan, 0.0, np.nan], [-2.0, -2.0, -2.0], [1.5, np.nan, -1.5, 4.0],
    ]
    v = np.array([x for g in groups for x in g], dtype=T)
    k = np.array([i for i, g in enumerate(groups) for _ in g], dtype=np.int32)
    add(f"special.{tag}", st, v, k)

# deviation cases: the exact product is in range, the sequential one overflows / underflows part-way
for st, tag, big in ((FLOAT64, "f64", 1e200), (FLOAT32, "f32", 1e30)):
    T = NPT[st]
    groups = [[big, big, 1 / big, 1 / big],               # reference: inf
              [1 / big, 1 / big, big, big],               # reference: 0
              [big, big, 1 / big, 1 / big, 0.0],          # reference: inf * 0 = NaN -> NA; exact: 0
              [-big, big, 1 / big, -1 / big, 3.0]]        # reference: -inf ... ; exact: 3
    v = np.array([x for g in groups for x in g], dtype=T)
    k = np.array([i for i, g in enumerate(groups) for _ in g], dtype=np.int32)
    add(f"deviation.{tag}", st, v, k, deviation=True)



# ---- cov / corr ----------------------------------------------------------------------------------------------
def add2(name, op, sx, x, sy, y, k1=None, k2=None, s=None, mode="by", i=None, bcast=False):
    if sx == BOOL:
        x = np.where(x == NA[BOOL], NA[BOOL], x != 0).astype(np.int8)
    if sy == BOOL:
        y = np.where(y == NA[BOOL], NA[BOOL], y != 0).astype(np.int8)
    cols, stypes = {"x": pylist(x, sx), "y": pylist(y, sy)}, {"x": DTST[sx], "y": DTST[sy]}
    for nm, c in (("k1", k1), ("k2", k2), ("s", s)):
        if c is not None:
            cols[nm] = pylist(c, INT32)
            stypes[nm] = dt.int32
    DT = dt.Frame(cols, stypes=stypes)
    fn = dt.cov if op == "cov" else dt.corr
    rows = slice(None) if i is None else slice(*i)
    j = [fn([f.x, f.y], f.y)] if bcast else {"r": fn(f.x, f.y)}
    if mode == "by":
        R = DT[rows, j, by(f.k1)]
    elif mode == "by2":
        R = DT[rows, j, by(f.k1, f.k2)]
    elif mode == "bysort":
        R = DT[rows, j, by(f.k1), sort(f.s)]
    elif mode == "none":
        R = DT[rows, j]
    else:                                                   # bykey: x is the by() column
        R = DT[rows, {"r": fn(f.k1, f.y)}, by(f.k1)]
    manifest.append({"name": name, "op": op, "stype": sx, "stype2": sy, "mode": mode, "i": i, "bcast": bcast,
                     "deviation": False, "nrows": int(R.nrows), "names": list(R.names),
                     "out_stype": str(R.stypes[-1])})
    arrays[name + ".x"] = np.ascontiguousarray(x, dtype=NPT[sx])
    arrays[name + ".y"] = np.ascontiguousarray(y, dtype=NPT[sy])
    for nm, c in (("k1", k1), ("k2", k2), ("s", s)):
        if c is not None:
            arrays[name + "." + nm] = np.ascontiguousarray(c, dtype=np.int32)
    for nm in R.names:
        arrays[name + ".out_" + nm] = to_np(R, nm)


def values2(st, n, na=0.1):
    if st in (FLOAT32, FLOAT64):
        v = np.round(rng.standard_normal(n) * 10, 3).astype(NPT[st])
        v[rng.random(n) < na] = np.nan
        return v
    return values(st, n, na)


TAGS = {BOOL: "bool", INT8: "i8", INT16: "i16", INT32: "i32", INT64: "i64", FLOAT32: "f32", FLOAT64: "f64"}
for op in ("cov", "corr"):
    for sx in ALL:
        for sy in ALL:
            n = 200
            y = values2(sy, n)
            if sy == INT64:
                y = rng.integers(-1000, 1000, n).astype(np.int64); y[rng.random(n) < 0.1] = NA[INT64]
            x = values2(sx, n)
            if sx == INT64:
                x = rng.integers(-1000, 1000, n).astype(np.int64); x[rng.random(n) < 0.1] = NA[INT64]
            add2(f"{op}.{TAGS[sx]}.{TAGS[sy]}", op, sx, x, sy, y, keys(n, 6))
    for sx, sy in ((FLOAT64, FLOAT64), (INT32, FLOAT32), (FLOAT32, FLOAT32)):
        tag = f"{TAGS[sx]}.{TAGS[sy]}"
        n = 300
        add2(f"{op}.by2.{tag}", op, sx, values2(sx, n), sy, values2(sy, n), keys(n, 3), keys(n, 4), mode="by2")
        add2(f"{op}.bysort.{tag}", op, sx, values2(sx, n), sy, values2(sy, n), keys(n, 5),
             s=rng.integers(-9, 10, n).astype(np.int32), mode="bysort")
        add2(f"{op}.none.{tag}", op, sx, values2(sx, n), sy, values2(sy, n), mode="none")
        add2(f"{op}.islice.{tag}", op, sx, values2(sx, n), sy, values2(sy, n), keys(n, 7), i=[1, None, 2])
        add2(f"{op}.bykey.{tag}", op, sx, values2(sx, 40), sy, values2(sy, 40), keys(40, 4), mode="bykey")
        add2(f"{op}.bcast.{tag}", op, sx, values2(sx, n), sy, values2(sy, n), keys(n, 5), bcast=True)
    # NA in x only, in y only, in both; groups with 0, 1 and 2 valid pairs; constant x / constant y; all-NA group
    N = np.nan
    groups = [([N, 1.0, 2.0], [1.0, N, 3.0]),          # no valid pair (NA in x, NA in y)
              ([N, N, 2.0], [N, 5.0, 3.0]),            # one valid pair
              ([1.0, 2.0, N], [3.0, 5.0, 7.0]),        # two valid pairs
              ([0.1, 0.1, 0.1, 0.1], [1.0, 2.0, 4.0, 8.0]),   # constant x: cov 0, corr NA
              ([1.0, 2.5, -3.0, 7.0], [0.3, 0.3, 0.3, 0.3]),  # constant y
              ([N, N], [N, N]),                        # all NA
              ([1.0, 2.0, 3.0, 4.0, 5.0], [5.0, 4.0, 3.5, 2.0, 1.0])]
    x = np.array([a for g in groups for a in g[0]])
    y = np.array([b for g in groups for b in g[1]])
    k = np.array([i for i, g in enumerate(groups) for _ in g[0]], dtype=np.int32)
    add2(f"{op}.napattern.f64", op, FLOAT64, x, FLOAT64, y, k)
    add2(f"{op}.napattern.f32", op, FLOAT32, x.astype(np.float32), FLOAT32, y.astype(np.float32), k)
    # offsets of 1e8 plus small noise: the one-pass formula would cancel away every digit
    n = 400
    x = 1e8 + np.round(rng.standard_normal(n), 4)
    y = -3e8 + 0.5 * (x - 1e8) + np.round(rng.standard_normal(n) * 0.1, 4)
    add2(f"{op}.offset.f64", op, FLOAT64, x, FLOAT64, y, keys(n, 4, na=0))

# a list that does not broadcast: the reference's ValueError text.  Raised late in a long session, this error crashed
# the reference's process (a segmentation fault inside its error path), so it is taken from a fresh interpreter.
import subprocess  # noqa: E402
import sys  # noqa: E402
broadcast_error = subprocess.run([sys.executable, "-c", """
import datatable as dt
from datatable import f
DT = dt.Frame(a=[1.0, 2.0], b=[2.0, 1.0], c=[0.5, 1.5])
try:
    DT[:, dt.corr([f.a, f.b], [f.a, f.b, f.c])]
except ValueError as e:
    print(e)
"""], capture_output=True, text=True, check=True).stdout.strip()

np.savez_compressed(os.path.join(HERE, "golden_v5.npz"), **arrays)
json.dump({"generator": "tests/golden/make_golden_v5.py", "datatable_version": dt.__version__,
           "broadcast_error": broadcast_error, "cases": manifest},
          open(os.path.join(HERE, "golden_v5.json"), "w"), indent=0)
print(len(manifest), "cases")
