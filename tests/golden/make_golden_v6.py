#!/usr/bin/env python
"""
Generates tests/golden/golden_v6.{npz,json} by running the *reference itself* (the unmodified build staged by
oracle/build_ref.sh) on dt.qcut:

    PYTHONPATH=oracle/_ref python tests/golden/make_golden_v6.py

    dt.qcut   Qcut_ColumnImpl (column/qcut.h:78-155), FExpr_Qcut (expr/fexpr_qcut.cc:64-158)

Every case stores the frame's columns (x, and where the query needs them y, ka, kb, s), the query (`mode`: none, by,
by2, bysort, sort, bykey = qcut of the by() column; `i`: a slice [start, stop, step] or an integer; `j`: one, list,
all = f[:], dict, dictlist, plain = [f.x, qcut(f.x)]; `q`: nquantiles) and what the reference returns: the output
names, stypes and columns.  The cases cover every accepted stype (bool, int8-64, float32/64, date32, time64), NA
first, in the middle and everywhere, -0.0 next to +0.0, +-inf, subnormals and several NaN bit patterns, constant
columns, one row and no rows, q = 1, 2 and 10 and q above the number of distinct values, V = 1 and 2 valid values,
one and two by() columns, by() + sort(), sort() alone, slices and integers for i, and the error texts.  The
reference cannot travel to the GPU box, so the vectors are committed.
"""
import json
import os

import numpy as np

import datatable as dt
from datatable import f, by, sort

HERE = os.path.dirname(os.path.abspath(__file__))
BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64 = 1, 2, 3, 4, 5, 6, 7, 17, 18
NPT = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
       FLOAT32: np.float32, FLOAT64: np.float64, DATE32: np.int32, TIME64: np.int64}
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
DTST = {BOOL: dt.bool8, INT8: dt.int8, INT16: dt.int16, INT32: dt.int32, INT64: dt.int64,
        FLOAT32: dt.float32, FLOAT64: dt.float64, DATE32: dt.int32, TIME64: dt.int64}
TAGS = {BOOL: "bool", INT8: "i8", INT16: "i16", INT32: "i32", INT64: "i64", FLOAT32: "f32", FLOAT64: "f64",
        DATE32: "date32", TIME64: "time64"}
arrays, manifest = {}, []
rng = np.random.default_rng(20261016)


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


def frame(cols):
    """cols: {name: (stype, array)}.  Float columns keep their bit patterns (NaN payloads, -0.0)."""
    DT = dt.Frame({nm: (a if st in (FLOAT32, FLOAT64) else pylist(a, st)) for nm, (st, a) in cols.items()},
                  stypes={nm: DTST[st] for nm, (st, _) in cols.items()})
    for nm, (st, _) in cols.items():
        if st == DATE32:
            DT[nm] = DT[:, dt.as_type(f[nm], dt.Type.date32)]
        elif st == TIME64:
            DT[nm] = DT[:, dt.as_type(f[nm], dt.Type.time64)]
    return DT


def query(DT, mode, i, j, q):
    if j == "one":
        J = dt.qcut(f.x, nquantiles=q)
    elif j == "list":
        J = dt.qcut([f.x, f.y], nquantiles=q)
    elif j == "tuple":
        J = dt.qcut((f.x, f.y), nquantiles=q)
    elif j == "all":
        J = dt.qcut(f[:], nquantiles=q)
    elif j == "dict":
        J = {"q": dt.qcut(f.x, nquantiles=q)}
    elif j == "dictlist":
        J = {"q": dt.qcut([f.x, f.y], nquantiles=q)}
    elif j == "plain":
        J = [f.x, dt.qcut(f.x, nquantiles=q)]
    else:                                                         # bykey: qcut of the by() column
        J = dt.qcut(f.ka, nquantiles=q)
    rows = slice(None) if i is None else (i if isinstance(i, int) else slice(*i))
    mods = {"none": (), "by": (by(f.ka),), "by2": (by(f.ka, f.kb),), "bysort": (by(f.ka), sort(f.s)),
            "sort": (sort(f.s),), "sortdesc": (sort(-f.s),)}[mode]
    return DT[(rows, J) + mods]


def add(name, cols, mode="none", i=None, j="one", q=None):
    DT = frame(cols)
    case = {"name": name, "mode": mode, "i": i, "j": j, "q": q, "stypes": {nm: st for nm, (st, _) in cols.items()}}
    try:
        R = query(DT, mode, i, j, q)
    except Exception as e:                                      # noqa: BLE001
        case.update(error=type(e).__name__, message=str(e))
    else:
        case.update(nrows=int(R.nrows), names=list(R.names), out_stypes=[str(s) for s in R.stypes])
        for nm in R.names:
            arrays[name + ".out_" + nm] = to_np(R, nm)
    for nm, (st, a) in cols.items():
        arrays[name + "." + nm] = np.ascontiguousarray(a, dtype=NPT[st])
    manifest.append(case)


def keys(n, ng, na=0.05):
    k = rng.integers(0, ng, n).astype(np.int32)
    k[rng.random(n) < na] = NA[INT32]
    return k


def values(st, n, na=0.1, distinct=12):
    if st == BOOL:
        v = rng.integers(0, 2, n).astype(np.int8)
    elif st in (FLOAT32, FLOAT64):
        v = rng.choice(np.linspace(-3, 3, distinct), n).astype(NPT[st])
    else:
        v = rng.integers(-distinct // 2, distinct // 2 + 1, n).astype(NPT[st])
        if st in (INT64, TIME64):
            v = v * 10**12 + 7
    mask = rng.random(n) < na
    if st in (FLOAT32, FLOAT64):
        v[mask] = np.nan
    else:
        v[mask] = NA[st]
    return v


ALL = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64)
n = 200
for st in ALL:
    tag = TAGS[st]
    add(f"none.{tag}", {"x": (st, values(st, n))})
    add(f"none_q3.{tag}", {"x": (st, values(st, n))}, q=3)
    add(f"by.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 9))})
    add(f"by2.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 3)), "kb": (INT32, keys(n, 4))}, mode="by2")
    add(f"bysort.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 5)),
                          "s": (INT32, rng.integers(-9, 10, n).astype(np.int32))}, mode="bysort")
    add(f"sort.{tag}", {"x": (st, values(st, n)), "s": (INT32, keys(n, 20))}, mode="sort")
    add(f"islice_by.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 7))}, mode="by", i=[1, None, 2])
    add(f"islice.{tag}", {"x": (st, values(st, n))}, i=[3, 150, 2])
    add(f"bykey.{tag}", {"x": (st, values(st, 40)), "ka": (INT32, keys(40, 4))}, mode="by", j="bykey")

# NA first, NA in the middle, all NA, NA only in some groups
for st in (INT32, FLOAT64):
    tag = TAGS[st]
    na = np.nan if st == FLOAT64 else NA[st]
    add(f"nafirst.{tag}", {"x": (st, np.array([na, 1, 2, 3, 2, 1], NPT[st]))})
    add(f"namiddle.{tag}", {"x": (st, np.array([4, 1, na, na, 2, 5, 1], NPT[st]))})
    add(f"allna.{tag}", {"x": (st, np.full(6, na, NPT[st]))})
    add(f"allna_by.{tag}", {"x": (st, np.array([na, 1, na, na, 3, na], NPT[st])),
                            "ka": (INT32, np.array([0, 1, 0, 2, 1, 2], np.int32))}, mode="by")

# +-0.0, +-inf, subnormals, NaN bit patterns
for st in (FLOAT32, FLOAT64):
    tag, T = TAGS[st], NPT[st]
    tiny = np.finfo(T).smallest_subnormal
    nan2 = np.array([0x7FF0000000000123 if st == FLOAT64 else 0x7F800123], dtype=np.uint64 if st == FLOAT64 else np.uint32).view(T)[0]
    nneg = -np.array([np.nan], T)[0]
    add(f"zeros.{tag}", {"x": (st, np.array([0.5, np.nan, -0.0, 0.0, 3.0, 0.0, 7.0], T))})
    add(f"zeros_by.{tag}", {"x": (st, np.array([0.5, np.nan, -0.0, 0.0, 3.0, 0.0, 7.0], T)),
                            "ka": (INT32, np.array([2, 1, 2, 1, 2, 1, 1], np.int32))}, mode="by")
    add(f"special.{tag}", {"x": (st, np.array([np.inf, -np.inf, tiny, -tiny, 0.0, -0.0, np.nan, nan2, nneg, 1.0,
                                                -np.inf, tiny, np.finfo(T).max, -np.finfo(T).max], T))})
    add(f"special_q2.{tag}", {"x": (st, np.array([np.inf, nan2, -0.0, tiny, nneg, 0.0, -np.inf], T))}, q=2)
    v = rng.choice(np.array([0.0, -0.0, np.nan, nan2, nneg, 1.5], T), 300)
    add(f"zeros_dense_by.{tag}", {"x": (st, v), "ka": (INT32, keys(300, 6))}, mode="by")

# constant columns, one row, no rows; q = 1, 2, 10 and above the number of distinct values; V = 1 and 2
for st in (INT32, FLOAT64):
    tag = TAGS[st]
    na = np.nan if st == FLOAT64 else NA[st]
    add(f"const.{tag}", {"x": (st, np.full(5, 3, NPT[st]))})
    add(f"const_na.{tag}", {"x": (st, np.array([3, na, 3, 3], NPT[st]))})       # V = 1 with an NA group
    add(f"v2.{tag}", {"x": (st, np.array([3, 8, 3, 8, 8], NPT[st]))})
    add(f"v2_na.{tag}", {"x": (st, np.array([na, 8, 3, na, 8], NPT[st]))})
    add(f"onerow.{tag}", {"x": (st, np.array([5], NPT[st]))})
    add(f"onerow_na.{tag}", {"x": (st, np.array([na], NPT[st]))})
    add(f"empty.{tag}", {"x": (st, np.zeros(0, NPT[st]))})
    for q in (1, 2, 10, 50, 2**31 - 1):
        add(f"q{q}.{tag}", {"x": (st, values(st, 60, distinct=6))}, q=q)
        add(f"q{q}_by.{tag}", {"x": (st, values(st, 60, distinct=6)), "ka": (INT32, keys(60, 3))}, mode="by", q=q)

# many distinct values: bins spread over 0 .. q-1
add("distinct.f64", {"x": (FLOAT64, rng.standard_normal(500))}, q=7)
add("distinct_by.i64", {"x": (INT64, rng.integers(-2**62, 2**62, 500, dtype=np.int64)), "ka": (INT32, keys(500, 4))},
    mode="by", q=100)

# j forms
x, y, g = values(FLOAT64, 50), values(INT32, 50), keys(50, 3)
xy = {"x": (FLOAT64, x), "y": (INT32, y)}
xyg = {"x": (FLOAT64, x), "y": (INT32, y), "ka": (INT32, g)}
add("j.list", xy, j="list", q=[2, 3])
add("j.tuple", xy, j="tuple", q=(4, 5))
add("j.list_default", xy, j="list")
add("j.list_by", xyg, mode="by", j="list", q=[3, 6])
add("j.all", xyg, j="all")
add("j.all_by", xyg, mode="by", j="all", q=[2, 3])
add("j.dict", xyg, mode="by", j="dict", q=4)
add("j.dict_none", xy, j="dict")
add("j.dictlist", xy, j="dictlist")
add("j.dictlist_by", xyg, mode="by", j="dictlist", q=[5, 2])
add("j.plain_by", xyg, mode="by", j="plain", q=3)
add("j.plain", xy, j="plain")
s = {"x": (FLOAT64, x), "s": (INT32, keys(50, 8))}
add("sortdesc.f64", s, mode="sortdesc")
add("sort_islice.f64", s, mode="sort", i=[1, None, 2])
add("sort_int.f64", s, mode="sort", i=3)
add("by_int.f64", xyg, mode="by", i=0)
add("by_int_neg.f64", xyg, mode="by", i=-1)
add("none_int.f64", xy, i=7)
add("by2_bykey.i32", {"x": (INT32, y), "ka": (INT32, g), "kb": (INT32, keys(50, 2))}, mode="by2", j="bykey")

# errors (ValueError / TypeError texts as Python sees them).  Raised late in a long session, an error can crash the
# reference's process (a segmentation fault inside its error path), so each is taken from a fresh interpreter.
import subprocess  # noqa: E402
import sys  # noqa: E402


def add_error(name, j, q):
    r = subprocess.run([sys.executable, "-c", f"""
import datatable as dt
from datatable import f
DT = dt.Frame(x=[1.5, None, 0.0], y=[1, 2, 3])
J = dt.qcut([f.x, f.y] if {j == "list"} else f.x, nquantiles={q!r})
try:
    DT[:, J]
except Exception as e:
    print(type(e).__name__); print(e)
"""], capture_output=True, text=True, check=True).stdout.strip().split("\n", 1)
    manifest.append({"name": name, "mode": "none", "i": None, "j": j, "q": q, "stypes": {"x": FLOAT64, "y": INT32},
                     "error": r[0], "message": r[1]})
    arrays[name + ".x"] = np.array([1.5, np.nan, 0.0])
    arrays[name + ".y"] = np.array([1, 2, 3], np.int32)


add_error("err.zero", "one", 0)
add_error("err.negative", "one", -3)
add_error("err.list_len", "list", [2])
add_error("err.list_elem", "list", [2, 0])
add_error("err.too_large", "one", 2**31)
add_error("err.float", "one", 2.5)
add_error("err.bool", "one", True)

np.savez_compressed(os.path.join(HERE, "golden_v6.npz"), **arrays)
json.dump({"generator": "tests/golden/make_golden_v6.py", "datatable_version": dt.__version__, "cases": manifest},
          open(os.path.join(HERE, "golden_v6.json"), "w"), indent=0)
print(len(manifest), "cases")
