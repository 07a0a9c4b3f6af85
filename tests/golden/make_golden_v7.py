#!/usr/bin/env python
"""
Generates tests/golden/golden_v7.{npz,json} by running the *reference itself* (the unmodified build staged by
oracle/build_ref.sh) on the cumulative functions:

    PYTHONPATH=oracle/_ref python tests/golden/make_golden_v7.py

    dt.cumsum / dt.cumprod   CumSumProd_ColumnImpl (column/cumsumprod.h), FExpr_CumSumProd (expr/fexpr_cumsumprod.cc)
    dt.cummin / dt.cummax    CumMinMax_ColumnImpl (column/cumminmax.h), FExpr_CumMinMax (expr/fexpr_cumminmax.cc)

Every case stores the frame's columns (x, and where the query needs them y, ka, kb, s), the query (`fn`: cumsum,
cumprod, cummin or cummax; `rev`: reverse=; `mode`: none, by, by2, bysort, sort, sortdesc; `i`: a slice
[start, stop, step] or an integer; `j`: one, list, tuple, all = f[:], dict, dictlist, plain = [f.x, fn(f.x)],
withqcut = [fn(f.x), qcut(f.x)], bykey = fn of the by() column) and what the reference returns: the output names,
stypes and columns.  The cases cover every accepted stype, NA first, in the middle, last and everywhere, a group of
one row and no rows, int64 wrap-around, +-inf, inf and -inf in one group, 0 and inf in one group, subnormals, runs of
-0.0 and +0.0, every query shape and j form, the inputs of the reference's own tests (tests/dt/test-cumsum.py,
test-cumprod.py, test-cumminmax.py) and the error texts.  The reference cannot travel to the GPU box, so the vectors
are committed.
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
FNS = {"cumsum": dt.cumsum, "cumprod": dt.cumprod, "cummin": dt.cummin, "cummax": dt.cummax}
arrays, manifest = {}, []
rng = np.random.default_rng(20261017)


def pylist(a, st):
    if st in (FLOAT32, FLOAT64):
        return [None if np.isnan(x) else float(x) for x in a.tolist()]
    return [None if x == NA[st] else (bool(x) if st == BOOL else int(x)) for x in a.tolist()]


def to_np(fr, name):
    """A result column as its stype's storage: float bit patterns kept (-0.0), NA as the stype's sentinel."""
    col = fr[:, name]
    st = col.stypes[0]
    if st in (dt.float32, dt.float64):
        if col.nrows == 0:                                      # the reference's to_numpy() crashes on 0 rows
            return np.zeros(0, np.float32 if st == dt.float32 else np.float64)
        return col.to_numpy().reshape(-1).astype(np.float32 if st == dt.float32 else np.float64)
    if st in (dt.stype.date32, dt.stype.time64):
        st = dt.int32 if st == dt.stype.date32 else dt.int64
        col = col[:, dt.as_type(f[0], st)]
    lst = col.to_list()[0]
    npdt = {dt.bool8: np.int8, dt.int8: np.int8, dt.int16: np.int16, dt.int32: np.int32, dt.int64: np.int64}[st]
    na = -128 if st == dt.bool8 else np.iinfo(npdt).min
    return np.array([na if x is None else int(x) for x in lst], dtype=npdt)


def frame(cols):
    """cols: {name: (stype, array)}.  Float columns keep their bit patterns (-0.0)."""
    DT = dt.Frame({nm: (a if st in (FLOAT32, FLOAT64) else pylist(a, st)) for nm, (st, a) in cols.items()},
                  stypes={nm: DTST[st] for nm, (st, _) in cols.items()})
    for nm, (st, _) in cols.items():
        if st == DATE32:
            DT[nm] = DT[:, dt.as_type(f[nm], dt.Type.date32)]
        elif st == TIME64:
            DT[nm] = DT[:, dt.as_type(f[nm], dt.Type.time64)]
    return DT


def query(DT, fn, rev, mode, i, j):
    F = FNS[fn]
    if j == "one":
        J = F(f.x, reverse=rev)
    elif j == "list":
        J = F([f.x, f.y], reverse=rev)
    elif j == "tuple":
        J = F((f.x, f.y), reverse=rev)
    elif j == "all":
        J = F(f[:], reverse=rev)
    elif j == "dict":
        J = {"c": F(f.x, reverse=rev)}
    elif j == "dictlist":
        J = {"c": F([f.x, f.y], reverse=rev)}
    elif j == "plain":
        J = [f.x, F(f.x, reverse=rev)]
    elif j == "withqcut":
        J = [F(f.x, reverse=rev), dt.qcut(f.y)]
    else:                                                         # bykey: fn of the by() column
        J = F(f.ka, reverse=rev)
    rows = slice(None) if i is None else (i if isinstance(i, int) else slice(*i))
    mods = {"none": (), "by": (by(f.ka),), "by2": (by(f.ka, f.kb),), "bysort": (by(f.ka), sort(f.s)),
            "sort": (sort(f.s),), "sortdesc": (sort(-f.s),)}[mode]
    return DT[(rows, J) + mods]


def add(name, cols, fn, rev=False, mode="none", i=None, j="one"):
    DT = frame(cols)
    case = {"name": name, "fn": fn, "rev": rev, "mode": mode, "i": i, "j": j,
            "stypes": {nm: st for nm, (st, _) in cols.items()}}
    R = query(DT, fn, rev, mode, i, j)
    case.update(nrows=int(R.nrows), names=list(R.names), out_stypes=[str(s) for s in R.stypes])
    for nm in R.names:
        arrays[name + ".out_" + nm] = to_np(R, nm)
    for nm, (st, a) in cols.items():
        arrays[name + "." + nm] = np.ascontiguousarray(a, dtype=NPT[st])
    manifest.append(case)


def add_all(name, cols, fns=tuple(FNS), revs=(False, True), **kw):
    for fn in fns:
        for rev in revs:
            add(f"{name}.{fn}{'.rev' if rev else ''}", cols, fn, rev, **kw)


def keys(n, ng, na=0.05):
    k = rng.integers(0, ng, n).astype(np.int32)
    k[rng.random(n) < na] = NA[INT32]
    return k


def values(st, n, na=0.1):
    if st == BOOL:
        v = rng.integers(0, 2, n).astype(np.int8)
    elif st in (FLOAT32, FLOAT64):
        v = rng.choice(np.linspace(-3, 3, 13), n).astype(NPT[st])
    else:
        v = rng.integers(-6, 7, n).astype(NPT[st])
        if st in (INT64, TIME64):
            v = v * 10**12 + 7
    mask = rng.random(n) < na
    if st in (FLOAT32, FLOAT64):
        v[mask] = np.nan
    else:
        v[mask] = NA[st]
    return v


NUMERIC = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
n = 60
# every op x reverse over every accepted stype, without and with by()
for st in NUMERIC + (DATE32, TIME64):
    tag = TAGS[st]
    fns = tuple(FNS) if st in NUMERIC else ("cummin", "cummax")
    add_all(f"none.{tag}", {"x": (st, values(st, n))}, fns=fns)
    add_all(f"by.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 5))}, fns=fns, mode="by")

# the query shapes, each op in both directions
for st in (INT32, FLOAT64):
    tag = TAGS[st]
    add_all(f"by2.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 3)), "kb": (INT32, keys(n, 3))}, mode="by2")
    add_all(f"bysort.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 4)),
                              "s": (INT32, rng.integers(-9, 10, n).astype(np.int32))}, mode="bysort")
    add_all(f"sort.{tag}", {"x": (st, values(st, n)), "s": (INT32, keys(n, 20))}, mode="sort")
    add_all(f"sortdesc.{tag}", {"x": (st, values(st, n)), "s": (INT32, keys(n, 20))}, mode="sortdesc")
    add_all(f"islice_by.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 5))}, mode="by", i=[1, None, 2])
    add_all(f"islice.{tag}", {"x": (st, values(st, n))}, i=[3, 50, 2])
    add_all(f"int_by.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 5))}, mode="by", i=-1)
    add_all(f"int.{tag}", {"x": (st, values(st, n))}, i=7)
    add_all(f"bykey.{tag}", {"x": (st, values(st, 30)), "ka": (INT32, keys(30, 4))}, mode="by", j="bykey")

# NA first, in the middle, last, everywhere; NA only in some groups; one row; no rows
for st in (INT32, FLOAT64):
    tag = TAGS[st]
    na = np.nan if st == FLOAT64 else NA[st]
    add_all(f"nafirst.{tag}", {"x": (st, np.array([na, na, 1, 2, 3, 2, 1], NPT[st]))})
    add_all(f"namiddle.{tag}", {"x": (st, np.array([4, 1, na, na, 2, 5, 1], NPT[st]))})
    add_all(f"nalast.{tag}", {"x": (st, np.array([4, 1, 2, 5, na, na], NPT[st]))})
    add_all(f"allna.{tag}", {"x": (st, np.full(6, na, NPT[st]))})
    add_all(f"na_by.{tag}", {"x": (st, np.array([na, 1, na, na, 3, na, 2], NPT[st])),
                             "ka": (INT32, np.array([0, 1, 0, 2, 1, 2, 3], np.int32))}, mode="by")
    add_all(f"onerow.{tag}", {"x": (st, np.array([5], NPT[st]))})
    add_all(f"onerow_na.{tag}", {"x": (st, np.array([na], NPT[st]))})
    add_all(f"onerow_by.{tag}", {"x": (st, np.array([5, na, 3], NPT[st])), "ka": (INT32, np.array([1, 2, 3], np.int32))},
            mode="by")
    add_all(f"empty.{tag}", {"x": (st, np.zeros(0, NPT[st]))})

# int64 wrap-around
big = np.array([2**62, 2**62, 2**62, -5, 2**62, 3], np.int64)
add_all("wrap.i64", {"x": (INT64, big)}, fns=("cumsum",))
add_all("wrap_prod.i64", {"x": (INT64, np.array([2**32, 2**31 + 1, 3, -7, 2**40, 5], np.int64))}, fns=("cumprod",))
add_all("wrap_by.i64", {"x": (INT64, big), "ka": (INT32, np.array([0, 1, 0, 1, 0, 1], np.int32))},
        fns=("cumsum", "cumprod"), mode="by")
add_all("extremes.i64", {"x": (INT64, np.array([2**63 - 1, -2**63 + 1, 5, 2**63 - 1, -2**63 + 1], np.int64))})

# +-inf, inf and -inf in one group, 0 and inf in one group, subnormals
for st in (FLOAT32, FLOAT64):
    tag, T = TAGS[st], NPT[st]
    tiny = np.finfo(T).smallest_subnormal
    add_all(f"inf.{tag}", {"x": (st, np.array([1.0, np.inf, 2.0, np.nan, 3.0], T))})
    add_all(f"ninf.{tag}", {"x": (st, np.array([1.0, -np.inf, -2.0, np.nan, 3.0], T))})
    add_all(f"infninf.{tag}", {"x": (st, np.array([1.0, np.inf, 2.0, -np.inf, 3.0, np.nan, 1.0], T))})
    add_all(f"zeroinf.{tag}", {"x": (st, np.array([2.0, 0.0, 3.0, np.inf, 1.0, np.nan, 4.0], T))})
    add_all(f"infzero.{tag}", {"x": (st, np.array([2.0, -np.inf, 3.0, -0.0, 1.0], T))})
    add_all(f"subnormal.{tag}", {"x": (st, np.array([tiny, tiny, -tiny, 3 * tiny, np.nan, tiny * 1024], T))})
    add_all(f"specials_by.{tag}", {"x": (st, np.array([np.inf, 1.0, -np.inf, 0.0, np.inf, tiny, -0.0, 2.0], T)),
                                   "ka": (INT32, np.array([0, 1, 0, 1, 1, 2, 2, 0], np.int32))}, mode="by")
    # runs of -0.0 and +0.0: the later of equal values wins in cummin / cummax; a sum of zeros keeps the sign rule
    add_all(f"zeros.{tag}", {"x": (st, np.array([-0.0, 0.0, -0.0, -0.0, np.nan, 0.0, 0.0, -0.0, 1.0, -0.0], T))})
    add_all(f"zeros2.{tag}", {"x": (st, np.array([-0.0, -0.0, np.nan, -0.0, 0.0, -1.0, 0.0, -0.0], T))})
    add_all(f"zeros_na.{tag}", {"x": (st, np.array([np.nan, -0.0, np.nan, -0.0], T))})
    v = rng.choice(np.array([0.0, -0.0, np.nan, 1.5, -1.5], T), 80)
    add_all(f"zeros_by.{tag}", {"x": (st, v), "ka": (INT32, keys(80, 4))}, mode="by")

# the inputs of the reference's own tests (tests/dt/test-cumsum.py, test-cumprod.py, test-cumminmax.py)
add_all("ka.small", {"x": (INT32, np.arange(5, dtype=np.int32)), "y": (FLOAT64, np.array([-1, 1, np.nan, 2, 5.5]))},
        j="list")
add_all("ka.groupby", {"ka": (INT32, np.array([2, 1, 1, 1, 2], np.int32)),
                       "x": (FLOAT64, np.array([1.5, -1.5, np.inf, 2, 3]))}, mode="by")
add_all("ka.grouped_column", {"ka": (INT32, np.array([2, 1, NA[INT32], 1, 2], np.int32)),
                              "x": (INT32, np.array([2, 1, NA[INT32], 1, 2], np.int32))}, mode="by", j="bykey")
add_all("ka.minmax", {"x": (INT32, np.array([3, NA[INT32], 1, 4, NA[INT32], 1, 5, 9, 2, 6], np.int32)),
                      "y": (FLOAT64, np.array([2.5, -1.5, np.nan, 0.5, -3.0, 7.0, np.nan, 2.0, -4.5, 1.0]))}, j="list")
add_all("ka.bool", {"x": (BOOL, np.array([1, 0, NA[BOOL], 1, 1, 0], np.int8))})
add_all("ka.prod", {"x": (INT32, np.array([1, 2, NA[INT32], 4, -5], np.int32)),
                    "y": (FLOAT64, np.array([1.5, np.nan, -2.0, 0.5, 4.0]))}, j="list")

# j forms (cumsum and cummax, both directions) -- x is float64, y int32
x, y, g = values(FLOAT64, 40), values(INT32, 40), keys(40, 3)
xy = {"x": (FLOAT64, x), "y": (INT32, y)}
xyg = {"x": (FLOAT64, x), "y": (INT32, y), "ka": (INT32, g)}
for fns in (("cumsum", "cummax"),):
    add_all("j.list", xy, fns=fns, j="list")
    add_all("j.tuple", xy, fns=fns, j="tuple")
    add_all("j.list_by", xyg, fns=fns, mode="by", j="list")
    add_all("j.all", xy, fns=fns, j="all")
    add_all("j.all_by", xyg, fns=fns, mode="by", j="all")
    add_all("j.dict", xyg, fns=fns, mode="by", j="dict")
    add_all("j.dict_none", xy, fns=fns, j="dict")
    add_all("j.dictlist", xy, fns=fns, j="dictlist")
    add_all("j.dictlist_by", xyg, fns=fns, mode="by", j="dictlist")
    add_all("j.plain", xy, fns=fns, j="plain")
    add_all("j.plain_by", xyg, fns=fns, mode="by", j="plain")
    add_all("j.withqcut", xy, fns=fns, j="withqcut")
    add_all("j.withqcut_by", xyg, fns=fns, mode="by", j="withqcut")
add_all("j.all_by.cumprod", {"x": (INT16, values(INT16, 40)), "y": (FLOAT32, values(FLOAT32, 40)), "ka": (INT32, g)},
        fns=("cumprod", "cummin"), mode="by", j="all")

# errors (TypeError texts as Python sees them), each from a fresh interpreter
import subprocess  # noqa: E402
import sys  # noqa: E402


def add_error(name, fn, xst, rev):
    xdef = {"f64": "dt.Frame(x=[1.5, None, 0.0])", "date32": "dt.Frame(x=[1, 2, 3], stype=dt.int32)",
            "time64": "dt.Frame(x=[1, 2, 3], stype=dt.int64)", "str": "dt.Frame(x=['a', 'b', 'c'])"}[xst]
    conv = {"date32": "DT['x'] = DT[:, dt.as_type(f.x, dt.Type.date32)]",
            "time64": "DT['x'] = DT[:, dt.as_type(f.x, dt.Type.time64)]"}.get(xst, "")
    r = subprocess.run([sys.executable, "-c", f"""
import datatable as dt
from datatable import f
DT = {xdef}
{conv}
try:
    DT[:, dt.{fn}(f.x, reverse={rev!r})]
except Exception as e:
    print(type(e).__name__); print(e)
"""], capture_output=True, text=True, check=True).stdout.strip().split("\n", 1)
    manifest.append({"name": name, "fn": fn, "rev": rev, "xstype": xst, "error": r[0], "message": r[1]})


for fn in FNS:
    add_error(f"err.rev_int.{fn}", fn, "f64", 2)
    add_error(f"err.rev_str.{fn}", fn, "f64", "yes")
    add_error(f"err.str.{fn}", fn, "str", False)
add_error("err.date32.cumsum", "cumsum", "date32", False)
add_error("err.time64.cumsum", "cumsum", "time64", True)
add_error("err.date32.cumprod", "cumprod", "date32", True)
add_error("err.time64.cumprod", "cumprod", "time64", False)

np.savez_compressed(os.path.join(HERE, "golden_v7.npz"), **arrays)
json.dump({"generator": "tests/golden/make_golden_v7.py", "datatable_version": dt.__version__, "cases": manifest},
          open(os.path.join(HERE, "golden_v7.json"), "w"), indent=0)
print(len(manifest), "cases")
