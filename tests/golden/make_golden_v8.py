#!/usr/bin/env python
"""
Generates tests/golden/golden_v8.{npz,json} by running the *reference itself* (the unmodified build staged by
oracle/build_ref.sh) on the grouped row functions:

    PYTHONPATH=oracle/_ref python tests/golden/make_golden_v8.py

    dt.shift                 compute_lag_rowindex / Head_Func_Shift (expr/head_func_shift.cc), Shift_ColumnImpl
                             (column/shift.h)
    dt.fillna (no value)     FExpr_FillNA::fill_rowindex (expr/fexpr_fillna.cc)
    dt.cumcount / dt.ngroup  CumcountNgroup_ColumnImpl (column/cumcountngroup.h), FExpr_CumcountNgroup
                             (expr/fexpr_cumcountngroup.cc)

Every case stores the frame's columns (x, and where the query needs them y, ka, kb, s), the query (`fn`: shift,
fillna, cumcount, ngroup or mix; `rev`: reverse=; `n`: shift's n; `mode`, `i` and `j` as tests/window_reference.py:
make_j builds them) and what the reference returns: the output names, stypes and columns.  The cases cover every
function and direction, shift's n in {0, +-1, +-2, +-3, +-group size, +-(group size + 1), a large n}, every accepted
stype, NA first, in the middle, last and everywhere, one row and no rows, -0.0 next to +0.0, +-inf, every query shape
and j form, an `i` slice that drops groups, a by() column as the argument, the inputs of the reference's own tests
(tests/dt/test-shift.py, test-fillna.py, test-cumcountngroup.py; string columns and expressions left out) and the
error texts.  Shifts whose reference result comes from int32 / size_t overflow (|n| beyond the positions) are left
out.  The reference cannot travel to the GPU box, so the vectors are committed.
"""
import json
import os
import subprocess
import sys

import numpy as np

import datatable as dt
from datatable import f

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from window_reference import query  # noqa: E402

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64 = 1, 2, 3, 4, 5, 6, 7, 17, 18
NPT = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
       FLOAT32: np.float32, FLOAT64: np.float64, DATE32: np.int32, TIME64: np.int64}
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
DTST = {BOOL: dt.bool8, INT8: dt.int8, INT16: dt.int16, INT32: dt.int32, INT64: dt.int64,
        FLOAT32: dt.float32, FLOAT64: dt.float64, DATE32: dt.int32, TIME64: dt.int64}
TAGS = {BOOL: "bool", INT8: "i8", INT16: "i16", INT32: "i32", INT64: "i64", FLOAT32: "f32", FLOAT64: "f64",
        DATE32: "date32", TIME64: "time64"}
arrays, manifest = {}, []
rng = np.random.default_rng(20261018)


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


def add(name, cols, fn, rev=False, n=1, mode="none", i=None, j="one"):
    assert not any(c["name"] == name for c in manifest), name
    DT = frame(cols)
    case = {"name": name, "fn": fn, "rev": rev, "n": n, "mode": mode, "i": i, "j": j,
            "stypes": {nm: st for nm, (st, _) in cols.items()}}
    R = query(dt, case, DT)
    case.update(nrows=int(R.nrows), names=list(R.names), out_stypes=[str(s) for s in R.stypes])
    for nm in R.names:
        arrays[name + ".out_" + nm] = to_np(R, nm)
    for nm, (st, a) in cols.items():
        arrays[name + "." + nm] = np.ascontiguousarray(a, dtype=NPT[st])
    manifest.append(case)


def shifts(nmax, nrows, grouped):
    """shift's n: 0, +-1, +-2, +-3, +-nmax, +-(nmax + 1) (nmax: the largest group) and +-10**6.  Without by() a lead
    of more than the selected rows reads past the column in the reference (nrows - |n| wraps in size_t): those leads
    are left out."""
    ns = [0, 1, -1, 2, -2, 3, -3, nmax, -nmax, nmax + 1, -(nmax + 1), 10**6, -10**6]
    return list(dict.fromkeys(k for k in ns if grouped or k >= -nrows))


def add_all(name, cols, fns=("shift", "fillna", "cumcount", "ngroup"), grouped=False, **kw):
    """Every function and direction; shift over shifts(), the others at n = 1."""
    nrows = len(next(iter(cols.values()))[1])
    nmax = int(np.unique(cols["ka"][1], return_counts=True)[1].max()) if grouped and nrows else nrows
    for fn in fns:
        if fn == "shift":
            for n in shifts(nmax, nrows, grouped):
                add(f"{name}.shift{n:+d}", cols, fn, False, n, **kw)
        else:
            for rev in (False, True):
                add(f"{name}.{fn}{'.rev' if rev else ''}", cols, fn, rev, **kw)


def keys(n, ng, na=0.05):
    k = rng.integers(0, ng, n).astype(np.int32)
    k[rng.random(n) < na] = NA[INT32]
    return k


def values(st, n, na=0.25):
    if st == BOOL:
        v = rng.integers(0, 2, n).astype(np.int8)
    elif st in (FLOAT32, FLOAT64):
        v = rng.choice(np.array([-2.5, -1.0, -0.0, 0.0, 0.5, 3.0, np.inf, -np.inf]), n).astype(NPT[st])
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
ALLST = NUMERIC + (DATE32, TIME64)
n = 40
# every function x direction over every accepted stype, without and with by()
for st in ALLST:
    tag = TAGS[st]
    add_all(f"none.{tag}", {"x": (st, values(st, n))}, fns=("shift", "fillna"))
    add_all(f"by.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 4))}, fns=("shift", "fillna"),
            grouped=True, mode="by")
add_all("none.nullary", {"x": (INT32, values(INT32, n))}, fns=("cumcount", "ngroup"))
add_all("by.nullary", {"x": (INT32, values(INT32, n)), "ka": (INT32, keys(n, 4))}, fns=("cumcount", "ngroup"),
        grouped=True, mode="by")

# the query shapes, every function in both directions; shift at +1, -1, +2 and -2 (a lead only where the selected
# rows are at least that many)
def add_shape(name, cols, nsel=None, **kw):
    add_all(name, cols, fns=("fillna", "cumcount", "ngroup"), **kw)
    for s in (1, -1, 2, -2):
        if nsel is None or s >= -nsel:
            add(f"{name}.shift{s:+d}", cols, "shift", False, s, **kw)


for st in (INT32, FLOAT64):
    tag = TAGS[st]
    add_shape(f"by2.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 3)), "kb": (INT32, keys(n, 3))},
              mode="by2")
    add_shape(f"bysort.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 4)),
                                "s": (INT32, rng.integers(-9, 10, n).astype(np.int32))}, mode="bysort")
    add_shape(f"sort.{tag}", {"x": (st, values(st, n)), "s": (INT32, keys(n, 20))}, mode="sort")
    add_shape(f"sortdesc.{tag}", {"x": (st, values(st, n)), "s": (INT32, keys(n, 20))}, mode="sortdesc")
    add_shape(f"islice_by.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 5))}, mode="by",
              i=[1, None, 2])
    add_shape(f"islice.{tag}", {"x": (st, values(st, n))}, i=[3, 35, 2])
    add_shape(f"int_by.{tag}", {"x": (st, values(st, n)), "ka": (INT32, keys(n, 5))}, mode="by", i=-1)
    add_shape(f"int.{tag}", {"x": (st, values(st, n))}, nsel=1, i=7)
    add_shape(f"islice_sort.{tag}", {"x": (st, values(st, n)), "s": (INT32, keys(n, 20))}, mode="sort",
              i=[2, 30])
# an `i` slice that drops groups: groups of 1 .. 4 rows, rows 2 and 3 of every group kept
kd = np.repeat(np.arange(8, dtype=np.int32), [1, 4, 2, 3, 1, 4, 1, 3])
add_shape("islice_drops", {"x": (FLOAT64, values(FLOAT64, len(kd))), "ka": (INT32, rng.permutation(kd))},
          mode="by", i=[2, 4])
add_shape("int_drops", {"x": (INT32, values(INT32, len(kd))), "ka": (INT32, rng.permutation(kd))},
          mode="by", i=3)

# a by() column as the argument
for st in (INT32, FLOAT64):
    ka = keys(30, 4, na=0.2)
    kk = {"x": (st, values(st, 30)), "ka": (INT32, ka)}
    for s in (1, -1, 2):
        add(f"bykey.{TAGS[st]}.shift{s:+d}", kk, "shift", n=s, mode="by", j="bykey")
    for rev in (False, True):
        add(f"bykey.{TAGS[st]}.fillna{'.rev' if rev else ''}", kk, "fillna", rev, mode="by", j="bykey")

# NA first, in the middle, last, everywhere; NA only in some groups; one row; no rows
for st in (INT32, FLOAT64):
    tag = TAGS[st]
    na = np.nan if st == FLOAT64 else NA[st]
    add_all(f"nafirst.{tag}", {"x": (st, np.array([na, na, 1, 2, 3, 2, 1], NPT[st]))})
    add_all(f"namiddle.{tag}", {"x": (st, np.array([4, 1, na, na, 2, 5, 1], NPT[st]))})
    add_all(f"nalast.{tag}", {"x": (st, np.array([4, 1, 2, 5, na, na], NPT[st]))})
    add_all(f"allna.{tag}", {"x": (st, np.full(6, na, NPT[st]))})
    add_all(f"na_by.{tag}", {"x": (st, np.array([na, 1, na, na, 3, na, 2, na], NPT[st])),
                             "ka": (INT32, np.array([0, 1, 0, 2, 1, 2, 3, 1], np.int32))}, grouped=True, mode="by")
    add_all(f"onerow.{tag}", {"x": (st, np.array([5], NPT[st]))})
    add_all(f"onerow_na.{tag}", {"x": (st, np.array([na], NPT[st]))})
    add_all(f"onerow_by.{tag}", {"x": (st, np.array([5, na, 3], NPT[st])), "ka": (INT32, np.array([1, 2, 3], np.int32))},
            grouped=True, mode="by")
    # (fillna over no rows without by() crashes the reference: left out)
    add_all(f"empty.{tag}", {"x": (st, np.zeros(0, NPT[st]))}, fns=("shift", "cumcount", "ngroup"))

# -0.0 next to +0.0, +-inf, NaN
for st in (FLOAT32, FLOAT64):
    tag, T = TAGS[st], NPT[st]
    z = np.array([-0.0, np.nan, 0.0, np.nan, -0.0, np.inf, np.nan, -np.inf, np.nan, -0.0, 0.0], T)
    add_all(f"zeros.{tag}", {"x": (st, z)})
    add_all(f"zeros_by.{tag}", {"x": (st, z), "ka": (INT32, np.array([0, 1, 0, 1, 0, 1, 1, 0, 0, 1, 1], np.int32))},
            grouped=True, mode="by")

# the inputs of the reference's own tests (tests/dt/test-shift.py, test-fillna.py, test-cumcountngroup.py)
add_all("ts.shift_by", {"ka": (INT32, np.array([1, 2, 1, 1, 2, 1, 2], np.int32)),
                        "x": (INT32, np.arange(7, dtype=np.int32))}, fns=("shift",), grouped=True, mode="by")
add("ts.shift_by_with_i", {"ka": (INT32, np.array([1, 2, 1, 2, 1, 2, 1, 2], np.int32)),
                           "x": (INT32, np.arange(8, dtype=np.int32))}, "shift", mode="by", i=[1, None])
add("ts.shift_group_column", {"ka": (INT32, np.array([1, 2, 1, 2, 1, 2, 1, 2], np.int32)),
                              "x": (INT32, np.arange(8, dtype=np.int32))}, "shift", mode="by", j="bykey")
for s in (1, 3, -2, 100):
    add(f"ts.shift_frame{s:+d}", {"x": (INT32, np.array([5, 3, 2, 17, 9, NA[INT32], 0], np.int32)),
                                  "y": (FLOAT64, np.array([1.5, -2.5, np.nan, 0.0, 7.0, 3.25, -0.0]))},
        "shift", n=s, j="frame")
fl = {"x": (INT32, np.array([NA[INT32], 1, NA[INT32], NA[INT32], 5, NA[INT32], 2], np.int32)),
      "y": (FLOAT64, np.array([np.nan, np.nan, 2.5, np.nan, -1.0, np.nan, np.nan])),
      "ka": (INT32, np.array([1, 1, 2, 2, 1, 2, 1], np.int32))}
add_all("ts.fillna_list", fl, fns=("fillna",), j="list")
add_all("ts.fillna_by", fl, fns=("fillna",), mode="by", j="all")
add_all("ts.cumcount_void", {"x": (INT8, np.full(10, NA[INT8], np.int8))}, fns=("cumcount", "ngroup"))
add_all("ts.cumcount_trivial", {"x": (INT64, np.array([0], np.int64))}, fns=("cumcount", "ngroup"))
cc = {"x": (INT32, np.array([1, 1, 2, 2, 2, 3, 1, 3], np.int32)), "ka": (INT32, np.array([1, 1, 2, 2, 2, 3, 1, 3], np.int32)),
      "kb": (INT32, np.array([5, 6, 5, 5, 6, 5, 6, 6], np.int32))}
add_all("ts.cumcount_by", cc, fns=("cumcount", "ngroup"), grouped=True, mode="by")
add_all("ts.cumcount_by2", cc, fns=("cumcount", "ngroup"), grouped=True, mode="by2")

# j forms -- x is float64, y int32
x, y, g = values(FLOAT64, 30), values(INT32, 30), keys(30, 3)
xy = {"x": (FLOAT64, x), "y": (INT32, y)}
xyg = {"x": (FLOAT64, x), "y": (INT32, y), "ka": (INT32, g)}
JF = {"shift": ("list", "tuple", "all", "dict", "plain", "withqcut", "withcum"),
      "fillna": ("list", "tuple", "all", "dict", "dictlist", "plain", "withqcut", "withcum"),
      "cumcount": ("list", "tuple", "dict", "plain", "withqcut", "withcum", "both"),
      "ngroup": ("list", "tuple", "dict", "plain", "withqcut", "withcum", "both")}
for fn, forms in JF.items():
    for jf in forms:
        for mode, cols in (("none", xy), ("by", xyg)):
            for rev in ((False,) if fn == "shift" else (False, True)):
                for s in ((1, -2) if fn == "shift" else (1,)):
                    add(f"j.{jf}.{mode}.{fn}{'.rev' if rev else ''}{f'{s:+d}' if fn == 'shift' else ''}", cols, fn,
                        rev, s, mode=mode, j=jf)
# the four together, as a user writes them: DT[:, {"lag": shift(f.x), "filled": fillna(f.x), "i": cumcount(),
# "g": ngroup()}, by(f.ka)]
for mode, cols in (("none", xy), ("by", xyg), ("bysort", dict(xyg, s=(INT32, keys(30, 7))))):
    for rev in (False, True):
        add(f"mix.{mode}{'.rev' if rev else ''}", cols, "mix", rev, 1, mode=mode, j="dict")
add("mix.by.lead", xyg, "mix", False, -1, mode="by", j="dict")


# errors (exception type and text as Python sees them), each from a fresh interpreter
def add_error(name, expr):
    r = subprocess.run([sys.executable, "-c", f"""
import datatable as dt
from datatable import f
try:
    dt.Frame(x=[1.5, None, 0.0], y=[1, 2, 3])[:, {expr}]
    print("none"); print("")
except Exception as e:
    print(type(e).__name__); print(e)
"""], capture_output=True, text=True, check=True).stdout.strip().split("\n", 1)
    assert r[0] != "none", expr
    manifest.append({"name": name, "expr": expr, "error": r[0], "message": r[1]})


ERRS = {"shift.noargs": "dt.shift()", "shift.none": "dt.shift(None)", "shift.n_only": "dt.shift(n=3)",
        "shift.int": "dt.shift(3)", "shift.float": "dt.shift(12.5)", "shift.str": "dt.shift('hi')",
        "shift.module": "dt.shift(dt)", "shift.list": "dt.shift([f.x, f.y])", "shift.tuple": "dt.shift((f.x,))",
        "shift.dict": "dt.shift({'a': f.x})", "shift.n_str": "dt.shift(f.x, n='one')",
        "shift.n_float": "dt.shift(f.x, n=0.0)", "shift.n_bool": "dt.shift(f.x, n=True)",
        "shift.n_range": "dt.shift(f.x, n=range(3))", "shift.n_list": "dt.shift(f.x, n=[1, 2, 3])",
        "shift.n_big": "dt.shift(f.x, n=2**31)", "shift.n_small": "dt.shift(f.x, n=-2**31 - 1)",
        "shift.n_before_cols": "dt.shift(None, n='x')",
        "fillna.value_reverse": "dt.fillna(f.x, value=1, reverse=True)",
        "fillna.value_reverse_false": "dt.fillna(f.x, value=0, reverse=False)",
        "fillna.reverse_int": "dt.fillna(f.x, reverse=1)", "fillna.reverse_str": "dt.fillna(f.x, reverse='yes')",
        "cumcount.int": "dt.cumcount(1)", "cumcount.str": "dt.cumcount('False')",
        "cumcount.float": "dt.cumcount(reverse=2.5)", "ngroup.str": "dt.ngroup('True')", "ngroup.int": "dt.ngroup(0)"}
for nm, ex in ERRS.items():
    add_error(f"err.{nm}", ex)

np.savez_compressed(os.path.join(HERE, "golden_v8.npz"), **arrays)
json.dump({"generator": "tests/golden/make_golden_v8.py", "datatable_version": dt.__version__, "cases": manifest},
          open(os.path.join(HERE, "golden_v8.json"), "w"), indent=0)
print(len(manifest), "cases")
