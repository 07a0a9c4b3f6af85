#!/usr/bin/env python
"""
Generates tests/golden/golden_v12.{npz,json} by running the *reference itself* (the unmodified build staged by
oracle/build_ref.sh) on dt.cut:

    PYTHONPATH=oracle/_ref python tests/golden/make_golden_v12.py

    dt.cut   CutNbins_ColumnImpl / CutBins_ColumnImpl (column/cut.h:91-281), FExpr_Cut (expr/fexpr_cut.cc:88-302)

Every case stores the frame's columns, the query and what the reference returns (output names, stypes, columns), or
the error it raises:
    mode   none, sort (sort(f.s)), sortdesc (sort(-f.s)), sortlast / sortremove (sort(f.x, na_position=...)), by
           (by(f.s): an error), join (join(J), J's columns stored as J.<name>)
    i      None, ["slice", [a, b, c]], ["int", k], ["bool", "b"] (f.b), ["frame", "isel"] (an int32 Frame with NA),
           ["list", [...]], ["range", [a, b, c]]
    j      one = cut(f.x), list = cut([f.x, f.y]), tuple, all = cut(f[:]), dict = {"c": cut(f.x)}, dictlist, plain =
           [f.x, cut(f.x)], qcut = [cut(f.x), qcut(f.x)], cumsum = [cut(f.x), cumsum(f.y)], shift = [cut(f.x),
           shift(f.x)], self = cut(DT), other = cut(Frame(z=...)) (column z stored as other.z), joincol = cut(g.v),
           joinlist = cut([f.x, g.v])
    kw     nbins (int, list or tuple), bins (a list of {"key", "stype"}: 1-column edge Frames), right_closed
The reference cannot travel to the GPU box, so the vectors are committed.
"""
import json
import os

# datatable before numpy: with numpy loaded first, the reference's process crashes (a segmentation fault) in the error
# path of a ValueError raised by cut()
import datatable as dt
from datatable import f, g, by, sort, join

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64 = 1, 2, 3, 4, 5, 6, 7, 17, 18
NPT = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
       FLOAT32: np.float32, FLOAT64: np.float64, DATE32: np.int32, TIME64: np.int64}
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
DTST = {BOOL: dt.bool8, INT8: dt.int8, INT16: dt.int16, INT32: dt.int32, INT64: dt.int64,
        FLOAT32: dt.float32, FLOAT64: dt.float64, DATE32: dt.int32, TIME64: dt.int64}
TAGS = {BOOL: "bool", INT8: "i8", INT16: "i16", INT32: "i32", INT64: "i64", FLOAT32: "f32", FLOAT64: "f64",
        DATE32: "date32", TIME64: "time64"}
NUMERIC = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
arrays, manifest = {}, []
rng = np.random.default_rng(20261018)


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


def query(DT, case, J=None, other=None, bins=None):
    kw = {}
    if case["nbins"] is not None:
        kw["nbins"] = tuple(case["nbins"]) if case.get("nbins_tuple") else case["nbins"]
    if bins is not None:
        kw["bins"] = bins
    if case["right_closed"] is not None:
        kw["right_closed"] = case["right_closed"]
    cut = lambda c: dt.cut(c, **kw)           # noqa: E731
    J_ = {"one": lambda: cut(f.x), "list": lambda: cut([f.x, f.y]), "tuple": lambda: cut((f.x, f.y)),
          "all": lambda: cut(f[:]), "dict": lambda: {"c": cut(f.x)}, "dictlist": lambda: {"c": cut([f.x, f.y])},
          "plain": lambda: [f.x, cut(f.x)], "qcut": lambda: [cut(f.x), dt.qcut(f.x)],
          "cumsum": lambda: [cut(f.x), dt.cumsum(f.y)], "shift": lambda: [cut(f.x), dt.shift(f.x)],
          "self": lambda: cut(DT), "other": lambda: cut(other), "joincol": lambda: cut(g.v),
          "joinlist": lambda: cut([f.x, g.v])}[case["j"]]()
    i = case["i"]
    if i is None:
        rows = slice(None)
    else:
        kind, p = i
        rows = {"slice": lambda: slice(*p), "int": lambda: p, "bool": lambda: f[p],
                "frame": lambda: dt.Frame(pylist(arrays[case["name"] + "." + p], INT32), stype=dt.int32),
                "list": lambda: list(p), "range": lambda: range(*p)}[kind]()
    mods = {"none": (), "sort": (sort(f.s),), "sortdesc": (sort(-f.s),),
            "sortlast": (sort(f.x, na_position="last"),), "sortremove": (sort(f.x, na_position="remove"),),
            "by": (by(f.s),), "join": (join(J),) if J is not None else ()}[case["mode"]]
    return DT[(rows, J_) + mods]


def add(name, cols, mode="none", i=None, j="one", nbins=None, bins=None, right_closed=None, nbins_tuple=False,
        jcols=None, other=None):
    """bins: a list of (stype, array) edge columns; jcols: J's columns {name: (stype, array)}, keyed by k;
    other: the column z of the Frame for j = other."""
    case = {"name": name, "mode": mode, "i": i, "j": j, "nbins": nbins, "nbins_tuple": nbins_tuple,
            "right_closed": right_closed, "stypes": {nm: st for nm, (st, _) in cols.items()}}
    for nm, (st, a) in cols.items():
        arrays[name + "." + nm] = np.ascontiguousarray(a, dtype=NPT[st])
    if i is not None and i[0] == "frame":
        arrays[name + ".isel"] = np.ascontiguousarray(i[2], dtype=np.int32)
        case["i"] = i = ["frame", "isel"]
    bf = None
    if bins is not None:
        case["bins"] = []
        bf = []
        for k, (st, a) in enumerate(bins):
            key = f"{name}.bins{k}"
            arrays[key] = np.ascontiguousarray(a, dtype=NPT[st])
            case["bins"].append({"key": key, "stype": st})
            bf.append(frame({"C0": (st, np.asarray(a, dtype=NPT[st]))}))
    J = None
    if jcols is not None:
        case["jstypes"] = {nm: st for nm, (st, _) in jcols.items()}
        for nm, (st, a) in jcols.items():
            arrays[name + ".J." + nm] = np.ascontiguousarray(a, dtype=NPT[st])
        J = frame(jcols)
        J.key = "k"
    O = None
    if other is not None:
        case["other_stype"] = other[0]
        arrays[name + ".other.z"] = np.ascontiguousarray(other[1], dtype=NPT[other[0]])
        O = frame({"z": other})
    DT = frame(cols)
    try:
        R = query(DT, case, J, O, bf)
    except Exception as e:                                      # noqa: BLE001
        case.update(error=type(e).__name__, message=str(e))
    else:
        case.update(nrows=int(R.nrows), names=list(R.names), out_stypes=[str(s) for s in R.stypes])
        for nm in R.names:
            arrays[name + ".out_" + nm] = to_np(R, nm)
    manifest.append(case)


def values(st, n, na=0.1, distinct=None):
    if st == BOOL:
        v = rng.integers(0, 2, n).astype(np.int8)
    elif st in (FLOAT32, FLOAT64):
        v = (rng.standard_normal(n) * 50).astype(NPT[st]) if distinct is None else \
            rng.choice(np.linspace(-3, 3, distinct), n).astype(NPT[st])
    else:
        hi = {INT8: 100, INT16: 30000, INT32: 2**30, INT64: 2**62, DATE32: 10**5, TIME64: 10**15}[st]
        v = rng.integers(-hi, hi, n).astype(NPT[st]) if distinct is None else \
            rng.integers(-distinct // 2, distinct // 2 + 1, n).astype(NPT[st])
    mask = rng.random(n) < na
    v[mask] = np.nan if st in (FLOAT32, FLOAT64) else NA[st]
    return v


n = 200
# every numeric stype, nbins and bins, both closures
for st in NUMERIC:
    tag = TAGS[st]
    add(f"nbins.{tag}", {"x": (st, values(st, n))})
    add(f"nbins3_open.{tag}", {"x": (st, values(st, n))}, nbins=3, right_closed=False)
    add(f"nbins7.{tag}", {"x": (st, values(st, n, distinct=9))}, nbins=7)
    e = np.sort(rng.choice(np.arange(-40, 41), 9, replace=False)).astype(np.float64)
    if st == BOOL:
        e = np.array([-1.0, 0.0, 0.5, 1.0, 2.0])
    add(f"bins.{tag}", {"x": (st, values(st, n, distinct=60))}, bins=[(FLOAT64, e)])
    add(f"bins_open.{tag}", {"x": (st, values(st, n, distinct=60))}, bins=[(FLOAT64, e)], right_closed=False)

# int64 beyond 2^53, at min+1 and max
big = np.array([2**53 + 1, 2**53 + 3, 2**60 + 7, -2**63 + 1, 2**63 - 1, NA[INT64], 0, -2**62, 2**53], np.int64)
add("i64_extreme", {"x": (INT64, big)})
add("i64_extreme_open", {"x": (INT64, big)}, nbins=1000, right_closed=False)
add("i64_beyond53", {"x": (INT64, 2**55 + rng.integers(-50, 50, 100).astype(np.int64))}, nbins=13)
add("i64_beyond53_bins", {"x": (INT64, 2**55 + rng.integers(-50, 50, 100).astype(np.int64))},
    bins=[(INT64, np.array([2**55 - 40, 2**55 - 3, 2**55, 2**55 + 8, 2**55 + 40], np.int64))])
add("i64_edges_minmax", {"x": (INT64, big)}, bins=[(INT64, np.array([-2**63 + 1, 0, 2**63 - 1], np.int64))])

# float specials: subnormals, signed zeros, NaN payloads, infinities, huge ranges
for st in (FLOAT32, FLOAT64):
    tag, T = TAGS[st], NPT[st]
    tiny = np.finfo(T).smallest_subnormal
    big_ = np.finfo(T).max
    nan2 = np.array([0x7FF0000000000123 if st == FLOAT64 else 0x7F800123],
                    dtype=np.uint64 if st == FLOAT64 else np.uint32).view(T)[0]
    nneg = -np.array([np.nan], T)[0]
    add(f"subnormal.{tag}", {"x": (st, np.array([tiny, 0.0, 3 * tiny, -tiny, np.nan, 2 * tiny], T))})
    add(f"subnormal_only.{tag}", {"x": (st, np.array([tiny, 2 * tiny, 5 * tiny, 4 * tiny], T))}, nbins=4)
    add(f"zero_tiny.{tag}", {"x": (st, np.array([0.0, tiny, -0.0], T))})                 # a overflows to inf
    add(f"zeros.{tag}", {"x": (st, np.array([-0.0, 0.0, 0.0, -0.0], T))})
    add(f"zeros_mixed.{tag}", {"x": (st, np.array([-0.0, 1.5, 0.0, np.nan, nan2, nneg, -2.5], T))}, nbins=4)
    add(f"zeros_open.{tag}", {"x": (st, np.array([-0.0, 1.5, 0.0, 3.0], T))}, nbins=4, right_closed=False)
    add(f"inf.{tag}", {"x": (st, np.array([1.0, np.inf, 2.0], T))})
    add(f"ninf.{tag}", {"x": (st, np.array([-np.inf, 1.0, 2.0], T))})
    add(f"bigrange.{tag}", {"x": (st, np.array([-big_, big_, 0.0, 1.0, -1e30], T))})
    add(f"bigrange_open.{tag}", {"x": (st, np.array([-big_, big_, 0.0, 1e30], T))}, right_closed=False)
    add(f"nan_patterns.{tag}", {"x": (st, np.array([nan2, 1.0, nneg, np.nan, 4.0], T))}, nbins=3)
    add(f"bins_special.{tag}", {"x": (st, np.array([np.inf, -np.inf, np.nan, nan2, 0.0, -0.0, tiny, -tiny, 1.0,
                                                   2.0, 3.0, big_], T))},
        bins=[(FLOAT64, np.array([-np.inf, -1.0, 0.0, 1.0, 2.0, np.inf]))])
    add(f"bins_special_open.{tag}", {"x": (st, np.array([np.inf, -np.inf, np.nan, 0.0, -0.0, tiny, 1.0, 2.0], T))},
        bins=[(FLOAT64, np.array([-np.inf, -1.0, 0.0, 1.0, 2.0, np.inf]))], right_closed=False)
add("f64_1e308", {"x": (FLOAT64, np.array([-1e308, 1e308, 0.0, 5e307, -3e307]))}, nbins=5)
add("f64_1e308_open", {"x": (FLOAT64, np.array([-1e308, 1e308, 0.0, 5e307]))}, nbins=5, right_closed=False)
add("f64_cancel", {"x": (FLOAT64, 1e300 * (1 + np.arange(20) * 2.0**-52))}, nbins=2**31 - 1)

# constant columns, one row, no rows, all NA
for st in (BOOL, INT32, INT64, FLOAT32, FLOAT64):
    tag, na = TAGS[st], (np.nan if st in (FLOAT32, FLOAT64) else NA[st])
    add(f"const.{tag}", {"x": (st, np.full(5, 1, NPT[st]))})
    add(f"const_open.{tag}", {"x": (st, np.full(5, 1, NPT[st]))}, nbins=4, right_closed=False)
    add(f"const_na.{tag}", {"x": (st, np.array([1, na, 1], NPT[st]))}, nbins=3)
    add(f"onerow.{tag}", {"x": (st, np.array([1], NPT[st]))})
    add(f"onerow_na.{tag}", {"x": (st, np.array([na], NPT[st]))})
    add(f"empty.{tag}", {"x": (st, np.zeros(0, NPT[st]))})
    add(f"empty_bins.{tag}", {"x": (st, np.zeros(0, NPT[st]))}, bins=[(FLOAT64, np.array([0.0, 1.0]))])
    add(f"allna.{tag}", {"x": (st, np.full(7, na, NPT[st]))})

# nbins 1, 2, 3, 10, more than the rows, 2^31 - 1; both closures
for nb in (1, 2, 3, 10, 50, 2**31 - 1):
    for st in (INT32, FLOAT64):
        for rc in (True, False):
            add(f"nb{nb}_{'rc' if rc else 'open'}.{TAGS[st]}", {"x": (st, values(st, 20, distinct=15))}, nbins=nb,
                right_closed=rc)
    add(f"nb{nb}_wide.f64", {"x": (FLOAT64, values(FLOAT64, 300))}, nbins=nb)

# per-column nbins: lists, tuples, one value for every column
x, y = values(FLOAT64, 60), values(INT32, 60)
xy = {"x": (FLOAT64, x), "y": (INT32, y)}
add("nbins_list", xy, j="list", nbins=[2, 5])
add("nbins_tuple", xy, j="list", nbins=[3, 4], nbins_tuple=True)
add("nbins_one_for_all", xy, j="list", nbins=[7])
add("nbins_list_open", xy, j="tuple", nbins=[6, 2], right_closed=False)

# bins: 2 edges, 1000 edges, more than the shared-memory sample holds; int / float32 / bool / infinite edges;
# values on the edges, below the first and above the last
add("bins2", {"x": (FLOAT64, values(FLOAT64, 100))}, bins=[(FLOAT64, np.array([-10.0, 10.0]))])
add("bins2_open", {"x": (FLOAT64, np.array([-10.0, 10.0, 0.0, -11.0, 11.0, np.nan]))},
    bins=[(FLOAT64, np.array([-10.0, 10.0]))], right_closed=False)
e1000 = np.cumsum(rng.random(1000) + 0.01) - 250.0
v = np.concatenate([rng.uniform(-300, 300, 2000), e1000[::7], [e1000[0], e1000[-1], -1e9, 1e9, np.nan]])
add("bins1000", {"x": (FLOAT64, v)}, bins=[(FLOAT64, e1000)])
add("bins1000_open", {"x": (FLOAT64, v)}, bins=[(FLOAT64, e1000)], right_closed=False)
e5000 = np.cumsum(rng.random(5000) + 0.001) - 1250.0
v = np.concatenate([rng.uniform(-1300, 1300, 3000), e5000[::3], e5000[4090:4110], [e5000[0], e5000[-1], np.nan]])
add("bins5000", {"x": (FLOAT64, v)}, bins=[(FLOAT64, e5000)])
add("bins5000_open", {"x": (FLOAT64, v)}, bins=[(FLOAT64, e5000)], right_closed=False)
e9001 = np.arange(9001, dtype=np.float64) * 0.5 - 1000.0
v = np.concatenate([rng.integers(-1100, 4000, 3000) * 0.25, [np.nan, -1000.0, 3500.0]])
add("bins9001.f64", {"x": (FLOAT64, v)}, bins=[(FLOAT64, e9001)])
add("bins9001_open.i32", {"x": (INT32, rng.integers(-1100, 3600, 3000).astype(np.int32))},
    bins=[(FLOAT64, e9001)], right_closed=False)
add("bins_int_edges", {"x": (INT32, rng.integers(-20, 20, 200).astype(np.int32))},
    bins=[(INT32, np.array([-15, -3, 0, 2, 9, 15], np.int32))])
add("bins_int_edges_open", {"x": (INT32, rng.integers(-20, 20, 200).astype(np.int32))},
    bins=[(INT32, np.array([-15, -3, 0, 2, 9, 15], np.int32))], right_closed=False)
add("bins_i8_edges", {"x": (FLOAT32, rng.uniform(-5, 5, 100).astype(np.float32))},
    bins=[(INT8, np.array([-4, -1, 0, 3], np.int8))])
add("bins_f32_edges", {"x": (FLOAT64, rng.uniform(-2, 2, 200))},
    bins=[(FLOAT32, np.array([-1.7, -0.1, 0.1, 0.3, 1.9], np.float32))])
add("bins_f32_edges_f32", {"x": (FLOAT32, np.array([-1.7, -0.1, 0.1, 0.3, 1.9, 0.2, 0.0], np.float32))},
    bins=[(FLOAT32, np.array([-1.7, -0.1, 0.1, 0.3, 1.9], np.float32))])
add("bins_bool_edges", {"x": (BOOL, values(BOOL, 50))}, bins=[(BOOL, np.array([0, 1], np.int8))])
add("bins_bool_edges_open", {"x": (FLOAT64, np.array([-0.5, 0.0, 0.5, 1.0, 1.5]))},
    bins=[(BOOL, np.array([0, 1], np.int8))], right_closed=False)
add("bins_inf_edges", {"x": (FLOAT64, np.array([-np.inf, -1e308, 0.0, 1e308, np.inf, 5.0]))},
    bins=[(FLOAT64, np.array([-np.inf, 0.0, np.inf]))])
add("bins_inf_edges_open", {"x": (FLOAT64, np.array([-np.inf, -1e308, 0.0, 1e308, np.inf, 5.0]))},
    bins=[(FLOAT64, np.array([-np.inf, 0.0, np.inf]))], right_closed=False)
add("bins_per_column", xy, j="list", bins=[(FLOAT64, np.array([-50.0, 0.0, 50.0])),
                                           (INT64, np.array([-2**30, 0, 2**29, 2**30], np.int64))])
add("bins_per_column_open", xy, j="list", bins=[(FLOAT64, np.array([-50.0, 0.0, 50.0])),
                                                (INT32, np.array([-2**30, 0, 2**29, 2**30], np.int32))],
    right_closed=False)

# query shapes
s = values(INT32, 60, distinct=20)
xs = {"x": (FLOAT64, x), "y": (INT32, y), "s": (INT32, s)}
b = rng.integers(0, 2, 60).astype(np.int8)
b[::11] = NA[BOOL]
xsb = dict(xs, b=(BOOL, b))
for mode in ("sort", "sortdesc", "sortlast", "sortremove"):
    add(f"{mode}.nbins", xs, mode=mode, nbins=4)
    add(f"{mode}.bins", xs, mode=mode, bins=[(FLOAT64, np.array([-60.0, -5.0, 0.0, 20.0, 80.0]))])
    add(f"{mode}.list", xs, mode=mode, j="list", nbins=[3, 5])
add("sort_islice", xs, mode="sort", i=["slice", [3, 50, 2]], nbins=6)
add("sort_int", xs, mode="sort", i=["int", 4])
add("sort_plain", xs, mode="sort", j="plain", nbins=3)
add("sort_self", xs, mode="sortdesc", j="self", nbins=3)
for nm, i in (("islice", ["slice", [5, 45, 3]]), ("islice_neg", ["slice", [None, None, -2]]), ("iint", ["int", 7]),
              ("iint_neg", ["int", -3]), ("ibool", ["bool", "b"]),
              ("iframe", ["frame", None, np.array([3, NA[INT32], 0, 59, 17, 17, NA[INT32], 8], np.int32)]),
              ("ilist", ["list", [5, 0, 9, 9, 33]]), ("irange", ["range", [2, 58, 5]]), ("irange_neg", ["range", [50, 3, -4]])):
    add(f"{nm}.nbins", xsb, i=i, nbins=5)
    add(f"{nm}.bins", xsb, i=i, bins=[(FLOAT64, np.array([-70.0, -10.0, 0.0, 10.0, 70.0]))], right_closed=False)
    add(f"{nm}.list", xsb, i=i, j="list")
add("ibool_allfalse", dict(xs, b=(BOOL, np.zeros(60, np.int8))), i=["bool", "b"], nbins=3)
add("iframe_allna", xs, i=["frame", None, np.full(4, NA[INT32], np.int32)])

# j forms
for j in ("one", "list", "tuple", "all", "dict", "dictlist", "plain", "qcut", "cumsum", "shift", "self"):
    add(f"j.{j}", xy, j=j)
    add(f"j.{j}_bins", xy, j=j, bins=[(FLOAT64, np.array([-100.0, 0.0, 100.0]))] * (2 if j in ("list", "tuple",
                                                                                                "dictlist", "all",
                                                                                                "self") else 1))
add("j.other", xy, j="other", other=(FLOAT32, values(FLOAT32, 60)), nbins=4)
add("j.other_i32", xy, j="other", other=(INT32, values(INT32, 60)), bins=[(INT32, np.array([-2**30, 0, 2**30]))])
add("j.all_i", xy, j="all", i=["slice", [10, 20]], nbins=[2, 3])

# join(J): the joined frame's columns
kx = rng.integers(0, 12, 80).astype(np.int32)
kx[::9] = NA[INT32]
jc = {"k": (INT32, np.arange(10, dtype=np.int32)), "v": (FLOAT64, values(FLOAT64, 10))}
add("join.joincol", {"x": (FLOAT64, values(FLOAT64, 80)), "k": (INT32, kx)}, mode="join", j="joincol", jcols=jc)
add("join.joinlist", {"x": (FLOAT64, values(FLOAT64, 80)), "k": (INT32, kx)}, mode="join", j="joinlist", jcols=jc,
    nbins=[3, 4])
add("join.bins", {"x": (FLOAT64, values(FLOAT64, 80)), "k": (INT32, kx)}, mode="join", j="joincol", jcols=jc,
    bins=[(FLOAT64, np.array([-100.0, 0.0, 100.0]))])

# the reference's own tests' inputs
add("ref.small", {"x": (INT32, np.array([3, NA[INT32], 4, 1, 5, 4], np.int32))}, nbins=5)
add("ref.small_open", {"x": (INT32, np.array([3, NA[INT32], 4, 1, 5, 4], np.int32))}, nbins=5, right_closed=False)
add("ref.bool", {"x": (BOOL, np.array([1, 0, NA[BOOL], 1], np.int8))}, nbins=2)

# errors raised when the query runs
e3 = np.array([0.0, 1.0, 2.0])
add("err.by", xs, mode="by")
add("err.by_bins", xs, mode="by", bins=[(FLOAT64, e3)])
add("err.nbins_len", xy, j="list", nbins=[2, 3, 4])
add("err.nbins_len_one", xy, j="one", nbins=[2, 3])
add("err.bins_len", xy, j="list", bins=[(FLOAT64, e3)])
add("err.bins_len_one", xy, j="one", bins=[(FLOAT64, e3), (FLOAT64, e3)])
for st in (DATE32, TIME64):
    add(f"err.{TAGS[st]}", {"x": (st, values(st, 10))})
    add(f"err.{TAGS[st]}_bins", {"x": (st, values(st, 10))}, bins=[(FLOAT64, e3)])
    add(f"err.{TAGS[st]}_second", {"x": (FLOAT64, values(FLOAT64, 10)), "y": (st, values(st, 10))}, j="list")
add("err.other_rows", xy, j="other", other=(FLOAT64, values(FLOAT64, 59)))
add("err.self_islice", xy, j="self", i=["slice", [1, None]])
# errors raised by cut() itself
add("err.nbins_zero", xy, nbins=0)
add("err.nbins_negative", xy, nbins=-4)
add("err.nbins_float", xy, nbins=2.5)
add("err.nbins_bool", xy, nbins=True)
add("err.nbins_large", xy, nbins=2**31)
add("err.nbins_small", xy, nbins=-2**31 - 1)
add("err.nbins_list_zero", xy, j="list", nbins=[3, 0])
add("err.nbins_list_float", xy, j="list", nbins=[3, 1.5])
add("err.right_closed_int", xy, right_closed=1)
add("err.right_closed_str", xy, right_closed="yes")
add("err.both", xy, nbins=3, bins=[(FLOAT64, e3)])
add("err.bins_one_edge", xy, bins=[(FLOAT64, np.array([1.0]))])
add("err.bins_no_edge", xy, bins=[(FLOAT64, np.zeros(0))])
add("err.bins_na", xy, bins=[(FLOAT64, np.array([0.0, np.nan, 2.0]))])
add("err.bins_na_first", xy, bins=[(INT32, np.array([NA[INT32], 1, 2], np.int32))])
add("err.bins_equal", xy, bins=[(FLOAT64, np.array([0.0, 1.0, 1.0]))])
add("err.bins_decreasing", xy, bins=[(FLOAT64, np.array([0.5, 0.25]))])
add("err.bins_i64_collide", xy, bins=[(INT64, np.array([2**53, 2**53 + 1], np.int64))])
add("err.bins_i64_collide_late", xy, bins=[(INT64, np.array([-5, 2**60, 2**60 + 2, 2**61], np.int64))])
add("err.bins_second_frame", xy, j="list", bins=[(FLOAT64, e3), (FLOAT64, np.array([3.0, -1e-7]))])
add("err.bins_date32", xy, bins=[(DATE32, np.array([0, 1], np.int32))])
add("err.bins_inf_equal", xy, bins=[(FLOAT64, np.array([-np.inf, np.inf, np.inf]))])

np.savez_compressed(os.path.join(HERE, "golden_v12.npz"), **arrays)
json.dump({"generator": "tests/golden/make_golden_v12.py", "datatable_version": dt.__version__, "cases": manifest},
          open(os.path.join(HERE, "golden_v12.json"), "w"), indent=0)
print(len(manifest), "cases,", sum(1 for c in manifest if "error" in c), "errors")
