"""
A numpy restatement of CutNbins_ColumnImpl and CutBins_ColumnImpl (column/cut.h:91-281) as FExpr_Cut::evaluate_n runs
them (expr/fexpr_cut.cc:88-170), and the golden_v12 query shapes it is checked against (tests/test_oracle_golden_v12.py)
and the engine with it (tests/test_gpu_cut.py).  It shares no code with the engine.

Values are scaled in float64 as the reference computes them: a multiply, then an add, each rounded (numpy runs them as
two operations), truncated as x86-64 converts a double to int32 (INT32_MIN for NaN and out-of-range values), and the
shift added with int32 wrap-around.  Explicit edges are an np.searchsorted.
"""
import json
import os

import numpy as np

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64 = 1, 2, 3, 4, 5, 6, 7, 17, 18
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
NA_INT32 = -2**31
FLT_EPSILON = 2.0**-23
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def as_float64(v, st):
    """(values as float64, valid mask): int64 rounds to nearest, NaN and the integer sentinels are NA."""
    v = np.asarray(v)
    if st in (FLOAT32, FLOAT64):
        with np.errstate(invalid="ignore"):                       # float32 NaN payloads
            x = v.astype(np.float64)
        return x, ~np.isnan(x)
    return v.astype(np.float64), v != NA[st]


def _trunc_i32(r):
    """static_cast<int32_t>(r) on x86-64: truncation; NaN and values outside the int32 range give INT32_MIN."""
    t = np.trunc(r)
    ok = (t >= -2.0**31) & (t < 2.0**31)
    return np.where(ok, np.where(ok, t, 0).astype(np.int64), NA_INT32)


def cut_nbins(v, st, nbins, right_closed=True, bounds=None):
    """Equal-width bins of column v (its rows as evaluated): int32, NA as INT32_MIN.  bounds: the (min, max) of the
    valid values of the whole column when v is a piece of it."""
    x, valid = as_float64(v, st)
    out = np.full(len(x), NA_INT32, dtype=np.int32)
    if bounds is None and not valid.any():
        return out
    mn, mx = (x[valid].min(), x[valid].max()) if bounds is None else bounds
    if np.isinf(mn) or np.isinf(mx):
        return out
    rc = 1 if right_closed else 0
    shift = 0
    with np.errstate(all="ignore"):
        if mn == mx:
            a, b = np.float64(0.0), np.float64((nbins - rc) // 2)
        else:
            a = np.float64((1 - FLT_EPSILON) * nbins) / np.float64(mx - mn)
            b = -a * mn
            if not right_closed:
                b = -a * mx
                shift = nbins - 1
        r = np.add(np.multiply(a, x[valid]), b)
    bins = (_trunc_i32(r) + shift) & 0xFFFFFFFF
    out[valid] = bins.astype(np.uint32).view(np.int32)
    return out


def cut_bins(v, st, edges, right_closed=True):
    """Bins of column v between the float64 edges: v in (e[0], e[-1]] (right-closed) or [e[0], e[-1])."""
    x, valid = as_float64(v, st)
    e = np.asarray(edges, dtype=np.float64)
    c = np.searchsorted(e, x, side="left" if right_closed else "right")      # #{e < v} or #{e <= v}
    ok = valid & (c >= 1) & (c <= len(e) - 1)
    return np.where(ok, c - 1, NA_INT32).astype(np.int32)


def at_rows(v, st, rows):
    """Column v seen through a RowIndex: an index < 0 is an NA row."""
    v = np.asarray(v)
    if rows is None:
        return v
    rows = np.asarray(rows, dtype=np.int64)
    na = np.float64("nan") if st in (FLOAT32, FLOAT64) else NA[st]
    return np.where(rows >= 0, v[np.clip(rows, 0, max(len(v) - 1, 0))] if len(v) else na, na).astype(v.dtype)


def cut_column(v, st, nbins=10, edges=None, right_closed=True):
    return cut_nbins(v, st, nbins, right_closed) if edges is None else cut_bins(v, st, edges, right_closed)


# ---- golden_v12 -----------------------------------------------------------------------------------------------------
def load_golden():
    cases = json.load(open(os.path.join(GOLDEN, "golden_v12.json")))["cases"]
    arr = dict(np.load(os.path.join(GOLDEN, "golden_v12.npz")))
    return cases, arr


def case_edges(case, arr):
    """The cases's bin edges as float64 arrays (int64 rounded to nearest), or None."""
    if "bins" not in case:
        return None
    return [np.asarray(arr[b["key"]]).astype(np.float64) for b in case["bins"]]


def case_rows(case, arr, orc):
    """The RowIndex of the case's query (None = every row in place), formed on the host; sort() by the C oracle."""
    name, mode, i = case["name"], case["mode"], case["i"]
    n = len(arr[name + ".x"])
    if mode in ("sort", "sortdesc", "sortlast", "sortremove"):
        key = "s" if mode in ("sort", "sortdesc") else "x"
        na_pos = {"sortlast": orc.NA_LAST, "sortremove": orc.NA_REMOVE}.get(mode, orc.NA_FIRST)
        flags = [orc.SORT_ONLY | (orc.DESCENDING if mode == "sortdesc" else 0)]
        order, _, _ = orc.group([arr[name + "." + key]], flags, na_pos)
        order = np.asarray(order, dtype=np.int64)
        if i is not None:
            start, stop, step = [i[1], i[1] + 1 if i[1] != -1 else None, 1] if i[0] == "int" else i[1]
            order = order[slice(start, stop, step)]
        return order
    if i is None:
        return None
    kind, p = i
    if kind == "slice":
        return np.arange(n)[slice(*p)]
    if kind == "int":
        return np.array([p % n])
    if kind == "bool":
        return np.flatnonzero(arr[name + "." + p] == 1)
    if kind == "frame":
        sel = arr[name + ".isel"].astype(np.int64)
        return np.where(sel == NA[INT32], -1, sel)
    if kind == "list":
        return np.array([k % n for k in p], dtype=np.int64)
    return np.array([k % n for k in range(*p)], dtype=np.int64)                # range


def j_sources(case):
    """[(output index, source)] of the case's cut outputs: source = ("x", col), ("J", col) or ("frame", col)
    (the Frame's own column, no RowIndex)."""
    j = case["j"]
    cols = {"one": ["x"], "dict": ["x"], "qcut": ["x"], "cumsum": ["x"], "shift": ["x"], "list": ["x", "y"],
            "tuple": ["x", "y"], "dictlist": ["x", "y"], "all": list(case["stypes"])}.get(j)
    if cols is not None:
        return [(k, ("x", c)) for k, c in enumerate(cols)]
    if j == "plain":
        return [(1, ("x", "x"))]
    if j == "self":
        return [(k, ("frame", c)) for k, c in enumerate(case["stypes"])]
    if j == "other":
        return [(0, ("other", "z"))]
    if j == "joincol":
        return [(0, ("J", "v"))]
    return [(0, ("x", "x")), (1, ("J", "v"))]                       # joinlist


def source_column(case, arr, src, rows):
    """(values at the query's rows, stype) of a cut input."""
    name = case["name"]
    kind, c = src
    if kind == "frame":
        return arr[name + "." + c], case["stypes"][c]
    if kind == "other":
        return arr[name + ".other.z"], case["other_stype"]
    if kind == "J":
        k = arr[name + ".k"].astype(np.int64)
        jk = arr[name + ".J.k"].astype(np.int64)
        pos = {int(key): r for r, key in enumerate(jk)}
        idx = np.array([pos.get(int(key), -1) if key != NA[INT32] else -1 for key in k], dtype=np.int64)
        st = case["jstypes"][c]
        return at_rows(at_rows(arr[name + ".J." + c], st, idx), st, rows), st
    st = case["stypes"][c]
    return at_rows(arr[name + "." + c], st, rows), st


def expected_cuts(case, arr, orc):
    """[(output index, int32 bins)] the restatement gives for the case's cut outputs."""
    rows = case_rows(case, arr, orc)
    edges = case_edges(case, arr)
    nb = case["nbins"]
    nbs = nb if isinstance(nb, list) else [10 if nb is None else nb]
    rc = True if case["right_closed"] is None else case["right_closed"]
    out = []
    for k, (idx, src) in enumerate(j_sources(case)):
        v, st = source_column(case, arr, src, rows)
        out.append((idx, cut_column(v, st, nbs[k % len(nbs)], None if edges is None else edges[k], rc)))
    return out


def frame_query(dtb, case, arr, device=False):
    """The case's query on the Frame of module dtb (datatable_b200)."""
    name = case["name"]
    f, g = dtb.f, dtb.g

    def mk(cols, stypes):
        fr = dtb.Frame(cols, stypes=stypes)
        return fr.to_device() if device else fr

    DT = mk({nm: arr[name + "." + nm] for nm in case["stypes"]}, case["stypes"])
    kw = {}
    if case["nbins"] is not None:
        kw["nbins"] = tuple(case["nbins"]) if case.get("nbins_tuple") else case["nbins"]
    if "bins" in case:
        kw["bins"] = [mk({"C0": arr[b["key"]]}, {"C0": b["stype"]}) for b in case["bins"]]
    if case["right_closed"] is not None:
        kw["right_closed"] = case["right_closed"]
    cut = lambda c: dtb.cut(c, **kw)           # noqa: E731
    J = None
    if "jstypes" in case:
        J = mk({nm: arr[name + ".J." + nm] for nm in case["jstypes"]}, case["jstypes"])
        J.key = "k"
    other = None
    if "other_stype" in case:
        other = mk({"z": arr[name + ".other.z"]}, {"z": case["other_stype"]})
    j = {"one": lambda: cut(f.x), "list": lambda: cut([f.x, f.y]), "tuple": lambda: cut((f.x, f.y)),
         "all": lambda: cut(f[:]), "dict": lambda: {"c": cut(f.x)}, "dictlist": lambda: {"c": cut([f.x, f.y])},
         "plain": lambda: [f.x, cut(f.x)], "qcut": lambda: [cut(f.x), dtb.qcut(f.x)],
         "cumsum": lambda: [cut(f.x), dtb.cumsum(f.y)], "shift": lambda: [cut(f.x), dtb.shift(f.x)],
         "self": lambda: cut(DT), "other": lambda: cut(other), "joincol": lambda: cut(g.v),
         "joinlist": lambda: cut([f.x, g.v])}[case["j"]]()
    i = case["i"]
    if i is None:
        rows = slice(None)
    else:
        kind, p = i
        rows = {"slice": lambda: slice(*p), "int": lambda: p, "bool": lambda: f[p],
                "frame": lambda: mk({"C0": arr[name + ".isel"]}, {"C0": INT32}),
                "list": lambda: list(p), "range": lambda: range(*p)}[kind]()
    mods = {"none": (), "sort": (dtb.sort(f.s),), "sortdesc": (dtb.sort(-f.s),),
            "sortlast": (dtb.sort(f.x, na_position="last"),), "sortremove": (dtb.sort(f.x, na_position="remove"),),
            "by": (dtb.by(f.s),), "join": (dtb.join(J),) if J is not None else ()}[case["mode"]]
    return DT[(rows, j) + mods]
