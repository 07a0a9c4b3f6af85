"""
A numpy restatement of the reference's grouped row functions shift, fillna, cumcount and ngroup, and the golden_v8
query shapes it is checked against (tests/test_oracle_golden_v8.py) and the engine with it (tests/test_gpu_window.py).

    lag_rowindex         compute_lag_rowindex (expr/head_func_shift.cc:40-64): shift under by()
    shift_rowindex       Shift_ColumnImpl (column/shift.h:37-88): shift of the whole selected column without by()
    fill_rowindex        FExpr_FillNA::fill_rowindex (expr/fexpr_fillna.cc:66-118)
    cumcount_ngroup      CumcountNgroup_ColumnImpl::materialize (column/cumcountngroup.h:48-66)

Each returns, per position of the grouped order, the source position (-1 = NA) or the int64 result, written as the
reference's loops are.  The *_fast forms give the same results with whole-array operations for inputs of millions of
rows; tests/test_oracle_golden_v8.py checks the two against each other.  Positions are int64 here, so the rule "a
source outside the group is NA" holds for every shift; the reference computes them in int32 / size_t, and its results
where that overflows are not pinned.
"""
import json
import os

import numpy as np

from cumulative_reference import (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64, NA, NPT, FLOATS,
                                  by_names, case_groups)

__all__ = ["BOOL", "INT8", "INT16", "INT32", "INT64", "FLOAT32", "FLOAT64", "DATE32", "TIME64", "NA", "NPT", "FLOATS",
           "case_groups", "load_golden", "make_j", "j_columns", "expected_columns", "row_fn", "row_fn_fast",
           "lag_rowindex", "shift_rowindex", "fill_rowindex", "cumcount_ngroup"]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NULLARY = ("cumcount", "ngroup")


def _valid(v, st):
    return ~np.isnan(v) if st in FLOATS else v != NA[st]


def _na_like(st):
    return np.nan if st in FLOATS else NA[st]


# ---- the reference's loops ------------------------------------------------------------------------------------------
def lag_rowindex(offsets, shift):
    """compute_lag_rowindex<shift > 0>: per group [j0, j2), position j takes j - shift, NA (-1) for the first
    min(shift, size) positions; a lead (shift < 0) takes j + |shift|, NA for the last |shift| positions."""
    n = int(offsets[-1]) if len(offsets) else 0
    idx = np.empty(n, np.int64)
    for g in range(len(offsets) - 1):
        j0, j2 = int(offsets[g]), int(offsets[g + 1])
        if shift > 0:
            j1 = min(j2, j0 + shift)
            idx[j0:j1] = -1
            idx[j1:j2] = np.arange(j1, j2) - shift
        else:
            j1 = max(j0, j2 + shift)
            idx[j0:j1] = np.arange(j0, j1) - shift
            idx[j1:j2] = -1
    return idx


def shift_rowindex(nrows, shift):
    """Shift_ColumnImpl<LAG>::_elem over one column of nrows rows: i < shift -> NA, else i - shift (LAG); i >= nrows -
    |shift| -> NA, else i + |shift| (lead), with nrows - |shift| taken as 0 where |shift| > nrows."""
    i = np.arange(nrows, dtype=np.int64)
    if shift > 0:
        return np.where(i < shift, -1, i - shift)
    return np.where(i >= max(nrows + shift, 0), -1, i - shift)


def fill_rowindex(valid, offsets, reverse):
    """fill_rowindex<REVERSE>: per group, the position of the latest valid row so far (REVERSE: scanning from the
    group's end); before the first valid row the group's first (last) position, itself NA."""
    n = int(offsets[-1]) if len(offsets) else 0
    idx = np.empty(n, np.int64)
    for g in range(len(offsets) - 1):
        i1, i2 = int(offsets[g]), int(offsets[g + 1])
        fill_id = i2 - 1 if reverse else i1
        for i in (range(i2 - 1, i1 - 1, -1) if reverse else range(i1, i2)):
            fill_id = i if valid[i] else fill_id
            idx[i] = fill_id
    return idx


def cumcount_ngroup(offsets, cumcount, reverse):
    n = int(offsets[-1]) if len(offsets) else 0
    ng = len(offsets) - 1
    out = np.empty(n, np.int64)
    for gi in range(ng):
        i1, i2 = int(offsets[gi]), int(offsets[gi + 1])
        i = np.arange(i1, i2, dtype=np.int64)
        if reverse:
            out[i1:i2] = (i2 - i - 1) if cumcount else ng - gi - 1
        else:
            out[i1:i2] = (i - i1) if cumcount else gi
    return out


def _take(vals, st, idx):
    out = np.full(len(idx), _na_like(st), NPT[st])
    ok = idx >= 0
    out[ok] = vals[idx[ok]]
    return out


def row_fn(fn, vals, st, offsets, grouped, rev=False, n=1):
    """fn over the values already in the grouped order (`vals`, one per position; None for cumcount / ngroup) and the
    groups `offsets`, as the reference evaluates it: `grouped` = the query has by() (has_groupby); without it shift
    runs Shift_ColumnImpl over the selected rows, cumcount is 0 .. n-1 (reversed) and ngroup 0, and fillna runs in
    the one group of the selected rows."""
    offsets = np.asarray(offsets, dtype=np.int64)
    if fn in NULLARY:
        if not grouped:
            offsets = np.array([0, offsets[-1]] if len(offsets) > 1 and offsets[-1] else [0], np.int64)
        return cumcount_ngroup(offsets, fn == "cumcount", rev)
    if fn == "shift":
        if n == 0:
            return vals.copy()
        return _take(vals, st, lag_rowindex(offsets, n) if grouped else shift_rowindex(len(vals), n))
    return _take(vals, st, fill_rowindex(_valid(vals, st), offsets, rev))


# ---- whole-array forms ----------------------------------------------------------------------------------------------
def row_fn_fast(fn, vals, st, offsets, rev=False, n=1):
    """fn inside every group of `offsets` (one group [0, n] stands for a query without by()) with whole-array numpy
    operations: shift takes position p - n where that lies in p's group, fillna the latest (reverse: earliest) valid
    position of the group at or before (after) p, cumcount and ngroup the position in the group and the group."""
    offsets = np.asarray(offsets, dtype=np.int64)
    npos = int(offsets[-1]) if len(offsets) > 1 else 0
    ng = len(offsets) - 1
    gid = np.repeat(np.arange(ng, dtype=np.int64), np.diff(offsets))
    p = np.arange(npos, dtype=np.int64)
    start, end = offsets[:-1][gid], offsets[1:][gid]
    if fn == "cumcount":
        return end - 1 - p if rev else p - start
    if fn == "ngroup":
        return ng - 1 - gid if rev else gid
    if fn == "shift":
        src = p - np.int64(n)
        return _take(vals, st, np.where((src >= start) & (src < end), src, -1))
    valid = _valid(vals, st)
    if rev:
        last = np.minimum.accumulate(np.where(valid, p, npos)[::-1])[::-1]
        return _take(vals, st, np.where(last < end, last, -1))
    last = np.maximum.accumulate(np.where(valid, p, -1))
    return _take(vals, st, np.where(last >= start, last, -1))


# ---- golden_v8 ------------------------------------------------------------------------------------------------------
def load_golden():
    cases = json.load(open(os.path.join(GOLDEN, "golden_v8.json")))["cases"]
    arr = dict(np.load(os.path.join(GOLDEN, "golden_v8.npz")))
    return cases, arr


def _call(M, fn, cols, rev, n):
    if fn == "shift":
        return M.shift(cols, n=n)
    if fn == "fillna":
        return M.fillna(cols, reverse=rev)
    return getattr(M, fn)(reverse=rev)


def make_j(M, case, DT):
    """The j of a golden case, built from module M (the reference's datatable or datatable_b200) for the frame DT.
    fn: shift, fillna, cumcount, ngroup, or mix (the four together in a dict); j: one, list, tuple, all = f[:], dict,
    dictlist, plain = [f.x, fn], withqcut = [fn, qcut(f.y)], withcum = [fn, cumsum(f.y)], bykey = fn of the by()
    column, both = [cumcount, ngroup], frame = shift(DT, n)."""
    fn, rev, n, j, f = case["fn"], case["rev"], case["n"], case["j"], M.f
    F = (lambda cols=None: _call(M, fn, cols, rev, n))
    if fn == "mix":
        return {"lag": M.shift(f.x, n=n), "filled": M.fillna(f.x, reverse=rev), "i": M.cumcount(reverse=rev),
                "g": M.ngroup(reverse=rev)}
    nullary = fn in NULLARY
    x, y = (None, None) if nullary else (f.x, f.y)
    if j == "one":
        return F(x)
    if j == "list":
        return F([f.x, f.y]) if fn == "fillna" else [F(x), F(y)]
    if j == "tuple":
        return F((f.x, f.y)) if fn == "fillna" else (F(x), F(y))
    if j == "all":
        return F(f[:])
    if j == "dict":
        return {"c": F(x)}
    if j == "dictlist":
        return {"c": F([f.x, f.y])}
    if j == "plain":
        return [f.x, F(x)]
    if j == "withqcut":
        return [F(x), M.qcut(f.y)]
    if j == "withcum":
        return [F(x), M.cumsum(f.y)]
    if j == "both":
        return [M.cumcount(reverse=rev), M.ngroup(reverse=not rev)]
    if j == "frame":
        return None                                                # shift(DT, n): the query is the call itself
    return F(f.ka)                                                 # bykey


def query(M, case, DT):
    J = make_j(M, case, DT)
    if case["j"] == "frame":
        return M.shift(DT, case["n"])
    f, i = M.f, case["i"]
    rows = slice(None) if i is None else (i if isinstance(i, int) else slice(*i))
    mods = {"none": (), "by": (M.by(f.ka),), "by2": (M.by(f.ka, f.kb),), "bysort": (M.by(f.ka), M.sort(f.s)),
            "sort": (M.sort(f.s),), "sortdesc": (M.sort(-f.s),)}[case["mode"]]
    return DT[(rows, J) + mods]


def j_columns(case):
    """[(kind, source column or None, reverse)] of the case's j in output order; kind: shift, fillna, cumcount,
    ngroup, plain, qcut or cumsum."""
    fn, rev, j = case["fn"], case["rev"], case["j"]
    if fn == "mix":
        return [("shift", "x", False), ("fillna", "x", rev), ("cumcount", None, rev), ("ngroup", None, rev)]
    src = (lambda c: None) if fn in NULLARY else (lambda c: c)
    if j in ("one", "dict"):
        return [(fn, src("x"), rev)]
    if j in ("list", "tuple", "dictlist"):
        return [(fn, src("x"), rev), (fn, src("y"), rev)]
    if j in ("all", "frame"):
        return [(fn, nm, rev) for nm in case["stypes"] if nm not in by_names(case)]
    if j == "plain":
        return [("plain", "x", rev), (fn, src("x"), rev)]
    if j == "withqcut":
        return [(fn, src("x"), rev), ("qcut", "y", rev)]
    if j == "withcum":
        return [(fn, src("x"), rev), ("cumsum", "y", rev)]
    if j == "both":
        return [("cumcount", None, rev), ("ngroup", None, not rev)]
    return [(fn, "ka", rev)]                                       # bykey


def expected_columns(case, arr, orc, loop=True, qcut=None, cum=None):
    """[(name, values)] the restatement gives for the case: by() columns first, then j.  qcut / cum: the restatements
    of qcut (tests/qcut_reference.py: qcut_groups) and cumsum (tests/cumulative_reference.py: cum_groups) for the j
    forms that put one next to the row function.  loop: the reference's loops, else the whole-array forms."""
    order, offsets = case_groups(case, arr, orc)
    rows = (lambda c: c) if order is None else (lambda c: c[np.asarray(order, dtype=np.int64)])
    name = case["name"]
    grouped = case["mode"] in ("by", "by2", "bysort")
    out = [rows(arr[name + "." + k]) for k in by_names(case)]
    for kind, src, rev in j_columns(case):
        st = case["stypes"].get(src)
        v = None if src is None else arr[name + "." + src]
        if kind == "plain":
            out.append(rows(v))
        elif kind == "qcut":
            out.append(qcut(v, st, order, offsets, 10))
        elif kind == "cumsum":
            out.append(cum("cumsum", v, st, order, offsets, False))
        elif loop:
            out.append(row_fn(kind, None if v is None else rows(v), st, offsets, grouped, rev, case["n"]))
        else:
            out.append(row_fn_fast(kind, None if v is None else rows(v), st, offsets, rev, case["n"]))
    return list(zip(case["names"], out))
