"""
A numpy restatement of CumSumProd_ColumnImpl::materialize (column/cumsumprod.h) and CumMinMax_ColumnImpl::materialize
(column/cumminmax.h) run inside every group, as FExpr_CumSumProd / FExpr_CumMinMax do, and the golden_v7 query shapes
it is checked against (tests/test_oracle_golden_v7.py) and the engine with it (tests/test_gpu_cumulative.py).

`cum_loop` is the reference's loop, row by row in the output column's own type.  `cum_groups` gives the same result
with whole-group numpy operations, for inputs of millions of rows; tests/test_oracle_golden_v7.py checks the two
against each other.
"""
import json
import os

import numpy as np

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64 = 1, 2, 3, 4, 5, 6, 7, 17, 18
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
NPT = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
       FLOAT32: np.float32, FLOAT64: np.float64, DATE32: np.int32, TIME64: np.int64}
FLOATS = (FLOAT32, FLOAT64)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def out_stype(fn, st):
    """fexpr_cumsumprod.cc / fexpr_cumminmax.cc: evaluate1; None = TypeError."""
    if fn in ("cumsum", "cumprod"):
        return INT64 if st in (BOOL, INT8, INT16, INT32, INT64) else (st if st in FLOATS else None)
    return st if st in NPT else None


def _valid(v, st):
    return ~np.isnan(v) if st in FLOATS else v != NA[st]


def cum_loop(fn, v, st, reverse=False):
    """One group, the reference's loop: values in the output stype, NA rows add 0 / multiply by 1 (sum, prod) or
    repeat the previous result (min, max; NA before the first valid row)."""
    ost = out_stype(fn, st)
    T = NPT[ost]
    n = len(v)
    out = np.empty(n, T)
    valid = _valid(v, st)
    idx = range(n - 1, -1, -1) if reverse else range(n)
    with np.errstate(over="ignore", invalid="ignore"):
        if fn in ("cumsum", "cumprod"):
            neutral = T(0) if fn == "cumsum" else T(1)
            prev = None
            for i in idx:
                x = T(v[i]) if valid[i] else neutral
                prev = x if prev is None else (prev + x if fn == "cumsum" else prev * x)
                out[i] = prev
        else:
            prev, res_valid = None, False
            for i in idx:
                if prev is None:
                    res_valid = bool(valid[i])
                    out[i] = v[i] if res_valid else NA.get(ost, np.nan)
                elif valid[i]:
                    keep = res_valid and (prev < v[i] if fn == "cummin" else prev > v[i])
                    out[i] = prev if keep else v[i]
                    res_valid = True
                else:
                    out[i] = prev
                prev = out[i]
    return out


def _cum_fast(fn, v, st):
    """cum_loop (forward) with whole-array numpy operations: integer sums and products wrap as numpy's int64 does;
    float sums and products run in order in the column's type (np.cumsum / np.cumprod accumulate sequentially); min /
    max take the latest row whose value equals the running extreme."""
    ost = out_stype(fn, st)
    T = NPT[ost]
    valid = _valid(v, st)
    with np.errstate(over="ignore", invalid="ignore"):
        if fn in ("cumsum", "cumprod"):
            c = np.where(valid, v, 0 if fn == "cumsum" else 1).astype(T)
            return (np.cumsum if fn == "cumsum" else np.cumprod)(c, dtype=T)
        if st in FLOATS:
            w = np.where(valid, v, np.inf if fn == "cummin" else -np.inf)
        else:
            info = np.iinfo(NPT[st])
            w = np.where(valid, v, info.max if fn == "cummin" else info.min)
        m = (np.minimum if fn == "cummin" else np.maximum).accumulate(w)
        take = valid & (v == m)
        last = np.maximum.accumulate(np.where(take, np.arange(len(v)), -1))
        out = np.where(last >= 0, v[np.maximum(last, 0)], NA.get(ost, np.nan)).astype(T)
    return out


def cum_groups(fn, v, st, order, offsets, reverse=False, loop=False):
    """fn inside every group of (order, offsets): one value per RowIndex position (the grouped order, GtoALL)."""
    offsets = np.asarray(offsets, dtype=np.int64)
    n = int(offsets[-1]) if len(offsets) else 0
    vals = np.asarray(v)[np.arange(n) if order is None else np.asarray(order, dtype=np.int64)]
    out = np.empty(n, NPT[out_stype(fn, st)])
    for g in range(len(offsets) - 1):
        a, b = offsets[g], offsets[g + 1]
        seg = vals[a:b]
        if loop:
            out[a:b] = cum_loop(fn, seg, st, reverse)
        else:
            out[a:b] = _cum_fast(fn, seg[::-1], st)[::-1] if reverse else _cum_fast(fn, seg, st)
    return out


# ---- golden_v7 ------------------------------------------------------------------------------------------------------
def load_golden():
    cases = json.load(open(os.path.join(GOLDEN, "golden_v7.json")))["cases"]
    arr = dict(np.load(os.path.join(GOLDEN, "golden_v7.npz")))
    return cases, arr


def int_slice(i):
    """An integer i is the slice [i, i+1) (fexpr_literal_int.cc:146-192)."""
    if isinstance(i, int):
        return [i, i + 1 if i != -1 else None, 1]
    return list(i) + [None] * (3 - len(i))


def by_names(case):
    return {"by": ["ka"], "by2": ["ka", "kb"], "bysort": ["ka"]}.get(case["mode"], [])


def j_columns(case):
    """[(kind, source column)] of the case's j, in output order (kind: cum | plain | qcut)."""
    j = case["j"]
    if j in ("one", "dict"):
        return [("cum", "x")]
    if j in ("list", "tuple", "dictlist"):
        return [("cum", "x"), ("cum", "y")]
    if j == "all":
        return [("cum", nm) for nm in case["stypes"] if nm not in by_names(case)]
    if j == "plain":
        return [("plain", "x"), ("cum", "x")]
    if j == "withqcut":
        return [("cum", "x"), ("qcut", "y")]
    return [("cum", "ka")]                                        # bykey


def case_groups(case, arr, orc):
    """(order, offsets) of the case's query, formed by the C oracle `orc`: the RowIndex (None = identity) and the
    groups the function runs in (one group without by())."""
    name, mode = case["name"], case["mode"]
    n = len(arr[name + "." + next(iter(case["stypes"]))])
    i = case["i"]
    if mode == "none":
        rows = np.arange(n, dtype=np.int32)
        if i is not None:
            rows = rows[[i % n]] if isinstance(i, int) else rows[slice(*i)]
        order = None if i is None else rows
        return order, np.array([0, len(rows)] if len(rows) else [0], dtype=np.int32)
    keys = [arr[name + "." + k] for k in by_names(case)]
    flags = [0] * len(keys)
    if mode in ("bysort", "sort", "sortdesc"):
        keys.append(arr[name + ".s"])
        flags.append(orc.SORT_ONLY | (orc.DESCENDING if mode == "sortdesc" else 0))
    order, offsets, _ = orc.group(keys, flags, orc.NA_FIRST)
    if offsets is None:
        offsets = np.array([0, len(order)] if len(order) else [0], dtype=np.int32)
    if i is not None:
        pos, offsets = orc.slice_groups(offsets, *int_slice(i))
        order = order[pos]
    return order, np.asarray(offsets, dtype=np.int32)


def expected_columns(case, arr, orc, loop=True, qcut=None):
    """[(name, values)] the restatement gives for the case: by() columns first, then j.  qcut: the qcut restatement
    (tests/qcut_reference.py: qcut_groups) for the j form that puts one next to the cumulative function."""
    order, offsets = case_groups(case, arr, orc)
    rows = (lambda c: c) if order is None else (lambda c: c[np.asarray(order, dtype=np.int64)])
    name = case["name"]
    out = [rows(arr[name + "." + k]) for k in by_names(case)]
    for kind, src in j_columns(case):
        v = arr[name + "." + src]
        if kind == "plain":
            out.append(rows(v))
        elif kind == "qcut":
            out.append(qcut(v, case["stypes"][src], order, offsets, 10))
        else:
            out.append(cum_groups(case["fn"], v, case["stypes"][src], order, offsets, case["rev"], loop=loop))
    return list(zip(case["names"], out))
