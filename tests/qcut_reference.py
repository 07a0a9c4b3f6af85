"""
A numpy restatement of Qcut_ColumnImpl::materialize (column/qcut.h:78-155) and of FExpr_Qcut::evaluate_n's loop over
the groups (expr/fexpr_qcut.cc:118-146), and the golden_v6 query shapes it is checked against
(tests/test_oracle_golden_v6.py) and the engine with it (tests/test_gpu_qcut.py).

Values are told apart as group() tells them: by bit pattern (-0.0 and +0.0 are two values), every NaN is the NA value,
NA first.  The bin is computed in float64 as the reference computes it, a multiply and an add, each rounded.
"""
import json
import os

import numpy as np

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64 = 1, 2, 3, 4, 5, 6, 7, 17, 18
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
NA_INT32 = -2**31
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def value_ranks(vals, st):
    """(na mask, rank of every valid value among the distinct valid values in group()'s order)."""
    vals = np.asarray(vals)
    if st in (FLOAT32, FLOAT64):
        na = np.isnan(vals)
        ui, sign = (np.uint32, np.uint32(1 << 31)) if st == FLOAT32 else (np.uint64, np.uint64(1 << 63))
        bits = vals.view(ui)
        image = np.where(bits & sign, ~bits, bits | sign)         # order-preserving image: -0.0 sorts below +0.0
    else:
        na = vals == NA[st]
        image = vals.astype(np.int64)
    ranks = np.zeros(len(vals), dtype=np.int64)
    if (~na).any():
        _, inv = np.unique(image[~na], return_inverse=True)
        ranks[~na] = inv.reshape(-1)
    return na, ranks


def qcut_column(vals, st, q):
    """Qcut_ColumnImpl::materialize on one column: int32 bins, NA as INT32_MIN."""
    n = len(vals)
    out = np.full(n, NA_INT32, dtype=np.int32)
    if n == 0:
        return out
    na, ranks = value_ranks(vals, st)
    has_na = bool(na.any())
    V = int(ranks[~na].max()) + 1 if (~na).any() else 0
    if V <= 1:                                                    # one group (qcut.h:90-105) or one valid value
        a, b = 0.0, float((q - 1) // 2)
    else:
        a = q * (1 - 2.0**-23) / float(V - 1)
        b = -a * float(has_na)
    i = (ranks + int(has_na)).astype(np.float64)
    bins = (a * i + b)                                            # numpy: two operations, each rounded
    out[~na] = np.trunc(bins[~na]).astype(np.int32)
    return out


def qcut_groups(v, st, order, offsets, q):
    """qcut inside every group of (order, offsets): bins in the grouped order (GtoALL), one per RowIndex position."""
    offsets = np.asarray(offsets, dtype=np.int64)
    n = int(offsets[-1]) if len(offsets) else 0
    rows = np.arange(n) if order is None else np.asarray(order, dtype=np.int64)
    out = np.empty(n, dtype=np.int32)
    for g in range(len(offsets) - 1):
        p0, p1 = offsets[g], offsets[g + 1]
        out[p0:p1] = qcut_column(np.asarray(v)[rows[p0:p1]], st, q)
    return out


# ---- golden_v6 ------------------------------------------------------------------------------------------------------
def load_golden():
    cases = json.load(open(os.path.join(GOLDEN, "golden_v6.json")))["cases"]
    arr = dict(np.load(os.path.join(GOLDEN, "golden_v6.npz")))
    return cases, arr


def int_slice(i):
    """An integer i is the slice [i, i+1) (fexpr_literal_int.cc:146-192)."""
    if isinstance(i, int):
        return [i, i + 1 if i != -1 else None, 1]
    return list(i) + [None] * (3 - len(i))


def by_names(case):
    return {"by": ["ka"], "by2": ["ka", "kb"], "bysort": ["ka"]}.get(case["mode"], [])


def j_columns(case):
    """[(kind, source column, nquantiles)] of the case's j, in output order (kind: qcut | plain)."""
    j, q = case["j"], case["q"]
    if j in ("one", "dict"):
        srcs = ["x"]
    elif j in ("list", "tuple", "dictlist"):
        srcs = ["x", "y"]
    elif j == "all":
        srcs = [nm for nm in case["stypes"] if nm not in by_names(case)]
    elif j == "plain":
        return [("plain", "x", None), ("qcut", "x", 10 if q is None else q)]
    else:                                                         # bykey
        srcs = ["ka"]
    qs = list(q) if isinstance(q, (list, tuple)) else [10 if q is None else q] * len(srcs)
    return [("qcut", s, qq) for s, qq in zip(srcs, qs)]


def case_groups(case, arr, orc):
    """(order, offsets, grouped) of the case's query, formed by the C oracle `orc`: the RowIndex (None = identity),
    the groups qcut runs in (one group without by()) and whether there is a Groupby."""
    name, mode = case["name"], case["mode"]
    n = len(arr[name + ".x"])
    i = case["i"]
    if mode == "none":
        rows = np.arange(n, dtype=np.int32)
        if i is not None:
            rows = rows[[i % n]] if isinstance(i, int) else rows[slice(*i)]
        order = None if i is None else rows
        return order, np.array([0, len(rows)] if len(rows) else [0], dtype=np.int32), False
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
    return order, np.asarray(offsets, dtype=np.int32), mode in ("by", "by2", "bysort")


def expected_columns(case, arr, orc):
    """[(name, values)] the restatement gives for the case: by() columns first, then j."""
    order, offsets, grouped = case_groups(case, arr, orc)
    rows = (lambda c: c) if order is None else (lambda c: c[np.asarray(order, dtype=np.int64)])
    name = case["name"]
    out = [rows(arr[name + "." + k]) for k in by_names(case)]
    for kind, src, q in j_columns(case):
        v = arr[name + "." + src]
        if kind == "plain":
            out.append(rows(v))
        elif grouped:
            out.append(qcut_groups(v, case["stypes"][src], order, offsets, q))
        else:
            n = int(offsets[-1]) if len(offsets) > 1 else 0
            out.append(qcut_groups(v, case["stypes"][src], order, np.array([0, n] if n else [0]), q))
    return list(zip(case["names"], out))
