"""A numpy restatement of what the reference's reducers give for a group without rows, and of the stypes of their
results (expr/fexpr_sumprod.cc, fexpr_mean.cc, fexpr_minmax.cc, fexpr_count*.cc, head_reduce_unary.cc,
head_reduce_binary.cc).

    sum               0 (int64 over bool8 / integers, the column's own float stype otherwise)
    prod              1 (the same stypes as sum)
    count, countna,
    nunique, count()  0 (int64)
    mean, sd          NA (float64, float32 over float32)
    min, max, first,
    last              NA of the column's own stype
    median            NA: float64 (float32 over float32) for an empty group among others; over a frame or selection
                      of zero rows the reference returns an NA column of the argument's own stype (compute_median,
                      head_reduce_unary.cc:493-496), and the Frame follows it
    cov, corr         NA (float32 when both columns are float32, else float64)
"""
import numpy as np

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64 = 1, 2, 3, 4, 5, 6, 7
FLOATS = (FLOAT32, FLOAT64)
NPT = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
       FLOAT32: np.float32, FLOAT64: np.float64}
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63}
# the C-ABI's op codes (include/dtb200.h)
SUM, MEAN, MIN, MAX, COUNT, COUNTNA, NROWS, FIRST, LAST, SD, MEDIAN, NUNIQUE, PROD, COV, CORR = range(1, 16)
OPS = {"sum": SUM, "prod": PROD, "mean": MEAN, "min": MIN, "max": MAX, "count": COUNT, "count0": NROWS,
       "countna": COUNTNA, "first": FIRST, "last": LAST, "sd": SD, "median": MEDIAN, "nunique": NUNIQUE, "cov": COV,
       "corr": CORR}                                  # in the order of tests/golden/make_golden_v13.py's red.*.all


def na_of(st):
    return np.nan if st in FLOATS else NA[st]


def out_stype(op, st, st2=FLOAT64):
    """The stype of reducer op over a column of stype st (cov / corr: and st2) in a Groupby with groups."""
    if op in (COUNT, COUNTNA, NROWS, NUNIQUE):
        return INT64
    if op in (SUM, PROD):
        return st if st in FLOATS else INT64
    if op in (MEAN, SD, MEDIAN):
        return FLOAT32 if st == FLOAT32 else FLOAT64
    if op in (MIN, MAX, FIRST, LAST):
        return st
    return FLOAT32 if st == FLOAT32 and st2 == FLOAT32 else FLOAT64


def empty_group(op, st, st2=FLOAT64, zero_rows=False):
    """(the one-element result of reducer op over a group without rows, its stype).  zero_rows: the reducer's
    argument has no rows at all (a frame or a selection of zero rows), where median keeps the argument's stype."""
    ost = st if (op == MEDIAN and zero_rows) else out_stype(op, st, st2)
    if op in (COUNT, COUNTNA, NROWS, NUNIQUE, SUM):
        v = 0
    elif op == PROD:
        v = 1
    else:
        v = na_of(ost)
    return np.array([v], dtype=NPT[ost]), ost


def reduce_rows(op, vals, st):
    """Reducer op over the values `vals` (a numpy array of stype st, NA sentinels included) of one group: the
    restatement for groups whose positions lie beyond the value column (read as NA)."""
    valid = ~np.isnan(vals) if st in FLOATS else vals != NA[st]
    x = vals[valid]
    ost = out_stype(op, st)
    if op == NROWS:
        return np.array([len(vals)], np.int64), INT64
    if op == COUNTNA:
        return np.array([len(vals) - len(x)], np.int64), INT64
    if len(x) == 0:
        return empty_group(op, st)
    raise NotImplementedError("only groups without valid values are restated here")
