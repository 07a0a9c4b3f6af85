"""natural_join (frame/join.cc:199-236, 386-458) restated in numpy, vectorised over the X rows, shared by
tests/test_oracle_golden_v9.py and tests/test_gpu_join_sets.py.  It shares no conversion code with the oracle.

- set_xrow: every X value is converted to J's type once, as static_cast<TJ>(newval) does: numpy astype on the typed
  array (int64 -> float32 is one rounding, not one through float64).  An X row cannot match when, in any key column,
  J's type is integral and the X value is integral but outside J's type (numeric_limits<TJ>: J's NA sentinel is in
  range), or is a float that does not survive the round trip through J's type (a fraction, +-inf, out of range).
- binsearch: start = 0, end = nj - 1; while start < end: mid = (start + end) >> 1, r = cmp_jrow(mid); r > 0: end =
  mid, r < 0: start = mid + 1, r == 0: the row is mid.  At start == end the row is start if cmp_jrow(start) == 0.
  Every X row runs this at once, one numpy step per halving of the range.
- cmp_jrow, column by column, first non-zero: sign(J - X) in J's type when both are valid, else jvalid - xvalid
  (NA == NA, NA < every valid value).

The number of steps is about log2(nj): 1e7 X rows against J of 2^20 + 1 rows take about ten seconds.
"""
import numpy as np

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64 = 1, 2, 3, 4, 5, 6, 7, 17, 18
NPT = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
       FLOAT32: np.float32, FLOAT64: np.float64, DATE32: np.int32, TIME64: np.int64}
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
NA_INDEX = -2**31
FLOATS = (FLOAT32, FLOAT64)


def na_mask(a, st):
    return np.isnan(a) if st in FLOATS else a == NA[st]


def x_in_j_type(x, xst, jst):
    """(valid, value in J's type, cannot match) of every X value: set_xrow"""
    valid = ~na_mask(x, xst)
    if jst in FLOATS:
        with np.errstate(over="ignore"):                       # float64 beyond float32's range becomes +-inf
            return valid, x.astype(NPT[jst]), np.zeros(len(x), bool)
    info = np.iinfo(NPT[jst])
    if xst in FLOATS:
        v = x.astype(np.float64)                               # float32 -> float64 is exact
        ok = np.isfinite(v) & (np.trunc(v) == v) & (v >= float(info.min)) & (v < -float(info.min))
        xj = np.where(ok, v, 0.0).astype(np.int64)
    else:
        xj = x.astype(np.int64)
        ok = (xj >= info.min) & (xj <= info.max)
    return valid, xj, valid & ~ok


def join_index(xcols, xst, jcols, jst):
    """int32[nx]: the row of J (sorted ascending by its key columns, NA first, unique) every X row matches, or
    NA_INDEX."""
    nx, nj = len(xcols[0]), len(jcols[0])
    out = np.full(nx, NA_INDEX, np.int32)
    if nx == 0 or nj == 0:
        return out
    xs, bad = [], np.zeros(nx, bool)
    for x, sx, sj in zip(xcols, xst, jst):
        valid, xj, b = x_in_j_type(np.asarray(x), sx, sj)
        xs.append((valid, xj))
        bad |= b
    js = []
    for j, sj in zip(jcols, jst):
        j = np.asarray(j)
        js.append((~na_mask(j, sj), j if sj in FLOATS else j.astype(np.int64)))

    def cmp(rows, mid):
        """cmp_jrow(mid[i]) for X row rows[i]"""
        r = np.zeros(len(rows), np.int8)
        for (xvalid, xj), (jvalid, jv) in zip(xs, js):
            todo = r == 0
            xv, jvv = xvalid[rows], jvalid[mid]
            both = xv & jvv
            a, b = jv[mid], xj[rows]
            sign = (a > b).astype(np.int8) - (a < b).astype(np.int8)
            r = np.where(todo, np.where(both, sign, jvv.astype(np.int8) - xv.astype(np.int8)), r)
        return r

    rows = np.flatnonzero(~bad)
    start = np.zeros(len(rows), np.int64)
    end = np.full(len(rows), nj - 1, np.int64)
    while len(rows):
        live = start < end
        if not live.all():                                      # start == end: one last comparison
            done = rows[~live]
            hit = cmp(done, start[~live]) == 0
            out[done[hit]] = start[~live][hit]
            rows, start, end = rows[live], start[live], end[live]
            if not len(rows):
                break
        mid = (start + end) >> 1
        r = cmp(rows, mid)
        eq = r == 0
        out[rows[eq]] = mid[eq]
        end = np.where(r > 0, mid, end)
        start = np.where(r < 0, mid + 1, start)
        rows, start, end = rows[~eq], start[~eq], end[~eq]
    return out
