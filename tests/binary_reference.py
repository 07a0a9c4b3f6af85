"""cov / corr per group, three ways, shared by tests/test_oracle_golden_v5.py and tests/test_gpu_prod_cov_corr.py:

- `welford`: the reference restated literally (expr/head_reduce_binary.cc:114-200): both columns cast to T (float32
  when both are float32, else float64), only rows where both values are valid, Welford's recurrence in T;
- `exact_cov_corr`: exact rational sums of the pairs (the inputs widened to float64 exactly, as the engine reads
  them), the square root of corr taken in `decimal` at 60 digits;
- `cov_ok` / `corr_ok`: the engine's error bound around the exact result.

The bound.  The engine shifts every pair by the group's first valid pair (px, py) and folds in float64, in any order:
    a_i = fl(x_i - px),  mx' = fl(sum a_i) / m,  dx_i = fl(a_i - mx')   (likewise b_i, my', dy_i)
    sxy = fl(sum dx_i dy_i),  sxx = fl(sum dx_i^2),  syy = fl(sum dy_i^2).
With u = 2^-53, A_i = |x_i - px| + |mx| and B_i = |y_i - py| + |my| (mx, my: the exact means of x - px, y - py):
|a_i - (x_i - px)| <= u |x_i - px|; the computed mean mx' is within gamma(m + 1) sum|a_i| / m of mx (a sum in any
order, Higham Lemma 3.1 / (4.4), then a division); so |dx_i - (x_i - mean x)| <= gamma(m + 3) A_i, and so on for dy.
Then each product adds one rounding and the final sum gamma(m - 1) of the sum of |terms|, so
    |sxy - Sxy| <= gamma(3m + 8) * sum A_i B_i,   |sxx - Sxx| <= gamma(3m + 8) * sum A_i^2,
where Sxy = sum (x_i - mean x)(y_i - mean y) exactly (the shift changes nothing exactly).  cov = sxy / (m - 1) adds one
rounding, corr = sxy / sqrt(sxx syy) four (product, sqrt, division, and the output), and |d corr| <= |d sxy| /
sqrt(Sxx Syy) + |corr| (|d sxx| / (2 Sxx) + |d syy| / (2 Syy)) to first order; the bound doubles that first-order
term to cover the second.  Results rounded to float32 add 2^-24 relative.
"""
import decimal
from fractions import Fraction

import numpy as np

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64 = 1, 2, 3, 4, 5, 6, 7
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63}


def gamma(k):
    k = Fraction(k)
    return k / 2**53 / (1 - k / 2**53)


def out_dtype2(sx, sy):
    return np.float32 if sx == FLOAT32 and sy == FLOAT32 else np.float64


def valid_pairs(x, sx, y, sy, order, offsets):
    """[(x values, y values) of group g's rows where both are valid, in RowIndex order]"""
    idx = np.arange(len(x)) if order is None else np.asarray(order, dtype=np.int64)
    xo, yo = x[idx], y[idx]
    okx = ~np.isnan(xo) if sx in (FLOAT32, FLOAT64) else xo != NA[sx]
    oky = ~np.isnan(yo) if sy in (FLOAT32, FLOAT64) else yo != NA[sy]
    ok = okx & oky
    offsets = np.asarray(offsets, dtype=np.int64)
    return [(xo[a:b][ok[a:b]], yo[a:b][ok[a:b]]) for a, b in zip(offsets[:-1], offsets[1:])]


def welford(groups, sx, sy, corr):
    """head_reduce_binary.cc:114-138 (cov) and :168-200 (corr), in T."""
    T = out_dtype2(sx, sy)
    out = np.empty(len(groups), dtype=T)
    with np.errstate(all="ignore"):
        for gi, (xs, ys) in enumerate(groups):
            m1 = m2 = cov = v1 = v2 = T(0)
            n = 0
            for a, b in zip(xs.tolist(), ys.tolist()):
                a, b = T(a), T(b)
                n += 1
                d1, d2 = T(a - m1), T(b - m2)
                m1 = T(m1 + T(d1 / T(n)))
                m2 = T(m2 + T(d2 / T(n)))
                t1, t2 = T(a - m1), T(b - m2)
                cov = T(cov + T(t1 * d2))
                v1 = T(v1 + T(t1 * d1))
                v2 = T(v2 + T(t2 * d2))
            if corr:
                vv = T(v1 * v2)
                out[gi] = T(cov / T(np.sqrt(vv))) if n > 1 and vv > 0 else np.nan
            else:
                out[gi] = T(cov / T(n - 1)) if n > 1 else np.nan
    return out


def _fr(a):
    return [Fraction(float(t)) for t in np.asarray(a, dtype=np.float64).tolist()]


def exact_sums(xs, ys):
    """(m, Sxy, Sxx, Syy, sum A_i B_i, sum A_i^2, sum B_i^2) with the pivot of the engine (the first pair)."""
    X, Y = _fr(xs), _fr(ys)
    m = len(X)
    if m == 0:
        return 0, 0, 0, 0, 0, 0, 0
    mx, my = sum(X) / m, sum(Y) / m
    Sxy = sum((a - mx) * (b - my) for a, b in zip(X, Y))
    Sxx = sum((a - mx) ** 2 for a in X)
    Syy = sum((b - my) ** 2 for b in Y)
    px, py = X[0], Y[0]
    smx, smy = abs(mx - px), abs(my - py)
    A = [abs(a - px) + smx for a in X]
    B = [abs(b - py) + smy for b in Y]
    return m, Sxy, Sxx, Syy, sum(a * b for a, b in zip(A, B)), sum(a * a for a in A), sum(b * b for b in B)


def _sqrt(fr):
    with decimal.localcontext() as ctx:
        ctx.prec = 60
        return Fraction(decimal.Decimal(fr.numerator).sqrt() / decimal.Decimal(fr.denominator).sqrt())


def exact_cov_corr(xs, ys, corr):
    """The exact result (a Fraction) or None for NA."""
    m, Sxy, Sxx, Syy, _, _, _ = exact_sums(xs, ys)
    if m <= 1:
        return None
    if not corr:
        return Sxy / (m - 1)
    if Sxx * Syy == 0:
        return None
    return Sxy / _sqrt(Sxx * Syy)


def result_ok(got, xs, ys, corr, out_dt):
    """Whether the engine's result `got` for one group is the exact cov / corr within the bound (NA exactly)."""
    m, Sxy, Sxx, Syy, SAB, SAA, SBB = exact_sums(xs, ys)
    g = float(got)
    na = m <= 1 or (corr and Sxx * Syy == 0)
    if na:
        return np.isnan(g)
    if np.isnan(g):
        return False
    G = gamma(3 * m + 8)
    u_out = Fraction(1, 2**24) if out_dt == np.float32 else Fraction(1, 2**53)
    if not corr:
        want = Sxy / (m - 1)
        tol = G * SAB / (m - 1) + (abs(want) + G * SAB / (m - 1)) * (u_out + Fraction(1, 2**52))
        return abs(Fraction(g) - want) <= tol
    root = _sqrt(Sxx * Syy)
    want = Sxy / root
    first = G * SAB / root + abs(want) * (G * SAA / (2 * Sxx) + G * SBB / (2 * Syy))
    tol = 2 * first + (abs(want) + 2 * first) * (u_out + 4 * Fraction(1, 2**53)) + Fraction(1, 10**40)
    return abs(Fraction(g) - want) <= tol


def one_pass_cov(xs, ys):
    """The textbook one-pass formula (sum xy - sum x sum y / m) / (m - 1) in float64: what the bound must reject."""
    x, y = np.asarray(xs, dtype=np.float64), np.asarray(ys, dtype=np.float64)
    m = len(x)
    return (np.sum(x * y) - np.sum(x) * np.sum(y) / m) / (m - 1)


def two_pass_cov(xs, ys, rng=None):
    """The engine's method in float64, over the pairs in a shuffled order (pivot = the first pair of that order)."""
    x, y = np.asarray(xs, dtype=np.float64), np.asarray(ys, dtype=np.float64)
    p = np.arange(len(x)) if rng is None else rng.permutation(len(x))
    a, b = x - x[0], y - y[0]
    a, b = a[p], b[p]
    mx, my = np.sum(a) / len(a), np.sum(b) / len(b)
    return np.sum((a - mx) * (b - my)) / (len(a) - 1)
