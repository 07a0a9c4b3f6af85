"""The per-group product, three ways, shared by tests/test_oracle_golden_v5.py and tests/test_gpu_prod_cov_corr.py:

- `seq_prod`: the reference restated literally (column/sumprod.h:34-59): start at 1, multiply the valid values in
  RowIndex order, in the column's own type (int64 wrapping modulo 2^64, float32, float64);
- `exact_prod`: the exact product, from integer significands times a power of two;
- `prod_ok`: the engine's error bound around the exact product (include/dtb200.h at dtb_reduce).

The bound.  The engine multiplies the float64 significands, each in [1, 2) and exact, of the m valid finite non-zero
values of a group: m - 1 products, each rounded once (relative error <= u = 2^-53), and rescales by 2 exactly.  So
its significand is the exact one times prod(1 + d_i), |prod(1 + d_i) - 1| <= gamma(m - 1), gamma(k) = k u / (1 - k u)
(Higham, Accuracy and Stability of Numerical Algorithms, Lemma 3.1), in any order.  The exponent is an exact integer
sum, and the result is rounded once to the output type: relative error <= u_out (float64 2^-53, float32 2^-24) in the
normal range, absolute error <= half the smallest subnormal below it.  Hence
    |got - exact| <= (gamma(m - 1) (1 + u_out) + u_out) |exact| + eta_out.
A zero and an infinity in one group give NA, a zero alone gives 0 and an infinity alone inf, each signed by the
parity of the negative values (-0.0 and -inf included).
"""
import json
import os
from fractions import Fraction

import numpy as np

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64 = 1, 2, 3, 4, 5, 6, 7
NPT = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
       FLOAT32: np.float32, FLOAT64: np.float64}
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63}
U = 2.0 ** -53
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def gamma(k):
    return k * U / (1 - k * U)


def out_dtype(st):
    return {FLOAT32: np.float32, FLOAT64: np.float64}.get(st, np.int64)


def valid_values(v, st, order, offsets):
    """[valid values of group g in RowIndex order] (order None = identity)."""
    vo = v if order is None else v[np.asarray(order, dtype=np.int64)]
    ok = ~np.isnan(vo) if st in (FLOAT32, FLOAT64) else vo != NA[st]
    offsets = np.asarray(offsets, dtype=np.int64)
    return [vo[a:b][ok[a:b]] for a, b in zip(offsets[:-1], offsets[1:])]


def seq_prod(groups, st):
    """The reference's loop: result = 1; result *= value, in the column's type."""
    if st not in (FLOAT32, FLOAT64):
        out = []
        for g in groups:
            r = 1
            for x in g.tolist():
                r = (r * int(x)) % 2**64
            out.append(r - 2**64 if r >= 2**63 else r)
        return np.array(out, dtype=np.int64)
    T = NPT[st]
    out = np.empty(len(groups), dtype=T)
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        for i, g in enumerate(groups):
            r = T(1)
            for x in g:
                r = T(r * x)
            out[i] = r
    return out


def int_prod(vals):
    """Exact integer product modulo 2^64, as int64."""
    r = 1
    for x in vals.tolist():
        r = (r * int(x)) % 2**64
    return r - 2**64 if r >= 2**63 else r


def exact_prod(vals):
    """("na" | "zero" | "inf" | "finite", negative?, exact |product| as a Fraction (finite only), m)."""
    x = np.asarray(vals, dtype=np.float64)
    neg = bool(np.count_nonzero(np.signbit(x)) % 2)
    zero, inf = bool(np.any(x == 0)), bool(np.any(np.isinf(x)))
    if zero and inf:
        return "na", neg, None, len(x)
    if zero or inf:
        return ("zero" if zero else "inf"), neg, None, len(x)
    sig, e2 = 1, 0
    for t in np.abs(x).tolist():
        n, d = t.as_integer_ratio()                    # d is a power of two
        sig *= n
        e2 -= d.bit_length() - 1
    return "finite", neg, (Fraction(sig) * Fraction(2) ** e2), len(x)


def prod_ok(got, vals, out_dt):
    """Whether one engine result `got` (a numpy scalar of out_dt) is the product of `vals` within the bound."""
    kind, neg, ex, m = exact_prod(vals)
    g = float(got)
    if kind == "na":
        return np.isnan(g)
    if kind == "zero":
        return g == 0 and bool(np.signbit(g)) == neg
    if kind == "inf":
        return np.isinf(g) and bool(np.signbit(g)) == neg
    if np.isnan(g) or bool(np.signbit(g)) != neg:
        return False
    fi = np.finfo(out_dt)
    if ex > Fraction(float(fi.max)) * (1 + Fraction(2) ** -20):
        return np.isinf(g)
    if np.isinf(g):
        return False
    u_out = Fraction(1, 2**53) if out_dt == np.float64 else Fraction(1, 2**24)
    eta = Fraction(float(fi.smallest_subnormal)) / 2
    k = max(m - 1, 0)
    gam = Fraction(k, 2**53) / (1 - Fraction(k, 2**53))
    return abs(Fraction(abs(g)) - ex) <= (gam * (1 + u_out) + u_out) * ex + eta


def load_golden():
    with open(os.path.join(GOLDEN, "golden_v5.json")) as fh:
        meta = json.load(fh)
    with np.load(os.path.join(GOLDEN, "golden_v5.npz")) as z:
        arr = {k: z[k] for k in z.files}
    return meta["cases"], arr


def case_query(case, arr):
    """(value column, key columns, key flags) of a golden case as group() takes them; SORT_ONLY = 4."""
    name = case["name"]
    v = arr[name + ".v"]
    if case["mode"] == "none":
        return v, [], []
    if case["mode"] == "bykey":
        return arr[name + ".k1"], [arr[name + ".k1"]], [0]
    if case["mode"] == "by2":
        return v, [arr[name + ".k1"], arr[name + ".k2"]], [0, 0]
    if case["mode"] == "bysort":
        return v, [arr[name + ".k1"], arr[name + ".s"]], [0, 4]
    return v, [arr[name + ".k1"]], [0]
