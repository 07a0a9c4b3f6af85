"""CPU: the literal restatements of the reference's per-group product (tests/prod_reference.py) and of its cov / corr
(tests/binary_reference.py) reproduce every golden_v5 case bit for bit, and the engine's error bounds (`prod_ok`,
`result_ok`) are tight enough to mean something.

golden_v5 comes from the unmodified reference (tests/golden/make_golden_v5.py).  Groups are formed by the C oracle
(oracle/dt_oracle.c, pinned to the reference by tests/test_oracle_golden*.py).
"""
import numpy as np
import pytest

from oracle import oracle as orc
import json
import os

import datatable_b200 as dtb
from binary_reference import one_pass_cov, result_ok, two_pass_cov, valid_pairs, welford
from prod_reference import (FLOAT32, FLOAT64, GOLDEN, case_query, int_prod, load_golden, out_dtype, prod_ok, seq_prod,
                            valid_values)

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if c["op"] == "prod"]
CASES2 = [c for c in ALL_CASES if c["op"] != "prod"]


def ref_groups(case):
    """(order, offsets) of the case's query: group() of its key columns, then its slice inside every group."""
    v, keys, flags = case_query(case, ARR)
    n = len(v)
    if not keys:
        return None, np.array([0, n], dtype=np.int32)
    order, offsets, _ = orc.group(keys, flags, orc.NA_FIRST)
    if case["i"] is not None:
        pos, offsets = orc.slice_groups(offsets, *case["i"])
        order = order[pos]
    return order, offsets


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_restatement_reproduces_golden(case):
    v, _, _ = case_query(case, ARR)
    st = 4 if case["mode"] == "bykey" else case["stype"]
    want = ARR[case["name"] + ".out_" + case["names"][-1]]
    if len(v) == 0:
        assert len(want) == 0
        return
    order, offsets = ref_groups(case)
    got = seq_prod(valid_values(v, st, order, offsets), st)
    assert got.dtype == want.dtype
    if got.dtype.kind == "f":
        ui = np.uint32 if got.dtype == np.float32 else np.uint64
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan)
        assert np.array_equal(got[~nan].view(ui), want[~nan].view(ui))
    else:
        assert np.array_equal(got, want)


def groups2(case):
    """(order, offsets) of a cov / corr case's query, as ref_groups does for prod."""
    name = case["name"]
    x = ARR[name + ".x"]
    if case["mode"] == "none":
        return None, np.array([0, len(x)], dtype=np.int32)
    keys = [ARR[name + ".k1"]] + ([ARR[name + ".k2"]] if case["mode"] == "by2" else []) + \
        ([ARR[name + ".s"]] if case["mode"] == "bysort" else [])
    flags = [0, 4] if case["mode"] == "bysort" else [0] * len(keys)
    order, offsets, _ = orc.group(keys, flags, orc.NA_FIRST)
    if case["i"] is not None:
        pos, offsets = orc.slice_groups(offsets, *case["i"])
        order = order[pos]
    return order, offsets


def outputs2(case):
    """[(x, stype of x, y, stype of y, output column name)] of a cov / corr case: corr(x, y) or, broadcast, corr([x, y], y)."""
    name, x, y = case["name"], ARR[case["name"] + ".x"], ARR[case["name"] + ".y"]
    if case["bcast"]:
        return [(x, case["stype"], y, case["stype2"], case["names"][-2]), (y, case["stype2"], y, case["stype2"], case["names"][-1])]
    return [(x, case["stype"], y, case["stype2"], case["names"][-1])]


@pytest.mark.parametrize("case", CASES2, ids=[c["name"] for c in CASES2])
def test_binary_restatement_reproduces_golden(case):
    order, offsets = groups2(case)
    for x, sx, y, sy, col in outputs2(case):
        want = ARR[case["name"] + ".out_" + col]
        if case["mode"] == "bykey":                         # a by() column as an argument: all NA (make_na_result)
            assert np.all(np.isnan(want))
            continue
        got = welford(valid_pairs(x, sx, y, sy, order, offsets), sx, sy, case["op"] == "corr")
        assert got.dtype == want.dtype
        ui = np.uint32 if got.dtype == np.float32 else np.uint64
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan)
        assert np.array_equal(got[~nan].view(ui), want[~nan].view(ui))


def test_binary_golden_covers_what_it_claims():
    names = {c["name"] for c in CASES2}
    tags = ("bool", "i8", "i16", "i32", "i64", "f32", "f64")
    for op in ("cov", "corr"):
        assert all(f"{op}.{a}.{b}" in names for a in tags for b in tags)
        for mode in ("by2", "bysort", "none", "islice", "bykey", "bcast"):
            assert f"{op}.{mode}.f64.f64" in names
    # NA in x only / y only; 0, 1, 2 valid pairs; constant x (cov exactly 0, corr NA); constant y; all NA
    assert np.isnan(ARR["cov.napattern.f64.out_r"][[0, 1, 5]]).all() and ARR["cov.napattern.f64.out_r"][3] == 0.0
    assert np.isnan(ARR["corr.napattern.f64.out_r"][[0, 1, 3, 4, 5]]).all()
    assert [c["names"] for c in CASES2 if c["name"] == "corr.bcast.f64.f64"] == [["k1", "C0", "C1"]]


def test_broadcast_error_text_matches_the_reference():
    with open(os.path.join(GOLDEN, "golden_v5.json")) as fh:
        want = json.load(fh)["broadcast_error"]
    with pytest.raises(ValueError) as e:
        dtb.corr([dtb.f.a, dtb.f.b], [dtb.f.a, dtb.f.b, dtb.f.c])
    assert str(e.value) == want
    assert len(dtb.cov([dtb.f.a, dtb.f.b], dtb.f.c)) == 2 and len(dtb.corr(dtb.f.a, [dtb.f.b, dtb.f.c])) == 2


def test_cov_bound_accepts_two_pass_any_order_and_rejects_one_pass_on_offset_data():
    rng = np.random.default_rng(9)
    for m in (2, 10, 500):
        x = 1e8 + rng.standard_normal(m)
        y = -1e8 + 0.3 * (x - 1e8) + rng.standard_normal(m) * 0.01
        for _ in range(3):
            assert result_ok(two_pass_cov(x, y, rng), x, y, False, np.float64)
        if m >= 10:
            assert not result_ok(one_pass_cov(x, y), x, y, False, np.float64)
        assert not result_ok(two_pass_cov(x, y) * (1 + 1e-6), x, y, False, np.float64)
    x = np.array([0.1] * 5); y = np.arange(5.0)
    assert result_ok(0.0, x, y, False, np.float64) and result_ok(np.nan, x, y, True, np.float64)
    assert not result_ok(1e-3, x, y, False, np.float64)


def test_golden_covers_what_it_claims():
    names = {c["name"] for c in CASES}
    for tag in ("bool", "i8", "i16", "i32", "i64", "f32", "f64"):
        for mode in ("rand", "by2", "bysort", "none", "islice", "fewvalid", "allna", "bykey", "empty"):
            assert f"{mode}.{tag}" in names
    assert [c["out_stype"] for c in CASES if c["name"] == "rand.f32"] == ["stype.float32"]
    assert [c["out_stype"] for c in CASES if c["name"] == "rand.bool"] == ["stype.int64"]
    # groups without valid rows give 1, never NA
    assert ARR["allna.f64.out_p"].tolist() == [1.0] and ARR["allna.i32.out_p"].tolist() == [1]
    assert ARR["fewvalid.i8.out_p"].tolist() == [1, 3, 1, 1]
    dev = [c for c in CASES if c["deviation"]]
    assert len(dev) == 2
    for c in dev:
        v, _, _ = case_query(c, ARR)
        order, offsets = ref_groups(c)
        want = ARR[c["name"] + ".out_p"]
        for vals, w in zip(valid_values(v, c["stype"], order, offsets), want):
            # the reference's running product left the range although the exact product is inside it
            assert not prod_ok(w, vals, want.dtype.type)


def test_product_bound_accepts_any_order_and_rejects_a_dropped_row():
    rng = np.random.default_rng(5)
    for m in (2, 17, 300, 2000):
        x = rng.choice([-1.0, 1.0], m) * np.exp2(rng.uniform(-30, 30, m)) * (1 + rng.random(m))
        for _ in range(3):
            p = np.float64(1.0)
            for t in rng.permutation(x):           # float64 products in a shuffled order stay inside the bound
                p = p * t
            assert prod_ok(p, x, np.float64)
        q = np.float64(1.0)
        for t in x[1:]:
            q = q * t
        if abs(x[0]) != 1.0:
            assert not prod_ok(q, x, np.float64)  # one row dropped
        assert not prod_ok(-p, x, np.float64)     # wrong sign
        # float32 output: one more rounding, at 2^-24
        assert prod_ok(np.float32(p), x, np.float32)


def test_product_bound_special_values():
    assert prod_ok(np.float64(np.nan), np.array([0.0, np.inf]), np.float64)
    assert prod_ok(np.float64(-0.0), np.array([-0.0, 2.0]), np.float64)
    assert not prod_ok(np.float64(0.0), np.array([-0.0, 2.0]), np.float64)
    assert prod_ok(np.float64(np.inf), np.array([-np.inf, -1.0]), np.float64)
    assert prod_ok(np.float64(1.0), np.array([1e200, 1e200, 1e-200, 1e-200]), np.float64)
    assert not prod_ok(np.float64(np.inf), np.array([1e200, 1e200, 1e-200, 1e-200]), np.float64)
    assert prod_ok(np.float64(np.inf), np.array([1e200, 1e200]), np.float64)                 # beyond the range
    assert prod_ok(np.float32(np.inf), np.array([1e30, 1e30]), np.float32)
    assert prod_ok(np.float64(5e-324), np.array([2.0 ** -1000, 2.0 ** -74]), np.float64)    # subnormal result


def test_int_prod_wraps():
    assert int_prod(np.array([2**62, 4], dtype=np.int64)) == 0
    assert int_prod(np.array([2**63 - 1, 2**63 - 1], dtype=np.int64)) == 1
    assert int_prod(np.array([-3, 5], dtype=np.int64)) == -15
    assert out_dtype(FLOAT32) == np.float32 and out_dtype(FLOAT64) == np.float64 and out_dtype(1) == np.int64
