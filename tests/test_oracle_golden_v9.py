"""CPU: the numpy join restatement (tests/join_reference.py) and the CPU oracle reproduce every golden_v9 join case,
and the oracle's set selection and largest-group scan, over columns promoted to the highest input stype, reproduce
every golden_v9 set-operation and column-statistics case.

golden_v9 comes from the unmodified reference (tests/golden/make_golden_v9.py).  The join cases include int64 X
values beyond 2^53 against float32 keys, where a conversion that rounds twice (int64 -> float64 -> float32) matches
the wrong row: 2^60 + 2^36 + 1 becomes 2^60 that way, and 2^60 + 2^37 in one rounding.
"""
import json
import os

import numpy as np
import pytest

from oracle import oracle as orc
from join_reference import (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64, NA, NPT, na_mask,
                            join_index)

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = json.load(open(os.path.join(G, "golden_v9.json")))["cases"]
ARR = dict(np.load(os.path.join(G, "golden_v9.npz")))
NUMERIC = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
JOINS = [c for c in CASES if c["kind"] == "join"]
SETS = [c for c in CASES if c["kind"] == "sets"]
STATS = [c for c in CASES if c["kind"] == "stats"]
PLAIN = {DATE32: INT32, TIME64: INT64}                  # the oracle compares dates and times as their storage


def A(case, key):
    return ARR[f"{case['name']}.{key}"]


def join_inputs(case):
    nk = len(case["xst"])
    return [A(case, f"x{i}") for i in range(nk)], [A(case, f"jsorted{i}") for i in range(nk)]


def test_golden_covers_the_ground():
    pairs = {(c["xst"][0], c["jst"][0]) for c in JOINS if len(c["xst"]) == 1}
    assert pairs >= {(x, j) for x in NUMERIC for j in NUMERIC} | {(DATE32, DATE32), (TIME64, TIME64)}
    assert {c["size"] for c in JOINS if "size" in c} >= {0, 1, 2, 3, 7, 8, 9, 1023, 1024, 1025, 4095, 4096, 4097}
    assert {len(c["xst"]) for c in JOINS} == {1, 2, 3, 4}
    assert not any("key_error" in c for c in JOINS)                   # -0.0 and +0.0 are distinct keys
    assert any(c["name"].startswith("jzero") for c in JOINS)
    assert {c["K"] for c in SETS} == set(range(1, 11))
    assert {tuple(c["sts"]) for c in SETS} >= {(INT32, FLOAT32), (INT64, FLOAT32), (BOOL, INT8), (INT8, FLOAT64),
                                               (FLOAT32, FLOAT64)}
    assert any(c["kind"] == "unique" for c in CASES)
    assert {c["sts"][0] for c in STATS} == set(NUMERIC)


def test_int64_against_float32_rounds_once():
    """The case the double rounding gets wrong, read straight from the reference's answer."""
    case = next(c for c in JOINS if c["name"] == "join.i64.f32")
    x, j = A(case, "x0"), A(case, "jsorted0")
    idx = A(case, "index")
    r = np.flatnonzero(x == 2**60 + 2**36 + 1)[0]
    assert j[idx[r]] == np.float32(2**60 + 2**37) and np.float32(2**60) in j


@pytest.mark.parametrize("group", sorted({c["name"].split(".")[0] for c in JOINS}))
def test_join_reference_reproduces_golden(group):
    bad = []
    for case in JOINS:
        if case["name"].split(".")[0] != group:
            continue
        xs, js = join_inputs(case)
        got = join_index(xs, case["xst"], js, case["jst"])
        if not np.array_equal(got, A(case, "index")):
            bad.append(case["name"])
    assert not bad, bad


@pytest.mark.parametrize("group", sorted({c["name"].split(".")[0] for c in JOINS}))
def test_oracle_join_reproduces_golden(group):
    bad = []
    for case in JOINS:
        if case["name"].split(".")[0] != group:
            continue
        xs, js = join_inputs(case)
        got = orc.join_index(xs, [PLAIN.get(s, s) for s in case["xst"]], js, [PLAIN.get(s, s) for s in case["jst"]])
        if not np.array_equal(got, A(case, "index")):
            bad.append(case["name"])
    assert not bad, bad


def test_join_reference_agrees_with_oracle_on_random_wide_keys():
    """Two restatements that share no code, on 3000 rows of two key columns with planted hits and NAs."""
    rng = np.random.default_rng(9)
    for xst, jst in ((INT64, FLOAT32), (FLOAT64, INT32), (INT32, FLOAT64), (FLOAT32, INT64), (INT16, INT8)):
        if INT64 in (xst, jst):        # float32 holds these exactly; the near misses round onto them or not
            base = rng.integers(-2**22, 2**22, 400) * 2**40
            near = base + rng.integers(-2**40, 2**40, 400)
        else:
            base = rng.integers(-300, 300, 400)
            near = base + rng.choice([-1, 1, 0.5], 400)
        j0 = np.unique(base.astype(NPT[jst]))
        j1 = rng.integers(0, 3, len(j0)).astype(np.int32)
        j1[::7] = NA[INT32]
        o, _, _ = orc.group([j0, j1], [0, 0], orc.NA_FIRST)
        j0, j1 = j0[o], j1[o]
        x0 = np.concatenate([base, near]).astype(NPT[xst])[rng.integers(0, 2 * len(base), 3000)]
        x1 = rng.integers(-1, 3, 3000).astype(np.int32)
        x1[x1 < 0] = NA[INT32]
        want = orc.join_index([x0, x1], [xst, INT32], [j0, j1], [jst, INT32])
        assert np.array_equal(join_index([x0, x1], [xst, INT32], [j0, j1], [jst, INT32]), want), (xst, jst)
        assert (want >= 0).sum() > 100


def same(got, want):
    """dtype and bits equal; any NaN is NA"""
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    if got.dtype.kind != "f":
        return np.array_equal(got, want)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint8), want[~nan].view(np.uint8))


def common_stype(sts):
    """Type::common for numeric types (types/typeimpl_numeric.cc:36-41): the highest stype"""
    return max(sts, key=list(NUMERIC).index)


def promote(ins, sts):
    """rbind under the common stype: every value cast once from its own type, NA to NA"""
    st = common_stype(sts)
    out = []
    for a, s in zip(ins, sts):
        b = a.astype(NPT[st])
        b[na_mask(a, s)] = np.nan if st in (FLOAT32, FLOAT64) else NA[st]
        out.append(b)
    return (np.concatenate(out) if out else np.zeros(0, NPT[st])), st


@pytest.mark.parametrize("group", sorted({c["name"].split(".")[0] for c in SETS}))
def test_set_operations_reproduce_golden(group):
    bad = []
    for case in SETS:
        if case["name"].split(".")[0] != group:
            continue
        ins = [A(case, f"in{i}") for i in range(case["K"])]
        cat, st = promote(ins, case["sts"])
        cs = np.cumsum([len(a) for a in ins])
        for op, mode in (("union", orc.SET_UNION), ("intersect", orc.SET_INTERSECT), ("setdiff", orc.SET_SETDIFF),
                         ("symdiff", orc.SET_SYMDIFF)):
            want = A(case, op)
            if len(cat):
                o, offs, _ = orc.group([cat], [0], orc.NA_FIRST, stypes=[st])
                got = cat[orc.set_select(mode if case["K"] > 1 else orc.SET_UNION, o, offs, cs)]
            else:
                got = cat
            if st != case["out_st"][op] or not same(got, want):
                bad.append(f"{case['name']} {op}")
    assert not bad, bad


def test_unique_of_mixed_columns_reproduces_golden():
    for case in (c for c in CASES if c["kind"] == "unique"):
        cat, st = promote([A(case, f"c{i}") for i in range(len(case["sts"]))], case["sts"])
        o, offs, _ = orc.group([cat], [0], orc.NA_FIRST, stypes=[st])
        got = cat[o[offs[:-1]]]
        assert st == case["out_st"], case["name"]
        assert same(got, A(case, "out")), case["name"]


def test_column_stats_reproduce_golden():
    bad = []
    for case in STATS:
        for i, st in enumerate(case["sts"]):
            a = A(case, f"c{i}")
            nu, size, mode = 0, 0, a[:0]
            if len(a):
                o, offs, ng = orc.group([a], [0], orc.NA_FIRST, stypes=[st])
                skip = int(na_mask(a[o[:1]], st)[0])
                nu = ng - skip
                idx, size = orc.largest_group(offs, skip)
                mode = a[o[offs[idx:idx + 1]]] if size else mode
            if not size:
                mode = np.array([np.nan if st in (FLOAT32, FLOAT64) else NA[st]], NPT[st])
            want = A(case, f"mode{i}")
            if (nu, size) != (A(case, "nunique")[i], A(case, "nmodal")[i]) or not same(mode, want):
                bad.append(f"{case['name']} c{i}")
    assert not bad, bad
