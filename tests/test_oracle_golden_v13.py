"""CPU: golden_v13 (queries over zero rows, from the unmodified reference, tests/golden/make_golden_v13.py) restated
with numpy and tests/zero_rows_reference.py: what a group without rows reduces to, one result row for a reducer j
without by() and none with it; an empty result's names and stypes; the engine's own output stypes (a host function of
the library) against the restatement; and the cases' call-time errors raised by the Frame before any library call."""
import json
import os

import numpy as np
import pytest

import zero_rows_reference as zr

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = json.load(open(os.path.join(G, "golden_v13.json")))["cases"]
ARR = dict(np.load(os.path.join(G, "golden_v13.npz")))
BY_NAME = {c["name"]: c for c in CASES}
ALL_ST = (zr.BOOL, zr.INT8, zr.INT16, zr.INT32, zr.INT64, zr.FLOAT32, zr.FLOAT64)
TAG = {zr.BOOL: "bool8", zr.INT8: "int8", zr.INT16: "int16", zr.INT32: "int32", zr.INT64: "int64",
       zr.FLOAT32: "float32", zr.FLOAT64: "float64"}
# The reference dies in fillna over zero rows, and qcut under by() over zero rows raises KeyError('stype.void'): the
# Frame returns the empty result there (tests/test_gpu_zero_rows.py)
REFERENCE_FAULTS = {c["name"] for c in CASES
                    if "reference_crash" in c or c.get("error") == ["KeyError", "stype.void"]}


def A(case, key):
    return ARR[f"{case['name']}.{key}"]


def same(got, want):
    got, want = np.asarray(got), np.asarray(want)
    return got.dtype == want.dtype and got.shape == want.shape and \
        np.array_equal(got, want, equal_nan=got.dtype.kind == "f")


def test_golden_covers_the_ground():
    names = set(BY_NAME)
    for st in ALL_ST:
        t = TAG[st]
        for nm in list(zr.OPS) + ["all"]:
            assert f"red.{t}.{nm}" in names
        for nm in ("cumsum", "cumprod", "cummin", "cummax", "shift", "fillna", "cumcount", "ngroup", "qcut",
                   "cut_nbins", "cut_bins"):
            assert f"row.{t}.{nm}" in names and f"row.{t}.{nm}_by" in names
        for na in ("first", "last", "remove"):
            assert f"by.{t}.sort_{na}" in names
        for op in ("union", "intersect", "setdiff", "symdiff"):
            assert f"set.{t}.{op}_ae" in names
    for sel in ("false", "allna", "list", "range", "slice", "frame", "join_mask"):
        for j in ("reducers", "rowfns", "cols"):
            assert f"sel.{sel}.{j}" in names
    for pre in ("iby.", "join.x_empty", "join.j_empty", "stat."):
        assert any(n.startswith(pre) for n in names), pre
    assert all(c["name"].startswith("row.") for c in CASES if "error" in c or "reference_crash" in c)
    assert {c["name"].split(".")[2] for c in CASES if "reference_crash" in c} == {"fillna", "fillna_by", "fillna_rev",
                                                                                  "fillna_rev_by"}


@pytest.mark.parametrize("st", ALL_ST, ids=lambda s: TAG[s])
def test_reducers_over_a_zero_row_frame(st):
    """Without by(), one result row: the empty group's value of every reducer, alone and all in one j."""
    allc = BY_NAME[f"red.{TAG[st]}.all"]
    assert allc["nrows"] == 1 and len(allc["names"]) == len(zr.OPS)
    for i, (nm, op) in enumerate(zr.OPS.items()):
        case = BY_NAME[f"red.{TAG[st]}.{nm}"]
        want, wst = zr.empty_group(op, st, zr.FLOAT64, zero_rows=True)
        assert case["nrows"] == 1 and case["stypes"] == [wst], nm
        assert case["names"] == [{"count0": "count", "cov": "C0", "corr": "C0"}.get(nm, "v")]
        assert same(A(case, "r0"), want), nm
        assert allc["stypes"][i] == wst and same(A(allc, f"r{i}"), want), nm


@pytest.mark.parametrize("st", ALL_ST, ids=lambda s: TAG[s])
def test_reducer_values_follow_numpy(st):
    """The empty group's sum and product are numpy's, and its count is the length of the empty slice."""
    e = np.zeros(0, dtype=zr.NPT[st])
    assert A(BY_NAME[f"red.{TAG[st]}.sum"], "r0")[0] == np.sum(e)
    assert A(BY_NAME[f"red.{TAG[st]}.prod"], "r0")[0] == np.prod(e)
    assert A(BY_NAME[f"red.{TAG[st]}.count0"], "r0")[0] == len(e)


@pytest.mark.parametrize("st", ALL_ST, ids=lambda s: TAG[s])
def test_engine_stypes_match_the_restatement(st):
    """The library's output stype of every reducer (dtb_reduce_out_stype, dtb_reduce2_out_stype) is the restated one;
    only median over zero rows differs, which the Frame replaces by the argument's stype."""
    from datatable_b200 import engine
    for nm, op in zr.OPS.items():
        if op in (zr.COV, zr.CORR):
            assert engine.reduce2_out_stype(op, st, zr.FLOAT64) == zr.out_stype(op, st, zr.FLOAT64)
            assert engine.reduce2_out_stype(op, st, st) == zr.out_stype(op, st, st)
        elif op != zr.NROWS:
            assert engine.reduce_out_stype(op, st) == zr.out_stype(op, st), nm


@pytest.mark.parametrize("case", [c for c in CASES if c["name"].startswith(("by.", "iby.")) and "error" not in c],
                         ids=lambda c: c["name"])
def test_grouped_zero_rows_are_empty(case):
    """With by() or sort() over zero rows (or a slice that empties every group): no group, so no row, with the
    restated names and stypes."""
    X = case["x"]
    assert case["nrows"] == 0
    for i in range(len(case["names"])):
        col = A(case, f"r{i}")
        if len(col):
            # first / last / median over zero rows make a column of one NA row (compute_firstlast, compute_median,
            # head_reduce_unary.cc:169-176, 493-496) that the reference's 0-row frame still holds; its 0 rows are
            # what the Frame returns
            assert "dt.first(" in case["query"] or "dt.median(" in case["query"]
            assert len(col) == 1 and same(col, np.array([zr.na_of(case["stypes"][i])], col.dtype)), case["name"]
    q = case["query"]
    if ":, :, sort(" in q or "100:, :, sort(" in q:
        assert case["names"] == list(X) and case["stypes"] == list(X.values())
    elif q.endswith("f.v, by(f.k)]"):
        assert case["names"] == ["k", "v"] and case["stypes"] == [X["k"], X["v"]]
    elif "by.bykey" in case["name"] or case["name"].endswith(".bykey"):
        assert case["names"] == ["v", "w"] and case["stypes"] == [X["v"], zr.out_stype(zr.SUM, X["w"])]
    elif case["name"].endswith(".reducers") and case["name"].startswith("by."):
        st = X["v"]
        ops = [zr.SUM, zr.NROWS, zr.FIRST, zr.MIN, zr.MEDIAN, zr.SD, zr.PROD, zr.NUNIQUE]
        assert case["stypes"] == [X["k"]] + [zr.empty_group(op, st, zero_rows=True)[1] for op in ops]


@pytest.mark.parametrize("case", [c for c in CASES if c["name"].startswith("sel.")], ids=lambda c: c["name"])
def test_empty_selections(case):
    """An empty selection of a non-empty frame: a reducer j gives one row of empty-group values, the other j kinds
    no row of the selected columns' stypes."""
    X = {**case["x"], **case["j"]}
    jn = case["name"].split(".")[2]
    if jn == "reducers" and "join" not in case["name"]:
        ops = [(zr.SUM, "v"), (zr.NROWS, "v"), (zr.FIRST, "q"), (zr.LAST, "b"), (zr.MEDIAN, "q"), (zr.PROD, "q"),
               (zr.SD, "w"), (zr.MIN, "w"), (zr.MAX, "q"), (zr.MEAN, "b"), (zr.COUNTNA, "v"), (zr.NUNIQUE, "q"),
               (zr.COV, "v")]
        assert case["nrows"] == 1
        for i, (op, col) in enumerate(ops):
            want, wst = zr.empty_group(op, X[col], X["q"] if op == zr.COV else zr.FLOAT64, zero_rows=True)
            assert case["stypes"][i] == wst and same(A(case, f"r{i}"), want), (case["name"], i)
    elif jn == "reducers":
        assert case["nrows"] == 1 and case["names"] == ["price", "count", "v"]
        assert same(A(case, "r0"), np.array([0.0])) and same(A(case, "r1"), np.array([0], np.int64))
        assert same(A(case, "r2"), np.array([np.nan]))
    else:
        assert case["nrows"] == 0
        if jn in ("cols", "all"):
            assert case["stypes"] == [X[n] for n in case["names"]]
        for i in range(len(case["names"])):
            assert len(A(case, f"r{i}")) == 0


def test_joins_and_sets_with_an_empty_operand():
    c = BY_NAME["join.j_empty"]                       # every X row unmatched: J's columns are NA
    assert c["nrows"] == 50 and same(A(c, "r0"), A(c, "x.k")) and np.isnan(A(c, "r1")).all()
    c = BY_NAME["join.j_empty_sum"]
    assert same(A(c, "r0"), np.array([0.0])) and same(A(c, "r1"), np.array([0], np.int64))
    assert same(A(c, "r2"), np.array([50], np.int64))
    c = BY_NAME["join.x_empty_sum"]
    assert same(A(c, "r0"), np.array([0.0])) and same(A(c, "r1"), np.array([0], np.int64))
    for st in ALL_ST:
        t = TAG[st]
        a = A(BY_NAME[f"set.{t}.union_ae"], "s.a.v")
        uniq = np.unique(a[~np.isnan(a)]) if st in zr.FLOATS else np.unique(a[a != zr.NA[st]])
        na = np.isnan(a).any() if st in zr.FLOATS else (a == zr.NA[st]).any()
        sorted_unique = np.concatenate([np.array([zr.na_of(st)], zr.NPT[st]), uniq]) if na else uniq   # NA first
        for op, want in (("union_ae", sorted_unique), ("union_ea", sorted_unique), ("setdiff_ae", sorted_unique),
                         ("symdiff_ae", sorted_unique), ("symdiff_ea", sorted_unique)):
            c = BY_NAME[f"set.{t}.{op}"]
            assert c["stypes"] == [st] and same(A(c, "r0"), want), (t, op)
        for op in ("intersect_ae", "intersect_ea", "setdiff_ea", "union_ee", "intersect_ee", "setdiff_ee",
                   "symdiff_ee", "unique"):
            c = BY_NAME[f"set.{t}.{op}"]
            assert c["nrows"] == 0 and c["stypes"] == [st], (t, op)
        c = BY_NAME[f"stat.{t}.nunique"]
        assert c["nrows"] == 1 and all(same(A(c, f"r{i}"), np.array([0], np.int64)) for i in range(3))
        c = BY_NAME[f"stat.{t}.nmodal"]
        assert c["nrows"] == 1 and all(same(A(c, f"r{i}"), np.array([0], np.int64)) for i in range(3))
        c = BY_NAME[f"stat.{t}.mode"]
        assert c["stypes"] == [st, zr.FLOAT64, zr.INT32]
        assert all(same(A(c, f"r{i}"), np.array([zr.na_of(s)], zr.NPT[s])) for i, s in enumerate(c["stypes"]))


def frames(case):
    import datatable_b200 as dtb
    X = dtb.Frame({nm: A(case, f"x.{nm}") for nm in case["x"]}, stypes=case["x"])
    return {"X": X, "S": {}, "dt": dtb, "f": dtb.f, "g": dtb.g, "join": dtb.join, "by": dtb.by, "sort": dtb.sort,
            "np": np}


@pytest.mark.parametrize("case", [c for c in CASES if "error" in c and c["name"] not in REFERENCE_FAULTS],
                         ids=lambda c: c["name"])
def test_errors_before_the_device(case, monkeypatch):
    """The reference's error type and text, raised while the query is resolved: no library call runs."""
    env = frames(case)
    from datatable_b200 import engine

    def untouched(*a, **k):
        raise AssertionError("the device was touched")
    for fn in ("mask_rows", "int_rows", "join_gather", "join_index", "group", "gather", "Groupby", "cut", "qcut"):
        monkeypatch.setattr(engine, fn, untouched)
    etype, msg = case["error"]
    with pytest.raises({"NotImplementedError": NotImplementedError}[etype]) as e:
        eval(case["query"], env)
    assert e.value.args[0] == msg
