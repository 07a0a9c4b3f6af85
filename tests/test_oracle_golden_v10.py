"""CPU: golden_v10 (DT[i, j, join(J), by(), sort()] from the unmodified reference, tests/golden/make_golden_v10.py)
restated with numpy: J sorted by its key (the oracle's group()), the join by tests/join_reference.py, J's columns
gathered into X's row order, then the oracle's group() and reducers over those columns.  The restatement covers the
reducer queries under by() (f. or g. keys) and the queries that only select rows and columns; the other shapes are
checked on the GPU (tests/test_gpu_join_groupby.py).  Also: the query's argument errors (g. without a join, a
missing g. column) are raised before the device is touched.
"""
import json
import os

import numpy as np
import pytest

from oracle import oracle as orc
from join_reference import BOOL, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64, NA, NPT, join_index

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = json.load(open(os.path.join(G, "golden_v10.json")))["cases"]
ARR = dict(np.load(os.path.join(G, "golden_v10.npz")))
PLAIN = {DATE32: INT32, TIME64: INT64}                  # the oracle compares dates and times as their storage
OPS = {"sum": orc.SUM, "mean": orc.MEAN, "min": orc.MIN, "max": orc.MAX, "count": orc.COUNT}


def A(case, key):
    return ARR[f"{case['name']}.{key}"]


def joined(case):
    """{"f.x": X's column x, "g.x": J's column x in X's row order (NA where no row of J matches)}, {ref: stype}"""
    keys = case["jkey"]
    xs = {f"f.{nm}": A(case, f"x.{nm}") for nm in case["x"]}
    sts = {f"f.{nm}": st for nm, st in case["x"].items()}
    jraw = {nm: A(case, f"j.{nm}") for nm in case["j"]}
    nj = len(jraw[keys[0]])
    order = (orc.group([jraw[k] for k in keys], [0] * len(keys), orc.NA_FIRST,
                       stypes=[PLAIN.get(case["j"][k], case["j"][k]) for k in keys])[0] if nj else np.zeros(0, np.int32))
    js = {nm: a[order] for nm, a in jraw.items()}
    idx = join_index([xs[f"f.{k}"] for k in keys], [case["x"][k] for k in keys], [js[k] for k in keys],
                     [case["j"][k] for k in keys])
    for nm, st in case["j"].items():
        v = np.full(len(idx), np.nan if st in (FLOAT32, FLOAT64) else NA[st], NPT[st])
        hit = idx >= 0
        v[hit] = js[nm][idx[hit]]
        xs[f"g.{nm}"], sts[f"g.{nm}"] = v, st
    return xs, sts


def same(got, want, rtol=0.0):
    """dtype and shape equal; integers exact; floats within rtol (NaN is NA)"""
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    if got.dtype.kind != "f":
        return np.array_equal(got, want)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.allclose(got[~nan], want[~nan], rtol=rtol, atol=0)


def test_golden_covers_the_ground():
    names = {c["name"] for c in CASES}
    jst = {c["j"]["k"] for c in CASES if c["name"].startswith("jst.")}
    assert jst == {BOOL, 2, 3, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64}
    for prefix in ("gap.", "sparse.", "multi.", "mixed.i32_f64", "mixed.f64_i32", "empty.x", "empty.j", "dense."):
        assert any(n.startswith(prefix) for n in names), prefix
    assert {len(c["jkey"]) for c in CASES} == {1, 2, 3}
    assert {c["name"] for c in CASES if "error" in c} == {"query.err_nojoin", "query.err_missing", "query.f_fallback"}
    assert sum("restate" in c for c in CASES) >= 40


@pytest.mark.parametrize("case", [c for c in CASES if "restate" in c], ids=lambda c: c["name"])
def test_reducers_by_restated(case):
    cols, sts = joined(case)
    by_ = case["restate"]["by"]
    n = len(cols[by_[0]])
    want = [A(case, f"r{i}") for i in range(len(case["names"]))]
    assert case["nrows"] == len(want[0])
    if n == 0:
        assert all(len(w) == 0 for w in want)
        return
    order, offsets, ng = orc.group([cols[r] for r in by_], [0] * len(by_), orc.NA_FIRST,
                                   stypes=[PLAIN.get(sts[r], sts[r]) for r in by_])
    assert ng == case["nrows"], case["name"]
    for i, r in enumerate(by_):                                  # the keys: first row of every group
        assert same(cols[r][order[offsets[:-1]]], want[i]), (case["name"], r)
    for i, (op, r) in enumerate(case["restate"]["red"], start=len(by_)):
        if r is None:
            got = np.diff(offsets).astype(np.int64)
        else:
            st = sts[r]
            got = orc.reduce(OPS[op], cols[r], order, offsets, stype=PLAIN.get(st, st))
        assert same(got, want[i], rtol=1e-6 if got.dtype.kind == "f" else 0), (case["name"], op, r)


SELECTS = {                    # case -> (rows of X, the result columns as f. / g. references)
    "query.all": (slice(None), None),
    "query.plain": (slice(None), ["f.a", "g.price", "g.k", "f.k", "g.region", "f.region"]),
    "query.i_slice": (slice(5, 40, 3), ["f.qty", "g.price", "g.region"]),
    "query.i_int": (slice(7, 8), None),
    "query.i_neg": (slice(-1, None), None),
}


@pytest.mark.parametrize("name", list(SELECTS))
def test_row_and_column_selection_restated(name):
    case = next(c for c in CASES if c["name"] == name)
    cols, _ = joined(case)
    rows, refs = SELECTS[name]
    if refs is None:                                             # j = :  X's columns, then J's non-key columns
        refs = [f"f.{nm}" for nm in case["x"]] + [f"g.{nm}" for nm in case["j"] if nm not in case["jkey"]]
    assert len(refs) == len(case["names"])
    for i, r in enumerate(refs):
        assert same(cols[r][rows], A(case, f"r{i}")), (name, r)


def test_f_name_falls_back_to_the_join_frame():
    """The reference's KeyError for f.x where only J has x; the engine reads J's x (a documented deviation)."""
    case = next(c for c in CASES if c["name"] == "query.f_fallback")
    assert case["error"][0] == "KeyError" and "price" not in case["x"] and "price" in case["j"]


def _frames(case):
    import datatable_b200 as dtb
    X = dtb.Frame({nm: A(case, f"x.{nm}") for nm in case["x"]}, stypes=case["x"])
    J = dtb.Frame({nm: A(case, f"j.{nm}") for nm in case["j"]}, stypes=case["j"])
    return dtb, X, J


@pytest.mark.parametrize("name", ["query.err_nojoin", "query.err_missing"])
def test_argument_errors_before_the_device(name, monkeypatch):
    """The reference's error type and text, raised while the query is resolved: neither the join nor group() runs."""
    dtb, X, J = _frames(next(c for c in CASES if c["name"] == name))
    from datatable_b200 import engine

    def untouched(*a, **k):
        raise AssertionError("the device was touched")
    for fn in ("join_gather", "join_index", "group", "gather"):
        monkeypatch.setattr(engine, fn, untouched)
    case = next(c for c in CASES if c["name"] == name)
    J._key = tuple(case["jkey"])               # setting a key sorts J on the device; the error comes before the join
    etype, msg = case["error"]
    with pytest.raises({"KeyError": KeyError, "ValueError": ValueError}[etype]) as e:
        eval(case["query"], {"X": X, "J": J, "dt": dtb, "f": dtb.f, "g": dtb.g, "join": dtb.join, "by": dtb.by,
                             "sort": dtb.sort})
    assert e.value.args[0].replace("`", "") == msg


def test_g_namespace():
    import datatable_b200 as dtb
    assert repr(dtb.g.x) == "g.x" and repr(-dtb.g["x"]) == "-g.x" and repr(dtb.f.x) == "f.x"
    assert (-dtb.g.x).frame == 1 and dtb.f.x.frame == 0
