"""GPU: DT[i, j, join(J), by(), sort()] -- group, sort and reduce over the joined frame's columns (g.) -- and
dtb_join_gather, the join lookup that also reads J's columns.

- golden_v10 (tests/golden/make_golden_v10.py, from the unmodified reference) through Frame, with host and with
  device frames: names, stypes and row counts equal; integer, order and group columns bit for bit; float columns to
  the bounds of tests/helpers.assert_reducer_equal (1e-6 relative, float32 sums 2e-4).
- median and qcut of a g. column (the reference crashes on them) against the same function over the joined column
  added to X as a plain column.
- engine.join_gather against join_index followed by gather, bit for bit, at 1e7 X rows: J of 1e3 and 1e6 rows with
  dense keys (the direct-address lookup), dense keys with one gap and sparse keys (the binary search).
"""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = json.load(open(os.path.join(G, "golden_v10.json")))["cases"]
ARR = dict(np.load(os.path.join(G, "golden_v10.npz")))
FLOAT32 = 6


def A(case, key):
    return ARR[f"{case['name']}.{key}"]


def host(a):
    return a.cpu().numpy() if hasattr(a, "cpu") else np.asarray(a)


def frames(case, device):
    import datatable_b200 as dtb
    X = dtb.Frame({nm: A(case, f"x.{nm}") for nm in case["x"]}, stypes=case["x"])
    J = dtb.Frame({nm: A(case, f"j.{nm}") for nm in case["j"]}, stypes=case["j"])
    if device:
        X, J = X.to_device(), J.to_device()
    J.key = case["jkey"]
    return X, J


def run(case, X, J):
    import datatable_b200 as dtb
    return eval(case["query"], {"X": X, "J": J, "dt": dtb, "f": dtb.f, "g": dtb.g, "join": dtb.join, "by": dtb.by,
                                "sort": dtb.sort})


def mismatch(got, want, st, op):
    """None when got matches the reference's column, else what differs"""
    got = host(got)
    if got.dtype != want.dtype or got.shape != want.shape:
        return f"{got.dtype}{got.shape} != {want.dtype}{want.shape}"
    if got.dtype.kind != "f":
        return None if np.array_equal(got, want) else "values"
    nan = np.isnan(want)
    if not np.array_equal(np.isnan(got), nan):
        return "NA pattern"
    g, w = got[~nan].astype(np.float64), want[~nan].astype(np.float64)
    rtol = 2e-4 if st == FLOAT32 and op in ("sum", "cumsum") else 1e-6
    inf = np.isinf(w)
    if not np.array_equal(g[inf], w[inf]):
        return "infinities"
    err = np.abs(g[~inf] - w[~inf])
    return None if np.all(err <= rtol * np.abs(w[~inf]) + 1e-12) else f"max abs err {err.max()}"


def op_of(case):
    q = case["query"]
    return "cumsum" if "cumsum" in q else ("sum" if "sum(" in q else None)


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("prefix", sorted({c["name"].split(".")[0] for c in CASES}))
def test_golden_through_frame(prefix, device):
    bad = []
    for case in CASES:
        if case["name"].split(".")[0] != prefix:
            continue
        X, J = frames(case, device)
        if "error" in case:
            if case["name"] == "query.f_fallback":           # f.x resolves to J's x where X has none (README)
                R, W = run(case, X, J), run({**case, "query": case["query"].replace("f.", "g.")}, X, J)
                if R.names != W.names or any(mismatch(R.column(n), host(W.column(n)), 0, None) for n in R.names):
                    bad.append(case["name"])
                continue
            try:
                run(case, X, J)
                bad.append(case["name"] + " raised nothing")
            except Exception as e:                            # noqa: BLE001
                if type(e).__name__ != case["error"][0] or e.args[0].replace("`", "") != case["error"][1]:
                    bad.append(f"{case['name']}: {type(e).__name__}: {e}")
            continue
        R = run(case, X, J)
        if list(R.names) != case["names"] or list(R.stypes) != case["stypes"] or R.nrows != case["nrows"]:
            bad.append(f"{case['name']}: {R.names} {R.stypes} {R.nrows}")
            continue
        for i, nm in enumerate(R.names):
            if device != (hasattr(R.column(nm), "is_cuda") and R.column(nm).is_cuda):
                bad.append(f"{case['name']} {nm}: result in the wrong memory")
            why = mismatch(R.column(nm), A(case, f"r{i}"), case["stypes"][i], op_of(case))
            if why:
                bad.append(f"{case['name']} {nm}: {why}")
    assert not bad, bad


@pytest.mark.parametrize("device", [False, True])
def test_sorted_functions_of_g_columns(device):
    """median / qcut of g.w equal median / qcut of the joined column w made a column of X"""
    import datatable_b200 as dtb
    from datatable_b200 import f, g, join, by
    case = next(c for c in CASES if c["name"] == "query.all")
    X, J = frames(case, device)
    plain = X[:, :, join(J)]                                 # X's columns, then J's non-key columns
    for q_g, q_f in ((lambda D: D[:, dtb.median(g.w), join(J), by(f.a)], lambda D: D[:, dtb.median(f.w), by(f.a)]),
                     (lambda D: D[:, dtb.qcut(g.price, 3), join(J), by(f.a)],
                      lambda D: D[:, dtb.qcut(f.price, 3), by(f.a)])):
        R, W = q_g(X), q_f(plain)
        assert R.names == W.names and R.stypes == W.stypes
        for nm in R.names:
            assert np.array_equal(host(R.column(nm)), host(W.column(nm)), equal_nan=True), nm


def _keys(layout, nj, rng):
    if layout == "dense":
        return np.arange(nj, dtype=np.int32) + 1000
    if layout == "gap":
        k = np.arange(nj + 1, dtype=np.int32) + 1000
        return np.delete(k, nj // 2)
    return np.sort(rng.choice(np.arange(-2**30, 2**30, 97, dtype=np.int64), nj, replace=False)).astype(np.int32)


@pytest.mark.parametrize("layout", ["dense", "gap", "sparse"])
@pytest.mark.parametrize("nj", [1000, 1_000_000])
def test_join_gather_matches_index_then_gather(layout, nj):
    import torch
    from datatable_b200 import engine, _lib
    rng = np.random.default_rng(nj + len(layout))
    n = 10_000_000
    jk = _keys(layout, nj, rng)
    jk[0] = -2**31 if layout == "dense" else jk[0]             # a leading NA key for the dense layout
    jk = np.sort(jk)                                          # NA first
    pool = np.concatenate([jk, jk[1:20] + 1, [-2**31, 2**31 - 1, 0]]).astype(np.int32)
    xk = torch.from_numpy(rng.choice(pool, n)).cuda()
    jkd = torch.from_numpy(jk).cuda()
    vals = [(torch.from_numpy(rng.random(nj)).cuda(), _lib.FLOAT64),
            (torch.from_numpy(rng.integers(-2**31 + 1, 2**31, nj).astype(np.int32)).cuda(), _lib.INT32),
            (torch.from_numpy(rng.integers(-127, 128, nj).astype(np.int8)).cuda(), _lib.INT8),
            (torch.from_numpy(rng.integers(-2**15 + 1, 2**15, nj).astype(np.int16)).cuda(), _lib.INT16),
            (torch.from_numpy(rng.random(nj).astype(np.float32)).cuda(), _lib.FLOAT32)]
    index = engine.join_index([xk], [jkd])
    got_index, got = engine.join_gather([xk], [jkd], [engine.Col(v, st) for v, st in vals], index=True)
    assert torch.equal(got_index, index)
    assert int((index >= 0).sum()) > n // 2
    for (v, st), o in zip(vals, got):
        want = engine.gather(engine.Col(v, st), index)
        assert o.dtype == want.dtype and torch.equal(o.view(torch.uint8), want.view(torch.uint8)), st
    # more value columns than one launch takes: the later ones come from a repeated lookup
    many = engine.join_gather([xk], [jkd], [engine.Col(vals[0][0], _lib.FLOAT64)] * 20)
    assert all(torch.equal(m.view(torch.uint8), got[0].view(torch.uint8)) for m in many)
