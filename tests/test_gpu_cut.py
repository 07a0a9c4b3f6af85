"""GPU: dt.cut (dtb_cut, engine.cut, the Frame's cut()) against the reference's goldens (golden_v12) and, on large
seeded inputs, bit for bit against the numpy restatement in tests/cut_reference.py.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from cut_reference import (FLOAT32, FLOAT64, INT8, INT32, INT64, NA, at_rows, case_edges, case_rows, cut_bins,
                           cut_column, cut_nbins, frame_query, j_sources, load_golden)

pytestmark = pytest.mark.gpu

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if "error" not in c]
STYPES = {"stype.int32": INT32, "stype.float64": FLOAT64, "stype.float32": FLOAT32, "stype.int64": INT64}


@pytest.fixture(scope="module")
def eng():
    import torch
    torch.cuda.set_device(0)
    from datatable_b200 import engine
    return engine, torch


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _same(got, want):
    got, want = _np(got), np.asarray(want)
    if want.dtype.kind == "f":
        nan = np.isnan(want)
        return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan], want[~nan])
    return got.dtype == want.dtype and np.array_equal(got, want)


@pytest.mark.parametrize("order64", [False, True], ids=["i32", "i64"])
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_engine_cut_golden(eng, case, device, order64):
    """engine.cut of every cut output of the case that reads the query's frame, through the query's RowIndex."""
    engine, torch = eng
    rows = case_rows(case, ARR, orc)
    edges = case_edges(case, ARR)
    nb = case["nbins"]
    nbs = nb if isinstance(nb, list) else [10 if nb is None else nb]
    rc = True if case["right_closed"] is None else case["right_closed"]
    put = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if device else (lambda a: a)
    order = None
    if rows is not None:
        order = np.where(rows < 0, -1 if order64 else NA[INT32], rows).astype(np.int64 if order64 else np.int32)
    for k, (idx, (kind, src)) in enumerate(j_sources(case)):
        if kind == "J":
            continue
        st = case["stypes"][src] if kind in ("x", "frame") else case["other_stype"]
        v = ARR[case["name"] + "." + src] if kind != "other" else ARR[case["name"] + ".other.z"]
        got = engine.cut(put(v), None if (order is None or kind != "x") else put(order), nbs[k % len(nbs)],
                         None if edges is None else edges[k], rc, stype=st)
        assert engine.is_tensor(got) == device
        assert _same(got, ARR[case["name"] + ".out_" + case["names"][idx]]), case["names"][idx]


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("case", ALL_CASES, ids=[c["name"] for c in ALL_CASES])
def test_frame_cut_golden(eng, case, device):
    import datatable_b200 as dtb
    if "error" in case:
        with pytest.raises(Exception) as ei:
            frame_query(dtb, case, ARR, device)
        assert (type(ei.value).__name__, str(ei.value)) == (case["error"], case["message"])
        return
    R = frame_query(dtb, case, ARR, device)
    assert list(R.names) == case["names"]
    assert R.nrows == case["nrows"]
    for nm, st in zip(case["names"], case["out_stypes"]):
        if st in STYPES:
            assert R._stypes[nm] == STYPES[st]
            assert _same(R.to_numpy(nm), ARR[case["name"] + ".out_" + nm]), nm


# ---- large seeded cases against the restatement --------------------------------------------------------------------
def _column(rng, st, n):
    if st in (FLOAT32, FLOAT64):
        v = (rng.standard_normal(n) * 1e3).astype(np.float64 if st == FLOAT64 else np.float32)
        v[rng.random(n) < 0.01] = np.nan
        v[:: 7919] = -0.0
    elif st == INT64:
        v = rng.integers(-2**62, 2**62, n, dtype=np.int64)
        v[rng.random(n) < 0.01] = NA[INT64]
    else:
        dt_ = np.int8 if st == INT8 else np.int32
        v = rng.integers(np.iinfo(dt_).min + 1, np.iinfo(dt_).max, n, dtype=dt_)
        v[rng.random(n) < 0.01] = NA[st]
    return v


@pytest.mark.parametrize("st", [INT8, INT32, INT64, FLOAT32, FLOAT64])
@pytest.mark.parametrize("order_kind", ["identity", "i32", "i64"])
def test_large_nbins(eng, st, order_kind):
    engine, torch = eng
    rng = np.random.default_rng(1000 + st)
    n = 20_000_000
    v = _column(rng, st, n)
    vd = torch.from_numpy(v).cuda()
    rows = None
    od = None
    if order_kind != "identity":
        rows = np.flatnonzero(rng.random(n) < 0.5)             # a density-0.5 mask selection
        rng.shuffle(rows)
        rows[:: 1009] = -1                                      # NA rows
        o = rows.astype(np.int64) if order_kind == "i64" else np.where(rows < 0, NA[INT32], rows).astype(np.int32)
        od = torch.from_numpy(o).cuda()
    for nbins, rc in ((10, True), (1000, False), (2**31 - 1, True), (7, False)):
        got = engine.cut(vd, od, nbins, None, rc, stype=st).cpu().numpy()
        want = cut_nbins(at_rows(v, st, rows), st, nbins, rc)
        assert np.array_equal(got, want), (nbins, rc)


@pytest.mark.parametrize("nedges", [2, 1000, 4096, 4097, 8193, 100_000])
@pytest.mark.parametrize("rc", [True, False])
def test_large_bins(eng, nedges, rc):
    """Both sides of the shared-memory limit (4096 edges): every k-th edge staged, the window searched in L2."""
    engine, torch = eng
    rng = np.random.default_rng(nedges)
    n = 10_000_000
    e = np.sort(rng.choice(np.unique(rng.standard_normal(nedges * 2) * 1e3), nedges, replace=False))
    v = _column(rng, FLOAT64, n)
    v[: 2 * nedges: 2] = e                                     # values on the edges
    vd = torch.from_numpy(v).cuda()
    rows = rng.integers(-5, n, n // 2)
    od = torch.from_numpy(np.where(rows < 0, NA[INT32], rows).astype(np.int32)).cuda()
    got = engine.cut(vd, None, edges=e, right_closed=rc).cpu().numpy()
    assert np.array_equal(got, cut_bins(v, FLOAT64, e, rc))
    got = engine.cut(vd, od, edges=e, right_closed=rc).cpu().numpy()
    assert np.array_equal(got, cut_bins(at_rows(v, FLOAT64, np.where(rows < 0, -1, rows)), FLOAT64, e, rc))
    vi = _column(rng, INT32, n)
    got = engine.cut(torch.from_numpy(vi).cuda(), None, edges=e, right_closed=rc).cpu().numpy()
    assert np.array_equal(got, cut_bins(vi, INT32, e, rc))


def test_negative_int64_indices_are_na_rows(eng):
    """Every int64 index < 0 (or >= nrows) is an NA row: it is left out of the statistics and gives NA."""
    engine, torch = eng
    v = np.array([4.0, -1.0, 2.5, 10.0, 7.0])
    order = np.array([0, -2, 1, -1, 3, np.iinfo(np.int64).min, 4, 5, -3, 2], dtype=np.int64)
    for rc in (True, False):
        got = engine.cut(torch.from_numpy(v).cuda(), torch.from_numpy(order).cuda(), 4, None, rc).cpu().numpy()
        rows = np.where((order >= 0) & (order < len(v)), order, -1)
        want = cut_nbins(at_rows(v, FLOAT64, rows), FLOAT64, 4, rc)
        assert np.array_equal(got, want)
        assert (got[[1, 3, 5, 7, 8]] == NA[INT32]).all()


def test_frame_large_mask(eng):
    """The Frame over a boolean selection of 2e7 rows: the statistics are those of the selected rows."""
    import datatable_b200 as dtb
    engine, torch = eng
    rng = np.random.default_rng(7)
    n = 20_000_000
    x = _column(rng, FLOAT64, n)
    b = (rng.random(n) < 0.5).astype(np.int8)
    fr = dtb.Frame({"x": torch.from_numpy(x).cuda(), "b": torch.from_numpy(b).cuda()}, stypes={"b": dtb._lib.BOOL})
    R = fr[dtb.f.b, dtb.cut(dtb.f.x, nbins=100)]
    assert np.array_equal(R.to_numpy("x"), cut_nbins(x[b == 1], FLOAT64, 100))


def test_1e9_rows(eng):
    """A 1e9-row float64 device column: the restatement on a strided sample, and the histogram of the bins against
    np.bincount of the restatement over the whole column, computed on the host in chunks."""
    engine, torch = eng
    n, nbins = 1_000_000_000, 1000
    gen = torch.Generator(device="cuda").manual_seed(12)
    vd = torch.randn(n, dtype=torch.float64, device="cuda", generator=gen)
    vd[::997] = float("nan")
    out = engine.cut(vd, None, nbins)
    torch.cuda.synchronize()
    got_hist = torch.bincount(out[out >= 0].long(), minlength=nbins).cpu().numpy()
    got_na = int((out < 0).sum())
    got_sample = out[::9973].cpu().numpy()
    del out
    valid = ~torch.isnan(vd)
    bounds = (float(vd[valid].min()), float(vd[valid].max()))
    del valid
    v_sample = vd[::9973].cpu().numpy()
    assert np.array_equal(got_sample, cut_nbins(v_sample, FLOAT64, nbins, bounds=bounds))
    want_hist = np.zeros(nbins, dtype=np.int64)
    want_na = 0
    step = 50_000_000
    for a in range(0, n, step):
        w = cut_nbins(vd[a:a + step].cpu().numpy(), FLOAT64, nbins, bounds=bounds)
        want_na += int((w < 0).sum())
        want_hist += np.bincount(w[w >= 0], minlength=nbins)
    assert got_na == want_na == len(range(0, n, 997))
    assert np.array_equal(got_hist, want_hist)
