"""GPU: DT[i, j] with `i` a boolean or integer column, a list or a range.

- dtb_mask_rows bit for bit against np.flatnonzero: sizes at the 4096-row rounds and 32768-row tiles +-1, densities
  0, 1e-6, 0.5, 1 - 1e-6 and 1, clustered runs, bytes other than 0 / 1 / -128, host and device masks, a mask that
  starts one byte into its buffer, and 1e9 rows;
- dtb_int_rows against numpy for every integer stype;
- the Frame against every golden_v11 case (tests/golden/make_golden_v11.py), host and device frames;
- seeded frames up to 1e8 rows against tests/rows_reference.py.
"""
import json
import os

import numpy as np
import pytest

import rows_reference as rr

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = json.load(open(os.path.join(G, "golden_v11.json")))["cases"]
ARR = dict(np.load(os.path.join(G, "golden_v11.npz")))
BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64 = 1, 2, 3, 4, 5, 6, 7
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63}
NPT = {INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64}

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    torch.cuda.set_device(0)
    return torch


def _mask(rng, n, density, clustered=False):
    if clustered:                                   # runs of selected and unselected rows, 1 .. 5000 rows long
        lens = rng.integers(1, 5000, n // 1000 + 2)
        m = np.repeat(np.arange(len(lens)) % 2, lens)[:n]
        m = np.concatenate([m, np.zeros(n - len(m), m.dtype)]).astype(np.int8)
    else:
        m = (rng.random(n) < density).astype(np.int8)
    na = rng.random(n) < 0.01
    m[na & (m == 0)] = -128
    return m


def _rows(engine, torch, m, device):
    out = engine.mask_rows(torch.from_numpy(m).cuda() if device else m)
    return out.cpu().numpy() if device else out


SIZES = [0, 1, 15, 16, 17, 4095, 4096, 4097, 32767, 32768, 32769, 65535, 65537, 1_000_003]


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_mask_rows_against_flatnonzero(torch, device):
    from datatable_b200 import engine
    rng = np.random.default_rng(11)
    for n in SIZES:
        for density in (0.0, 1e-6, 0.5, 1 - 1e-6, 1.0):
            m = _mask(rng, n, density)
            got = _rows(engine, torch, m, device)
            assert got.dtype == np.int32 and np.array_equal(got, rr.mask_rows(m)), (n, density)
        m = _mask(rng, n, 0, clustered=True)
        assert np.array_equal(_rows(engine, torch, m, device), rr.mask_rows(m)), (n, "clustered")


def test_mask_rows_any_byte_and_offsets(torch):
    from datatable_b200 import engine
    rng = np.random.default_rng(12)
    for n in (33, 4097, 32769, 100_001):
        m = rng.integers(-128, 128, n + 3).astype(np.int8)
        d = torch.from_numpy(m).cuda()
        for off in (0, 1, 3):                      # a view that starts off bytes into its buffer
            got = engine.mask_rows(d[off:off + n]).cpu().numpy()
            assert np.array_equal(got, rr.mask_rows(m[off:off + n])), (n, off)


def test_mask_rows_1e9(torch):
    from datatable_b200 import engine
    n = 1_000_000_000
    rng = np.random.default_rng(13)
    m = (rng.random(n, dtype=np.float32) < 1e-3).astype(np.int8)
    m[::7919] = -128
    got = engine.mask_rows(torch.from_numpy(m).cuda()).cpu().numpy()
    assert np.array_equal(got, rr.mask_rows(m))
    full = torch.ones(n, dtype=torch.int8, device="cuda")
    got = engine.mask_rows(full)
    assert got.numel() == n and int(got[-1]) == n - 1 and bool((got[1:] - got[:-1] == 1).all())


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("st", [INT8, INT16, INT32, INT64])
def test_int_rows_against_numpy(torch, st, device):
    from datatable_b200 import engine
    rng = np.random.default_rng(14)
    for n in (0, 1, 7, 4099, 1_000_001):
        a = rng.integers(0, 120, n).astype(NPT[st])
        a[rng.random(n) < 0.1] = NA[st]
        rows, lo, hi, nna = engine.int_rows(torch.from_numpy(a).cuda() if device else a, st)
        rows = rows.cpu().numpy() if device else rows
        want = rr.int_rows(a, NA[st])
        assert rows.dtype == np.int32 and np.array_equal(rows.astype(np.int64), np.where(want < 0, -2**31, want))
        valid = a[a != NA[st]]
        assert nna == n - len(valid)
        if len(valid):
            assert (lo, hi) == (int(valid.min()), int(valid.max()))


# ---- the Frame against the goldens -----------------------------------------------------------------------------------
def A(case, key):
    return ARR[f"{case['name']}.{key}"]


def _env(case, device):
    import datatable_b200 as dtb

    def fr(cols, prefix):
        F = dtb.Frame({nm: A(case, f"{prefix}.{nm}") for nm in cols}, stypes=cols)
        return F.to_device() if device else F
    env = {"X": fr(case["x"], "x"), "S": {s: fr(cols, f"s.{s}") for s, cols in case["s"].items()},
           "A": {nm: A(case, f"a.{nm}") for nm in case["a"]}, "dt": dtb, "f": dtb.f, "g": dtb.g, "join": dtb.join,
           "by": dtb.by, "sort": dtb.sort, "np": np}
    if case["name"] == "err.frame_keyed":
        env["S"]["s"].key = "C0"
    if case["j"]:
        env["J"] = fr(case["j"], "j")
        env["J"].key = case["jkey"]
    return env


def _same(got, want, rtol):
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    if got.dtype.kind != "f":
        return np.array_equal(got, want)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.allclose(got[~nan], want[~nan], rtol=rtol, atol=0)


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
# DT[True, :] keeps its NotImplementedError.
@pytest.mark.parametrize("case", [c for c in CASES if c["name"] not in ("err.bool_literal",)],
                         ids=lambda c: c["name"])
def test_frame_against_golden(torch, case, device):
    env = _env(case, device)
    if "error" in case or "reference_crash" in case:
        etype, msg = case["error"] if "error" in case else rr.SOURCE_ERRORS[case["name"]]
        with pytest.raises(Exception) as e:
            eval(case["query"], env)
        assert etype in [t.__name__ for t in type(e.value).__mro__], (type(e.value), etype)
        assert e.value.args[0].replace("`", "") == msg.replace("`", "")
        return
    R = eval(case["query"], env)
    assert list(R.names) == case["names"] and R.nrows == case["nrows"]
    for i, nm in enumerate(R.names):
        assert R.stypes[i] == case["stypes"][i], (case["name"], nm)
        assert _same(R.to_numpy(nm), A(case, f"r{i}"), 1e-9), (case["name"], nm)


# ---- seeded frames at scale --------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [10_000_019, 100_000_000])
def test_seeded_frames_against_the_restatement(torch, n):
    import datatable_b200 as dtb
    rng = np.random.default_rng(n)
    m = _mask(rng, n, 0.3)
    v = rng.integers(-1000, 1000, n).astype(np.float64)
    DT = dtb.Frame({"m": m, "v": v}, stypes={"m": BOOL, "v": FLOAT64}).to_device()
    ri = rr.mask_rows(m)
    got = DT[dtb.f.m, dtb.f.v].to_numpy("v")
    assert np.array_equal(got, v[ri])
    assert DT[dtb.f.m, dtb.sum(dtb.f.v)].to_numpy("v")[0] == v[ri].sum()          # integer values: exact
    cs = DT[dtb.f.m, dtb.cumsum(dtb.f.v)].to_numpy("v")
    assert np.array_equal(cs, np.cumsum(v[ri]))
    idx = rng.integers(0, n, n // 10).astype(np.int64)
    idx[::101] = NA[INT64]
    ri2 = rr.int_rows(idx, NA[INT64])
    R = DT[dtb.Frame({"i": idx}, stypes={"i": INT64}), dtb.f.v]
    assert np.array_equal(R.to_numpy("v"), rr.gather(v, ri2, np.nan), equal_nan=True)
    sel = [5, -1, None, slice(10, 20, 3), range(n - 1, n - 10, -4)]
    assert np.array_equal(DT[sel, dtb.f.v].to_numpy("v"), v[rr.rows(sel, n)])
