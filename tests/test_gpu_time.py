"""GPU: the time functions (dtb_time_part, engine.time_part, datatable_b200.time through the Frame) against the
reference's goldens (golden_v14) and, over every date32 day in [-1e6, 1e6] and 1e7 random values of the whole int32 and
int64 ranges, bit for bit against the numpy restatement in tests/time_reference.py.
"""
import numpy as np
import pytest

from oracle import oracle as orc
from time_reference import (CODE, DATE32, FLOAT64, INT32, INT64, NA, PARTS, TIME64, at_rows, case_rows, frame_query,
                            j_parts, joined, load_golden, time_part)

pytestmark = pytest.mark.gpu

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if "error" not in c]
PLAIN = [c for c in CASES if c["mode"] in ("none", "sort", "sortdesc", "join")]
STYPES = {"stype.int32": INT32, "stype.int64": INT64, "stype.float64": FLOAT64, "stype.date32": DATE32,
          "stype.time64": TIME64}


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
        return np.array_equal(np.isnan(got), nan) and np.allclose(got[~nan], want[~nan], rtol=1e-12, atol=1e-12)
    return got.dtype == want.dtype and np.array_equal(got, want)


@pytest.mark.parametrize("order64", [False, True], ids=["i32", "i64"])
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_engine_against_golden(eng, device, order64):
    """engine.time_part of every time-part output of every case without by(), through the query's RowIndex (negative
    entries: NA rows), with host or device buffers.  A failure names every case that differs."""
    engine, torch = eng
    put = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if device else (lambda a: a)
    bad = []
    for case in PLAIN:
        rows = case_rows(case, ARR, orc)
        order = None
        if rows is not None:
            order = np.where(rows < 0, -1 if order64 else NA[INT32], rows).astype(np.int64 if order64 else np.int32)
        for idx, part, (kind, c) in j_parts(case):
            if kind == "J":
                v, st = joined(case, ARR, c)
            else:
                v, st = ARR[case["name"] + "." + c], case["stypes"][c]
            got = engine.time_part(CODE[part], put(v), None if order is None else put(order), stype=st)
            if engine.is_tensor(got) != device or not _same(got, ARR[case["name"] + ".out_" + case["names"][idx]]):
                bad.append((case["name"], idx))
    assert not bad, bad


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_frame_against_golden(eng, device):
    """Every golden case through the Frame: names, stypes and values, or the error with the reference's text."""
    import datatable_b200 as dtb
    bad = []
    for case in ALL_CASES:
        if case.get("call"):
            continue
        try:
            R = frame_query(dtb, case, ARR, device)
        except Exception as e:                                   # noqa: BLE001
            if (type(e).__name__, str(e)) != (case.get("error"), case.get("message")):
                bad.append((case["name"], type(e).__name__, str(e)))
            continue
        if "error" in case:
            bad.append((case["name"], "no error"))
            continue
        if list(R.names) != case["names"] or R.nrows != case["nrows"]:
            bad.append((case["name"], list(R.names), R.nrows))
            continue
        for nm, st in zip(case["names"], case["out_stypes"]):
            if R._stypes[nm] != STYPES[st] or not _same(R.to_numpy(nm), ARR[case["name"] + ".out_" + nm]):
                bad.append((case["name"], nm))
    assert not bad, bad


def test_reducer_next_to_a_time_part(eng):
    """A reducer in the same j, or a time part as a reducer's argument, is refused as for every row function."""
    import datatable_b200 as dtb
    f, T = dtb.f, dtb.time
    DT = dtb.Frame({"d": np.array([1, 400, 800], np.int32), "v": np.array([1.0, 2.0, 3.0])}, stypes={"d": DATE32})
    for q in ((slice(None), [T.year(f.d), dtb.sum(f.v)]), (slice(None), [T.year(f.d), dtb.sum(f.v)], dtb.by(f.d)),
              (slice(None), dtb.sum(T.year(f.d))), (slice(None), dtb.sum(T.year(f.d)), dtb.by(T.year(f.d)))):
        with pytest.raises(NotImplementedError):
            DT[q]


@pytest.mark.parametrize("order_kind", ["identity", "i32", "i64"])
def test_every_day_and_random_values(eng, order_kind):
    """Every date32 day in [-1e6, 1e6] and 1e7 random values over the whole int32 and int64 ranges, every part, bit for
    bit against the restatement.  Through a RowIndex the values are read through a shuffled order with entries < 0."""
    engine, torch = eng
    rng = np.random.default_rng(14)
    days = np.concatenate([np.arange(-10**6, 10**6 + 1), rng.integers(-2**31 + 1, 2**31, 10**7)]).astype(np.int32)
    days[::1001] = NA[DATE32]
    times = rng.integers(-2**63 + 1, 2**63 - 1, 10**7, dtype=np.int64, endpoint=True)
    times[: 2 * 10**6] //= 10**4                              # instants within the years 1677 .. 2262 too
    times[::997] = NA[TIME64]
    for st, v in ((DATE32, days), (TIME64, times)):
        vd = torch.from_numpy(v).cuda()
        rows, od = None, None
        if order_kind != "identity":
            rows = rng.permutation(len(v)).astype(np.int64)
            rows[::1009] = -1
            o = rows if order_kind == "i64" else np.where(rows < 0, NA[INT32], rows).astype(np.int32)
            od = torch.from_numpy(o).cuda()
        src = at_rows(v, st, rows)
        for part in (PARTS if st == TIME64 else PARTS[:4]):
            got = engine.time_part(CODE[part], vd, od, stype=st).cpu().numpy()
            assert np.array_equal(got, time_part(part, src, st)), (st, part)


def test_misaligned_device_column(eng):
    """A device column that starts off a 16-byte boundary takes the element-by-element identity path."""
    engine, torch = eng
    v = np.arange(-5000, 5003, dtype=np.int64) * 3_600_000_000_123
    vd = torch.from_numpy(v).cuda()
    for off in (1, 2, 3):
        got = engine.time_part(CODE["hour"], vd[off:], None, stype=TIME64).cpu().numpy()
        assert np.array_equal(got, time_part("hour", v[off:], TIME64))


def test_by_year_sum_1e8_rows(eng):
    """DT[:, sum(f.v), by(year(f.d))] over 1e8 device rows equals grouping a year column computed on the host."""
    import datatable_b200 as dtb
    engine, torch = eng
    rng = np.random.default_rng(8)
    n = 100_000_000
    d = rng.integers(-40000, 40000, n).astype(np.int32)
    d[::4099] = NA[DATE32]
    v = rng.integers(-1000, 1000, n).astype(np.int64)
    y = time_part("year", d, DATE32)
    D = dtb.Frame({"d": torch.from_numpy(d).cuda(), "v": torch.from_numpy(v).cuda()}, stypes={"d": DATE32})
    Y = dtb.Frame({"d": torch.from_numpy(y).cuda(), "v": torch.from_numpy(v).cuda()})
    got = D[:, dtb.sum(dtb.f.v), dtb.by(dtb.time.year(dtb.f.d))]
    want = Y[:, dtb.sum(dtb.f.v), dtb.by(dtb.f.d)]
    assert got.names == want.names == ("d", "v")
    assert np.array_equal(got.to_numpy("d"), want.to_numpy("d"))
    assert np.array_equal(got.to_numpy("v"), want.to_numpy("v"))
    assert got._stypes["d"] == INT32
