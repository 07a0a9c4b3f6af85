"""CPU: the numpy restatement of the cumulative functions (tests/cumulative_reference.py) reproduces every golden_v7
case, its whole-group form agrees with its row-by-row form, the Frame checks cumsum / cumprod / cummin / cummax's
arguments with the reference's error texts before any library call, and dtb_cumulative returns its argument codes
before any GPU work.

golden_v7 comes from the unmodified reference (tests/golden/make_golden_v7.py).  Groups are formed by the C oracle
(oracle/dt_oracle.c, pinned to the reference by tests/test_oracle_golden*.py).
"""
import ctypes

import numpy as np
import pytest

from oracle import oracle as orc
import datatable_b200 as dtb
from datatable_b200 import _lib
from cumulative_reference import (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64, NA, NPT,
                                  cum_groups, expected_columns, load_golden)
from qcut_reference import qcut_groups

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if "error" not in c]
ERRORS = [c for c in ALL_CASES if "error" in c]
FNS = {"cumsum": dtb.cumsum, "cumprod": dtb.cumprod, "cummin": dtb.cummin, "cummax": dtb.cummax}


def test_golden_covers_the_ground():
    assert {c["stypes"]["x"] for c in CASES} == {BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64}
    assert {(c["fn"], c["rev"]) for c in CASES} == {(fn, r) for fn in FNS for r in (False, True)}
    assert {c["mode"] for c in CASES} == {"none", "by", "by2", "bysort", "sort", "sortdesc"}
    assert {c["j"] for c in CASES} == {"one", "list", "tuple", "all", "dict", "dictlist", "plain", "withqcut", "bykey"}
    assert any(c["nrows"] == 0 for c in CASES) and any(c["nrows"] == 1 for c in CASES)
    assert len(ERRORS) == 16


def _check(got, case):
    assert [nm for nm, _ in got] == case["names"]
    assert len(got) == len(case["out_stypes"])
    for nm, col in got:
        want = ARR[case["name"] + ".out_" + nm]
        assert len(col) == case["nrows"]
        assert col.dtype == want.dtype, nm
        if want.dtype.kind == "f":                                # bit for bit, -0.0 included; any NaN is NA
            assert np.array_equal(np.isnan(col), np.isnan(want)), nm
            ok = ~np.isnan(want)
            ui = np.uint32 if want.dtype == np.float32 else np.uint64
            assert np.array_equal(col[ok].view(ui), want[ok].view(ui)), nm
        else:
            assert np.array_equal(col, want), nm


FNREV = [(fn, rev) for fn in FNS for rev in (False, True)]
FNREV_IDS = [f"{fn}{'-rev' if rev else ''}" for fn, rev in FNREV]


def _failures(fn, rev, loop):
    bad = []
    for case in CASES:
        if case["fn"] != fn or case["rev"] != rev:
            continue
        try:
            _check(expected_columns(case, ARR, orc, loop=loop, qcut=qcut_groups), case)
        except AssertionError as e:                                # noqa: PERF203
            bad.append(f"{case['name']}: {e}")
    return bad


@pytest.mark.parametrize("fn,rev", FNREV, ids=FNREV_IDS)
def test_restatement_reproduces_golden(fn, rev):
    bad = _failures(fn, rev, loop=True)
    assert not bad, bad


@pytest.mark.parametrize("fn,rev", FNREV, ids=FNREV_IDS)
def test_whole_group_form_reproduces_golden(fn, rev):
    bad = _failures(fn, rev, loop=False)
    assert not bad, bad


@pytest.mark.parametrize("fn", list(FNS))
@pytest.mark.parametrize("st", [BOOL, INT8, INT32, INT64, FLOAT32, FLOAT64, DATE32])
def test_whole_group_form_matches_the_loop(fn, st):
    if fn in ("cumsum", "cumprod") and st == DATE32:
        pytest.skip("cumsum / cumprod refuse date32")
    rng = np.random.default_rng(st * 10 + len(fn))
    n = 3000
    if st in (FLOAT32, FLOAT64):
        v = rng.choice(np.array([0.0, -0.0, 1.5, -2.0, 0.75, np.inf, -np.inf, np.nan, 3.0], NPT[st]), n)
    else:
        v = rng.integers(-5, 6, n).astype(NPT[st]) if st != BOOL else rng.integers(0, 2, n).astype(np.int8)
        v[rng.random(n) < 0.2] = NA[st]
    offsets = np.unique(np.concatenate([[0, n], rng.integers(1, n, 40)])).astype(np.int32)
    order = rng.permutation(n).astype(np.int32)
    for rev in (False, True):
        a = cum_groups(fn, v, st, order, offsets, rev, loop=True)
        b = cum_groups(fn, v, st, order, offsets, rev, loop=False)
        if a.dtype.kind == "f":
            ui = np.uint32 if a.dtype == np.float32 else np.uint64
            a, b = np.where(np.isnan(a), np.nan, a).view(ui), np.where(np.isnan(b), np.nan, b).view(ui)
        assert np.array_equal(a, b)


def _error_frame(xst):
    if xst == "f64":
        return dtb.Frame({"x": np.array([1.5, np.nan, 0.0])})
    st = {"date32": DATE32, "time64": TIME64}[xst]
    return dtb.Frame({"x": np.array([1, 2, 3], dtype=NPT[st])}, stypes={"x": st})


@pytest.mark.parametrize("case", [c for c in ERRORS if c["xstype"] != "str"],
                         ids=[c["name"] for c in ERRORS if c["xstype"] != "str"])
def test_frame_argument_errors_match_reference(case):
    """The checks run before any library call (they pass on a machine without a GPU)."""
    fr = _error_frame(case["xstype"])
    exc = {"ValueError": ValueError, "TypeError": TypeError}[case["error"]]
    with pytest.raises(exc) as ei:
        fr[:, FNS[case["fn"]](dtb.f.x, reverse=case["rev"])]
    assert str(ei.value) == case["message"]


def test_frame_argument_errors_in_every_query_shape():
    fr = dtb.Frame({"x": np.array([1, 2], np.int32), "g": np.array([1, 1], np.int32)}, stypes={"x": DATE32})
    f = dtb.f
    for mods in ((), (dtb.by(f.g),), (dtb.sort(f.g),), (dtb.by(f.g), dtb.sort(f.x))):
        with pytest.raises(TypeError, match=r"^Invalid column of type date32 in cumsum\(f.x, reverse=False\)$"):
            fr[(slice(None), dtb.cumsum(f.x)) + mods]
        with pytest.raises(TypeError, match=r"^Invalid column of type date32 in cumprod\(f\[:\], reverse=True\)$"):
            fr[(slice(0, 1), {"c": dtb.cumprod(f[:], reverse=True)}) + mods]
    with pytest.raises(TypeError, match="Argument reverse in function datatable.cummax"):
        dtb.cummax(f.x, reverse=None)


def test_abi_argument_codes_before_any_gpu_work():
    v = np.array([1.0, 2.0, 3.0])
    offs = np.array([0, 3], dtype=np.int32)
    out = np.empty(3, dtype=np.float64)

    def call(op=_lib.OP_SUM, stype=_lib.FLOAT64, ng=1, offsets=ctypes.c_void_p(offs.ctypes.data)):
        col = _lib.dtb_col(ctypes.c_void_p(v.ctypes.data), stype, 0)
        return _lib.lib.dtb_cumulative(op, 0, col, 3, None, 0, offsets, ng, None, ctypes.c_void_p(out.ctypes.data))

    for op in (_lib.OP_MEAN, _lib.OP_COUNT, _lib.OP_NROWS, _lib.OP_COV, 0, 99):
        assert call(op=op) == _lib.EINVAL
    assert call(op=_lib.OP_SUM, stype=DATE32) == _lib.EINVAL
    assert call(op=_lib.OP_PROD, stype=TIME64) == _lib.EINVAL
    assert call(stype=21) == _lib.ENOTIMPL                       # str32 has no fixed width
    assert call(op=_lib.OP_MIN, stype=21) == _lib.ENOTIMPL
    assert call(ng=-1) == _lib.EINVAL
    assert call(offsets=None) == _lib.EINVAL
    assert _lib.lib.dtb_cumulative_out_stype(_lib.OP_SUM, BOOL) == INT64
    assert _lib.lib.dtb_cumulative_out_stype(_lib.OP_PROD, INT16) == INT64
    assert _lib.lib.dtb_cumulative_out_stype(_lib.OP_SUM, FLOAT32) == FLOAT32
    assert _lib.lib.dtb_cumulative_out_stype(_lib.OP_MIN, BOOL) == BOOL
    assert _lib.lib.dtb_cumulative_out_stype(_lib.OP_MAX, TIME64) == TIME64
    assert _lib.lib.dtb_cumulative_out_stype(_lib.OP_SUM, DATE32) == 0
    assert _lib.lib.dtb_cumulative_out_stype(_lib.OP_MEAN, FLOAT64) == 0
