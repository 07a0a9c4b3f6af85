"""CPU: the numpy restatement of shift / fillna / cumcount / ngroup (tests/window_reference.py) reproduces every
golden_v8 case, its whole-array form agrees with the reference's loops, the Frame checks the functions' arguments with
the reference's error texts before any library call, and dtb_shift / dtb_fillna / dtb_group_index return their
argument codes before any GPU work.

golden_v8 comes from the unmodified reference (tests/golden/make_golden_v8.py).  Groups are formed by the C oracle
(oracle/dt_oracle.c, pinned to the reference by tests/test_oracle_golden*.py).
"""
import ctypes

import numpy as np
import pytest

from oracle import oracle as orc
import datatable_b200 as dtb
from datatable_b200 import _lib
from cumulative_reference import cum_groups
from qcut_reference import qcut_groups
from window_reference import (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64, NA, NPT,
                              expected_columns, load_golden, row_fn, row_fn_fast)

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if "error" not in c]
ERRORS = [c for c in ALL_CASES if "error" in c]
FNS = ("shift", "fillna", "cumcount", "ngroup", "mix")


def test_golden_covers_the_ground():
    assert {c["stypes"]["x"] for c in CASES if c["fn"] in ("shift", "fillna")} == \
        {BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64}
    assert {(c["fn"], c["rev"]) for c in CASES} == {(fn, r) for fn in FNS for r in (False, True)} - {("shift", True)}
    assert {c["mode"] for c in CASES} == {"none", "by", "by2", "bysort", "sort", "sortdesc"}
    assert {c["j"] for c in CASES} == {"one", "list", "tuple", "all", "dict", "dictlist", "plain", "withqcut",
                                       "withcum", "bykey", "both", "frame"}
    assert {c["n"] for c in CASES if c["fn"] == "shift"} >= {0, 1, -1, 2, -2, 3, -3, 10**6, -10**6}
    assert any(c["nrows"] == 0 for c in CASES) and any(c["nrows"] == 1 for c in CASES)
    assert len(ERRORS) == 27


def _check(got, case):
    assert [nm for nm, _ in got] == case["names"]
    for nm, col in got:
        want = ARR[case["name"] + ".out_" + nm]
        assert len(col) == case["nrows"], nm
        assert col.dtype == want.dtype, nm
        if want.dtype.kind == "f":                                # bit for bit, -0.0 included; any NaN is NA
            assert np.array_equal(np.isnan(col), np.isnan(want)), nm
            ok = ~np.isnan(want)
            ui = np.uint32 if want.dtype == np.float32 else np.uint64
            assert np.array_equal(col[ok].view(ui), want[ok].view(ui)), nm
        else:
            assert np.array_equal(col, want), nm


def _failures(fn, loop):
    bad = []
    for case in CASES:
        if case["fn"] != fn:
            continue
        try:
            _check(expected_columns(case, ARR, orc, loop=loop, qcut=qcut_groups, cum=cum_groups), case)
        except AssertionError as e:                                # noqa: PERF203
            bad.append(f"{case['name']}: {e}")
    return bad


@pytest.mark.parametrize("fn", FNS)
def test_restatement_reproduces_golden(fn):
    bad = _failures(fn, loop=True)
    assert not bad, bad


@pytest.mark.parametrize("fn", FNS)
def test_whole_array_form_reproduces_golden(fn):
    bad = _failures(fn, loop=False)
    assert not bad, bad


def _same(a, b):
    if a.dtype.kind == "f":
        ui = np.uint32 if a.dtype == np.float32 else np.uint64
        return np.array_equal(np.where(np.isnan(a), np.nan, a).astype(a.dtype).view(ui),
                              np.where(np.isnan(b), np.nan, b).astype(b.dtype).view(ui))
    return np.array_equal(a, b)


@pytest.mark.parametrize("st", [BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64])
def test_whole_array_form_matches_the_loops(st):
    """Under by(), on random groups (lengths 1 .. ~200) with NA runs: every function, shift over n from -300 to 300
    and the extremes of int32."""
    rng = np.random.default_rng(st)
    n = 4000
    if st in (FLOAT32, FLOAT64):
        v = rng.choice(np.array([0.0, -0.0, 1.5, -2.0, np.inf, -np.inf, np.nan, np.nan], NPT[st]), n)
    else:
        v = rng.integers(-5, 6, n).astype(NPT[st]) if st != BOOL else rng.integers(0, 2, n).astype(np.int8)
        v[rng.random(n) < 0.4] = NA[st]
    offsets = np.unique(np.concatenate([[0, n], rng.integers(1, n, 60)])).astype(np.int64)
    for s in (0, 1, -1, 2, -7, 57, -200, 300, 2**31 - 1, -2**31):
        assert _same(row_fn_fast("shift", v, st, offsets, n=s), row_fn("shift", v, st, offsets, True, n=s)), s
    for rev in (False, True):
        assert _same(row_fn_fast("fillna", v, st, offsets, rev), row_fn("fillna", v, st, offsets, True, rev)), rev
        for fn in ("cumcount", "ngroup"):
            assert np.array_equal(row_fn_fast(fn, None, st, offsets, rev), row_fn(fn, None, st, offsets, True, rev))


def _error_frame():
    return dtb.Frame({"x": np.array([1.5, np.nan, 0.0]), "y": np.array([1, 2, 3], np.int32)})


@pytest.mark.parametrize("case", ERRORS, ids=[c["name"] for c in ERRORS])
def test_frame_argument_errors_match_reference(case):
    """The checks run before any library call (they pass on a machine without a GPU)."""
    DT = _error_frame()
    exc = {"ValueError": ValueError, "TypeError": TypeError}[case["error"]]
    with pytest.raises(exc) as ei:
        DT[:, eval(case["expr"], {"dt": dtb, "f": dtb.f})]                 # noqa: S307  (the golden's own text)
    assert str(ei.value) == case["message"]


def test_frame_refusals_before_any_library_call():
    """What stays outside the GPU path raises NotImplementedError when the function is called."""
    f = dtb.f
    with pytest.raises(NotImplementedError):
        dtb.fillna(f.x, value=0)
    with pytest.raises(NotImplementedError):
        dtb.shift(dtb.sum(f.x))
    with pytest.raises(NotImplementedError):
        dtb.fillna([f.x, dtb.cumsum(f.x)])
    assert dtb.cumcount(None).reverse is False and dtb.fillna(f.x, reverse=None).reverse is False
    assert dtb.shift(f.x, n=None).n == 1


def test_abi_argument_codes_before_any_gpu_work():
    v = np.array([1.0, 2.0, 3.0])
    offs = np.array([0, 3], dtype=np.int32)
    out = np.empty(3, dtype=np.float64)
    oi = np.empty(3, dtype=np.int64)
    po = ctypes.c_void_p(offs.ctypes.data)

    def col(stype=_lib.FLOAT64):
        return _lib.dtb_col(ctypes.c_void_p(v.ctypes.data), stype, 0)

    def shift(stype=_lib.FLOAT64, ng=1, offsets=po, nrows=3):
        return _lib.lib.dtb_shift(col(stype), nrows, None, 0, offsets, ng, 1, None, ctypes.c_void_p(out.ctypes.data))

    def fill(stype=_lib.FLOAT64, ng=1, offsets=po, nrows=3):
        return _lib.lib.dtb_fillna(0, col(stype), nrows, None, 0, offsets, ng, None, ctypes.c_void_p(out.ctypes.data))

    for call in (shift, fill):
        assert call(stype=21) == _lib.ENOTIMPL                      # str32 has no fixed width
        assert call(stype=0) == _lib.ENOTIMPL
        assert call(ng=-1) == _lib.EINVAL
        assert call(offsets=None) == _lib.EINVAL
        assert call(nrows=-1) == _lib.EINVAL
    for kind in (0, 3, -1, 99):
        assert _lib.lib.dtb_group_index(kind, 0, po, 1, None, ctypes.c_void_p(oi.ctypes.data)) == _lib.EINVAL
    assert _lib.lib.dtb_group_index(_lib.GROUP_CUMCOUNT, 0, po, -1, None, ctypes.c_void_p(oi.ctypes.data)) == _lib.EINVAL
    assert _lib.lib.dtb_group_index(_lib.GROUP_NGROUP, 1, None, 1, None, ctypes.c_void_p(oi.ctypes.data)) == _lib.EINVAL
