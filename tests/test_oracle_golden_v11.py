"""CPU: golden_v11 (DT[i, j] with `i` a boolean or integer column, a list or a range, from the unmodified reference,
tests/golden/make_golden_v11.py) restated with tests/rows_reference.py; every argument error of those forms raised by
the Frame before the device is touched; and the argument checks of dtb_mask_rows / dtb_int_rows, which come before
any CUDA call."""
import ctypes
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


def A(case, key):
    return ARR[f"{case['name']}.{key}"]


def na_of(a, st):
    return np.nan if st in (FLOAT32, FLOAT64) else NA[st]


def restated_rows(case):
    """The RowIndex of the case's selector (its `restate` source text) by tests/rows_reference.py."""
    n = len(A(case, f"x.{next(iter(case['x']))}"))

    def M(nm):
        return ("mask", A(case, f"x.{nm}"))

    def F(nm):
        st = case["s"][nm]["C0"]
        a = A(case, f"s.{nm}.C0")
        return ("mask", a) if st == BOOL else ("ints", a, NA[st])

    def N(nm):
        a = A(case, f"a.{nm}")
        return ("mask", a) if a.dtype == np.bool_ else ("ints", a, None)

    sel = eval(case["restate"]["sel"], {"M": M, "F": F, "N": N})
    return rr.rows(list(sel) if isinstance(sel, tuple) and sel and not isinstance(sel[0], str) else sel, n)


def test_golden_covers_the_ground():
    names = {c["name"] for c in CASES}
    for prefix in ("mask.", "frame.", "numpy.", "list.", "range.", "j.", "join.", "err.by_", "err.so_"):
        assert any(n.startswith(prefix) for n in names), prefix
    assert {c["s"]["s"]["C0"] for c in CASES if c["name"].startswith("frame.")} >= {BOOL, INT8, INT16, INT32, INT64}
    assert all(c["name"].startswith("err.") for c in CASES if "error" in c or "reference_crash" in c)
    assert {c["name"] for c in CASES if "reference_crash" in c} <= set(rr.SOURCE_ERRORS)
    assert sum("restate" in c for c in CASES) >= 30


@pytest.mark.parametrize("case", [c for c in CASES if "restate" in c], ids=lambda c: c["name"])
def test_selection_restated(case):
    ri = restated_rows(case)
    cols = case["restate"]["cols"] or list(case["x"])
    assert case["nrows"] == len(ri) and case["names"] == cols, case["name"]
    for i, nm in enumerate(cols):
        st = case["x"][nm]
        got = rr.gather(A(case, f"x.{nm}"), ri, na_of(None, st))
        want = A(case, f"r{i}")
        assert got.dtype == want.dtype and np.array_equal(got, want, equal_nan=got.dtype.kind == "f"), (case["name"], nm)


def expected_error(case):
    if "error" in case:
        return tuple(case["error"])
    return rr.SOURCE_ERRORS[case["name"]][0], rr.SOURCE_ERRORS[case["name"]][1].replace("`", "")


def frames(case):
    import datatable_b200 as dtb
    X = dtb.Frame({nm: A(case, f"x.{nm}") for nm in case["x"]}, stypes=case["x"])
    S = {snm: dtb.Frame({cn: A(case, f"s.{snm}.{cn}") for cn in cols}, stypes=cols) for snm, cols in case["s"].items()}
    if case["name"] == "err.frame_keyed":
        S["s"]._key = ("C0",)                  # setting a key sorts on the device; the refusal needs only the flag
    env = {"X": X, "S": S, "A": {nm: A(case, f"a.{nm}") for nm in case["a"]}, "dt": dtb, "f": dtb.f, "g": dtb.g,
           "join": dtb.join, "by": dtb.by, "sort": dtb.sort, "np": np}
    if case["j"]:
        J = dtb.Frame({nm: A(case, f"j.{nm}") for nm in case["j"]}, stypes=case["j"])
        J._key = tuple(case["jkey"])
        env["J"] = J
    return env


@pytest.mark.parametrize("case", [c for c in CASES if c["name"].startswith("err.") and c["name"] not in rr.DATA_ERRORS
                                  and c["name"] != "err.bool_literal"], ids=lambda c: c["name"])
def test_errors_before_the_device(case, monkeypatch):
    """The reference's error type and text, raised while the query is resolved: no library call runs."""
    env = frames(case)
    from datatable_b200 import engine

    def untouched(*a, **k):
        raise AssertionError("the device was touched")
    for fn in ("mask_rows", "int_rows", "join_gather", "join_index", "group", "gather", "Groupby"):
        monkeypatch.setattr(engine, fn, untouched)
    etype, msg = expected_error(case)
    with pytest.raises({"KeyError": KeyError, "ValueError": ValueError, "TypeError": TypeError,
                        "NotImplementedError": NotImplementedError}[etype]) as e:
        eval(case["query"], env)
    assert type(e.value).__name__ == etype or isinstance(e.value, {"ValueError": ValueError}.get(etype, ())), etype
    assert e.value.args[0].replace("`", "") == msg


def test_bool_literal_stays_outside():
    """DT[True, :] keeps its NotImplementedError (the reference's TypeError is pinned in the golden)."""
    case = next(c for c in CASES if c["name"] == "err.bool_literal")
    assert case["error"] == ["TypeError", "A boolean value cannot be used as a row selector"]
    with pytest.raises(NotImplementedError):
        eval(case["query"], frames(case))


def test_rows_reference_forms():
    m = np.array([1, 0, -128, 5, -1, 0], np.int8)
    assert rr.mask_rows(m).tolist() == [0, 3, 4]
    assert rr.rows([0, -1, None, slice(2, 4)], 6).tolist() == [0, 5, 2, 3]
    assert rr.rows(range(5, 0, -2), 6).tolist() == [5, 3, 1]
    assert rr.rows(("ints", np.array([3, NA[INT16], 3], np.int16), NA[INT16]), 6).tolist() == [3, -1, 3]


# ---- the C-ABI's argument checks, in their documented order, without a device ------------------------------------
def _lib():
    from datatable_b200 import _lib
    return _lib


def test_mask_rows_argument_errors():
    L = _lib()
    m = np.array([1, 0, 1], np.int8)
    out = np.zeros(3, np.int32)
    n = ctypes.c_int64(0)

    def call(stype=BOOL, data=m.ctypes.data, nrows=3, rows=out.ctypes.data, cap=3, nout=ctypes.byref(n)):
        rc = L.lib.dtb_mask_rows(L.dtb_col(ctypes.c_void_p(data), stype, 0), nrows, None, rows, cap, nout)
        return rc, L.lib.dtb_last_error().decode()

    E = L.EINVAL
    assert call(nout=None, stype=INT32) == (E, "nrows_out is NULL")
    assert call(stype=INT32, nrows=-1) == (E, "dtb_mask_rows takes a bool8 column, not stype 4")
    assert call(nrows=-1, cap=-1) == (E, "nrows must be in 0..INT32_MAX")
    assert call(nrows=2**31) == (E, "nrows must be in 0..INT32_MAX")
    assert call(cap=-1, data=None) == (E, "rows_capacity must be non-negative")
    assert call(data=None, rows=None) == (E, "mask data is NULL")
    assert call(rows=None) == (E, "rows_out is NULL")


def test_int_rows_argument_errors():
    L = _lib()
    s = np.array([1, 0, 1], np.int16)
    out = np.zeros(3, np.int32)
    lo, hi, nna = ctypes.c_int64(0), ctypes.c_int64(0), ctypes.c_int64(0)

    def call(stype=INT16, data=s.ctypes.data, nrows=3, rows=out.ctypes.data, mins=ctypes.byref(lo)):
        rc = L.lib.dtb_int_rows(L.dtb_col(ctypes.c_void_p(data), stype, 0), nrows, None, rows, mins, ctypes.byref(hi),
                                ctypes.byref(nna))
        return rc, L.lib.dtb_last_error().decode()

    E = L.EINVAL
    assert call(mins=None, stype=FLOAT64) == (E, "min_out / max_out / nacount_out is NULL")
    assert call(stype=FLOAT64, nrows=-1) == (E, "dtb_int_rows takes an int8, int16, int32 or int64 column, not stype 7")
    assert call(stype=BOOL) == (E, "dtb_int_rows takes an int8, int16, int32 or int64 column, not stype 1")
    assert call(nrows=-1, data=None) == (E, "nrows must be in 0..INT32_MAX")
    assert call(data=None, rows=None) == (E, "selector data is NULL")
    assert call(rows=None) == (E, "rows_out is NULL")
