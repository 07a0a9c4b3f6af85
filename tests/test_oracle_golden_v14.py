"""CPU: the numpy restatement of the time functions (tests/time_reference.py) reproduces every golden_v14 case, and the
Frame raises the functions' call-time errors with the reference's texts before any library call.

golden_v14 comes from the unmodified reference (tests/golden/make_golden_v14.py).  sort() orders and by() groups are
formed by the C oracle (oracle/dt_oracle.c, pinned to the reference by tests/test_oracle_golden*.py).
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
import datatable_b200 as dtb
from time_reference import PARTS, expected_parts, keyed_outputs, load_golden

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if "error" not in c]
PLAIN = [c for c in CASES if c["mode"] in ("none", "sort", "sortdesc", "join")]
KEYED = [c for c in CASES if c["mode"] not in ("none", "sort", "sortdesc", "join", "bypartjoin") and c["i"] is None]
CALL_ERRORS = [c for c in ALL_CASES if c.get("call")]
CALLS = {"noargs": lambda P: P(), "twoargs": lambda P: P(dtb.f.d, dtb.f.t), "kwarg": lambda P: P(**{"date": dtb.f.d}),
         "badkw": lambda P: P(foo=dtb.f.d), "dupkw": lambda P: P(dtb.f.d, **{"date": dtb.f.t})}


def test_golden_covers_the_ground():
    assert {c["part"] for c in CASES} == set(PARTS)
    assert {(c["name"].split(".")[1], c["part"]) for c in CASES if c["name"].startswith("edge.")} >= \
        {("date32", p) for p in PARTS[:4]} | {("time64", p) for p in PARTS}
    assert {c["mode"] for c in CASES} >= {"none", "sort", "sortdesc", "by", "bysort", "join", "bypart", "bypartneg",
                                          "bykpart", "sortpart", "sortpartneg", "bypart_t", "bypartjoin", "bypartsort"}
    assert {c["i"][0] for c in CASES if c["i"]} >= {"slice", "int", "bool", "frame", "list", "range"}
    assert {c["j"] for c in CASES} >= {"one", "list", "tuple", "all", "dict", "plain", "cut", "qcut", "cumsum",
                                       "shift", "fillna", "cumcount", "ngroup", "joincol", "joinlist", "parts",
                                       "bysum", "bycount", "byall", "bykeys"}
    assert len(CALL_ERRORS) == 15 and len(ALL_CASES) - len(CASES) == 35


def test_edges_are_pinned():
    """29 February of 1900 (none), 2000 and 2100 (none), years 0 and -1, the int32 ends and instants before 1970."""
    d = ARR["edge.date32.year.d"]
    got = {int(k): (int(y), int(m), int(dd)) for k, y, m, dd in zip(d, ARR["edge.date32.year.out_d"],
                                                                    ARR["edge.date32.month.out_d"],
                                                                    ARR["edge.date32.day.out_d"])}
    assert got[11016] == (2000, 2, 29) and got[-25509] == (1900, 2, 28) and got[47540] == (2100, 2, 28)
    assert got[-719468] == (0, 3, 1) and got[-719469] == (0, 2, 29) and got[-719834] == (-1, 3, 1)
    assert got[2**31 - 1][0] == -5877641                    # the int32 add of the conversion wraps
    t = ARR["edge.time64.hour.d"]
    h = dict(zip(t.tolist(), ARR["edge.time64.hour.out_d"].tolist()))
    assert h[-1] == 23 and h[-86400 * 10**9] == 0


@pytest.mark.parametrize("case", PLAIN, ids=[c["name"] for c in PLAIN])
def test_restatement_reproduces_golden(case):
    for idx, want in expected_parts(case, ARR, orc):
        nm = case["names"][idx]
        assert case["out_stypes"][idx] == "stype.int32"
        got = ARR[case["name"] + ".out_" + nm]
        assert got.dtype == np.int32 and np.array_equal(got, want), nm


@pytest.mark.parametrize("case", KEYED, ids=[c["name"] for c in KEYED])
def test_restatement_reproduces_keyed_golden(case):
    """by() / sort() with a time part as a key: the key column and the time parts of j, in the oracle's order."""
    for idx, want in keyed_outputs(case, ARR, orc):
        nm = case["names"][idx]
        assert case["out_stypes"][idx] == "stype.int32", nm
        assert np.array_equal(ARR[case["name"] + ".out_" + nm], want), nm


@pytest.mark.parametrize("case", CALL_ERRORS, ids=[c["name"] for c in CALL_ERRORS])
def test_frame_call_errors(case):
    with pytest.raises(Exception) as ei:
        CALLS[case["call"]](getattr(dtb.time, case["part"]))
    assert (type(ei.value).__name__, str(ei.value)) == (case["error"], case["message"])


def test_refusals_before_the_device():
    """An expression as the argument, and a negated part in j, are not on the GPU path; the other row functions are
    still refused as keys."""
    f, T = dtb.f, dtb.time
    for bad in (lambda: T.year(dtb.sum(f.d)), lambda: T.month(T.year(f.d)), lambda: T.day(-f.d),
                lambda: T.hour(dtb.qcut(f.t))):
        with pytest.raises(NotImplementedError):
            bad()
    DT = dtb.Frame({"d": np.array([1, 2], np.int32), "s": np.array([3, 1], np.int32)}, stypes={"d": dtb._lib.DATE32})
    with pytest.raises(TypeError, match="Unsupported key expression"):
        DT[:, f.s, dtb.by(dtb.cumsum(f.s))]
    with pytest.raises(NotImplementedError):
        DT[:, dtb.sum(T.year(f.d))]
    with pytest.raises(NotImplementedError):
        DT[:, dtb.cov(T.year(f.d), f.s)]
    with pytest.raises(NotImplementedError):
        DT[:, -T.year(f.d)]
    with pytest.raises(NotImplementedError):
        DT[:, f.s, dtb.by(T.year([f.d, f.s]))]
    with pytest.raises(TypeError, match=r"Function time\.year\(\) requires a date32 or time64 column, instead "
                                        r"received column of type int32"):
        DT[:, f.d, dtb.by(T.year(f.s))]


def test_kernels_have_no_division_call():
    """Every divisor is a constant: no time kernel's SASS calls a 64-bit division routine (or anything else)."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed")
    obj = os.path.join(os.path.dirname(dtb._lib.LIB_PATH), "dtb_time.o")
    sass = subprocess.run([tool, "-sass", obj], capture_output=True, text=True, check=True).stdout
    bodies = [b for b in re.split(r"\n\s*Function : ", sass)[1:] if "time_part" in b.split("\n", 1)[0]]
    assert len(bodies) == 48               # date32 x 4 parts + time64 x 8 parts, x (2 identity + 2 RowIndex) kernels
    for body in bodies:
        assert not re.search(r"\bCALL\b", body), body.split("\n", 1)[0]
