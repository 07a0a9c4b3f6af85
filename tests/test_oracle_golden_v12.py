"""CPU: the numpy restatement of cut (tests/cut_reference.py) reproduces every golden_v12 case, the Frame raises
cut()'s call-time errors with the reference's texts before any library call, and the emit kernel is built without a
fused multiply-add.

golden_v12 comes from the unmodified reference (tests/golden/make_golden_v12.py).  sort() orders are formed by the C
oracle (oracle/dt_oracle.c, pinned to the reference by tests/test_oracle_golden*.py).
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
import datatable_b200 as dtb
from cut_reference import expected_cuts, frame_query, load_golden

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if "error" not in c]
ERRORS = [c for c in ALL_CASES if "error" in c]
# errors cut() raises when it is called, before any query: these need no device
CALL_ERRORS = [c for c in ERRORS if c["name"].startswith(("err.nbins_zero", "err.nbins_negative", "err.nbins_float",
                                                          "err.nbins_bool", "err.nbins_large", "err.nbins_small",
                                                          "err.nbins_list", "err.right_closed", "err.both",
                                                          "err.bins_")) and not c["name"].startswith("err.bins_len")]


def test_golden_covers_the_ground():
    assert {c["stypes"]["x"] for c in CASES} >= {1, 2, 3, 4, 5, 6, 7}
    assert {c["mode"] for c in CASES} >= {"none", "sort", "sortdesc", "sortlast", "sortremove", "join"}
    assert {c["i"][0] for c in CASES if c["i"]} >= {"slice", "int", "bool", "frame", "list", "range"}
    assert {c["j"] for c in CASES} >= {"one", "list", "tuple", "all", "dict", "dictlist", "plain", "qcut", "cumsum",
                                       "shift", "self", "other", "joincol", "joinlist"}
    nedges = {len(ARR[b["key"]]) for c in CASES for b in c.get("bins", [])}
    assert min(nedges) == 2 and max(nedges) > 4096                # both sides of the shared-memory limit
    assert len(ERRORS) == 36 and len(CALL_ERRORS) == 22


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_restatement_reproduces_golden(case):
    for idx, want in expected_cuts(case, ARR, orc):
        nm = case["names"][idx]
        assert case["out_stypes"][idx] == "stype.int32"
        got = ARR[case["name"] + ".out_" + nm]
        assert got.dtype == np.int32 and np.array_equal(got, want), nm


@pytest.mark.parametrize("case", CALL_ERRORS, ids=[c["name"] for c in CALL_ERRORS])
def test_frame_call_errors(case):
    """The bins Frames and the query's frame stay on the host: cut() raises before any library call."""
    with pytest.raises(Exception) as ei:
        frame_query(dtb, case, ARR)
    assert type(ei.value).__name__ == case["error"]
    assert str(ei.value) == case["message"]


def test_argument_forms():
    f = dtb.f
    with pytest.raises(TypeError, match="requires exactly 1 positional argument, but none were given"):
        dtb.cut()
    with pytest.raises(TypeError, match="takes only one positional argument, but 2 were given"):
        dtb.cut(f.x, 3)
    with pytest.raises(TypeError, match="bins parameter must be a list or a tuple, instead got <class 'int'>"):
        dtb.cut(f.x, bins=5)
    with pytest.raises(TypeError, match="Expected a Frame, instead got <class 'list'>"):
        dtb.cut(f.x, bins=[[1, 2]])
    with pytest.raises(ValueError, match="needs exactly one column with the bin edges, instead for the frame 0 got: 2"):
        dtb.cut(f.x, bins=[dtb.Frame({"a": np.array([1, 2]), "b": np.array([3, 4])})])
    with pytest.raises(NotImplementedError):
        dtb.cut(dtb.qcut(f.x))                                    # nested row functions: not on the GPU path
    c = dtb.cut(f.x, right_closed=None, nbins=[4])
    assert c.right_closed is True and c.nbins == [4]
    assert dtb.cut(cols=f.x).nbins == [10]


@pytest.mark.parametrize("fn", ["qcut", "cumsum", "cummax"])
def test_frame_argument_is_cut_only(fn):
    """Only cut() takes a Frame as its argument: the other row functions still refuse one when the query is resolved,
    before any library call, and never read the query's own columns of the same names."""
    DT = dtb.Frame({"x": np.array([1.0, 2.0, 3.0]), "s": np.array([3, 1, 2], np.int32)})
    O = dtb.Frame({"x": np.array([9.0, 8.0, 7.0])})
    e = getattr(dtb, fn)(O)
    for q in ((slice(None), e), (slice(None), e, dtb.sort(dtb.f.s)), (slice(None, None, 2), e)):
        with pytest.raises(TypeError, match="Unsupported key expression"):
            DT[q]


def test_emit_kernel_has_no_fma():
    """int32(a * v + b) is a DMUL then a DADD in the emit kernel's SASS, never a DFMA."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed")
    obj = os.path.join(os.path.dirname(dtb._lib.LIB_PATH), "dtb_cut.o")
    sass = subprocess.run([tool, "-sass", obj], capture_output=True, text=True, check=True).stdout
    bodies = [b for b in re.split(r"\n\s*Function : ", sass) if b.split("\n", 1)[0].find("cut_emit_kernel") >= 0]
    assert len(bodies) == 18                                      # 6 element types x (identity, int32, int64 order)
    for body in bodies:
        ops = re.findall(r"\b(DFMA|DMUL|DADD)\b", body)
        assert "DFMA" not in ops and "DMUL" in ops and "DADD" in ops
