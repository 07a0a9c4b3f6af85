"""CPU: the numpy restatement of qcut (tests/qcut_reference.py) reproduces every golden_v6 case, the Frame checks
qcut()'s arguments with the reference's error texts before any library call, and the bin kernel is built without a
fused multiply-add.

golden_v6 comes from the unmodified reference (tests/golden/make_golden_v6.py).  Groups are formed by the C oracle
(oracle/dt_oracle.c, pinned to the reference by tests/test_oracle_golden*.py).
"""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
import datatable_b200 as dtb
from datatable_b200 import _lib
from qcut_reference import expected_columns, load_golden

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if "error" not in c]
ERRORS = [c for c in ALL_CASES if "error" in c]


def test_golden_covers_the_ground():
    stypes = {c["stypes"]["x"] for c in CASES}
    assert stypes == {1, 2, 3, 4, 5, 6, 7, 17, 18}
    assert {c["mode"] for c in CASES} >= {"none", "by", "by2", "bysort", "sort", "sortdesc"}
    assert {c["j"] for c in CASES} >= {"one", "list", "tuple", "all", "dict", "dictlist", "plain", "bykey"}
    assert {c["q"] for c in CASES if not isinstance(c["q"], list)} >= {None, 1, 2, 10, 50}
    assert len(ERRORS) == 7


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_restatement_reproduces_golden(case):
    got = expected_columns(case, ARR, orc)
    assert [nm for nm, _ in got] == case["names"]
    assert len(got) == len(case["out_stypes"])
    for nm, col in got:
        want = ARR[case["name"] + ".out_" + nm]
        assert len(col) == case["nrows"]
        if want.dtype.kind == "f":
            assert np.array_equal(np.isnan(col), np.isnan(want))
            assert np.array_equal(col[~np.isnan(want)], want[~np.isnan(want)])
        else:
            assert col.dtype == want.dtype, nm
            assert np.array_equal(col, want), nm


def _frame_args(case):
    fr = dtb.Frame({"x": ARR[case["name"] + ".x"], "y": ARR[case["name"] + ".y"]}, stypes=case["stypes"])
    f = dtb.f
    cols = [f.x, f.y] if case["j"] == "list" else f.x
    return fr, dtb.qcut(cols, nquantiles=case["q"])


@pytest.mark.parametrize("case", ERRORS, ids=[c["name"] for c in ERRORS])
def test_frame_argument_errors_match_reference(case):
    """The checks run before any library call (they pass on a machine without a GPU)."""
    fr, J = _frame_args(case)
    exc = {"ValueError": ValueError, "TypeError": TypeError}[case["error"]]
    with pytest.raises(exc) as ei:
        fr[:, J]
    assert str(ei.value) == case["message"]


def test_frame_argument_errors_in_every_query_shape():
    fr = dtb.Frame({"x": np.array([1.0, 2.0]), "g": np.array([1, 1], np.int32)})
    f = dtb.f
    msg = "Number of quantiles must be positive, instead got: 0"
    for mods in ((), (dtb.by(f.g),), (dtb.sort(f.g),), (dtb.by(f.g), dtb.sort(f.x))):
        with pytest.raises(ValueError, match=msg):
            fr[(slice(None), dtb.qcut(f.x, nquantiles=0)) + mods]
        with pytest.raises(ValueError, match=msg):
            fr[(slice(0, 1), {"q": dtb.qcut(f.x, nquantiles=0)}) + mods]
    # f[:] under by() leaves out the by() column: one column, so a list of two does not fit
    with pytest.raises(ValueError, match="i.e. 1, instead got: 2"):
        fr[:, dtb.qcut(f[:], nquantiles=[2, 3]), dtb.by(f.g)]


def test_abi_argument_codes_before_any_gpu_work():
    import ctypes
    v = np.array([1.0, 2.0, 3.0])
    offs = np.array([0, 3], dtype=np.int32)
    out = np.empty(3, dtype=np.int32)

    def call(stype=_lib.FLOAT64, ng=1, q=10, offsets=ctypes.c_void_p(offs.ctypes.data)):
        col = _lib.dtb_col(ctypes.c_void_p(v.ctypes.data), stype, 0)
        return _lib.lib.dtb_qcut(col, 3, None, offsets, ng, q, None, ctypes.c_void_p(out.ctypes.data))

    assert call(q=0) == _lib.EINVAL
    assert _lib.lib.dtb_last_error().decode() == "Number of quantiles must be positive, instead got: 0"
    assert call(q=-5) == _lib.EINVAL
    assert call(ng=-1) == _lib.EINVAL
    assert call(offsets=None) == _lib.EINVAL
    assert call(stype=21) == _lib.ENOTIMPL                       # str32 has no fixed width


def test_engine_rejects_nquantiles_outside_int32():
    with pytest.raises(ValueError):
        dtb.engine.qcut(np.zeros(3), None, np.array([0, 3], np.int32), 2**31)


def test_emit_kernel_rounds_multiply_and_add_separately():
    """int32(a * i + b) is a DMUL then a DADD in the bin kernel's SASS, never a DFMA."""
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump is not installed")
    sass = subprocess.run([tool, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    bodies = [b for b in re.split(r"\n\s*Function : ", sass) if b.split("\n", 1)[0].find("qcut_emit_kernel") >= 0]
    assert len(bodies) == 1
    ops = re.findall(r"\b(DFMA|DMUL|DADD)\b", bodies[0])
    assert "DFMA" not in ops
    assert "DMUL" in ops and "DADD" in ops
