"""CPU: the C-ABI library loads, exports every symbol include/dtb200.h declares, and fails loudly
(no CPU fallback) when no CUDA device is present."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "dtb200.h")).read()
    return sorted(set(re.findall(r"DTB_API\s+[\w\s\*]+?\b(dtb_\w+)\s*\(", src)))


def test_header_declares_expected_entry_points():
    syms = header_symbols()
    for s in ("dtb_group", "dtb_groupby_create", "dtb_reduce", "dtb_gather", "dtb_last_error"):
        assert s in syms


def test_library_exports_every_declared_symbol():
    from datatable_b200 import _lib
    dll = ctypes.CDLL(_lib.LIB_PATH)
    for s in header_symbols():
        assert hasattr(dll, s), f"libdtb200.so does not export {s}"
    assert sorted(_lib.EXPORTS) == header_symbols()


def test_pure_host_queries():
    from datatable_b200 import _lib
    L = _lib.lib
    assert L.dtb_abi_version() == 1
    assert [L.dtb_stype_size(s) for s in (1, 2, 3, 4, 5, 6, 7, 17, 18, 11, 21)] == [1, 1, 2, 4, 8, 4, 8, 4, 8, 0, 0]
    # reducer output stypes (fexpr_sumprod.cc:50-66, fexpr_mean.cc:49-78, fexpr_minmax.cc:50-72)
    assert L.dtb_reduce_out_stype(_lib.OP_SUM, _lib.INT8) == _lib.INT64
    assert L.dtb_reduce_out_stype(_lib.OP_SUM, _lib.FLOAT32) == _lib.FLOAT32
    assert L.dtb_reduce_out_stype(_lib.OP_MEAN, _lib.INT32) == _lib.FLOAT64
    assert L.dtb_reduce_out_stype(_lib.OP_MEAN, _lib.FLOAT32) == _lib.FLOAT32
    assert L.dtb_reduce_out_stype(_lib.OP_MIN, _lib.BOOL) == _lib.BOOL      # bool8 in, bool8 out (reference: stype.bool8)
    assert L.dtb_reduce_out_stype(_lib.OP_MAX, _lib.INT16) == _lib.INT16
    assert L.dtb_reduce_out_stype(_lib.OP_COUNT, _lib.FLOAT64) == _lib.INT64
    assert L.dtb_reduce_out_stype(_lib.OP_SUM, 11) == 0


def test_options_roundtrip():
    from datatable_b200 import engine
    assert engine.get_option("radix_bits") == 0
    engine.set_option("radix_bits", 7)
    assert engine.get_option("radix_bits") == 7
    engine.set_option("radix_bits", 0)
    with pytest.raises(ValueError):
        engine.set_option("radix_bits", 99)
    with pytest.raises(ValueError):
        engine.set_option("no_such_option", 1)


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    import datatable_b200 as d
    with pytest.raises(d.DtbCudaError):
        d.engine.group([np.arange(10, dtype=np.int32)])
    with pytest.raises(d.DtbCudaError):
        d.engine.gather(np.arange(10, dtype=np.float64), np.arange(3, dtype=np.int32))


def test_argument_validation_before_any_gpu_work():
    import datatable_b200 as d
    with pytest.raises(NotImplementedError):      # NotImplError "Unable to sort Column of stype" (sort.cc:673)
        d.engine.group([np.array(["a", "b"])])
    with pytest.raises(ValueError):
        d.engine.group([np.arange(3, dtype=np.int32), np.arange(4, dtype=np.int32)])
    # every entry point that takes key columns checks them before any library call: the library reads nrows rows of
    # each key column, so a shorter one would be read past its end
    short = [np.arange(4, dtype=np.int32), np.arange(3, dtype=np.int64)]
    for call in (d.engine.group, d.engine.group64, d.engine.Groupby):
        with pytest.raises(ValueError):
            call(short)
        with pytest.raises(ValueError):
            call([])
