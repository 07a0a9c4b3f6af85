"""CPU: dtb_time_part's argument checks (include/dtb200.h, dtb_time_part) return their codes in the documented order, on
the host before any CUDA call -- so the same with or without a device."""
import ctypes

import numpy as np
import pytest

from datatable_b200 import _lib

L = _lib.lib
STR32 = 21
V = np.array([1, 2, 3], dtype=np.int32)
OUT = np.zeros(3, dtype=np.int32)
EINVAL, ENOTIMPL = _lib.EINVAL, _lib.ENOTIMPL


def _call(part=_lib.TIME_YEAR, stype=_lib.DATE32, data=V, nrows=3, order=None, n=3, out=OUT):
    rc = L.dtb_time_part(part, _lib.dtb_col(ctypes.c_void_p(None if data is None else data.ctypes.data), stype, 0),
                         nrows, order, 0, n, None, ctypes.c_void_p(None if out is None else out.ctypes.data))
    return rc, L.dtb_last_error().decode()


@pytest.mark.parametrize("kw, code, msg", [
    (dict(part=0), EINVAL, "unknown time part 0"),
    (dict(part=9, stype=STR32), EINVAL, "unknown time part 9"),                        # the part before the stype
    (dict(stype=STR32), ENOTIMPL, "time functions cannot be applied to columns of stype 21"),
    (dict(stype=_lib.INT32, n=-1), EINVAL, "date32 or time64"),                          # the stype before the sizes
    (dict(stype=_lib.FLOAT64), EINVAL, "date32 or time64"),
    (dict(part=_lib.TIME_HOUR, n=-1), EINVAL, "need a time64 column"),                  # a clock part of date32
    (dict(part=_lib.TIME_NANOSECOND), EINVAL, "need a time64 column"),
    (dict(n=-1), EINVAL, "negative size"),
    (dict(nrows=-1, n=-1), EINVAL, "negative size"),
    (dict(data=None), EINVAL, "value column data is NULL"),
    (dict(data=None, n=2), EINVAL, "value column data is NULL"),
    (dict(n=2), EINVAL, "n must equal nrows_value"),
    (dict(out=None), EINVAL, "out is NULL"),
])
def test_argument_codes(kw, code, msg):
    rc, err = _call(**kw)
    assert rc == code
    assert msg in err
