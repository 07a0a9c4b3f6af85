"""CPU: dtb_cut's argument checks (include/dtb200.h, dtb_cut) return their codes in the documented order, on the host
before any CUDA call -- so the same with or without a device."""
import ctypes

import numpy as np
import pytest

from datatable_b200 import _lib

L = _lib.lib
STR32 = 21
V = np.array([1.0, 2.0, 3.0])
OUT = np.zeros(3, dtype=np.int32)
EINVAL, ENOTIMPL = _lib.EINVAL, _lib.ENOTIMPL


def _edges(*e):
    a = np.array(e, dtype=np.float64)
    return a, ctypes.c_void_p(a.ctypes.data), len(a)


def _call(stype=_lib.FLOAT64, data=V, nrows=3, order=None, n=3, nbins=10, edges=None, out=OUT):
    keep, ep, ne = edges if edges is not None else (None, None, 0)
    rc = L.dtb_cut(_lib.dtb_col(ctypes.c_void_p(None if data is None else data.ctypes.data), stype, 0), nrows, order, 0,
                   n, nbins, ep, ne, 1, None, ctypes.c_void_p(None if out is None else out.ctypes.data))
    return rc, L.dtb_last_error().decode()


@pytest.mark.parametrize("kw, code, msg", [
    (dict(nbins=0), EINVAL, "Number of bins must be positive"),
    (dict(nbins=-5, stype=STR32), EINVAL, "Number of bins must be positive"),          # nbins before the stype
    (dict(edges=_edges(1.0)), EINVAL, "at least two edges"),
    (dict(edges=_edges(np.nan, 1.0)), EINVAL, "NaN"),
    (dict(edges=_edges(0.0, np.nan)), EINVAL, "strictly increasing"),
    (dict(edges=_edges(0.0, 1.0, 1.0)), EINVAL, "strictly increasing: edges 1 and 2"),
    (dict(edges=_edges(2.0, 1.0), stype=STR32), EINVAL, "strictly increasing"),          # edges before the stype
    (dict(nbins=0, edges=_edges(0.0, 1.0), stype=STR32), ENOTIMPL, "stype 21"),          # nbins is ignored with edges
    (dict(stype=STR32), ENOTIMPL, "cut() cannot be applied to columns of stype 21"),
    (dict(stype=_lib.DATE32, n=-1), EINVAL, "numeric"),                                  # the stype before the sizes
    (dict(stype=_lib.TIME64), EINVAL, "numeric"),
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
