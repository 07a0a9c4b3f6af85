#!/usr/bin/env python3
"""Checks the ArrayView gather hook and the residency bracket of a patched reference build
(run with PYTHONPATH=oracle/_ref/patched).

* option sort.b200 on: DT[:, :, sort(f.k)] -- the reference's group() through dtb_group, then the
  materialisation of every ArrayView column through dtb_gather -- must equal the stock CPU result.
* the residency bracket around EvalContext::evaluate(): inside DT[:, sum(f.v), by(f.k)] with both options
  on, dtb_reduce finds the RowIndex and the offsets that dtb_group just produced already in HBM
  (dtb_last_call_stats().cache_hits of the reducer call >= 1: the RowIndex; the offsets too unless the
  reference's Buffer::resize moved them).
* no usable GPU: the engine's error must surface.
"""
import ctypes
import os
import sys
import time

import numpy as np
import datatable as dt
from datatable import f, by, sort

rng = np.random.default_rng(11)
n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 400_000
k = rng.integers(0, 5000, n).astype(np.int32)
v = rng.random(n); v[rng.random(n) < 0.05] = np.nan
w = rng.integers(-1000, 1000, n).astype(np.int16)
b = rng.random(n) < 0.3
DT = dt.Frame(k=k, v=v, w=w, b=b, x=rng.integers(-2**60, 2**60, n))


def sorted_frame():
    R = DT[:, :, sort(f.k)]
    R.materialize()
    return R.to_numpy()


want = sorted_frame()
dt.options.sort.b200 = True
try:
    t0 = time.perf_counter(); got = sorted_frame(); t_gpu = time.perf_counter() - t0
except Exception as e:
    assert "dtb200" in str(e), str(e)
    print("check_hook_views: no usable GPU here; the engine was reached and reported:", str(e).splitlines()[0])
    sys.exit(0)
finally:
    dt.options.sort.b200 = False
assert np.array_equal(got, want, equal_nan=True)
print(f"check_hook_views: sort + materialise of {DT.ncols} view columns on the engine == CPU path: ok")

# residency: the stats of the LAST engine call of the query (the reducer) count the cache hits
here = os.path.dirname(os.path.abspath(__file__))
lib = ctypes.CDLL(os.path.join(os.path.dirname(here), "datatable_b200", "lib", "libdtb200.so"))


class Stats(ctypes.Structure):
    _fields_ = [("kernels_launched", ctypes.c_int32), ("radix_passes", ctypes.c_int32), ("key_bits", ctypes.c_int32),
                ("cache_hits", ctypes.c_int32), ("scratch_bytes", ctypes.c_int64)]


dt.options.sort.b200 = True
dt.options.sort.b200_reducers = True
try:
    R = DT[:, dt.sum(f.v), by(f.k)]
    # the reducer ran inside evaluate() (eagerly, through dtb_reduce); the group-key column is still a lazy
    # view: read the stats of the reducer call before anything materialises it
    st = Stats(); lib.dtb_last_call_stats(ctypes.byref(st))
    R.materialize()
finally:
    dt.options.sort.b200 = False
    dt.options.sort.b200_reducers = False
assert st.cache_hits >= 1, st.cache_hits
print(f"check_hook_views: dtb_reduce reused {st.cache_hits} buffers left in HBM by dtb_group (residency bracket): ok")
