#!/usr/bin/env python3
"""Checks a reference build patched by apply_hook.py (run with PYTHONPATH=<scratch>/src).

* option sort.b200 exists and defaults to False; with it off, results are the stock CPU results;
* with it on, group() goes through libdtb200's dtb_group:
    - on a box with a GPU: the results must equal the stock CPU results (bit-exact RowIndex / offsets,
      sums within 1e-6 relative);
    - on a box without a usable GPU (this build container): the engine's own error must surface as a
      datatable exception -- there is no CPU fallback inside the library, and unsupported column types
      (strings) still take the reference's CPU path (DTB_ENOTIMPL falls through).
"""
import sys
import numpy as np
import datatable as dt
from datatable import f, by, sort

rng = np.random.default_rng(7)
n = 200_000
k = rng.integers(0, 1000, n).astype(np.int32)
x = rng.standard_normal(n)
v = rng.random(n)
DT = dt.Frame(k=k, x=x, v=v, idx=np.arange(n, dtype=np.int32))


def run():
    a = DT[:, {"s": dt.sum(f.v), "c": dt.count()}, by(f.k)].to_numpy()
    b = DT[:, f.idx, sort(-f.x, na_position="last")].to_numpy().ravel()
    c = DT[:, f.idx, by(f.k), sort(f.x)].to_numpy()
    return a, b, c


assert dt.options.sort.b200 is False, "option sort.b200 must exist and default to False"
want = run()
dt.options.sort.b200 = True
try:
    got = run()
except Exception as e:                       # no usable GPU: the engine's error is surfaced
    msg = str(e)
    assert "dtb200" in msg, msg
    print("check_hook: no usable GPU here; dtb_group was reached and reported:", msg.splitlines()[0])
    # string keys are outside the engine's scope: they must still work (CPU path) with the option on
    S = dt.Frame(s=["b", "a", None, "a"], v=[1, 2, 3, 4])
    r = S[:, dt.sum(f.v), by(f.s)].to_list()
    assert r == [[None, "a", "b"], [3, 6, 1]], r
    print("check_hook: string keys fall through to the reference's CPU path: ok")
    sys.exit(0)
finally:
    dt.options.sort.b200 = False
assert np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
assert np.array_equal(got[0][:, 0], want[0][:, 0]) and np.array_equal(got[0][:, 2], want[0][:, 2])
assert np.allclose(got[0][:, 1], want[0][:, 1], rtol=1e-6, atol=0)
print("check_hook: GPU path == CPU path on", n, "rows: ok")
