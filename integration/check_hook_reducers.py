#!/usr/bin/env python3
"""Checks the reducer hook of a patched reference build (option sort.b200_reducers; run with
PYTHONPATH=<scratch>/src or oracle/_ref/patched).

With the option on, sum/mean/min/max/count/countna of plain numeric columns go through dtb_reduce.
* GPU: results must equal the stock CPU results (ints/min/max/counts bit-exact, float sums/means 1e-6);
  with sort.b200 on as well the whole DT[:, reducers, by(k)] runs on the engine.
* no usable GPU: the engine's error must surface; reducers outside the engine's scope (prod, sd) and
  computed arguments (f.v * 2) must keep working through the reference's own columns.
"""
import sys
import numpy as np
import datatable as dt
from datatable import f, by

rng = np.random.default_rng(3)
n = 300_000
k = rng.integers(0, 5000, n).astype(np.int32)
v = rng.random(n); v[rng.random(n) < 0.05] = np.nan
w = rng.integers(-1000, 1000, n).astype(np.int16)
b = (rng.random(n) < 0.3)
DT = dt.Frame(k=k, v=v, w=w, b=b)
J = {"sv": dt.sum(f.v), "mv": dt.mean(f.v), "lo": dt.min(f.v), "hi": dt.max(f.v), "cv": dt.count(f.v),
     "sw": dt.sum(f.w), "mw": dt.mean(f.w), "lw": dt.min(f.w), "hw": dt.max(f.w), "sb": dt.sum(f.b),
     "pv": dt.prod(f.b), "s2": dt.sum(f.v * 2)}


def run():
    R = DT[:, J, by(f.k)]
    return R.names, R.to_numpy()


assert dt.options.sort.b200_reducers is False
names, want = run()
for group_too in (False, True):
    dt.options.sort.b200_reducers = True
    dt.options.sort.b200 = group_too
    try:
        _, got = run()
    except Exception as e:
        msg = str(e)
        assert "dtb200" in msg, msg
        print("check_hook_reducers: no usable GPU here; the engine was reached and reported:", msg.splitlines()[0])
        sys.exit(0)
    finally:
        dt.options.sort.b200_reducers = False
        dt.options.sort.b200 = False
    for j, nm in enumerate(names):
        a, c = got[:, j], want[:, j]
        if nm in ("sv", "mv", "mw", "s2"):
            assert np.allclose(a, c, rtol=1e-6, atol=0, equal_nan=True), nm
        else:
            assert np.array_equal(a, c, equal_nan=True), nm
    print(f"check_hook_reducers: engine == CPU for {len(names) - 1} reducers (group() on engine: {group_too}): ok")
