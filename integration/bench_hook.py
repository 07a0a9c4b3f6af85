#!/usr/bin/env python3
"""Times the PATCHED reference (oracle/_ref/patched on PYTHONPATH): its own
DT[:, dt.sum(f.v), by(f.k)] on host Frames with the engine options off (stock CPU path) and on
(group() -> dtb_group, sum -> dtb_reduce, residency bracket).  This is the drop-in end-to-end number:
the user's code and the reference's Frame objects are unchanged, only `dt.options.sort.b200*` flip.
Prints one JSON object.  Usage: bench_hook.py [rows_cpu] [rows_gpu]"""
import json
import sys
import time

import numpy as np
import datatable as dt
from datatable import f, by

rows_cpu = int(float(sys.argv[1])) if len(sys.argv) > 1 else 10_000_000
rows_gpu = int(float(sys.argv[2])) if len(sys.argv) > 2 else 100_000_000
rng = np.random.default_rng(42)
k = rng.integers(0, 1_000_000, rows_gpu, dtype=np.int32)
v = rng.random(rows_gpu)


def run(DT, on, reps):
    dt.options.sort.b200 = on
    dt.options.sort.b200_reducers = on
    try:
        ts, R = [], None
        for _ in range(reps):
            t0 = time.perf_counter()
            R = DT[:, dt.sum(f.v), by(f.k)]
            R.materialize()
            ts.append(time.perf_counter() - t0)
        return min(ts), R
    finally:
        dt.options.sort.b200 = False
        dt.options.sort.b200_reducers = False


out = {"query": "DT[:, dt.sum(f.v), by(f.k)] on host Frames of the patched reference, int32 keys (1e6 distinct), float64 values",
       "nthreads": int(dt.options.nthreads)}
DTs = dt.Frame(k=k[:rows_cpu], v=v[:rows_cpu])
t_off, R_off = run(DTs, False, 2)
try:
    t_on, R_on = run(DTs, True, 3)
    a, b = R_off.to_numpy(), R_on.to_numpy()
    same = bool(np.array_equal(a[:, 0], b[:, 0]) and np.allclose(a[:, 1], b[:, 1], rtol=1e-9))
    out["small"] = {"rows": rows_cpu, "cpu_s": t_off, "engine_s": t_on, "speedup": t_off / t_on, "results_equal": same,
                    "rows_per_s_engine": rows_cpu / t_on}
    DTb = dt.Frame(k=k, v=v)
    t_big, R_big = run(DTb, True, 3)
    out["large"] = {"rows": rows_gpu, "engine_s": t_big, "rows_per_s_engine": rows_gpu / t_big, "groups": int(R_big.nrows),
                    "note": "the stock CPU path is not timed at this size: it takes ~50 s at 3e7 rows on this box (bench.py --impl reference probes)"}
except Exception as e:                                                  # noqa: BLE001
    out["error"] = str(e).splitlines()[0][:200]
    out["small"] = {"rows": rows_cpu, "cpu_s": t_off}
print(json.dumps(out))
