#!/usr/bin/env python
"""Row selection by a boolean or integer column on one GPU (dtb_mask_rows, dtb_int_rows, DT[f.m, j]).

    python scripts/bench_row_select.py [--n 1000000000] [--reps 10] [--out results/h100_bench_row_select.json]

- the compaction of a bool8 mask of n rows at densities 0, 1e-6, 0.5, 1 - 1e-6 and 1, random and clustered (runs of
  1 .. 5000 rows): CUDA-event time per call and GB/s over its bytes model, 2 B per row (the mask read twice) plus 4 B
  per selected row (1 B per row when nothing is selected: the emit pass does not run); torch.nonzero on the same mask, in the same process, as a yardstick only;
- the integer path (statistics + int32 RowIndex) for int32 and int64 selectors of n / 10 rows;
- DT[f.m, f.v] and DT[f.m, dt.sum(f.v)] on a device frame at density 0.5.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import datatable_b200 as dtb                                   # noqa: E402
from datatable_b200 import engine                               # noqa: E402
from datatable_b200._lib import BOOL, INT32, INT64, FLOAT64     # noqa: E402


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), float(min(ms))


def mask(n, density, clustered, gen):
    if clustered:
        lens = torch.randint(1, 5000, (n // 2500 + 2,), generator=gen, device="cuda")
        runs = torch.arange(len(lens), device="cuda") % 2
        m = torch.repeat_interleave(runs, lens)[:n].to(torch.int8)
        return torch.cat([m, torch.zeros(n - m.numel(), dtype=torch.int8, device="cuda")])
    if density in (0.0, 1.0):
        return torch.full((n,), int(density), dtype=torch.int8, device="cuda")
    return (torch.rand(n, generator=gen, device="cuda") < density).to(torch.int8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_row_select.py needs a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    rec = {"gpu": smi[0] if smi else torch.cuda.get_device_name(), "n": args.n, "compaction": [], "int_rows": [],
           "frame": []}
    gen = torch.Generator(device="cuda").manual_seed(1)
    n = args.n
    for clustered in (False, True):
        for density in ((0.0, 1e-6, 0.5, 1 - 1e-6, 1.0) if not clustered else (0.5,)):
            m = mask(n, density, clustered, gen)
            k = engine.mask_rows(m).numel()
            med, best = timed(lambda: engine.mask_rows(m), args.reps)
            tmed, tbest = timed(lambda: torch.nonzero(m).view(-1), args.reps)
            byts = (2 * n if k else n) + 4 * k              # nothing selected: the emit pass does not run
            rec["compaction"].append({"density": density, "clustered": clustered, "selected": k, "ms": med,
                                      "ms_best": best, "GBps": byts / med / 1e6, "torch_nonzero_ms": tmed,
                                      "torch_nonzero_ms_best": tbest})
            print(json.dumps(rec["compaction"][-1]), flush=True)
            del m
    for st, dt_ in ((INT32, torch.int32), (INT64, torch.int64)):
        s = torch.randint(0, n, (n // 10,), generator=gen, device="cuda", dtype=torch.int64).to(dt_)
        med, best = timed(lambda: engine.int_rows(s, st), args.reps)
        rec["int_rows"].append({"stype": st, "rows": s.numel(), "ms": med, "ms_best": best})
        print(json.dumps(rec["int_rows"][-1]), flush=True)
        del s
    m = mask(n, 0.5, False, gen)
    v = torch.rand(n, generator=gen, device="cuda", dtype=torch.float64)
    DT = dtb.Frame({"m": m, "v": v}, stypes={"m": BOOL, "v": FLOAT64})
    for name, q in (("DT[f.m, f.v]", lambda: DT[dtb.f.m, dtb.f.v]),
                    ("DT[f.m, dt.sum(f.v)]", lambda: DT[dtb.f.m, dtb.sum(dtb.f.v)])):
        med, best = timed(q, max(3, args.reps // 2))
        rec["frame"].append({"query": name, "density": 0.5, "ms": med, "ms_best": best})
        print(json.dumps(rec["frame"][-1]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(rec, fh, indent=1)
    print(json.dumps({"gpu": rec["gpu"]}))


if __name__ == "__main__":
    main()
