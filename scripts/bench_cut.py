#!/usr/bin/env python
"""Times dt.cut over whole device-resident columns (dtb_cut) on one GPU.

    python scripts/bench_cut.py [--rows 1e9] [--out results]

For an int32 and a float64 column (1 % NA) of `rows` rows, seen through the identity and through a random int32
RowIndex (the rows of a density-0.5 mask, shuffled), it times with CUDA events on the current stream, 2 warm-up calls
and the median of 5:

    nbins10        equal-width bins: cut_stats (min / max of the rows) then cut_emit
    edges10 / 1000 explicit edges staged in shared memory: cut_bins
    edges20000     above the 4096-edge shared-memory limit: a sample of every 5th edge, then a window in L2

then, in a separate profiled pass, the per-kernel times of the engine's profile (cut_stats, cut_emit, cut_bins).  As
yardsticks only, on the same columns: torch.bucketize on the same edges, and torch.aminmax plus one elementwise pass
(the two HBM passes of nbins without the bin arithmetic), each timed with the gather through the RowIndex and, for
bucketize, the conversion to float64 that cut makes on the fly.  The model for the identity float64 nbins call is 20
bytes per row (8 read by the statistics, 8 read and 4 written by the emit): the script reports each call's bytes over
its time.  The card's name and power limit are read in the same run and written with the timings to
OUT/h100_bench_cut.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        limit = f"unknown ({e})"
    return name, limit


def timed(fn, warmup=2, reps=5):
    import torch
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms), ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1e9")
    ap.add_argument("--out", default=os.path.join(ROOT, "results"))
    args = ap.parse_args()
    import numpy as np
    import torch
    from datatable_b200 import engine, _lib
    torch.cuda.set_device(0)
    name, limit = card()
    n = int(float(args.rows))
    res = {"card": name, "power_limit": limit, "rows": n, "cases": []}
    g = torch.Generator(device="cuda").manual_seed(2026)
    rng = np.random.default_rng(2026)
    edges = {k: np.sort(rng.choice(np.unique(rng.standard_normal(3 * k)), k, replace=False)) for k in (10, 1000, 20000)}
    mask = torch.rand(n, device="cuda", generator=g) < 0.5
    ridx = torch.nonzero(mask).view(-1).to(torch.int32)
    del mask
    ridx = ridx[torch.randperm(ridx.numel(), device="cuda", generator=g)]
    for vname in ("int32", "float64"):
        if vname == "float64":
            v = torch.randn(n, device="cuda", generator=g, dtype=torch.float64)
            v[torch.rand(n, device="cuda", generator=g) < 0.01] = float("nan")
            scale = 1.0
        else:
            v = torch.randint(-2**30, 2**30, (n,), device="cuda", generator=g, dtype=torch.int32)
            v[torch.rand(n, device="cuda", generator=g) < 0.01] = -2**31
            scale = 2.0**30 / 3
        esz = v.element_size()
        for oname, o in (("identity", None), ("rowindex_i32", ridx)):
            m = n if o is None else o.numel()
            ib = 0 if o is None else 4
            calls = [("nbins10", lambda: engine.cut(v, o, 10), m * (2 * (ib + esz) + 4))]
            for k, e in edges.items():
                calls.append((f"edges{k}", lambda e=e: engine.cut(v, o, edges=e * scale), m * (ib + esz + 4)))
            for cname, fn, nbytes in calls:
                rec = {"value": vname, "rows": oname, "positions": m, "call": cname, "bytes": nbytes}
                try:
                    rec["ms"], rec["all_ms"] = timed(fn)
                    rec["GB_per_s"] = nbytes / rec["ms"] / 1e6
                    engine.set_option("profile", 1)
                    _lib.profile_records()
                    fn()
                    torch.cuda.synchronize()
                    rec["kernels_ms"] = _lib.profile_records()
                    engine.set_option("profile", 0)
                except Exception as ex:  # noqa: BLE001
                    rec["error"] = f"{type(ex).__name__}: {ex}"
                    engine.set_option("profile", 0)
                torch.cuda.empty_cache()
                print(json.dumps(rec), flush=True)
                res["cases"].append(rec)
            # yardsticks: torch's own kernels over the same positions, the RowIndex gather (and int32 -> float64 for
            # bucketize) timed with them, as cut pays for it
            gather = (lambda: v) if o is None else (lambda: torch.index_select(v, 0, o))
            e1000 = torch.from_numpy(edges[1000] * scale).cuda()

            def aminmax_elementwise():
                x = gather()
                return torch.aminmax(x), torch.mul(x, 3).to(torch.int32)
            ys = [("torch.bucketize_edges1000", lambda: torch.bucketize(gather().double(), e1000, out_int32=True)),
                  ("torch.aminmax+elementwise", aminmax_elementwise)]
            for cname, fn in ys:
                rec = {"value": vname, "rows": oname, "positions": m, "call": cname}
                rec["ms"], rec["all_ms"] = timed(fn)
                print(json.dumps(rec), flush=True)
                res["cases"].append(rec)
            torch.cuda.empty_cache()
        del v
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_bench_cut.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({"card": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
