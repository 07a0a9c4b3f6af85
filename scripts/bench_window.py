#!/usr/bin/env python
"""Times the grouped row functions shift, fillna, cumcount and ngroup (dtb_shift, dtb_fillna, dtb_group_index) next to
a gather and a cummax of the same column through the same RowIndex, on one GPU.

    python scripts/bench_window.py [--rows 1e8,1e9] [--out DIR]

Keys are shaped like the db-benchmark groupby question C2: one int32 key column with 1e6 distinct values, grouped
once (engine.group).  The value columns are float64 (uniform, 1 % NaN) and int32 (1000 distinct values, 1 % NA).  Two
groupings run over the same RowIndex: the C2 groups, and one group of all rows (its offsets [0, n]).  Each call is
timed with CUDA events on the current stream, 2 warm-up calls and the median of 5:

    gather                       engine.gather of the column through the RowIndex: the random reads and one write
    shift_p1, shift_m1           engine.shift, n = +1 and -1: the gather's random reads plus the group bounds
    fillna, fillna_reverse       engine.fillna: the cumulative scan's three kernels
    cummax                       engine.cumulative(OP_MAX): the same kernels as fillna, another state
    cumcount, ngroup             engine.group_index: no value reads, one 8-byte write per row

The card's name and power limit are read in the same run and written with the timings to DIR/bench_window.json.
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
    ap.add_argument("--rows", default="1e8,1e9")
    ap.add_argument("--out", default="bench_out")
    args = ap.parse_args()
    import torch
    from datatable_b200 import engine, _lib
    torch.cuda.set_device(0)
    name, limit = card()
    res = {"card": name, "power_limit": limit, "cases": []}
    g = torch.Generator(device="cuda")
    calls = (("gather", lambda v, o, f: engine.gather(v, o)),
             ("shift_p1", lambda v, o, f: engine.shift(v, o, f, 1)),
             ("shift_m1", lambda v, o, f: engine.shift(v, o, f, -1)),
             ("fillna", lambda v, o, f: engine.fillna(v, o, f)),
             ("fillna_reverse", lambda v, o, f: engine.fillna(v, o, f, reverse=True)),
             ("cummax", lambda v, o, f: engine.cumulative(_lib.OP_MAX, v, o, f)),
             ("cumcount", lambda v, o, f: engine.group_index(_lib.GROUP_CUMCOUNT, f)),
             ("ngroup", lambda v, o, f: engine.group_index(_lib.GROUP_NGROUP, f)))
    for n in [int(float(x)) for x in args.rows.split(",")]:
        g.manual_seed(n)
        k = torch.randint(0, 1_000_000, (n,), device="cuda", generator=g, dtype=torch.int32)
        order, offsets, ng = engine.group([k], [0], _lib.NA_FIRST)
        del k
        torch.cuda.empty_cache()
        one = torch.tensor([0, n], dtype=torch.int32, device="cuda")
        for vname in ("float64", "int32"):
            if vname == "float64":
                v = torch.rand(n, device="cuda", generator=g, dtype=torch.float64)
                v[torch.rand(n, device="cuda", generator=g) < 0.01] = float("nan")
            else:
                v = torch.randint(0, 1000, (n,), device="cuda", generator=g, dtype=torch.int32)
                v[torch.rand(n, device="cuda", generator=g) < 0.01] = -2**31
            for shape, f, groups in (("C2 groups", offsets, ng), ("one group", one, 1)):
                rec = {"shape": shape, "rows": n, "groups": groups, "value": vname}
                for cname, fn in calls:
                    try:
                        rec[cname + "_ms"], rec[cname + "_all_ms"] = timed(lambda: fn(v, order, f))
                    except Exception as e:  # noqa: BLE001  (recorded: e.g. out of device memory at the largest size)
                        rec[cname + "_error"] = f"{type(e).__name__}: {e}"
                    torch.cuda.empty_cache()
                print(json.dumps(rec), flush=True)
                res["cases"].append(rec)
            del v
            torch.cuda.empty_cache()
        del order, offsets, one
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_window.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({"card": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
