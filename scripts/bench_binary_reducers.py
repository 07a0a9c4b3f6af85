#!/usr/bin/env python
"""Times the per-group product, sd and cov / corr next to the per-group sum on the same groups, on one GPU.

    python scripts/bench_binary_reducers.py [--rows 1e8,1e9] [--out DIR]

Keys are shaped like the db-benchmark groupby question C4: two int32 key columns (1000 x 1000 values, at most 1e6
groups); the value columns v1, v2 are float64 with 1 % NaN.  The frame is grouped once (a Groupby handle), then each reducer
is timed with CUDA events on the current stream: 2 warm-up calls, the median of 5.

    sum            the handle's reducer: with device key columns and a small key domain it streams the rows by
                   group key (dtb_groupby_reduce)
    sum_rowindex   the same sum gathered through the RowIndex (dtb_reduce on the handle's RowIndex)
    prod           the handle's PROD: it always gathers through the RowIndex, so sum_rowindex is its yardstick
    sd             the handle's SD(v1): a pivot pass and two passes, each reading the RowIndex and one random value
                   sector per row
    cov, corr      dtb_groupby_reduce2(v1, v2): the same moment kernels over two random value sectors per row

A second case puts every row in one group under a random RowIndex (2e7 rows and the largest size asked for): every
tile's boundary slots then belong to the same group.  The card's name and power limit are read in the same run and
written with the timings to DIR/bench_binary_reducers.json.
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
    sizes = [int(float(x)) for x in args.rows.split(",")]
    g = torch.Generator(device="cuda")
    for n in sizes:
        g.manual_seed(n)
        k1 = torch.randint(0, 1000, (n,), device="cuda", generator=g, dtype=torch.int32)
        k2 = torch.randint(0, 1000, (n,), device="cuda", generator=g, dtype=torch.int32)
        v = torch.rand(n, device="cuda", generator=g, dtype=torch.float64) + 0.5
        v[torch.rand(n, device="cuda", generator=g) < 0.01] = float("nan")
        v2 = torch.rand(n, device="cuda", generator=g, dtype=torch.float64) - 0.5
        v2[torch.rand(n, device="cuda", generator=g) < 0.01] = float("nan")
        gb = engine.Groupby([k1, k2], [0, 0], _lib.NA_FIRST)
        order = gb.order()
        rec = {"shape": "C4 keys", "rows": n, "groups": gb.ngroups}
        rec["sum_ms"], _ = timed(lambda: gb.reduce(_lib.OP_SUM, v))
        rec["sum_rowindex_ms"], _ = timed(lambda: gb.reduce_ordered(_lib.OP_SUM, v, order))
        rec["prod_ms"], _ = timed(lambda: gb.reduce(_lib.OP_PROD, v))
        rec["sd_ms"], _ = timed(lambda: gb.reduce(_lib.OP_SD, v))
        rec["cov_ms"], _ = timed(lambda: gb.reduce2(_lib.OP_COV, v, v2))
        rec["corr_ms"], _ = timed(lambda: gb.reduce2(_lib.OP_CORR, v, v2))
        print(json.dumps(rec), flush=True)
        res["cases"].append(rec)
        del gb, order, k1, k2
        torch.cuda.empty_cache()
        for m in sorted({20_000_000, n}) if n == sizes[0] else [n]:
            order = torch.randperm(m, device="cuda", generator=g, dtype=torch.int32)
            offsets = torch.tensor([0, m], dtype=torch.int32, device="cuda")
            w, w2 = v[:m], v2[:m]
            rec = {"shape": "one group", "rows": m, "groups": 1}
            rec["sum_rowindex_ms"], _ = timed(lambda: engine.reduce(_lib.OP_SUM, w, order, offsets))
            rec["prod_ms"], _ = timed(lambda: engine.reduce(_lib.OP_PROD, w, order, offsets))
            rec["sd_ms"], _ = timed(lambda: engine.reduce(_lib.OP_SD, w, order, offsets))
            rec["cov_ms"], _ = timed(lambda: engine.reduce2(_lib.OP_COV, w, w2, order, offsets))
            rec["corr_ms"], _ = timed(lambda: engine.reduce2(_lib.OP_CORR, w, w2, order, offsets))
            print(json.dumps(rec), flush=True)
            res["cases"].append(rec)
            del order
            torch.cuda.empty_cache()
        del v, v2
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_binary_reducers.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({"card": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
