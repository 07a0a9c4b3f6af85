#!/usr/bin/env python
"""Times the keyed join that reads the joined frame's columns (dtb_join_gather) against the index-then-gather
composition it replaces, and the whole DT[:, j, join(P), by()] queries, on one GPU.

    python scripts/bench_join_groupby.py [--rows 1e8,1e9] [--out DIR]

X is shaped like the db-benchmark groupby question C2: an int32 key k with 1e6 distinct values and a float64 value
v, plus an int32 join key pk drawn from P's keys (every X row matches).  P, the keyed dimension frame, has 1e3 or 1e6
rows: pk (int32), region (int32, 10 values) and price (float64).  Its keys are dense (consecutive: the direct-address
lookup) or sparse (every 7919th integer: the binary search).  Each call is timed with CUDA events on the current
stream, 2 warm-up calls and the median of 5:

    index          engine.join_index: the int32 RowIndex of P's rows
    index_gather   join_index, then one engine.gather of P's price through it
    join_gather    engine.join_gather of price: the same lookup, the value written at the match, no index
    q_sum_g_by_f   X[:, dt.sum(g.price), join(P), by(f.k)]   (device frames)
    q_sum_f_by_g   X[:, dt.sum(f.v), join(P), by(g.region)]

join_gather saves the index's int32 write and read per X row; the direct-address lookup replaces about log2(nP)
dependent probes of P's keys with one.  The card's name and power limit are read in the same run and written with
the timings to DIR/bench_join_groupby.json.
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
    import datatable_b200 as dt
    from datatable_b200 import engine, _lib, f, g, join, by
    torch.cuda.set_device(0)
    name, limit = card()
    res = {"card": name, "power_limit": limit, "cases": []}
    gen = torch.Generator(device="cuda")
    for n in [int(float(x)) for x in args.rows.split(",")]:
        gen.manual_seed(n)
        k = torch.randint(0, 1_000_000, (n,), device="cuda", generator=gen, dtype=torch.int32)
        v = torch.rand(n, device="cuda", generator=gen, dtype=torch.float64)
        for npr in (1000, 1_000_000):
            for layout in ("dense", "sparse"):
                pk = torch.arange(npr, device="cuda", dtype=torch.int32) * (1 if layout == "dense" else 7919)
                region = torch.randint(0, 10, (npr,), device="cuda", generator=gen, dtype=torch.int32)
                price = torch.rand(npr, device="cuda", generator=gen, dtype=torch.float64)
                xpk = pk[torch.randint(0, npr, (n,), device="cuda", generator=gen)]
                P = dt.Frame({"pk": pk, "region": region, "price": price})
                P.key = "pk"
                X = dt.Frame({"k": k, "pk": xpk, "v": v})
                xc, jc = [engine.Col(xpk, _lib.INT32)], [engine.Col(pk, _lib.INT32)]
                pc = engine.Col(price, _lib.FLOAT64)
                rec = {"rows": n, "p_rows": npr, "p_keys": layout}
                try:
                    rec["index_ms"], rec["index_all_ms"] = timed(lambda: engine.join_index(xc, jc))
                    rec["index_gather_ms"], rec["index_gather_all_ms"] = timed(
                        lambda: engine.gather(pc, engine.join_index(xc, jc)))
                    rec["join_gather_ms"], rec["join_gather_all_ms"] = timed(lambda: engine.join_gather(xc, jc, [pc]))
                    want = engine.gather(pc, engine.join_index(xc, jc))
                    rec["join_gather_equal"] = bool(torch.equal(engine.join_gather(xc, jc, [pc])[0].view(torch.int64),
                                                                want.view(torch.int64)))
                    del want
                    rec["q_sum_g_by_f_ms"], rec["q_sum_g_by_f_all_ms"] = timed(
                        lambda: X[:, dt.sum(g.price), join(P), by(f.k)])
                    rec["q_sum_f_by_g_ms"], rec["q_sum_f_by_g_all_ms"] = timed(
                        lambda: X[:, dt.sum(f.v), join(P), by(g.region)])
                except Exception as e:  # noqa: BLE001  (recorded: e.g. out of device memory at the largest size)
                    rec["error"] = f"{type(e).__name__}: {e}"
                print(json.dumps({a: b for a, b in rec.items() if not a.endswith("_all_ms")}), flush=True)
                res["cases"].append(rec)
                del P, X, xpk, xc, jc, pc
                torch.cuda.empty_cache()
        del k, v
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_join_groupby.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({"card": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
