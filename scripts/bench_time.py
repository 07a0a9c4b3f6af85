#!/usr/bin/env python
"""Times the time functions (dtb_time_part) and a by() on a derived year key, over device-resident columns on one GPU.

    python scripts/bench_time.py [--rows 1e9] [--out results]

With CUDA events on the current stream, 2 warm-up calls and the median of 5:

    year / hour over a date32 / time64 column of `rows` rows (1 % NA), through the identity: the model is 8 bytes per
        row for date32 (4 read, 4 written) and 12 for time64 (8 read, 4 written);
    the same through a shuffled int32 RowIndex of every row: 4 more bytes per row for the index, and the values are
        read at random (one 32-byte sector per row);
    DT[:, sum(f.v), by(year(f.d))] end to end over device columns (d date32, v int64), against the same query on a
        stored int32 year column (by(f.y)), which leaves out only the derived key's pass.

Each call's bytes over its time are reported as GB/s.  The card's name and power limit are read in the same run and
written with the timings to OUT/h100_bench_time.json.
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
    import torch
    import datatable_b200 as dtb
    from datatable_b200 import engine, _lib
    torch.cuda.set_device(0)
    name, limit = card()
    n = int(float(args.rows))
    res = {"card": name, "power_limit": limit, "rows": n, "cases": []}
    g = torch.Generator(device="cuda").manual_seed(2026)

    def record(rec, fn, nbytes=None):
        rec["ms"], rec["all_ms"] = timed(fn)
        if nbytes:
            rec["bytes"] = nbytes
            rec["GB_per_s"] = nbytes / rec["ms"] / 1e6
        print(json.dumps(rec), flush=True)
        res["cases"].append(rec)

    perm = torch.randperm(n, device="cuda", generator=g).to(torch.int32)
    for st, part in ((_lib.DATE32, _lib.TIME_YEAR), (_lib.TIME64, _lib.TIME_YEAR), (_lib.TIME64, _lib.TIME_HOUR)):
        if st == _lib.DATE32:
            v = torch.randint(-50000, 50000, (n,), device="cuda", generator=g, dtype=torch.int32)
            v[torch.rand(n, device="cuda", generator=g) < 0.01] = -2**31
        else:
            v = torch.randint(-2**62, 2**62, (n,), device="cuda", generator=g, dtype=torch.int64)
            v[torch.rand(n, device="cuda", generator=g) < 0.01] = -2**63
        esz = v.element_size()
        label = {_lib.DATE32: "date32", _lib.TIME64: "time64"}[st]
        pname = {_lib.TIME_YEAR: "year", _lib.TIME_HOUR: "hour"}[part]
        record({"value": label, "part": pname, "rows": "identity"},
               lambda: engine.time_part(part, v, None, stype=st), n * (esz + 4))
        record({"value": label, "part": pname, "rows": "rowindex_i32_shuffled"},
               lambda: engine.time_part(part, v, perm, stype=st), n * (4 + esz + 4))
        del v
        torch.cuda.empty_cache()
    del perm
    torch.cuda.empty_cache()

    d = torch.randint(-50000, 50000, (n,), device="cuda", generator=g, dtype=torch.int32)
    d[torch.rand(n, device="cuda", generator=g) < 0.01] = -2**31
    val = torch.randint(-1000, 1000, (n,), device="cuda", generator=g, dtype=torch.int64)
    y = engine.time_part(_lib.TIME_YEAR, d, None, stype=_lib.DATE32)
    D = dtb.Frame({"d": d, "v": val}, stypes={"d": _lib.DATE32})
    Y = dtb.Frame({"y": y, "v": val})
    f = dtb.f
    a = D[:, dtb.sum(f.v), dtb.by(dtb.time.year(f.d))]
    b = Y[:, dtb.sum(f.v), dtb.by(f.y)]
    same = bool(torch.equal(a.column("d"), b.column("y")) and torch.equal(a.column("v"), b.column("v")))
    record({"query": "DT[:, sum(f.v), by(year(f.d))]", "ngroups": a.nrows, "same_as_stored_key": same},
           lambda: D[:, dtb.sum(f.v), dtb.by(dtb.time.year(f.d))])
    record({"query": "DT[:, sum(f.v), by(f.y)] (stored int32 year)", "ngroups": b.nrows},
           lambda: Y[:, dtb.sum(f.v), dtb.by(f.y)])
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "h100_bench_time.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({"card": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
