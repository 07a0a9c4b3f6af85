"""Per-launch radix pass times of C2 (1e9 int32 keys, 1e6 groups, sum(v) by(k)) and of the same keys sorted only,
next to the bytes each pass moves.

The radix passes carry only the key bits that later passes still read, in the narrowest of u8 / u16 / u32 / u64
(DESIGN.md 4.1).  This script sets the per-launch scatter and count times, taken from the engine's profile records
(CUDA events around every launch), against two byte models of the same passes: the full-width one that bench.py's
roofline keeps (4-byte keys in and out of every pass) and the narrowed one.

    python scripts/bench_narrow_keys.py [--root TREE] [--runs 3] [--steps 5] [--out FILE]

--root imports datatable_b200 from another checkout (for example the parent commit), so that two trees can be
compared in one process-per-tree sequence on the same card.  One JSON line per run goes to stdout and, with --out,
is appended to FILE.
"""
import argparse
import json
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def plan_passes(total_bits, width=8):
    """dtb_api.cu plan_passes: (shift, bits) of every pass."""
    np_ = max(1, -(-total_bits // width))
    base, extra, sh, out = total_bits // np_, total_bits % np_, 0, []
    for p in range(np_):
        b = max(1, base + (1 if p < extra else 0))
        out.append((sh, b))
        sh += b
    return out


def narrow_bytes(bits):
    return 1 if bits <= 8 else 2 if bits <= 16 else 4 if bits <= 32 else 8


def pass_bytes(total_bits, passes, narrowed, raw_bytes=4):
    """Algorithmic bytes per row of every pass whose last pass writes no keys: read (key [+ row id]), write
    (key + row id).  The first pass reads the raw column and no row id."""
    out = []
    for p, (sh, b) in enumerate(passes):
        first, last = p == 0, p == len(passes) - 1
        kin = raw_bytes if first else (narrow_bytes(total_bits - sh) if narrowed else 4)
        kout = 0 if last else (narrow_bytes(total_bits - sh - b) if narrowed else 4)
        out.append(kin + (0 if first else 4) + kout + 4)
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=os.path.dirname(HERE))
    ap.add_argument("--label", default=None)
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--groups", type=int, default=1_000_000)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_narrow_keys.py: no CUDA device")
    from datatable_b200 import engine, _lib

    n, G = args.rows, args.groups
    gen = torch.Generator(device="cuda"); gen.manual_seed(42)             # bench.py's C2 input
    k = torch.randint(0, G, (n,), generator=gen, device="cuda", dtype=torch.int32)
    v = torch.rand(n, generator=gen, device="cuda", dtype=torch.float64)
    torch.cuda.synchronize()

    def c2():
        engine.Groupby([k], [0], _lib.NA_FIRST, reducers=[(_lib.OP_SUM, v)]).close()

    def sort_only():
        engine.Groupby([k], [_lib.FLAG_SORT_ONLY], _lib.NA_FIRST).close()

    info = {"label": args.label or os.path.abspath(args.root), "card": card(),
            "device": torch.cuda.get_device_name(0), "rows": n, "groups": G}
    for run in range(args.runs):
        for name, fn in (("C2", c2), ("sort_only", sort_only)):
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            engine.set_option("profile", 1)
            _lib.profile_records(reset=True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            engine.set_option("profile", 0)
            recs = _lib.profile_records(reset=True)
            st = _lib.last_call_stats()
            passes = plan_passes(st["key_bits"])
            npass = len(passes)
            fam = {}
            for fam_name, ms in recs:
                fam.setdefault(fam_name, []).append(ms)
            per_pass = {}
            for f_ in ("radix_scatter", "radix_count"):
                t = fam.get(f_, [])
                per_pass[f_] = [round(sum(t[p::npass]) / max(1, len(t[p::npass])), 4) for p in range(npass)] \
                    if len(t) == npass * args.steps else t
            full = pass_bytes(st["key_bits"], passes, False)
            narrow = pass_bytes(st["key_bits"], passes, True)
            line = dict(info, run=run, case=name, ms_per_step=e0.elapsed_time(e1) / args.steps,
                        key_bits=st["key_bits"], passes=passes, radix_passes=st["radix_passes"],
                        scatter_ms_per_pass=per_pass["radix_scatter"], count_ms_per_pass=per_pass["radix_count"],
                        bytes_per_row_full=full, bytes_per_row_narrow=narrow,
                        kernel_ms_per_step={f_: round(sum(t) / args.steps, 4) for f_, t in fam.items()})
            s = per_pass["radix_scatter"]
            if len(s) == npass:
                line["scatter_GBps_full_model"] = [round(b * n / (ms / 1e3) / 1e9, 1) for b, ms in zip(full, s)]
                line["scatter_GBps_narrow_model"] = [round(b * n / (ms / 1e3) / 1e9, 1) for b, ms in zip(narrow, s)]
            print(json.dumps(line), flush=True)
            if args.out:
                with open(args.out, "a") as fh:
                    fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
