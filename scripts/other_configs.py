"""Timings of the non-headline BASELINE configs (C3, C4) at full size on one H100, with
size-independent correctness checks.  Not bench lines: reported in DESIGN.md."""
import sys, time, json
import torch
sys.path.insert(0, ".")
from datatable_b200 import engine, _lib
from datatable_b200._lib import FLAG_SORT_ONLY

n = int(float(sys.argv[1])) if len(sys.argv) > 1 else 1_000_000_000
out = {}
g = torch.Generator(device="cuda"); g.manual_seed(1)

def timeit(fn, reps=3):
    fn(); torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); r = fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return min(ts), r

# ---- C3: float64 column sort -> RowIndex (ARR32) ----
x = torch.randn(n, generator=g, device="cuda", dtype=torch.float64)
x[::1000] = float("nan")
ms, (order, offs, ng) = timeit(lambda: engine.group([x], [FLAG_SORT_ONLY], 1))
xs = engine.gather(x, order)
nn = int(torch.isnan(x).sum())
ok = bool(torch.isnan(xs[:nn]).all()) and bool((xs[nn + 1:] >= xs[nn:-1]).all())
out["C3_f64_sort"] = {"rows": n, "ms": ms, "rows_per_s": n / ms * 1e3, "alg_GBps(12B/row)": 12 * n / ms / 1e6,
                      "key_bits": _lib.last_call_stats()["key_bits"], "sorted_nan_first": ok}
del x, xs, order
torch.cuda.empty_cache()

# ---- C4: (int64, int32) keys, mean/min/max/count over 3 float64 columns ----
k1 = torch.randint(0, 1000, (n,), generator=g, device="cuda", dtype=torch.int64) << 33
k2 = torch.randint(0, 1000, (n,), generator=g, device="cuda", dtype=torch.int32)
vs = [torch.randn(n, generator=g, device="cuda", dtype=torch.float64) for _ in range(3)]
for v in vs:
    v[::100] = float("nan")
ops = [_lib.OP_MEAN, _lib.OP_MIN, _lib.OP_MAX, _lib.OP_COUNT]
def c4():
    gb = engine.Groupby([k1, k2], [0, 0], 1, reducers=[(op, v) for v in vs for op in ops])
    res = [gb.reduced(i) for i in range(12)]
    ngroups = gb.ngroups
    gb.close()
    return ngroups, res
ms, (ngroups, res) = timeit(c4, reps=2)
cnt_total = int(res[3].sum())
ok = (ngroups == 1_000_000 or n < 10_000_000) and cnt_total == int((~torch.isnan(vs[0])).sum())
mx = float(torch.nan_to_num(res[2], nan=-1e300).max()); ok = ok and mx == float(vs[0][~torch.isnan(vs[0])].max())
out["C4_2key_12reducers"] = {"rows": n, "ms": ms, "rows_per_s": n / ms * 1e3, "alg_GBps(40B/row)": 40 * n / ms / 1e6,
                             "ngroups": ngroups, "key_bits": 20, "checks_ok": bool(ok)}
print(json.dumps(out, indent=1))
