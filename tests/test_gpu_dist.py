"""GPU: the multi-GPU layer (datatable_b200/dist.py) on the engine's own kernels, against a single-process reference.

- dtb_dense_scatter + dtb_dense_compact against numpy: int32 / int64 keys, one block, several blocks and the largest
  table, presence patterns at the block edges, kmin at the type edges, partials that must keep their bits; and the
  documented argument refusals.
- dtb_lower_bound against np.searchsorted(side="left") on runs of duplicates, every stype, ±0.0 ties.
- groupby_partitioned (all three exchanges) and sort_partitioned in world 2 and world 3, ragged and with an empty
  rank.  Every rank runs the real kernels on its GPU (cuda:0 when only one is visible); the collectives run on a gloo
  group through a shim that stages device tensors through the host.  With two or more GPUs the same workers also run
  on NCCL without the shim, one process per GPU.
- The reference is computed here from the concatenated rows: group keys and their order from oracle.group (NA first,
  -0.0 and +0.0 distinct groups), per-group results from numpy; float sums bit for bit on multiples of 2^-8, and
  within a bound of math.fsum on uniform random values.
"""
import ctypes
import datetime
import math
import os
import socket
import traceback

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

DENSE_MAX = 1 << 22
SUM, MEAN, MIN, MAX, COUNT, COUNTNA, NROWS = 1, 2, 3, 4, 5, 6, 7


def same(got, want):
    """dtype, shape and bits equal (-0.0 is not +0.0); any NaN is NA"""
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    if got.dtype.kind != "f":
        return np.array_equal(got, want)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint8), want[~nan].view(np.uint8))


# ---------------------------------------------------------------------------------------------------------------
# dtb_dense_scatter / dtb_dense_compact
# ---------------------------------------------------------------------------------------------------------------
def _scatter(keys, kst, vals, kmin, table, present, size=None):
    from datatable_b200 import engine, _lib
    ptr = lambda t: ctypes.c_void_p(t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data)
    return _lib.lib.dtb_dense_scatter(ptr(keys), kst, ptr(vals), len(keys), int(kmin),
                                      len(table) if size is None else size, ptr(table), ptr(present),
                                      engine._stream())


def _err():
    from datatable_b200 import _lib
    return _lib.lib.dtb_last_error().decode("utf-8", "replace")


def _compact(table, present, kmin, kst, out_k, out_v, size=None):
    from datatable_b200 import engine, _lib
    ptr = lambda t: ctypes.c_void_p(t.data_ptr() if isinstance(t, torch.Tensor) else t.ctypes.data)
    ng = ctypes.c_int64(-1)
    rc = _lib.lib.dtb_dense_compact(ptr(table), ptr(present), len(table) if size is None else size, int(kmin), kst,
                                    ptr(out_k), ptr(out_v), ctypes.byref(ng), engine._stream())
    return rc, ng.value


SPECIAL_BITS = np.array([0x7FF8000000000123, 0xFFF0000000000001, 0x8000000000000000, 0x7FFFFFFFFFFFFFFF,
                         0, 0x7FF0000000000000, 1], np.uint64).view(np.int64)   # NaN payloads, -0.0, int64 min/max


def _patterns(size, rng):
    blk = np.arange(size) % 1024
    yield "none", np.zeros(size, bool)
    yield "all", np.ones(size, bool)
    yield "first", blk == 0
    yield "last", blk == 1023
    yield "1%", rng.random(size) < 0.01
    yield "99%", rng.random(size) < 0.99


@pytest.mark.parametrize("kdt", [np.int32, np.int64])
@pytest.mark.parametrize("size", [1024, 3 * 1024, DENSE_MAX])
def test_dense_scatter_compact(kdt, size):
    from datatable_b200 import _lib
    rng = np.random.default_rng(size + np.dtype(kdt).itemsize)
    kst = _lib.INT32 if kdt == np.int32 else _lib.INT64
    info = np.iinfo(kdt)
    kmins = [info.min + 1, -5, info.max - size + 1] if kdt == np.int32 else [-2**62, 2**62, info.min + 1]
    for kmin in kmins:
        for name, mask in _patterns(size, rng):
            x = np.flatnonzero(mask)
            vals = rng.integers(-2**63, 2**63 - 1, len(x), dtype=np.int64, endpoint=True)
            vals[:min(len(x), len(SPECIAL_BITS))] = SPECIAL_BITS[:len(x)]
            want_t = np.zeros(size, np.int64)
            want_t[x] = vals
            keys = (kmin + x).astype(kdt)
            # keys just outside the table are skipped (below kmin = min + 1 lies the NA key)
            outside = [k for k in (kmin - 1, kmin + size) if info.min <= k <= info.max]
            keys = np.concatenate([keys, np.array(outside, kdt)])
            vals = np.concatenate([vals, np.full(len(outside), 77, np.int64)])
            perm = rng.permutation(len(keys))
            keys, vals = keys[perm], vals[perm]
            table = torch.zeros(size, dtype=torch.int64, device="cuda")
            present = torch.zeros(size, dtype=torch.int32, device="cuda")
            kd, vd = torch.from_numpy(keys).cuda(), torch.from_numpy(vals).cuda()
            assert _scatter(kd, kst, vd, kmin, table, present) == _lib.OK, _err()
            where = (np.dtype(kdt).name, size, kmin, name)
            assert np.array_equal(present.cpu().numpy(), mask.astype(np.int32)), where
            assert np.array_equal(table.cpu().numpy(), want_t), where
            out_k = torch.full((size,), 3, dtype={np.int32: torch.int32, np.int64: torch.int64}[kdt], device="cuda")
            out_v = torch.full((size,), 3, dtype=torch.int64, device="cuda")
            rc, ng = _compact(table, present, kmin, kst, out_k, out_v)
            assert rc == _lib.OK and ng == len(x), where
            assert np.array_equal(out_k[:ng].cpu().numpy(), (kmin + x).astype(kdt)), where
            assert np.array_equal(out_v[:ng].cpu().numpy(), want_t[x]), where
            assert (out_k[ng:] == 3).all() and (out_v[ng:] == 3).all(), where      # nothing written past ng


def test_dense_refusals():
    from datatable_b200 import _lib
    big = DENSE_MAX + 2048
    table = torch.zeros(big, dtype=torch.int64, device="cuda")
    present = torch.zeros(big, dtype=torch.int32, device="cuda")
    keys = torch.arange(4, dtype=torch.int32, device="cuda")
    vals = torch.ones(4, dtype=torch.int64, device="cuda")
    out_k = torch.zeros(big, dtype=torch.int32, device="cuda")
    out_v = torch.zeros(big, dtype=torch.int64, device="cuda")
    for size in (1000, 1024 + 512, DENSE_MAX + 1024):
        assert _scatter(keys, _lib.INT32, vals, 0, table, present, size=size) == _lib.EINVAL, size
        assert "multiple of 1024" in _err()
        assert _compact(table, present, 0, _lib.INT32, out_k, out_v, size=size)[0] == _lib.EINVAL, size
        assert "multiple of 1024" in _err()
    h_table, h_present = np.zeros(1024, np.int64), np.zeros(1024, np.int32)
    h_keys, h_vals = np.arange(4, dtype=np.int32), np.ones(4, np.int64)
    t, p = table[:1024], present[:1024]
    assert _scatter(keys, _lib.INT32, vals, 0, h_table, p) == _lib.EINVAL
    assert _scatter(keys, _lib.INT32, vals, 0, t, h_present) == _lib.EINVAL
    assert _scatter(h_keys, _lib.INT32, vals, 0, t, p) == _lib.EINVAL
    assert _scatter(keys, _lib.INT32, h_vals, 0, t, p) == _lib.EINVAL
    assert _compact(h_table, p, 0, _lib.INT32, out_k, out_v)[0] == _lib.EINVAL
    assert _compact(t, h_present, 0, _lib.INT32, out_k, out_v)[0] == _lib.EINVAL
    assert _compact(t, p, 0, _lib.INT32, np.zeros(1024, np.int32), out_v)[0] == _lib.EINVAL
    assert _compact(t, p, 0, _lib.INT32, out_k, np.zeros(1024, np.int64))[0] == _lib.EINVAL
    for st in (_lib.INT8, _lib.INT16, _lib.BOOL, _lib.FLOAT32, _lib.FLOAT64):
        assert _scatter(keys, st, vals, 0, t, p) == _lib.ENOTIMPL, st
        assert _compact(t, p, 0, st, out_k, out_v)[0] == _lib.ENOTIMPL, st
    assert not present.any() and not table.any()                          # no refused call touched the device


# ---------------------------------------------------------------------------------------------------------------
# dtb_lower_bound
# ---------------------------------------------------------------------------------------------------------------
LB_TYPES = {"bool": np.int8, "int8": np.int8, "int16": np.int16, "int32": np.int32, "int64": np.int64,
            "float32": np.float32, "float64": np.float64}


@pytest.mark.parametrize("name", list(LB_TYPES))
def test_lower_bound_runs(name):
    from datatable_b200 import engine, _lib
    dt = LB_TYPES[name]
    st = {"bool": _lib.BOOL, "int8": _lib.INT8, "int16": _lib.INT16, "int32": _lib.INT32, "int64": _lib.INT64,
          "float32": _lib.FLOAT32, "float64": _lib.FLOAT64}[name]
    rng = np.random.default_rng(len(name))
    if name == "bool":
        distinct = np.array([0, 1], dt)
    elif dt in (np.float32, np.float64):
        distinct = np.concatenate([[-np.inf, np.finfo(dt).min, -1.5, 0.0, 1e-30, 2.5, np.finfo(dt).max, np.inf],
                                   rng.standard_normal(40)]).astype(dt)
    else:
        info = np.iinfo(dt)
        distinct = np.concatenate([[info.min + 1, info.min + 2, -1, 0, 1, info.max - 1, info.max],
                                   rng.integers(info.min + 1, info.max, 40)]).astype(dt)
    distinct = np.unique(distinct)
    for n_runs in (0, 1, 2, len(distinct)):
        for run in (1, 3, 1000):
            pick = np.sort(rng.choice(len(distinct), n_runs, replace=False)) if n_runs else np.zeros(0, int)
            lengths = rng.integers(1, run + 1, n_runs)
            s = np.repeat(distinct[pick], lengths)
            if dt in (np.float32, np.float64):
                zeros = np.flatnonzero(s == 0)
                s[zeros[rng.random(len(zeros)) < 0.5]] = -0.0            # ±0.0 ties inside one run
            if name == "bool":
                probes = np.array([0, 1], dt)
            elif dt in (np.float32, np.float64):
                with np.errstate(over="ignore"):                         # next after ±max is ±inf
                    probes = np.concatenate([distinct, np.nextafter(distinct, dt(-np.inf)),
                                             np.nextafter(distinct, dt(np.inf)), np.array([0.0, -0.0], dt)]).astype(dt)
            else:
                probes = np.concatenate([distinct, distinct - 1, distinct + 1,
                                         np.array([np.iinfo(dt).min, np.iinfo(dt).max], dt)]).astype(dt)
            want = np.searchsorted(s, probes, side="left").astype(np.int64)
            sc = engine.Col(torch.from_numpy(s).cuda(), st)
            vc = engine.Col(torch.from_numpy(probes).cuda(), st)
            out = torch.full((len(probes),), -7, dtype=torch.int64, device="cuda")
            _lib.check(_lib.lib.dtb_lower_bound(sc.c(), sc.nrows, vc.c(), vc.nrows, engine._stream(),
                                                ctypes.c_void_p(out.data_ptr())))
            assert np.array_equal(out.cpu().numpy(), want), (name, n_runs, run)


# ---------------------------------------------------------------------------------------------------------------
# world 2 / world 3 on the real kernels
# ---------------------------------------------------------------------------------------------------------------
class _StagedGloo:
    """What dist.py calls of torch.distributed, on a gloo group: device tensors are copied to the host, the gloo
    collective runs there, and the result is copied back into the device tensor."""
    ReduceOp = dist.ReduceOp
    is_available = staticmethod(dist.is_available)
    is_initialized = staticmethod(dist.is_initialized)
    get_rank = staticmethod(dist.get_rank)
    get_world_size = staticmethod(dist.get_world_size)

    @staticmethod
    def all_gather_into_tensor(out, inp, group=None):
        h = out.cpu()
        dist.all_gather_into_tensor(h, inp.cpu(), group=group)
        out.copy_(h)

    @staticmethod
    def all_reduce(t, op=dist.ReduceOp.SUM, group=None):
        h = t.cpu()
        dist.all_reduce(h, op=op, group=group)
        t.copy_(h)

    @staticmethod
    def all_to_all_single(out, inp, output_split_sizes=None, input_split_sizes=None, group=None):
        h = out.cpu()
        dist.all_to_all_single(h, inp.cpu(), output_split_sizes, input_split_sizes, group=group)
        out.copy_(h)


def _run_case(ddist, c, rank):
    if c["kind"] == "groupby":
        k = torch.from_numpy(c["keys"][rank]).cuda()
        v = torch.from_numpy(c["vals"][rank]).cuda()
        mk, mv = ddist.groupby_partitioned(k, v, c["op"], exchange=c["exchange"], key_range=c.get("key_range"))
        return mk.cpu().numpy(), mv.cpu().numpy(), ddist.LAST_MERGE_LAUNCHES
    k = torch.from_numpy(c["keys"][rank]).cuda()
    sk, sid = ddist.sort_partitioned(k, c["row0"][rank])
    return sk.cpu().numpy(), sid.cpu().numpy()


def _worker(rank, world, port, backend, cases, q):
    try:
        os.environ["MASTER_ADDR"] = "127.0.0.1"
        os.environ["MASTER_PORT"] = str(port)
        torch.cuda.set_device(rank if torch.cuda.device_count() > 1 else 0)
        dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=180))
        from datatable_b200 import dist as ddist, _lib
        if backend == "gloo":
            ddist.dist = _StagedGloo
        out = []
        for c in cases:
            try:                                  # a refusal is raised on every rank at the same point
                out.append(_run_case(ddist, c, rank))
            except _lib.DtbError as e:
                out.append(("raise", type(e).__name__, str(e)))
        q.put((rank, out))
    except BaseException:
        q.put((rank, "worker failed:\n" + traceback.format_exc()))
    finally:
        if dist.is_initialized():
            dist.destroy_process_group()


def _spawn(world, backend, cases):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, cases, q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        res = {}
        for _ in range(world):
            rank, out = q.get(timeout=900)
            assert not isinstance(out, str), f"rank {rank}: {out}"
            res[rank] = out
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
        return [res[r] for r in range(world)]
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
            p.join(timeout=30)


# -- case generation ----------------------------------------------------------------------------------------------
KEY_DTYPES = ("int8", "int16", "int32", "int64", "bool", "float32", "float64")
I32_NA = np.iinfo(np.int32).min


def _is_key(k, key):
    """k's rows that hold the group key `key`: NaN is one group, -0.0 and +0.0 are two"""
    if k.dtype.kind != "f":
        return k == key
    if np.isnan(key):
        return np.isnan(k)
    return (k == key) & (np.signbit(k) == np.signbit(key))


def _na_key(dt):
    return np.nan if np.dtype(dt).kind == "f" else np.iinfo(dt).min


def _keys(name, n, rng):
    if name == "bool":
        return rng.integers(0, 2, n).astype(np.bool_)
    if name in ("float32", "float64"):
        k = (rng.integers(-200, 200, n) / 4).astype(name)
        k[rng.random(n) < 0.03] = -0.0
        k[rng.random(n) < 0.01] = np.inf
        k[rng.random(n) < 0.01] = -np.inf
        return k
    hi = {"int8": 100, "int16": 3000, "int32": 50_000, "int64": 50_000}[name]
    k = rng.integers(-hi, hi, n).astype(name)
    if name == "int64":
        k += np.int64(2**40)                                  # a wide kmin that still fits a dense table
    return k


def _values(kind, n, rng):
    if kind == "f64":                                         # multiples of 2^-8 in [-256, 256]: sums are exact
        v = rng.integers(-2**16, 2**16, n, endpoint=True) / 256.0
        v[rng.random(n) < 0.05] = np.nan
    elif kind == "rand":                                      # uniform random: sums are compared with fsum
        v = rng.uniform(-1e3, 1e3, n)
        v[rng.random(n) < 0.05] = np.nan
    else:
        v = rng.integers(-10**6, 10**6, n).astype(np.int32)
        v[rng.random(n) < 0.05] = I32_NA
    return v


OPS = ((SUM, "f64"), (SUM, "i32"), (COUNT, "f64"), (COUNTNA, "i32"), (NROWS, "f64"), (MIN, "i32"), (MAX, "f64"),
       (MIN, "f64"), (SUM, "rand"))


def _groupby_cases(world, rng, sizes, exchanges=("allreduce", "allgather", "alltoall")):
    cases = []
    for ex in exchanges:
        for kname in KEY_DTYPES:
            for na in (("none",) if kname == "bool" else ("none", "one", "all")):
                keys = [_keys(kname, n, rng) for n in sizes]
                if na != "none":
                    for r, k in enumerate(keys):
                        if len(k) and (na == "all" or r == world - 1):
                            k[rng.random(len(k)) < 0.05] = _na_key(k.dtype)
                plant = None if kname == "bool" else keys[0][0]         # a group whose values are all NA
                for op, vk in OPS:
                    vals = [_values(vk, len(k), rng) for k in keys]
                    if plant is not None:
                        for k, v in zip(keys, vals):
                            v[_is_key(k, plant)] = np.nan if v.dtype.kind == "f" else I32_NA
                    cases.append(dict(kind="groupby", exchange=ex, op=op, keys=keys, vals=vals,
                                      label=f"{ex} {kname} na={na} op={op}/{vk}", plant=plant))
    return cases


def _span_cases(world, rng):
    """Key spans on either side of the dense table's limit, and caller-given key ranges."""
    cases = []
    for kname, base in (("int32", -2**31 + 1), ("int32", 12345), ("int64", -2**62), ("int64", 2**62)):
        for span in (DENSE_MAX, DENSE_MAX + 1):
            keys = []
            for r in range(world):
                k = (base + rng.integers(0, span, 300 + 50 * r)).astype(kname)
                keys.append(k)
            keys[0][0], keys[-1][-1] = base, base + span - 1                 # the span is exact
            vals = [_values("f64", len(k), rng) for k in keys]
            cases.append(dict(kind="groupby", exchange="allreduce", op=SUM, keys=keys, vals=vals,
                              label=f"span {kname} {base} {span}", launches=5 if span <= DENSE_MAX else 8))
    for kname, lo, hi, rng_, ok in (("int32", 0, 999, (0, 999), True), ("int32", 0, 999, (-5, 2000), True),
                                    ("int8", -100, 99, (-128, 127), True), ("int16", -3000, 2999, (-3000, 2999), True),
                                    ("int64", 2**40, 2**40 + 999, (2**40, 2**40 + 999), True),
                                    ("int32", 0, 999, (0, 500), False), ("int32", 0, 999, (10, 5), False),
                                    ("int32", 0, 999, (2**40, 2**40 + 5), False)):
        keys = [rng.integers(lo, hi + 1, 400 + 77 * r).astype(kname) for r in range(world)]
        vals = [_values("f64", len(k), rng) for k in keys]
        cases.append(dict(kind="groupby", exchange="allreduce", op=COUNT, keys=keys, vals=vals, key_range=rng_,
                          label=f"key_range {kname} {rng_}", refuse=not ok, launches=5 if ok else None))
    k = [rng.integers(0, 50, 100).astype(np.int32) for _ in range(world)]
    cases.append(dict(kind="groupby", exchange="allgather", op=MEAN, keys=k, vals=[x.astype(np.float64) for x in k],
                      label="mean has no merge rule", refuse="DtbNotImplError"))
    return cases


def _sort_cases(world, rng, sizes, base=0):
    cases = []
    for kname in ("int8", "int16", "int32", "int64", "float32", "float64"):
        keys = []
        for n in sizes:
            if kname.startswith("float"):
                k = (rng.integers(-20, 20, n) / 2).astype(kname)         # ties across ranks
                for val, p in ((np.nan, 0.05), (-0.0, 0.05), (np.inf, 0.02), (-np.inf, 0.02)):
                    k[rng.random(n) < p] = val
            else:                                                        # ties across ranks, NA and the edges
                info = np.iinfo(kname)
                k = rng.integers(-50, 50, n).astype(kname)
                edge = rng.random(n) < 0.2
                k[edge] = rng.choice(np.array([info.min, info.min + 1, info.max], kname), int(edge.sum()))
            keys.append(k)
        row0 = list(base + np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64))
        cases.append(dict(kind="sort", keys=keys, row0=[int(x) for x in row0], base=base, label=f"sort {kname} base={base}"))
    return cases


# -- the reference ------------------------------------------------------------------------------------------------
def _isna(a):
    return np.isnan(a) if a.dtype.kind == "f" else a == np.iinfo(a.dtype).min


def _ref_groupby(c):
    from oracle import oracle as orc
    k, v = np.concatenate(c["keys"]), np.concatenate(c["vals"])
    o, f, ng = orc.group([k], [0], orc.NA_FIRST)
    gk = k[o[f[:-1]]]
    if gk.dtype == np.bool_:
        gk = gk.astype(np.int8)                               # the engine's bool column is int8 0 / 1
    vs, starts, rows = v[o], f[:-1], np.diff(f).astype(np.int64)
    na = _isna(vs)
    cnt = np.add.reduceat((~na).astype(np.int64), starts)
    op = c["op"]
    if op == COUNT:
        return gk, cnt
    if op == COUNTNA:
        return gk, rows - cnt
    if op == NROWS:
        return gk, rows
    if op == SUM:
        if vs.dtype.kind == "f":
            return gk, np.add.reduceat(np.where(na, 0.0, vs), starts)
        return gk, np.add.reduceat(np.where(na, 0, vs).astype(np.int64), starts)
    if vs.dtype.kind == "f":
        m = (np.fmin if op == MIN else np.fmax).reduceat(vs, starts)
    else:
        fill = np.iinfo(vs.dtype).max if op == MIN else np.iinfo(vs.dtype).min
        m = (np.minimum if op == MIN else np.maximum).reduceat(np.where(na, fill, vs), starts)
        m[cnt == 0] = np.iinfo(vs.dtype).min
    return gk, m.astype(vs.dtype)


def _check_fsum(c, gk, gv, wk, world):
    from oracle import oracle as orc
    k, v = np.concatenate(c["keys"]), np.concatenate(c["vals"])
    o, f, ng = orc.group([k], [0], orc.NA_FIRST)
    assert same(gk, wk) and gv.dtype == np.float64 and len(gv) == ng, c["label"]
    vs = np.where(np.isnan(v[o]), 0.0, v[o])
    for g in range(ng):
        x = vs[f[g]:f[g + 1]]
        want = math.fsum(x)
        tol = (len(x) + world) * 2.0**-52 * float(np.abs(x).sum())
        assert abs(gv[g] - want) <= tol, (c["label"], g, gv[g], want)


def _check(cases, results, world):
    from oracle import oracle as orc
    for i, c in enumerate(cases):
        outs = [results[r][i] for r in range(world)]
        lab = c["label"]
        if c.get("refuse"):
            want = c["refuse"] if isinstance(c["refuse"], str) else "DtbValueError"
            assert all(isinstance(o[0], str) and o[1] == want for o in outs), (lab, [o[:2] for o in outs])
            continue
        raised = [o for o in outs if isinstance(o[0], str)]
        assert not raised, (lab, raised)
        if c["kind"] == "sort":
            kcat = np.concatenate(c["keys"])
            want_o = orc.group([kcat], [orc.SORT_ONLY], orc.NA_FIRST)[0]
            got_k = np.concatenate([o[0] for o in outs])
            got_id = np.concatenate([o[1] for o in outs])
            assert got_id.dtype == np.int64, lab
            assert np.array_equal(got_id, want_o.astype(np.int64) + c["base"]), lab
            assert same(got_k, kcat[want_o]), lab
            continue
        wk, wv = _ref_groupby(c)
        if c["exchange"] == "alltoall":
            got = [(np.concatenate([o[0] for o in outs]), np.concatenate([o[1] for o in outs]))]
        else:                                                 # every rank holds the full result
            got = [(o[0], o[1]) for o in outs]
            launches = {o[2] for o in outs}
            assert len(launches) == 1, (lab, launches)        # every rank took the same path
            if c.get("launches") is not None:
                assert launches == {c["launches"]}, (lab, launches)
        for gk, gv in got:
            if c["op"] == SUM and c["vals"][0].dtype == np.float64 and "rand" in lab:
                _check_fsum(c, gk, gv, wk, world)
                continue
            assert same(gk, wk), (lab, gk[:8], wk[:8], len(gk), len(wk))
            assert same(gv, wv), (lab, gv[:8], wv[:8])
        plant = c.get("plant")
        if plant is not None:                                 # the all-NA group is there with count 0 / sum 0 / min NA
            gi = np.flatnonzero(_is_key(wk, plant))
            assert len(gi) == 1, lab
            if c["op"] in (COUNT, SUM) and "rand" not in lab:
                assert wv[gi[0]] == 0, lab
            if c["op"] in (MIN, MAX):
                assert _isna(wv[gi]).all(), lab


def _cases(world, rng, sizes):
    return _groupby_cases(world, rng, sizes) + _span_cases(world, rng) + _sort_cases(world, rng, sizes) + \
        _sort_cases(world, rng, sizes, base=2**31 + 7)


@pytest.mark.parametrize("world,sizes", [(2, (700, 1300)), (3, (900, 0, 611))])
def test_dist_gloo_staged(world, sizes):
    rng = np.random.default_rng(world)
    cases = _cases(world, rng, sizes)
    _check(cases, _spawn(world, "gloo", cases), world)


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2,
                    reason="NCCL needs one GPU per rank")
def test_dist_nccl():
    for world in sorted({2, min(3, torch.cuda.device_count())}):
        sizes = (700, 1300, 0)[:world]
        rng = np.random.default_rng(10 + world)
        cases = _cases(world, rng, sizes)
        _check(cases, _spawn(world, "nccl", cases), world)
