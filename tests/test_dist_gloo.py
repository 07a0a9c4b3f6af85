"""CPU: the N>1 exchange logic of datatable_b200.dist under gloo with world_size 2.
The GPU kernels are replaced by the oracle here (tests may use the oracle as a checker/stand-in);
what is exercised is the host side: size exchange, padding, all-gather, un-padding, merge order."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


class OracleKernels:
    @staticmethod
    def group(keys):
        from oracle import oracle as orc
        o, f, ng = orc.group([keys.numpy()], [0], orc.NA_FIRST)
        return torch.from_numpy(o), torch.from_numpy(f), ng

    @staticmethod
    def sort(keys):
        from oracle import oracle as orc
        return torch.from_numpy(orc.group([keys.numpy()], [orc.SORT_ONLY], orc.NA_FIRST)[0])

    @staticmethod
    def reduce(op, v, order, offsets):
        from oracle import oracle as orc
        return torch.from_numpy(orc.reduce(op, v.numpy(), order.numpy(), offsets.numpy()))

    @staticmethod
    def take(src, idx):
        return src[idx.long()]

    @staticmethod
    def lower_bound(sorted_keys, values):
        # lower_bound_kernel's own bisection (dtb_next.cu), not np.searchsorted: on a run that is not ascending under
        # `<` (NaN first) the two differ, and the exchange must not depend on which one runs
        s = sorted_keys.tolist()
        out = []
        for x in values.tolist():
            lo, hi = 0, len(s)
            while lo < hi:
                mid = (lo + hi) >> 1
                if s[mid] < x:
                    lo = mid + 1
                else:
                    hi = mid
            out.append(lo)
        return torch.tensor(out, dtype=torch.int64)

    # numpy stand-ins of dtb_dense_scatter / dtb_dense_compact (include/dtb200.h)
    @staticmethod
    def dense_scatter(gkeys, part, kmin, table, present):
        x = gkeys.long() - kmin
        keep = (x >= 0) & (x < table.numel())          # the kernel skips a key outside the table
        table[x[keep]] = part[keep]
        present[x[keep]] = 1

    @staticmethod
    def dense_compact(table, present, kmin, key_dtype):
        x = torch.nonzero(present).flatten()
        return (x + kmin).to(key_dtype), table[x]


def _worker(rank, world, port, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from datatable_b200 import dist as ddist, _lib
        from oracle import oracle as orc
        rng = np.random.default_rng(100 + rank)
        n = 5000 + 777 * rank                      # ragged partitions -> different group counts per rank
        k = rng.integers(0, 300 + 50 * rank, n).astype(np.int32)
        v = rng.random(n)
        o, f, ng = orc.group([k], [0], orc.NA_FIRST)
        part = orc.reduce(orc.SUM, v, o, f)
        gkeys = k[o[f[:-1]]]
        mk, mv = ddist.merge_partials(torch.from_numpy(gkeys), torch.from_numpy(part), _lib.OP_SUM,
                                      kernels=OracleKernels)
        dk, dv = ddist.merge_partials_dense(torch.from_numpy(gkeys), torch.from_numpy(part), _lib.OP_SUM,
                                            kernels=OracleKernels)
        rk, rv = ddist.merge_partials_dense(torch.from_numpy(gkeys), torch.from_numpy(part), _lib.OP_SUM,
                                            kernels=OracleKernels, key_range=(0, 399))   # caller-known key range: no range collective
        assert torch.equal(rk, dk) and torch.allclose(rv, dv, rtol=1e-12)
        # MIN partials do not all-reduce: the dense entry point must fall back to the all-gather merge
        pmin = orc.reduce(orc.MIN, v, o, f)
        nk, nv = ddist.merge_partials_dense(torch.from_numpy(gkeys), torch.from_numpy(pmin), _lib.OP_MIN,
                                            kernels=OracleKernels)
        ak, av = ddist.merge_partials_alltoall(torch.from_numpy(gkeys), torch.from_numpy(part), _lib.OP_SUM,
                                               kernels=OracleKernels)
        k64 = rng.integers(-10**12, 10**12, n).astype(np.int64)
        k64[::9] = k64[0]                             # ties across ranks: stability must hold globally
        row0 = 0 if rank == 0 else 5000
        sk, sid = ddist.sort_partitioned(torch.from_numpy(k64), row0, kernels=OracleKernels)
        kf = rng.standard_normal(n); kf[::7] = np.nan; kf[::11] = -0.0; kf[1::11] = 0.0; kf[5] = np.inf; kf[6] = -np.inf
        fk, fid = ddist.sort_partitioned(torch.from_numpy(kf), row0, kernels=OracleKernels)
        q.put((rank, k, v, mk.numpy(), mv.numpy(), ak.numpy(), av.numpy(), k64, sk.numpy(), sid.numpy(),
               dk.numpy(), dv.numpy(), nk.numpy(), nv.numpy(), kf, fk.numpy(), fid.numpy()))
    finally:
        dist.destroy_process_group()


def _run_world2(worker):
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=worker, args=(r, 2, port, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = [q.get(timeout=120) for _ in range(2)]
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
            p.join(timeout=10)
    return sorted(res, key=lambda t: t[0])


I64_NA = np.iinfo(np.int64).min


def _na_worker(rank, world, port, q):
    """Group keys that hold the int64 NA or NaN, through the dense and the all-to-all merge."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from datatable_b200 import dist as ddist, _lib
        out = {}

        def t(a, dt):
            return torch.tensor(a, dtype=dt)
        # int64 NA on rank 0 only, then on every rank
        k = [[I64_NA, 0, 1, 2], [5, 6, 7]][rank]
        p = [[1.0, 2.0, 3.0, 4.0], [10.0, 20.0, 30.0]][rank]
        out["na_one"] = ddist.merge_partials_dense(t(k, torch.int64), t(p, torch.float64), _lib.OP_SUM,
                                                   kernels=OracleKernels)
        k = [[I64_NA, 0, 1], [I64_NA, 1, 9]][rank]
        p = [[1.0, 2.0, 3.0], [10.0, 20.0, 30.0]][rank]
        out["na_all"] = ddist.merge_partials_dense(t(k, torch.int64), t(p, torch.float64), _lib.OP_SUM,
                                                   kernels=OracleKernels)
        # float keys with NaN through the all-to-all: the NaN group must come out once, first
        k = [[np.nan, 1.0, 2.0, 3.0], [np.nan, 0.1, 0.2, 0.3, 1.0]][rank]
        p = [[1.0, 2.0, 3.0, 4.0], [10.0, 20.0, 30.0, 40.0, 50.0]][rank]
        out["nan_a2a"] = ddist.merge_partials_alltoall(t(k, torch.float64), t(p, torch.float64), _lib.OP_SUM,
                                                       kernels=OracleKernels)
        # a key outside the caller's key_range is refused on every rank rather than dropped
        k = [[0, 1, 2], [3, 4, 12]][rank]
        try:
            ddist.merge_partials_dense(t(k, torch.int32), t([1.0, 2.0, 3.0], torch.float64), _lib.OP_SUM,
                                       kernels=OracleKernels, key_range=(0, 9))
            out["outside"] = None
        except _lib.DtbValueError as e:
            out["outside"] = str(e)
        out = {name: v if isinstance(v, (str, type(None))) else (v[0].numpy(), v[1].numpy()) for name, v in out.items()}
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


def test_merge_partials_na_keys_world2():
    res = _run_world2(_na_worker)
    want_one = (np.array([I64_NA, 0, 1, 2, 5, 6, 7]), np.array([1.0, 2, 3, 4, 10, 20, 30]))
    want_all = (np.array([I64_NA, 0, 1, 9]), np.array([11.0, 2, 23, 30]))
    for rank, out in res:                            # every rank holds every group, NA included
        for name, (wk, wv) in (("na_one", want_one), ("na_all", want_all)):
            gk, gv = out[name]
            assert np.array_equal(gk, wk) and np.array_equal(gv, wv), (rank, name, gk, gv)
        assert out["outside"] is not None and "outside key_range" in out["outside"], (rank, out["outside"])
    gk = np.concatenate([out["nan_a2a"][0] for _, out in res])
    gv = np.concatenate([out["nan_a2a"][1] for _, out in res])
    assert np.isnan(gk[0]) and not np.isnan(gk[1:]).any(), gk
    assert np.array_equal(gk[1:], [0.1, 0.2, 0.3, 1.0, 2.0, 3.0]) and np.array_equal(gv, [11.0, 20, 30, 40, 52, 3, 4])


def test_merge_refusals_without_collectives():
    """An op without a merge rule and an empty key_range are refused before any local work or collective."""
    from datatable_b200 import dist as ddist, _lib
    k, p = torch.tensor([1, 2], dtype=torch.int32), torch.tensor([1.0, 2.0], dtype=torch.float64)
    for fn in (ddist.merge_partials, ddist.merge_partials_dense, ddist.merge_partials_alltoall):
        with pytest.raises(_lib.DtbNotImplError, match="no merge rule"):
            fn(k, p, _lib.OP_MEAN, kernels=OracleKernels)
    with pytest.raises(_lib.DtbNotImplError, match="no merge rule"):
        ddist.groupby_partitioned(k, p, _lib.OP_MEAN)
    with pytest.raises(_lib.DtbValueError, match="empty"):
        ddist.merge_partials_dense(k, p, _lib.OP_SUM, kernels=OracleKernels, key_range=(5, 4))


def test_merge_partials_world2():
    res = _run_world2(_worker)
    kall = np.concatenate([r[1] for r in res]); vall = np.concatenate([r[2] for r in res])
    uk = np.unique(kall)
    want = np.array([vall[kall == x].sum() for x in uk])
    for r in res:                                   # every rank holds the full merged result
        assert np.array_equal(r[3], uk)
        assert np.allclose(r[4], want, rtol=1e-12)
    wmin = np.array([vall[kall == x].min() for x in uk])
    for r in res:                                   # dense all-reduce merge == all-gather merge; MIN falls back
        assert np.array_equal(r[10], uk) and r[10].dtype == np.int32
        assert np.allclose(r[11], want, rtol=1e-12)
        assert np.array_equal(r[12], uk) and np.array_equal(r[13], wmin)
    # all-to-all variant: the ranks hold disjoint ascending key ranges that concatenate to the result
    ak = np.concatenate([r[5] for r in res]); av = np.concatenate([r[6] for r in res])
    assert np.array_equal(ak, uk) and np.allclose(av, want, rtol=1e-12)
    assert len(res[0][5]) > 0 and len(res[1][5]) > 0
    # distributed sort: concatenated slices == stable argsort of the concatenated column (global row ids)
    kcat = np.concatenate([r[7] for r in res])
    want_ids = np.argsort(kcat, kind="stable")
    got_ids = np.concatenate([r[9] for r in res]); got_keys = np.concatenate([r[8] for r in res])
    assert got_ids.dtype == np.int64
    assert np.array_equal(got_ids, want_ids) and np.array_equal(got_keys, kcat[want_ids])
    # float keys: NaN first, -inf, ..., -0.0 < +0.0, ..., +inf; ties by global row id (the oracle's float order)
    from oracle import oracle as orc
    fcat = np.concatenate([r[14] for r in res])
    want_f, _, _ = orc.group([fcat], [4], 1)                      # SORT_ONLY, NA first
    got_fid = np.concatenate([r[16] for r in res]); got_fk = np.concatenate([r[15] for r in res])
    assert np.array_equal(got_fid, want_f.astype(np.int64))
    assert np.array_equal(got_fk.view(np.int64)[~np.isnan(got_fk)], fcat[want_f].view(np.int64)[~np.isnan(fcat[want_f])])
    assert np.isnan(got_fk[:np.isnan(fcat).sum()]).all()
