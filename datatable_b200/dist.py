"""
Row-partitioned groupby over several GPUs of one box (one process per GPU,
torch.distributed / NCCL over NVLink).  The reference is single-process
(SURVEY.md 8e); this is the "final NCCL reduce of per-group partials" leg of
the north star: every rank groups and reduces its own row partition with the
single-GPU kernels, the per-group partials (key, partial) are exchanged with
one NCCL all-gather, and the same group()/reduce() kernels merge them.  Sums,
counts, minima and maxima are associative, so the merged result equals the
single-GPU result on the concatenated rows (float sums up to association).

Exchanges built on the same kernels:

* `merge_partials_dense`     the partials are scattered into a dense table indexed by key - kmin, the
                             tables are all-reduced IN PLACE by NCCL (one ncclAllReduce of <= 32 MB over
                             NVLink) and compacted back: no re-sort, no re-group.  For SUM-like partials
                             over a key range of at most 2^22 (C2); anything else falls back to:
* `merge_partials`           all-gather of (key, partial) lists; every rank ends with the full result.
                             Moves 12-16 bytes per *group*; right when ngroups is small (C2).
* `merge_partials_alltoall`  key-range all-to-all of the partial lists: rank r ends with the r-th key
                             range of the result (nothing is replicated); right when ngroups is large (C5).
* `sort_partitioned`         global ordering of a row-partitioned key column: local sort, sample
                             splitters, NCCL all-to-all of (key, global row id) runs, local merge-sort.
                             Rank r ends with the r-th key range of the global RowIndex (int64 row ids,
                             the ARR64 case the reference cannot represent, SURVEY.md mismatch 3).
"""
import ctypes

import torch
import torch.distributed as dist

from . import _lib, engine

_MERGE_OP = {_lib.OP_SUM: _lib.OP_SUM, _lib.OP_MIN: _lib.OP_MIN, _lib.OP_MAX: _lib.OP_MAX,
             _lib.OP_COUNT: _lib.OP_SUM, _lib.OP_NROWS: _lib.OP_SUM, _lib.OP_COUNTNA: _lib.OP_SUM}


def _merge_op(op):
    """The reducer that merges partials of `op`; refused before any work when the partials of `op` do not merge."""
    if op not in _MERGE_OP:
        raise _lib.DtbNotImplError(f"reducer {op} has no merge rule across ranks (sum, count, countna, nrows, min, max)")
    return _MERGE_OP[op]


def _bytes(x):
    """The raw bytes of a 1-d tensor.  All-gathers and all-to-alls only move data; moving it as bytes lets every key
    dtype travel on every backend (neither NCCL nor gloo has an int16 type)."""
    return x.contiguous().view(torch.uint8)


def local_groupby(k, v, op):
    """(group keys, partials) of this rank's partition; k, v are CUDA tensors."""
    order, offsets, ng = engine.group([k], [0], _lib.NA_FIRST)
    part = engine.reduce(op, v, order, offsets)
    first = engine.gather(engine.Col(order, _lib.INT32), offsets[:-1])
    gkeys = engine.gather(k, first)
    return gkeys, part


def _dense_key_stype(dtype):
    st = {torch.int32: _lib.INT32, torch.int64: _lib.INT64}.get(dtype)
    if st is None:
        raise _lib.DtbNotImplError(f"dense merge: group keys must be int32 or int64, not {dtype}")
    return st


def _dense_scatter(gkeys, part, kmin, table, present):
    st = _dense_key_stype(gkeys.dtype)
    _lib.check(_lib.lib.dtb_dense_scatter(ctypes.c_void_p(gkeys.data_ptr()), st, ctypes.c_void_p(part.data_ptr()),
                                          gkeys.numel(), int(kmin), table.numel(), ctypes.c_void_p(table.data_ptr()),
                                          ctypes.c_void_p(present.data_ptr()), engine._stream()))


def _dense_compact(table, present, kmin, key_dtype):
    st = _dense_key_stype(key_dtype)
    size = table.numel()
    out_k = torch.empty(size, dtype=key_dtype, device=table.device)
    out_v = torch.empty(size, dtype=table.dtype, device=table.device)
    ng = ctypes.c_int64(0)
    _lib.check(_lib.lib.dtb_dense_compact(ctypes.c_void_p(table.data_ptr()), ctypes.c_void_p(present.data_ptr()), size,
                                          int(kmin), st, ctypes.c_void_p(out_k.data_ptr()),
                                          ctypes.c_void_p(out_v.data_ptr()), ctypes.byref(ng), engine._stream()))
    return out_k[:ng.value], out_v[:ng.value]


class _EngineKernels:
    """The product path: libdtb200.so kernels.  (tests/ swap in an oracle-backed object to run the
    exchange logic under gloo on CPU.)"""
    dense_scatter = staticmethod(_dense_scatter)
    dense_compact = staticmethod(_dense_compact)
    group = staticmethod(lambda keys: engine.group([keys], [0], _lib.NA_FIRST))
    sort = staticmethod(lambda keys: engine.group([keys], [_lib.FLAG_SORT_ONLY], _lib.NA_FIRST)[0])
    reduce = staticmethod(lambda op, v, order, offsets: engine.reduce(op, v, order, offsets))
    take = staticmethod(lambda src, idx: engine.gather(src, idx))


def merge_partials(gkeys, part, op, group=None, kernels=_EngineKernels):
    """All-gather every rank's (key, partial) list and merge equal keys with the engine's kernels."""
    mop = _merge_op(op)
    world = dist.get_world_size(group)
    if world == 1:
        return gkeys, part
    n_local = torch.tensor([gkeys.numel()], dtype=torch.int64, device=gkeys.device)
    sizes = torch.empty(world, dtype=torch.int64, device=gkeys.device)
    dist.all_gather_into_tensor(sizes, n_local, group=group)
    sizes_h = sizes.tolist()
    cap = max(sizes_h)
    kpad = torch.zeros(cap, dtype=gkeys.dtype, device=gkeys.device); kpad[:gkeys.numel()] = gkeys
    ppad = torch.zeros(cap, dtype=part.dtype, device=part.device); ppad[:part.numel()] = part
    kall = torch.empty(world * cap, dtype=gkeys.dtype, device=gkeys.device)
    pall = torch.empty(world * cap, dtype=part.dtype, device=part.device)
    dist.all_gather_into_tensor(_bytes(kall), _bytes(kpad), group=group)
    dist.all_gather_into_tensor(_bytes(pall), _bytes(ppad), group=group)
    if any(sz != cap for sz in sizes_h):
        keep = torch.cat([torch.arange(r * cap, r * cap + sizes_h[r], device=gkeys.device) for r in range(world)])
        kall, pall = kall[keep].contiguous(), pall[keep].contiguous()
    order, offsets, ng = kernels.group(kall)
    merged = kernels.reduce(mop, pall, order, offsets)
    first = kernels.take(order, offsets[:-1])
    return kernels.take(kall, first), merged


DENSE_MAX = 1 << 22            # entries of the dense per-key table (32 MB of float64 partials)
LAST_MERGE_LAUNCHES = 0        # engine kernels launched by the last merge on this rank (bench.py's count)
_SUM_LIKE = (_lib.OP_SUM, _lib.OP_COUNT, _lib.OP_COUNTNA, _lib.OP_NROWS)


def merge_partials_dense(gkeys, part, op, group=None, kernels=_EngineKernels, key_range=None):
    """Merge every rank's (ascending group keys, SUM-like partials) through dense per-key tables that
    NCCL all-reduces in place; every rank ends with the full (keys, merged partials) lists.

    key_range=(kmin, kmax): the caller's bound on the group keys of ALL ranks (e.g. a dictionary-coded
    column); without it one small all-reduce learns the global range (two scalars: the only extra host
    round trip).  The partial table and the presence table travel in ONE all-reduce (presence as 0/1 in
    the partials' dtype).  Falls back to `merge_partials` for MIN/MAX partials (NA partials do not
    all-reduce), for float keys and for key ranges beyond DENSE_MAX.  int8 / int16 / bool keys go through the
    tables as int32.  An empty or inverted key_range, or a key outside it, raises DtbValueError on every rank."""
    global LAST_MERGE_LAUNCHES
    _merge_op(op)
    if key_range is not None and int(key_range[1]) < int(key_range[0]):
        raise _lib.DtbValueError(f"key_range {tuple(key_range)} is empty")
    world = dist.get_world_size(group)
    if world == 1:
        LAST_MERGE_LAUNCHES = 0
        return gkeys, part
    dev = gkeys.device
    if gkeys.dtype.is_floating_point or op not in _SUM_LIKE or part.element_size() != 8:
        LAST_MERGE_LAUNCHES = 8      # decided from what every rank shares: no range collective
        return merge_partials(gkeys, part, op, group, kernels)
    keys = gkeys if gkeys.dtype in (torch.int32, torch.int64) else gkeys.to(torch.int32)
    if key_range is not None:
        kmin, hi = int(key_range[0]), int(key_range[1])
    else:
        big = torch.iinfo(torch.int64).max
        if keys.numel():
            # -(-2^63) wraps: clamp the int64 NA key first, so that it makes the span too large for a table
            rng = torch.stack([-keys[0].to(torch.int64).clamp_min(-big), keys[-1].to(torch.int64)])
        else:
            rng = torch.tensor([-big, -big], dtype=torch.int64, device=dev)
        dist.all_reduce(rng, op=dist.ReduceOp.MAX, group=group)
        neg_lo, hi = rng.tolist()
        kmin = -neg_lo
    span = hi - kmin + 1
    if span > DENSE_MAX or span <= 0:
        LAST_MERGE_LAUNCHES = 8
        return merge_partials(gkeys, part, op, group, kernels) if span > 0 else (gkeys, part)
    size = (span + 1023) // 1024 * 1024
    both = torch.zeros(2 * size + 1, dtype=part.dtype, device=dev)    # [partials | presence | keys out of range]
    table = both[:size]
    present = torch.zeros(size, dtype=torch.int32, device=dev)
    kernels.dense_scatter(keys, part, kmin, table, present)
    both[size:2 * size] = present                                     # 0 / 1 in the partials' dtype
    if key_range is not None:                                         # the scatter drops them: count them instead
        info = torch.iinfo(keys.dtype)
        if kmin > info.max or hi < info.min:
            both[2 * size] = keys.numel()
        else:
            both[2 * size] = ((keys < max(kmin, info.min)) | (keys > min(hi, info.max))).sum()
    dist.all_reduce(both, op=dist.ReduceOp.SUM, group=group)
    present = (both[size:2 * size] != 0).to(torch.int32)
    LAST_MERGE_LAUNCHES = 5          # scatter + block sums + scan + compact + emit
    mk, mv = kernels.dense_compact(table, present, kmin, keys.dtype)
    if key_range is not None and both[2 * size].item() != 0:          # dtb_dense_compact has synchronised
        raise _lib.DtbValueError(f"{int(both[2 * size].item())} group keys lie outside key_range {tuple(key_range)}")
    return (mk if mk.dtype == gkeys.dtype else mk.to(gkeys.dtype)), mv


def groupby_partitioned(k, v, op=_lib.OP_SUM, group=None, exchange="allgather", key_range=None):
    """DT[:, op(f.v), by(f.k)] over a frame row-partitioned across the ranks of `group`.
    exchange="allreduce": dense per-key tables all-reduced in place (every rank gets all groups);
    "allgather": every rank gets all groups; "alltoall": rank r gets the r-th key range.
    key_range: the caller's bound on the keys of all ranks, for exchange="allreduce" (see merge_partials_dense)."""
    _merge_op(op)
    gkeys, part = local_groupby(k, v, op)
    if dist.is_available() and dist.is_initialized():
        if exchange == "alltoall":
            return merge_partials_alltoall(gkeys, part, op, group)
        if exchange == "allreduce":
            return merge_partials_dense(gkeys, part, op, group, key_range=key_range)
        return merge_partials(gkeys, part, op, group)
    return gkeys, part


# ---------------------------------------------------------------------------
# key-range all-to-all
# ---------------------------------------------------------------------------
def _lower_bound(sorted_keys, values):
    """Rows of the ascending tensor `sorted_keys` below each value: the engine's own kernel (dtb_lower_bound)."""
    out = torch.empty(values.numel(), dtype=torch.int64, device=sorted_keys.device)
    s, v = engine.Col(sorted_keys), engine.Col(values.to(sorted_keys.dtype).contiguous())
    _lib.check(_lib.lib.dtb_lower_bound(s.c(), s.nrows, v.c(), v.nrows, engine._stream(), ctypes.c_void_p(out.data_ptr())))
    return out


def _splitters(sorted_keys, world, group=None):
    """world-1 global splitters from evenly spaced samples of every rank's sorted keys.  The <= 4*world^2
    samples are gathered and ordered on the host (plumbing, a few hundred values)."""
    n = sorted_keys.numel()
    nsamp = 4 * world
    if n > 0:
        pos = (torch.arange(nsamp, device=sorted_keys.device, dtype=torch.int64) * (n - 1)) // (nsamp - 1)
        samp = sorted_keys[pos]
    else:
        samp = torch.zeros(nsamp, dtype=sorted_keys.dtype, device=sorted_keys.device)
    have = torch.tensor([1 if n > 0 else 0], dtype=torch.int64, device=sorted_keys.device)
    allsamp = torch.empty(world * nsamp, dtype=sorted_keys.dtype, device=sorted_keys.device)
    allhave = torch.empty(world, dtype=torch.int64, device=sorted_keys.device)
    dist.all_gather_into_tensor(_bytes(allsamp), _bytes(samp), group=group)
    dist.all_gather_into_tensor(allhave, have, group=group)
    samp_h, have_h = allsamp.cpu().numpy(), allhave.cpu().numpy()
    pool = sorted(samp_h.reshape(world, nsamp)[have_h.astype(bool)].reshape(-1).tolist())
    if not pool:
        return torch.zeros(world - 1, dtype=sorted_keys.dtype, device=sorted_keys.device)
    spl = [pool[(r * len(pool)) // world] for r in range(1, world)]
    return torch.tensor(spl, dtype=sorted_keys.dtype, device=sorted_keys.device)


LAST_EXCHANGE_BYTES = 0        # bytes this rank sent in the last all-to-all (bench.py reports NVLink GB/s)
LAST_EXCHANGE_EVENTS = None    # (start, end) CUDA events around the payload all-to-alls of the last exchange


def _exchange(sorted_keys, payloads, world, group=None, kernels=None):
    """Cut the locally sorted run at the global splitters and all-to-all the pieces.
    Returns (received keys, received payloads): source-rank-major, each piece still sorted."""
    global LAST_EXCHANGE_BYTES, LAST_EXCHANGE_EVENTS
    spl = _splitters(sorted_keys, world, group)
    lb = getattr(kernels, "lower_bound", None) or _lower_bound
    cuts = lb(sorted_keys, spl)                                   # rows with key < splitter go left
    bounds = torch.cat([torch.zeros(1, dtype=cuts.dtype, device=cuts.device), cuts,
                        torch.tensor([sorted_keys.numel()], dtype=cuts.dtype, device=cuts.device)])
    send = (bounds[1:] - bounds[:-1]).to(torch.int64)
    recv = torch.empty_like(send)
    dist.all_to_all_single(recv, send, group=group)
    send_l, recv_l = send.tolist(), recv.tolist()
    nrecv = sum(recv_l)
    rank = dist.get_rank(group)
    LAST_EXCHANGE_BYTES = (sum(send_l) - send_l[rank]) * (sorted_keys.element_size() + sum(p.element_size() for p in payloads))

    def a2a(x):
        out = torch.empty(nrecv, dtype=x.dtype, device=x.device)
        esz = x.element_size()
        dist.all_to_all_single(_bytes(out), _bytes(x), output_split_sizes=[c * esz for c in recv_l],
                               input_split_sizes=[c * esz for c in send_l], group=group)
        return out
    timed = sorted_keys.is_cuda
    if timed:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    out = a2a(sorted_keys), [a2a(p) for p in payloads]
    if timed:
        e1.record()
        LAST_EXCHANGE_EVENTS = (e0, e1)
    return out


def merge_partials_alltoall(gkeys, part, op, group=None, kernels=_EngineKernels):
    """Key-range all-to-all of per-group partials; `gkeys` must be ascending (as group() returns them).
    Rank r ends with the groups whose keys fall into the r-th global key range.  Float keys travel as their
    order-preserving integer images: a bisection by `<` is not monotone over a NaN-first run, so the NaN group
    could otherwise be cut to different sides on different ranks."""
    mop = _merge_op(op)
    world = dist.get_world_size(group)
    if world == 1:
        return gkeys, part
    if gkeys.dtype.is_floating_point:
        ik, mv = merge_partials_alltoall(_float_image(gkeys), part, op, group, kernels)
        return _float_unimage(ik, gkeys.dtype), mv
    rk, (rp,) = _exchange(gkeys, [part], world, group, kernels)
    if rk.numel() == 0:
        return rk, rp
    order, offsets, ng = kernels.group(rk)
    merged = kernels.reduce(mop, rp, order, offsets)
    first = kernels.take(order, offsets[:-1])
    return kernels.take(rk, first), merged


def _float_image(k):
    """Order-preserving signed-integer image of a float column: NaN (NA) first, -0.0 < +0.0 -- the order of the
    reference's float sort (sort.cc:778-845).  Elementwise plumbing; the sorting runs on the image."""
    it = torch.int64 if k.dtype == torch.float64 else torch.int32
    b = k.view(it)
    flip = torch.iinfo(it).max
    img = torch.where(b < 0, b ^ flip, b)
    return torch.where(torch.isnan(k), torch.full_like(img, torch.iinfo(it).min), img)


def _float_unimage(img, dtype):
    flip = torch.iinfo(img.dtype).max
    b = torch.where(img < 0, img ^ flip, img)
    out = b.view(dtype).clone()
    out[img == torch.iinfo(img.dtype).min] = float("nan")
    return out


def sort_partitioned(k, row_offset, group=None, kernels=_EngineKernels):
    """Global stable ordering of an integer or float key column row-partitioned over the ranks
    (rank r holds global rows [row_offset, row_offset + len(k))).

    Returns (keys, row_ids): this rank's slice of the globally sorted sequence -- rank 0 holds the
    smallest keys (NA / NaN first) -- with int64 GLOBAL row ids; concatenated over ranks this is the ARR64
    RowIndex.  Ties keep ascending global row id (local sorts are stable, the exchange is source-rank-major).
    Float keys travel as their order-preserving integer images."""
    if k.dtype.is_floating_point:
        ks, ids = sort_partitioned(_float_image(k), row_offset, group, kernels)
        return _float_unimage(ks, k.dtype), ids
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    order = kernels.sort(k)
    ks = kernels.take(k, order)
    ids = order.to(torch.int64) + int(row_offset)
    if world == 1:
        return ks, ids
    rk, (rid,) = _exchange(ks, [ids], world, group, kernels)
    if rk.numel() == 0:
        return rk, rid
    order2 = kernels.sort(rk)
    return kernels.take(rk, order2), kernels.take(rid, order2)
