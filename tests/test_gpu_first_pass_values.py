"""The radix passes that carry something besides keys and row ids.

A region sum's first pass carries the value column to its output slots.  These tests compare its sums with the exact
per-group sums (the bound of test_gpu_reducers_exact) for every value stype, for a value column that starts one
element into its buffer (not 16-byte aligned), and for n around a multiple of the 8192-row scatter tile.

A count-table last pass runs on 4096-row tiles.  Its RowIndex and offsets are compared bit for bit with ref_group at
sizes that are not a multiple of the tile, with keys whose low-bit regions start inside tiles.

Which path ran is read from the engine's verbose lines.
"""
import re

import numpy as np
import pytest

from helpers import BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64
from test_gpu_reducers_exact import _STATS, check_reducer, hard_values
from test_gpu_group_plan import FIRST, LAST, parse_plan, ref_group, to_np

ALL_ST = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
_REGION = re.compile(r"\[dtb200\]   reducer (\d+): region sum")
_LOW_BITS = re.compile(r"\[dtb200\]   round \d+: .* low_bits=(\d+)")


@pytest.fixture(autouse=True)
def _clear_stats():
    yield
    _STATS.clear()


def region_sum(capfd, k, v, st, offset=0):
    """sum(v) by(k) through a Groupby with the value column on the device starting `offset` elements into its
    buffer.  Returns the sums, whether the region sum ran, and the oracle's order and offsets."""
    import torch
    from datatable_b200 import engine, _lib
    from oracle import oracle as orc
    buf = torch.from_numpy(np.concatenate([np.zeros(offset, v.dtype), v])).cuda()
    col = engine.Col(buf[offset:], st)
    assert (col.ptr % 16 != 0) == (offset * v.dtype.itemsize % 16 != 0)
    capfd.readouterr()
    engine.set_option("verbose", 1)
    try:
        gb = engine.Groupby([torch.from_numpy(k).cuda()], [0], _lib.NA_FIRST, reducers=[(_lib.OP_SUM, col)])
        torch.cuda.synchronize()
    finally:
        engine.set_option("verbose", 0)
    err = capfd.readouterr().err
    try:
        got = gb.reduced(0).cpu().numpy()
    finally:
        gb.close()
    order, offsets, _ = orc.group([k], [0], orc.NA_FIRST)
    return got, {int(m) for m in _REGION.findall(err)} == {0}, order, offsets


def keys20(rng, n):
    k = rng.integers(0, 1 << 20, n).astype(np.int32)
    k[1], k[2] = 0, (1 << 20) - 1                                  # 20 key bits: the 7/7/6 plan
    return k


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("st", ALL_ST)
def test_region_sum_value_stypes(capfd, st, offset):
    """Every value stype, from an aligned column and from a view one element in."""
    rng = np.random.default_rng(900 + 10 * st + offset)
    n = 8192 * 20 + 4096
    k = keys20(rng, n)
    v = hard_values(rng, st, k)
    got, region, order, offsets = region_sum(capfd, k, v, st, offset)
    assert region
    check_reducer("sum", got, v, st, order, offsets, f"st={st} offset={offset}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [8192 * 13 - 1, 8192 * 13, 8192 * 13 + 1])
@pytest.mark.parametrize("st", (INT32, FLOAT64))
def test_region_sum_sizes_around_the_tile(capfd, n, st):
    """The last tile one row short, whole, and one row long."""
    rng = np.random.default_rng(n + st)
    k = keys20(rng, n)
    v = hard_values(rng, st, k)
    got, region, order, offsets = region_sum(capfd, k, v, st)
    assert region
    check_reducer("sum", got, v, st, order, offsets, f"n={n} st={st}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4096 * 50 + 1, 4096 * 77 + 2049, 300_007])
@pytest.mark.parametrize("shape", ["uniform", "clustered"])
def test_count_table_last_pass_tiles(capfd, n, shape):
    """A Groupby on device keys of 20 bits: three passes, the last one counting rows per group key with the low 14
    bits recovered from the rows' slots.  Clustered keys leave few distinct low-bit values, so many 4096-row tiles
    of the last pass straddle a low-bit boundary."""
    import torch
    from datatable_b200 import engine
    rng = np.random.default_rng(n)
    if shape == "uniform":
        k = keys20(rng, n)
    else:
        k = (rng.integers(0, 64, n) * 16411 + rng.integers(0, 3, n)).astype(np.int32)
        k[1], k[2] = 0, (1 << 20) - 1
    k[::97] = -2**31                                               # NA keys: one more value in the domain
    for na_pos in (FIRST, LAST):
        want = ref_group([k], [INT32], [0], na_pos)
        capfd.readouterr()
        engine.set_option("verbose", 1)
        try:
            g = engine.Groupby([engine.Col(torch.from_numpy(k).cuda(), INT32)], [0], na_pos)
        finally:
            engine.set_option("verbose", 0)
        err = capfd.readouterr().err
        try:
            p = parse_plan(err)
            assert p["nrounds"] == 1 and p["rounds"][0]["count_table"] == 1 and p["rounds"][0]["passes"] == 3, p
            assert [int(b) for b in _LOW_BITS.findall(err)] == [14], err
            assert g.ngroups == want[2]
            assert np.array_equal(to_np(g.order()), want[0]), f"n={n} {shape}: RowIndex"
            assert np.array_equal(to_np(g.offsets()), want[1]), f"n={n} {shape}: offsets"
        finally:
            g.close()
