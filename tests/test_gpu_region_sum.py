"""The region sum: a fused SUM over spread-out group keys, added up per digit region of the first radix pass.

When a Groupby's fused reducers include a SUM and the group keys have at most 13 bits above the first pass's digit
(12 to 20 key bits), the first pass carries the value column to its output slots and every region of that pass is
folded in a shared-memory table instead of one L2 atomic per row.  These tests compare those sums with the exact
per-group sums (the bound of test_gpu_reducers_exact: float64 accumulation in any order; integers exact modulo
2^64) over value stypes, key widths, NA keys, descending keys, sizes around the tile and chunk sizes, skewed keys
and reducers beside the sum, and check from the engine's verbose lines, its profile records and last_call_stats()
which path ran.
"""
import re

import numpy as np
import pytest

from helpers import BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64
from test_gpu_reducers_exact import _STATS, check_reducer, hard_values

ALL_ST = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
NA_I32 = -2**31
_REGION = re.compile(r"\[dtb200\]   reducer (\d+): region sum")


@pytest.fixture(autouse=True)
def _clear_stats():
    yield
    _STATS.clear()


def run(capfd, keys, reducers, flags=0, na="first", bucketed=1):
    """Groupby(keys, reducers) on the device with options verbose and profile on.  Returns (the reduced columns,
    the oracle's order and offsets, the reducers that took the region sum, the kernel families, the call stats)."""
    import torch
    from datatable_b200 import engine, _lib
    from oracle import oracle as orc
    na_lib = _lib.NA_FIRST if na == "first" else _lib.NA_LAST
    kd = torch.from_numpy(keys).cuda()
    dev = {}                                                 # one device column per array: reducers of one column
    for _, v, st in reducers:
        dev.setdefault(id(v), engine.Col(torch.from_numpy(v).cuda(), st))
    specs = [(op, dev[id(v)]) for op, v, _ in reducers]
    capfd.readouterr()
    _lib.profile_records()
    engine.set_option("verbose", 1)
    engine.set_option("profile", 1)
    engine.set_option("bucketed_reducers", bucketed)
    try:
        gb = engine.Groupby([kd], [flags], na_lib, reducers=specs)
        stats = _lib.last_call_stats()
        torch.cuda.synchronize()
    finally:
        engine.set_option("verbose", 0)
        engine.set_option("profile", 0)
        engine.set_option("bucketed_reducers", 1)
    err = capfd.readouterr().err
    fams = [name for name, _ in _lib.profile_records()]
    try:
        got = [gb.reduced(i).cpu().numpy() for i in range(len(reducers))]
        ng = gb.ngroups
    finally:
        gb.close()
    order, offsets, want_ng = orc.group([keys], [flags], orc.NA_FIRST if na == "first" else orc.NA_LAST)
    assert ng == want_ng
    region = {int(m) for m in _REGION.findall(err)}
    return got, order, offsets, region, fams, stats


def check(got, reducers, order, offsets, ctx):
    names = {1: "sum", 2: "mean", 3: "min", 4: "max"}
    for g, (op, v, st) in zip(got, reducers):
        check_reducer(names[op], g, v, st, order, offsets, ctx)


def keys_of(rng, n, bits, na=None):
    """n int32 keys of `bits` significant bits after normalisation (an NA key takes one more value: its domain is
    one smaller), NA keys on every 101st row."""
    hi = (1 << bits) - (1 if na else 0)
    k = rng.integers(0, hi, n).astype(np.int32)
    if na:
        k[::101] = NA_I32
    k[1], k[2] = 0, hi - 1                                   # the whole domain: bits is exact
    return k


# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("st", ALL_ST)
def test_value_stypes(capfd, st):
    """C2's shape, 20-bit keys, every value stype with its hard values (cancellation, extremes, NA, inf, wraps)."""
    from datatable_b200 import _lib
    rng = np.random.default_rng(700 + st)
    n = 200_001
    k = keys_of(rng, n, 20)
    v = hard_values(rng, st, k)
    reducers = [(_lib.OP_SUM, v, st)]
    got, order, offsets, region, fams, stats = run(capfd, k, reducers)
    assert region == {0}
    assert "reduce_direct" in fams and "region_sum" in fams and "reduce" not in fams, fams   # bench.py: reduce_direct
    # the carried value column (and the 256 digit bases) is the scratch a count of the same column does not take
    _, _, _, region_c, fams_c, stats_c = run(capfd, k, [(_lib.OP_COUNT, v, st)])
    assert region_c == set() and "region_sum" not in fams_c
    assert stats["scratch_bytes"] - stats_c["scratch_bytes"] == n * v.dtype.itemsize + 1024
    check(got, reducers, order, offsets, f"region st={st}")


@pytest.mark.gpu
@pytest.mark.parametrize("bits,na,desc", [(12, None, False), (17, None, False), (20, None, False), (22, None, False),
                                          (20, "first", False), (20, "last", False), (20, None, True),
                                          (17, "last", True), (12, "first", True)])
@pytest.mark.parametrize("st", (INT64, FLOAT64))
def test_key_widths_na_and_descending(capfd, bits, na, desc, st):
    """12 to 20 key bits take the region sum (at most 13 bits above the first digit); 22 bits do not."""
    from datatable_b200 import _lib
    rng = np.random.default_rng(bits * 10 + (na == "last") + 2 * desc)
    n = 120_007
    k = keys_of(rng, n, bits, na)
    v = hard_values(rng, st, k)
    reducers = [(_lib.OP_SUM, v, st)]
    got, order, offsets, region, fams, _ = run(capfd, k, reducers, flags=_lib.FLAG_DESCENDING if desc else 0,
                                               na=na or "first")
    assert region == (set() if bits > 20 else {0})
    check(got, reducers, order, offsets, f"bits={bits} na={na} desc={desc}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4_999, 8_192 * 3 + 17, 65_536 + 1, 1_000_003])
def test_sizes(capfd, n):
    """n below one scatter tile, not a multiple of the tile, one row past a count chunk, and a million rows."""
    from datatable_b200 import _lib
    rng = np.random.default_rng(n)
    k = keys_of(rng, n, 12 if n < 10_000 else 17)
    v = hard_values(rng, FLOAT64, k)
    reducers = [(_lib.OP_SUM, v, FLOAT64)]
    got, order, offsets, region, _, _ = run(capfd, k, reducers)
    assert region == {0}
    check(got, reducers, order, offsets, f"n={n}")


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["half_one_key", "power_law", "sorted"])
@pytest.mark.parametrize("st", (INT32, FLOAT64))
def test_skewed_keys(capfd, shape, st):
    """One key owns half the rows and a power-law head (hot keys), and sorted keys (the rows of a region arrive in key
    order): the warps fold repeated keys before the shared-memory add."""
    from datatable_b200 import _lib
    rng = np.random.default_rng(31 + st)
    n = 400_009
    k = rng.integers(0, 1_000_000, n).astype(np.int32)
    if shape == "half_one_key":
        k[::2] = 7
    elif shape == "power_law":
        k = (rng.random(n) ** 8 * 1_000_000).astype(np.int32)
        k[-1] = 999_999
    else:
        k.sort()
    v = hard_values(rng, st, k)
    reducers = [(_lib.OP_SUM, v, st)]
    got, order, offsets, region, fams, _ = run(capfd, k, reducers)
    assert region == {0}
    # a hot key: the kernel that also folds the hot keys' lanes in the warp
    assert ("region_sum_hot" in fams) == (shape != "sorted") and ("region_sum" in fams) == (shape == "sorted"), fams
    check(got, reducers, order, offsets, shape)


@pytest.mark.gpu
def test_sum_beside_other_reducers(capfd):
    """A sum next to min on another column (region sum + direct path), next to mean / min / max on another column
    (that column is bucketed: no region sum), and two sums of one column (bucketed, and with the bucketed reducers
    off both take the region sum)."""
    from datatable_b200 import _lib
    rng = np.random.default_rng(5)
    n = 300_007
    k = keys_of(rng, n, 20)
    a, b = hard_values(rng, FLOAT64, k), hard_values(rng, INT32, k)
    S, MEAN, MIN, MAX = _lib.OP_SUM, _lib.OP_MEAN, _lib.OP_MIN, _lib.OP_MAX
    cases = [([(MIN, b, INT32), (S, a, FLOAT64)], 1, {1}),
             ([(S, a, FLOAT64), (MEAN, b, INT32), (MIN, b, INT32), (MAX, b, INT32)], 1, set()),
             ([(S, b, INT32), (S, b, INT32)], 1, set()),
             ([(S, b, INT32), (MIN, a, FLOAT64), (S, b, INT32)], 0, {0, 2})]
    for reducers, bucketed, want in cases:
        got, order, offsets, region, _, _ = run(capfd, k, reducers, bucketed=bucketed)
        assert region == want, (len(reducers), bucketed, region)
        check(got, reducers, order, offsets, f"{len(reducers)} reducers, bucketed={bucketed}")


@pytest.mark.gpu
def test_few_groups_and_piecewise_keep_their_paths(capfd):
    """Few groups in a wide key domain (known only after the sort) keep the shared-memory small-table path, and the
    piecewise reducers (dtb_groupby_reduce_begin / _add / _end) never see a carried column."""
    import torch
    from datatable_b200 import engine, _lib
    from oracle import oracle as orc
    rng = np.random.default_rng(11)
    n = 200_003
    k = (rng.integers(0, 1500, n) * 699).astype(np.int32)                # 1500 groups over 20 bits
    v = hard_values(rng, FLOAT64, k)
    reducers = [(_lib.OP_SUM, v, FLOAT64)]
    got, order, offsets, region, fams, _ = run(capfd, k, reducers)
    assert region == set() and "reduce_direct" in fams and not {"region_sum", "region_sum_hot"} & set(fams)
    check(got, reducers, order, offsets, "few groups")

    k = keys_of(rng, n, 20)
    v = hard_values(rng, FLOAT64, k)
    capfd.readouterr()
    engine.set_option("verbose", 1)
    try:
        gb = engine.Groupby([torch.from_numpy(k).cuda()], [0], _lib.NA_FIRST)
        vd = torch.from_numpy(v).cuda()
        pcs = [(vd[a:b], a, None) for a, b in ((0, 1), (1, n // 3), (n // 3, n))]
        got = gb.reduce_pieces(_lib.OP_SUM, FLOAT64, pcs)
    finally:
        engine.set_option("verbose", 0)
    try:
        err = capfd.readouterr().err
        assert "region_sum" not in err and "region sum" not in err
        order, offsets, _ = orc.group([k], [0], orc.NA_FIRST)
        check_reducer("sum", got, v, FLOAT64, order, offsets, "pieces")
    finally:
        gb.close()
