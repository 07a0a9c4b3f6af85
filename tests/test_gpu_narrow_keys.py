"""Narrowed keys between radix passes, against the independent reference of test_gpu_group_plan.

Every pass but the last writes only the key bits later passes read, in the narrowest of 1 / 2 / 4 / 8 bytes, unless
the last pass writes the sorted keys; the last pass of a count table recovers the low bits the earlier passes
consumed from the rows' slots (at most 3 passes and 16 recovered bits, else the keys keep their width).  Every case
checks the RowIndex and Groupby bit for bit and the key bytes every pass reads and writes, from the verbose plan.
"""
import re

import numpy as np
import pytest

from test_gpu_group_plan import (INT32, INT64, FLOAT64, DESCENDING, SORT_ONLY, FIRST, LAST, NA_INT, ref_group,
                                 dev, to_np, assert_group_equal, plan, radix_bits, Plan)  # noqa: F401 (fixtures)

_WIDTHS = re.compile(r"\[dtb200\]   round \d+: .* count_table=(\d) key_bytes=([\d:,]+) low_bits=(\d+)")


def plan_passes(total, width):
    np_ = max(1, -(-total // width))
    base, extra, sh, out = total // np_, total % np_, 0, []
    for p in range(np_):
        b = max(1, base + (1 if p < extra else 0))
        out.append((sh, b))
        sh += b
    return out


def expect_widths(total, width, want_sorted, count_table):
    """(key bytes read:written per pass, low_bits) as plan_group sets them for a single-round plan."""
    kb = 4 if total <= 32 else 8
    pp = plan_passes(total, width)
    if kb == 8 and not want_sorted and not count_table and width == 8 and total > 32:
        lo, hi = plan_passes(total - 32, 8), plan_passes(32, 8)
        if len(lo) + len(hi) <= len(pp):
            pp = lo + [(total - 32 + s, b) for s, b in hi]
    n = len(pp)
    low = pp[-1][0] if count_table and n > 1 else 0
    narrow = not want_sorted and not (count_table and (n > 3 or low > 16))
    kin, kout = [], []
    for p, (s, b) in enumerate(pp):
        left = total - s - b
        kin.append(kb if p == 0 else kout[-1])
        if p == n - 1:
            kout.append(kb if want_sorted else 0)
        else:
            kout.append(kb if not narrow else 1 if left <= 8 else 2 if left <= 16 else 4 if left <= 32 else 8)
    return ",".join(f"{a}:{b}" for a, b in zip(kin, kout)), (low if narrow else 0)


def widths_of(err):
    m = _WIDTHS.findall(err[err.rfind("[dtb200] group:"):])
    assert len(m) == 1, err[-2000:]
    return int(m[0][0]), m[0][1], int(m[0][2])


class WPlan(Plan):
    def __call__(self, fn):
        from datatable_b200 import engine
        self.capfd.readouterr()
        engine.set_option("verbose", 1)
        try:
            out = fn()
        finally:
            engine.set_option("verbose", 0)
        err = self.capfd.readouterr().err
        self.ct, self.widths, self.low = widths_of(err)
        self.bits = int(re.findall(r"\[dtb200\] group: n=\d+ keys=\d+ bits=(\d+)", err)[-1])
        return out


WIDTHS = (8, 7, 5, 4)
KEY_BITS = range(5, 23)
BY_SORT = ((10, 14), (6, 10), (12, 8), (20, 2))


def check_all_paths(wp, cols, sts, flags, na_pos, width, ctx):
    """The count-table handle, engine.group (sorted keys written) and the sort-only call, each bit for bit, each
    with the key widths its plan implies."""
    from datatable_b200 import engine
    d = dev(cols, sts)
    want = ref_group(cols, sts, flags, na_pos)
    g = wp(lambda: engine.Groupby(d, flags, na_pos))
    assert wp.ct == 1, ctx
    assert (wp.widths, wp.low) == expect_widths(wp.bits, width, False, True), (ctx, wp.widths, wp.low)
    assert g.ngroups == want[2], ctx
    assert np.array_equal(to_np(g.order()), want[0]), f"{ctx}: handle RowIndex"
    assert np.array_equal(to_np(g.offsets()), want[1]), f"{ctx}: handle offsets"
    g.close()
    got = wp(lambda: engine.group(d, flags, na_pos))
    assert (wp.widths, wp.low) == expect_widths(wp.bits, width, True, False), (ctx, wp.widths)
    assert_group_equal(got, want, f"{ctx}: engine.group")
    so = [f | SORT_ONLY for f in flags]
    want = ref_group(cols, sts, so, na_pos)
    got = wp(lambda: engine.group(d, so, na_pos))
    assert (wp.widths, wp.low) == expect_widths(wp.bits, width, False, False), (ctx, wp.widths)
    assert_group_equal(got, want, f"{ctx}: sort only")


@pytest.fixture
def wplan(capfd):
    return WPlan(capfd)


def span_keys(rng, n, bits, na, shift=0):
    """int32 keys of exactly `bits` key bits (the NA slot counts), their low `shift` bits constant."""
    span = 2**bits - (2 if na else 1)
    c = (rng.integers(0, span, n, endpoint=True) << shift) - 1000
    c[:2] = [-1000, (span << shift) - 1000]
    if na:
        m = rng.random(n) < 0.03
        m[:2] = False
        c[m] = NA_INT[INT32]
    return c.astype(np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("width", WIDTHS)
@pytest.mark.parametrize("n", [1000, 70_001, 300_001])
def test_key_bits_5_to_22(wplan, radix_bits, width, n):
    """5- to 22-bit keys: the count table recovers every number of low bits it can (3 to 15 here, 16 below), and
    the plans of more than 3 passes fall back to full-width keys.  Fewer rows than a tile, a partial last tile, and
    several chunks; the small row counts put many region boundaries in one tile."""
    radix_bits(width)
    rng = np.random.default_rng(n * 10 + width)
    for bits in KEY_BITS:
        for na, na_pos, desc in ((False, FIRST, False), (True, FIRST, True), (True, LAST, False)):
            k = span_keys(rng, n, bits, na)
            check_all_paths(wplan, [k], [INT32], [DESCENDING if desc else 0], na_pos, width,
                            f"bits={bits} w={width} n={n} na={na} desc={desc}")


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [12, 17, 20])
def test_constant_low_bits(wplan, bits):
    """Keys whose low 3 bits never vary: they are dropped, so the first pass counts with the count kernel instead
    of folding the statistics histogram."""
    rng = np.random.default_rng(bits)
    for n in (4096 * 3, 200_003):
        k = span_keys(rng, n, bits, True, shift=3)
        check_all_paths(wplan, [k], [INT32], [0], LAST, 8, f"cshift bits={bits} n={n}")


@pytest.mark.gpu
@pytest.mark.parametrize("by_bits,sort_bits", BY_SORT)
def test_by_and_sort(wplan, by_bits, sort_bits):
    """by() + sort(): the group key is the composite above group_shift; up to 24 composite bits, 16 recovered."""
    from datatable_b200 import engine
    rng = np.random.default_rng(by_bits * 100 + sort_bits)
    for n in (3000, 250_001):
        k = span_keys(rng, n, by_bits, True)
        s = span_keys(rng, n, sort_bits, False)
        flags = [0, SORT_ONLY | DESCENDING]
        want = ref_group([k, s], [INT32, INT32], flags, FIRST)
        d = dev([k, s], [INT32, INT32])
        g = wplan(lambda: engine.Groupby(d, flags, FIRST))
        assert wplan.ct == 1 and wplan.bits == by_bits + sort_bits
        assert (wplan.widths, wplan.low) == expect_widths(wplan.bits, 8, False, True), (wplan.widths, wplan.low)
        assert g.ngroups == want[2]
        assert np.array_equal(to_np(g.order()), want[0]), f"by {by_bits} sort {sort_bits} n={n}: RowIndex"
        assert np.array_equal(to_np(g.offsets()), want[1]), f"by {by_bits} sort {sort_bits} n={n}: offsets"
        g.close()


def test_every_low_bits_value_reached():
    """The count-table cases above recover every number of low bits from 3 (the least with digits of at least 4
    bits) to 16, and some of their plans fall back to full-width keys."""
    lows = {expect_widths(b, w, False, True)[1] for w in WIDTHS for b in KEY_BITS}
    lows |= {expect_widths(b + s, 8, False, True)[1] for b, s in BY_SORT}
    assert set(range(3, 17)) <= lows, sorted(lows)
    assert any(len(plan_passes(b, w)) > 3 for w in WIDTHS for b in KEY_BITS)


@pytest.mark.gpu
@pytest.mark.parametrize("span_bits", [40, 64])
def test_sort_only_64bit(wplan, span_bits):
    """64-bit sort-only keys: each pass writes the bits left, 8 -> 4 -> 2 -> 1 bytes down the chain."""
    from datatable_b200 import engine
    rng = np.random.default_rng(span_bits)
    n = 70_001
    if span_bits == 64:
        k = rng.integers(-2**63 + 1, 2**63 - 1, n, dtype=np.int64, endpoint=True)
        k[:2] = [-2**63 + 1, 2**63 - 1]
        k[rng.random(n) < 0.02] = NA_INT[INT64]
    else:
        k = rng.integers(0, 2**40 - 2, n, endpoint=True).astype(np.int64) - 2**35
        k[:2] = [-2**35, 2**40 - 2 - 2**35]
        k[rng.random(n) < 0.02] = NA_INT[INT64]
    x = rng.standard_normal(n)
    x[::997] = np.nan
    for cols, sts in (([k], [INT64]), ([x], [FLOAT64])):
        for desc in (False, True):
            flags = [SORT_ONLY | (DESCENDING if desc else 0)]
            want = ref_group(cols, sts, flags, LAST)
            got = wplan(lambda: engine.group(dev(cols, sts), flags, LAST))
            assert wplan.bits > 32
            assert (wplan.widths, wplan.low) == expect_widths(wplan.bits, 8, False, False), wplan.widths
            assert wplan.widths.split(",")[-2].endswith(":1"), wplan.widths
            assert_group_equal(got, want, f"64-bit sort only st={sts[0]} desc={desc}")
