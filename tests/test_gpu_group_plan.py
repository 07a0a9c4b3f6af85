"""group()'s RowIndex and Groupby at every branch of the key planner, against an independent reference.

`ref_group` restates group() in numpy alone: every key column becomes (NA rank, uint64 image), one stable lexsort
orders the rows, and the groups are the runs of equal keys over the LEADING run of by() columns (sort.cc:1471-1482).
It does not use the C oracle.  The CPU tests pin it to the reference's own output (golden_v1, and golden_v4 with 4 to
8 keys and 2, 3 and 8 sort rounds) and to the oracle; the GPU tests compare the engine with it bit for bit.

Every planner case also asserts that it reached the branch it was built for.  The plan comes from the engine's
verbose lines (`[dtb200] group: ... rounds=`, one `key c:` line per column with its bits and cshift, one `round r:`
line per sort round with its passes, narrowing pass and whether the first pass took the folded histogram) and from
last_call_stats().  A case whose data no longer reaches its branch fails there.
"""
import glob
import json
import math
import os
import re

import numpy as np
import pytest

from conftest import ROOT, golden
from helpers import (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DESCENDING, SORT_ONLY, NA_POS,
                     case_flags)

DATE32, TIME64 = 17, 18
FIRST, LAST, REMOVE = NA_POS["first"], NA_POS["last"], NA_POS["remove"]
NP = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64, DATE32: np.int32,
      TIME64: np.int64, FLOAT32: np.float32, FLOAT64: np.float64}
NA_INT = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
WIDTH = {BOOL: 1, INT8: 8, INT16: 16, INT32: 32, INT64: 64, DATE32: 32, TIME64: 64, FLOAT32: 32, FLOAT64: 64}
ALL_STYPES = (BOOL, INT8, INT16, INT32, INT64, DATE32, TIME64, FLOAT32, FLOAT64)
SIGN = np.uint64(1 << 63)


# ---------------------------------------------------------------------------------------------------------------
# the reference
# ---------------------------------------------------------------------------------------------------------------
def key_image(a, st):
    """(NA mask, uint64 image) of a column: the image orders the valid values ascending.  Integers: the value with
    its sign bit flipped; floats: the IEEE sign-flip image (-0.0 below +0.0); any NaN is NA."""
    a = np.asarray(a)
    if st in (FLOAT32, FLOAT64):
        na = np.isnan(a)
        with np.errstate(invalid="ignore"):              # (signalling NaNs; they are NA anyway)
            b = a.astype(np.float64).view(np.uint64)      # float32 -> float64 is exact and keeps the order
        img = np.where((b >> np.uint64(63)) == 1, ~b, b | SIGN)
    else:
        na = a == NA_INT[st]
        img = a.astype(np.int64).view(np.uint64) ^ SIGN
    return na, np.where(na, np.uint64(0), img)


def ref_keys(cols, stypes, flags, na_pos):
    """Per column (NA rank, image): NA ranks first for first / remove and last for last, whatever the direction."""
    ranks, imgs = [], []
    for c, st, fl in zip(cols, stypes, flags):
        na, img = key_image(c, st)
        if fl & DESCENDING:
            img = ~img
        ranks.append(np.where(na, 2 if na_pos == LAST else 0, 1).astype(np.uint8))
        imgs.append(img)
    return ranks, imgs


def ref_group(cols, stypes, flags, na_pos):
    """(order int32, offsets int32 or None, ngroups or None) of group(cols, flags, na_pos)."""
    n = len(cols[0])
    ranks, imgs = ref_keys(cols, stypes, flags, na_pos)
    seq = []
    for r, im in zip(reversed(ranks), reversed(imgs)):
        seq += [im, r]                                    # np.lexsort: the last key is the primary one
    order = np.lexsort(seq).astype(np.int32)
    nby = 0
    while nby < len(flags) and not flags[nby] & SORT_ONLY:
        nby += 1
    if na_pos == REMOVE:
        if nby:
            raise ValueError("groups with na_position = remove are refused")
        if n == 1:                                        # one row returns before any NA is removed (sort.cc:1435)
            return order, None, None
        return order[int(np.count_nonzero(ranks[-1] == 0)):], None, None     # sort.cc:598-605
    if nby == 0:
        return order, None, None
    change = np.zeros(max(n - 1, 0), dtype=bool)
    for c in range(nby):
        r, im = ranks[c][order], imgs[c][order]
        change |= (r[1:] != r[:-1]) | (im[1:] != im[:-1])
    offsets = np.concatenate([[0], np.flatnonzero(change) + 1, [n]] if n else [[0]]).astype(np.int32)
    return order, offsets, len(offsets) - 1


def load_golden(prefix):
    g = os.path.join(ROOT, "tests", "golden")
    with open(os.path.join(g, prefix + ".json")) as fh:
        meta = json.load(fh)
    arr = {}
    for part in sorted(glob.glob(os.path.join(g, prefix + "_*.npz"))):
        with np.load(part) as z:
            arr.update((k, z[k]) for k in z.files)
    return meta["cases"], arr


def check_golden_cases(cases, arr):
    for case in cases:
        name = case["name"]
        keys = [arr[f"{name}__k{i}"] for i in range(len(case["kst"]))]
        order, offsets, ng = ref_group(keys, case["kst"], case_flags(case), NA_POS[case["na_position"]])
        assert np.array_equal(order, arr[f"{name}__order"]), f"{name}: RowIndex differs from the reference"
        if case["nby"] is None:
            assert offsets is None, name
        else:
            assert np.array_equal(offsets, arr[f"{name}__offsets"]), f"{name}: offsets differ from the reference"


def test_ref_group_reproduces_golden_v1():
    g = golden()
    check_golden_cases(g.cases, g.arr)


def test_ref_group_reproduces_golden_v4():
    cases, arr = load_golden("golden_v4")
    assert len(cases) > 100 and max(len(c["kst"]) for c in cases) == 8
    check_golden_cases(cases, arr)


# ---------------------------------------------------------------------------------------------------------------
# hard values
# ---------------------------------------------------------------------------------------------------------------
def f64_bits(b):
    return np.array([b], np.uint64).view(np.float64)[0]


def f32_bits(b):
    return np.array([b], np.uint32).view(np.float32)[0]


F64_HARD = [-0.0, 0.0, np.inf, -np.inf, np.finfo(np.float64).max, -np.finfo(np.float64).max, f64_bits(1),
            f64_bits(0x8000000000000001), 1.0]
F64_NANS = [np.nan, f64_bits(0x7FF0000000000001), f64_bits(0xFFF8000000000000), f64_bits(0xFFFFFFFFFFFFFFFF)]
F32_HARD = [-0.0, 0.0, np.inf, -np.inf, np.finfo(np.float32).max, -np.finfo(np.float32).max, f32_bits(1),
            f32_bits(0x80000001), 2.0**24 - 1, 2.0**24, 2.0**24 + 2, -(2.0**24)]
F32_NANS = [np.nan, f32_bits(0x7F800001), f32_bits(0xFFC00000), f32_bits(0xFFFFFFFF)]


def hard_values(st):
    """(valid hard values, NA spellings) of a stype."""
    if st == FLOAT64:
        return np.array(F64_HARD, np.float64), np.array(F64_NANS, np.float64)
    if st == FLOAT32:
        return np.array(F32_HARD, np.float32), np.array(F32_NANS, np.float32)
    if st == BOOL:
        return np.array([0, 1], np.int8), np.array([-128], np.int8)
    lo, hi = NA_INT[st] + 1, -NA_INT[st] - 1
    return np.array([lo, hi, 0, -1, 1, lo + 1, hi - 1], NP[st]), np.array([NA_INT[st]], NP[st])


def full_range(rng, st, n, na):
    """Values over the whole range of the stype with every hard value present; na = fraction of NA rows (every
    NA spelling of a float appears)."""
    good, nas = hard_values(st)
    if st in (FLOAT32, FLOAT64):
        ui = np.uint32 if st == FLOAT32 else np.uint64
        a = rng.integers(0, np.iinfo(ui).max, n, dtype=ui, endpoint=True).view(NP[st])
        bad = np.isnan(a)
        a[bad] = good[rng.integers(0, len(good), int(bad.sum()))]
    elif st == BOOL:
        a = rng.integers(0, 2, n).astype(np.int8)
    else:
        info = np.iinfo(NP[st])
        a = rng.integers(info.min + 1, info.max, n, dtype=NP[st], endpoint=True)
    pos = rng.choice(n, size=min(n, len(good)), replace=False)
    a[pos] = good[:len(pos)]
    if na:
        m = rng.random(n) < na
        m[pos] = False
        a[m] = nas[rng.integers(0, len(nas), int(m.sum()))]
    return a


def span_whole(col, st, at):
    """Writes the two values that make the column span its stype's whole range at rows at, at + 1."""
    good = hard_values(st)[0]
    col[at:at + 2] = good[2:4] if st in (FLOAT32, FLOAT64) else good[:2]      # floats: +-inf; integers: lo, hi


def pool(rng, st, n, na=True, k=None):
    """Few distinct hard values (the rows tie on this column); all of them span the stype's whole range."""
    good, nas = hard_values(st)
    vals = np.concatenate([good[:k] if k else good, nas if na else nas[:0]])
    a = vals[rng.integers(0, len(vals), n)]
    m = min(n, len(good[:k] if k else good))
    a[:m] = good[:m]
    return a.astype(NP[st])


# ---------------------------------------------------------------------------------------------------------------
# the oracle against the reference on shapes golden_v1 does not have
# ---------------------------------------------------------------------------------------------------------------
ORACLE_SHAPES = [
    ([INT64, FLOAT64, INT32, INT16], [0, SORT_ONLY, 0, SORT_ONLY]),                  # [by, sort, by, sort]
    ([INT64, FLOAT64, INT64], [0, SORT_ONLY, 0]),                                    # [by, sort, by]
    ([FLOAT32, INT64, INT8, BOOL, FLOAT64], [0, 0, SORT_ONLY | DESCENDING, 0, DESCENDING]),
    ([INT64, FLOAT64, INT64, FLOAT64, INT64, FLOAT64, INT64, FLOAT64], [0] * 4 + [SORT_ONLY] * 4),
    ([INT64, FLOAT64, INT64, FLOAT64, INT64, FLOAT64, INT64, FLOAT64], [SORT_ONLY | DESCENDING] * 8),
    ([INT16, INT64, FLOAT64, INT32, INT8, FLOAT32], [SORT_ONLY, 0, 0, 0, 0, 0]),     # [sort, by, ...]: no groups
]


@pytest.mark.parametrize("shape", range(len(ORACLE_SHAPES)))
def test_ref_group_agrees_with_oracle(shape):
    from oracle import oracle as orc
    sts, flags = ORACLE_SHAPES[shape]
    rng = np.random.default_rng(1000 + shape)
    for n in (1, 2, 700, 3001):
        cols = [pool(rng, st, n, k=3 + j % 3) for j, st in enumerate(sts)]
        for na_pos in (FIRST, LAST, REMOVE):
            if na_pos == REMOVE and not flags[0] & SORT_ONLY:
                continue
            want = orc.group(cols, flags, na_pos, stypes=sts)
            got = ref_group(cols, sts, flags, na_pos)
            assert np.array_equal(got[0], want[0]), f"n={n} na_pos={na_pos}: RowIndex"
            # one row: the reference returns a single group even for a sort (sort.cc:1435-1439); the engine keeps
            # the convention of sort-only calls and reports no Groupby
            assert (got[1] is None) == (want[1] is None or (n == 1 and bool(flags[0] & SORT_ONLY)))
            if got[1] is not None:
                assert np.array_equal(got[1], want[1]) and got[2] == want[2], f"n={n} na_pos={na_pos}: offsets"


def test_frame_refuses_by_with_sort_remove():
    """by() + sort(na_position="remove"): the RowIndex would be shorter than the Groupby it belongs to."""
    import datatable_b200 as dtb
    f, by, sort = dtb.f, dtb.by, dtb.sort
    DT = dtb.Frame({"k": np.array([1, 2, 1, 2], np.int32), "s": np.array([1.0, np.nan, 3.0, 4.0]),
                    "v": np.array([1.0, 2.0, 3.0, 4.0])})
    with pytest.raises(ValueError, match="remove"):
        DT[:, dtb.sum(f.v), by(f.k), sort(f.s, na_position="remove")]


# ---------------------------------------------------------------------------------------------------------------
# GPU: running group() and reading its plan
# ---------------------------------------------------------------------------------------------------------------
_GROUP = re.compile(r"\[dtb200\] group: n=(\d+) keys=(\d+) bits=(\d+) rounds=(\d+)")
_KEY = re.compile(r"\[dtb200\]   key (\d+): stype=(\d+) desc=(\d+) bits=(\d+) cshift=(\d+) lshift=(\d+)")
_ROUND = re.compile(r"\[dtb200\]   round (\d+): keys=(\d+) bits=(\d+) group_shift=(\d+) passes=(\d+) "
                    r"narrow_after=(-?\d+) fold=(\d) count_table=(\d)")


def parse_plan(err):
    """The plan of the last group() call in the verbose output, or None when it printed none (constant keys)."""
    i = err.rfind("[dtb200] group:")
    if i < 0:
        return None
    text = err[i:]
    m = _GROUP.search(text)
    keys = [dict(bits=int(k[3]), cshift=int(k[4]), lshift=int(k[5])) for k in _KEY.findall(text)]
    rounds = [dict(keys=int(r[1]), bits=int(r[2]), group_shift=int(r[3]), passes=int(r[4]), narrow_after=int(r[5]),
                   fold=int(r[6]), count_table=int(r[7])) for r in _ROUND.findall(text)]
    return dict(bits=int(m[3]), nrounds=int(m[4]), keys=keys, rounds=rounds)


class Plan:
    """Runs a call with option verbose on and keeps its plan and its call statistics."""

    def __init__(self, capfd):
        self.capfd = capfd

    def __call__(self, fn):
        from datatable_b200 import engine, _lib
        self.capfd.readouterr()
        engine.set_option("verbose", 1)
        try:
            out = fn()
        finally:
            engine.set_option("verbose", 0)
        self.plan = parse_plan(self.capfd.readouterr().err)
        self.stats = _lib.last_call_stats()
        return out


@pytest.fixture
def plan(capfd):
    return Plan(capfd)


@pytest.fixture
def radix_bits():
    """Sets option radix_bits for one test and restores the default."""
    from datatable_b200 import engine
    yield lambda w: engine.set_option("radix_bits", w)
    engine.set_option("radix_bits", 0)


def dev(cols, sts):
    import torch
    from datatable_b200 import engine
    return [engine.Col(torch.from_numpy(np.ascontiguousarray(c)).cuda(), st) for c, st in zip(cols, sts)]


def host(cols, sts):
    from datatable_b200 import engine
    return [engine.Col(np.ascontiguousarray(c), st) for c, st in zip(cols, sts)]


def to_np(x):
    return None if x is None else (x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x))


def assert_group_equal(got, want, ctx):
    order, offsets, ng = to_np(got[0]), to_np(got[1]), got[2]
    assert np.array_equal(order, want[0]), f"{ctx}: RowIndex differs ({np.count_nonzero(order != want[0]) if len(order) == len(want[0]) else 'length'})"
    assert (offsets is None) == (want[1] is None), f"{ctx}: groups requested / not requested"
    if want[1] is not None:
        assert ng == want[2], f"{ctx}: ngroups {ng} != {want[2]}"
        assert np.array_equal(offsets, want[1]), f"{ctx}: offsets differ"


def run_case(plan, cols, sts, flags, na_pos, ctx, device=True, also64=True):
    """engine.group (and group64) against ref_group; returns the plan of the group() call."""
    from datatable_b200 import engine
    want = ref_group(cols, sts, flags, na_pos)
    ecols = dev(cols, sts) if device else host(cols, sts)
    got = plan(lambda: engine.group(ecols, flags, na_pos))
    assert_group_equal(got, want, ctx)
    if also64:
        g64 = engine.group64(ecols, flags, na_pos)
        assert to_np(g64[0]).dtype == np.int64
        assert np.array_equal(to_np(g64[0]), to_np(got[0]).astype(np.int64)), f"{ctx}: group64 RowIndex"
        assert (g64[1] is None) == (got[1] is None) and g64[2] == got[2], f"{ctx}: group64 groups"
        if got[1] is not None:
            assert np.array_equal(to_np(g64[1]), to_np(got[1]).astype(np.int64)), f"{ctx}: group64 offsets"
    return plan.plan


def expect_passes(p, stats, width=8):
    """radix_passes = the sum of the rounds' passes, each as plan_passes / narrow_after give it."""
    total = 0
    for i, r in enumerate(p["rounds"]):
        b = r["bits"]
        if r["narrow_after"] >= 0:
            assert width == 8 and b > 32, r
            lo = math.ceil((b - 32) / 8)
            assert r["narrow_after"] == lo - 1 and r["passes"] == lo + 4, r
        else:
            assert r["passes"] == max(1, math.ceil(b / width)), r
        total += r["passes"]
    assert stats["radix_passes"] == total, (stats, p["rounds"])


def flag_of(kind, desc):
    return (SORT_ONLY if kind == "sort" else 0) | (DESCENDING if desc else 0)


# ---------------------------------------------------------------------------------------------------------------
# single raw key: the folded first-pass histogram
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("st", ALL_STYPES)
@pytest.mark.parametrize("na", ["first", "last", "none"])
@pytest.mark.parametrize("desc", [False, True])
@pytest.mark.parametrize("kind", ["sort", "by"])
def test_single_raw_key_folded_histogram(plan, st, na, desc, kind):
    rng = np.random.default_rng(st * 100 + ["first", "last", "none"].index(na) * 10 + desc * 2 + (kind == "by"))
    n = 65_537
    col = full_range(rng, st, n, 0.0 if na == "none" else 0.05)
    na_pos = LAST if na == "last" else FIRST
    flags = [flag_of(kind, desc)]
    p = run_case(plan, [col], [st], flags, na_pos, f"st={st} na={na} desc={desc} {kind}", device=(st % 2 == 0))
    # the whole range plus NA: the NA takes the slot the missing INT_MIN leaves, so the key keeps its width
    want_bits = 2 if (st == BOOL and na != "none") else WIDTH[st]
    assert p["nrounds"] == 1 and p["bits"] == want_bits and p["keys"][0]["cshift"] == 0, p
    assert p["rounds"][0]["fold"] == 1, p
    narrowed = kind == "sort" and want_bits > 32
    assert (p["rounds"][0]["narrow_after"] >= 0) == narrowed, p
    expect_passes(p, plan.stats)


@pytest.mark.gpu
@pytest.mark.parametrize("span_bits", [33, 40, 64])
@pytest.mark.parametrize("na", ["first", "last", "none"])
@pytest.mark.parametrize("w", [8, 4, 6, 7])
def test_narrowed_sort_only_passes(plan, radix_bits, span_bits, na, w):
    """int64 / time64 keys of 33, 40 and 64 bits, sort only: the low passes run on 64-bit words, the narrowing pass
    writes key >> (bits - 32), the rest run on 32-bit words.  33 bits = a span of 2^32 - 1 plus the NA slot."""
    radix_bits(w)
    rng = np.random.default_rng(span_bits * 10 + w)
    for st in (INT64, TIME64):
        for desc in (False, True):
            n = 65_537
            if span_bits == 64:
                col = full_range(rng, INT64, n, 0.0 if na == "none" else 0.03)
            else:
                span = 2**(span_bits - (0 if na == "none" else 1)) - 1
                base = -2**31 + 5
                col = base + rng.integers(0, span, n, endpoint=True)
                col[:2] = [base, base + span]
                if na != "none":
                    m = rng.random(n) < 0.03
                    m[:2] = False
                    col[m] = NA_INT[INT64]
            na_pos = LAST if na == "last" else FIRST
            p = run_case(plan, [col], [st], [flag_of("sort", desc)], na_pos, f"{span_bits} bits st={st} w={w}",
                         also64=False)
            assert p["nrounds"] == 1 and p["bits"] == span_bits and p["rounds"][0]["fold"] == 1, p
            assert (p["rounds"][0]["narrow_after"] >= 0) == (w == 8), p
            expect_passes(p, plan.stats, width=w)
            # a composite of the same width (two columns, so the count kernel rather than the fold)
            hi_bits = span_bits - 32
            k0 = rng.integers(0, 2**hi_bits - 1, n, endpoint=True).astype(np.int64)
            k0[0] = 2**hi_bits - 1
            k1 = full_range(rng, INT32, n, 0.0)
            p = run_case(plan, [k0, k1], [st, INT32], [flag_of("sort", desc), SORT_ONLY], FIRST,
                         f"{span_bits}-bit composite w={w}", also64=False)
            assert p["nrounds"] == 1 and p["bits"] == span_bits and p["rounds"][0]["fold"] == 0, p
            assert (p["rounds"][0]["narrow_after"] >= 0) == (w == 8), p
            expect_passes(p, plan.stats, width=w)


# ---------------------------------------------------------------------------------------------------------------
# constant low bits
# ---------------------------------------------------------------------------------------------------------------
def cshift_cases():
    """(name, stype, values, expected cshift): columns whose valid values share their low bits."""
    out = [
        ("i32_even", INT32, [0, 2, -2**31 + 2, 2**31 - 2, 6], 1),
        ("i32_x128", INT32, [0, 128, -2**31 + 128, 2**31 - 128, -128], 7),
        ("i32_top", INT32, [1, -2**31 + 1], 31),
        ("i8_top", INT8, [3, -125], 7),
        ("i16_top", INT16, [9, 9 - 2**15], 15),
        ("i64_top", INT64, [5, -2**63 + 5], 63),
        ("t64_x2", TIME64, [0, 2, 2**63 - 2, -2**63 + 2], 1),
        ("d32_x128", DATE32, [128, 256, -2**31 + 128], 7),
        ("f64_1_2", FLOAT64, [1.0, 2.0], 52),
        ("f32_1_2", FLOAT32, [1.0, 2.0], 23),
    ]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", cshift_cases(), ids=[c[0] for c in cshift_cases()])
@pytest.mark.parametrize("na", ["first", "last", "none"])
def test_constant_low_bits(plan, case, na):
    _, st, vals, cshift = case
    rng = np.random.default_rng(cshift * 7 + len(na))
    for n in (4097, 65_537):
        for desc in (False, True):
            for kind in ("sort", "by"):
                vals_ = np.array(vals, dtype=NP[st])
                col = vals_[rng.integers(0, len(vals_), n)]
                col[:len(vals_)] = vals_
                if na != "none":
                    nas = hard_values(st)[1]
                    m = rng.random(n) < 0.05
                    m[:len(vals_)] = False
                    col[m] = nas[rng.integers(0, len(nas), int(m.sum()))]
                p = run_case(plan, [col], [st], [flag_of(kind, desc)], LAST if na == "last" else FIRST,
                             f"{case[0]} n={n} desc={desc} {kind}", device=(n > 5000), also64=(n < 5000))
                assert p["keys"][0]["cshift"] == cshift and p["rounds"][0]["fold"] == 0, p
                expect_passes(p, plan.stats)


# ---------------------------------------------------------------------------------------------------------------
# one round: composites of at most 32 and at most 64 bits
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("sts,want_bits", [
    ((INT16, INT8, BOOL), 26),                      # 16 + 8 + 2: 32-bit words
    ((BOOL, DATE32), 34),                           # 2 + 32: 64-bit words
    ((INT32, INT16, INT8), 56),
    ((FLOAT32, INT16, INT8, BOOL, BOOL), 60),
])
@pytest.mark.parametrize("nby", [0, 1, 2, 3])
def test_single_round_composites(plan, sts, want_bits, nby):
    rng = np.random.default_rng(want_bits + nby)
    nby = min(nby, len(sts))
    for n in (4095, 65_536):
        cols = [pool(rng, st, n, k=3) for st in sts]
        for j, st in enumerate(sts):          # the full range in every column, so that the widths are exact
            span_whole(cols[j], st, n // 2)
        for na_pos in (FIRST, LAST):
            flags = [(0 if j < nby else SORT_ONLY) | (DESCENDING if (j + n) % 3 == 0 else 0) for j in range(len(sts))]
            if nby == 0:
                flags = [f | SORT_ONLY for f in flags]
            p = run_case(plan, cols, list(sts), flags, na_pos, f"{sts} nby={nby} n={n}", also64=(n < 5000))
            assert p["nrounds"] == 1 and p["bits"] == want_bits, p
            expect_passes(p, plan.stats)


# ---------------------------------------------------------------------------------------------------------------
# several rounds
# ---------------------------------------------------------------------------------------------------------------
def wide_col(rng, st, n):
    """A 64-bit-wide column with few distinct values: rows tie on it, so that the later columns decide."""
    return pool(rng, st, n, k=4)


# (name, stypes, flags: "b" by / "s" sort / "B" by descending / "S" sort descending, expected rounds)
ROUND_CASES = [
    # 2 rounds {f64} {i64}
    ("r2_by_boundary", [INT64, FLOAT64], "bs", 2),
    ("r2_all_by", [TIME64, FLOAT64], "bB", 2),
    ("r2_sort", [FLOAT64, INT64], "sS", 2),
    ("r2_sort_by", [INT64, FLOAT64], "sb", 2),
    # 3 rounds {i64} {i32, i32} {f64}
    ("r3_split_inside", [FLOAT64, INT32, INT32, INT64], "bbss", 3),
    ("r3_split_boundary", [FLOAT64, INT32, INT32, INT64], "bsss", 3),
    ("r3_split_boundary2", [FLOAT64, INT32, INT32, INT64], "bbbs", 3),
    ("r3_by_sort_by", [INT64, FLOAT64, INT64], "bsb", 3),
    ("r3_by_sort_by_desc", [FLOAT64, TIME64, INT64], "BSB", 3),
    ("r3_sort_by", [INT64, FLOAT64, INT64], "sbb", 3),
    # 3 rounds {bool} {i64} {i8, i16, i32}: splits inside the leading round and on its boundaries
    ("r3b_split1", [INT32, INT16, INT8, INT64, BOOL], "bssss", 3),
    ("r3b_split2", [INT32, INT16, INT8, INT64, BOOL], "bbsss", 3),
    ("r3b_split3", [INT32, INT16, INT8, INT64, BOOL], "bbbss", 3),
    ("r3b_by_sort_by", [INT32, INT16, INT8, INT64, BOOL], "bsbbb", 3),
    # 0-bit columns between wide ones: constant, all-NA
    ("r3_zero_bits", [INT64, "const", FLOAT64, "allna", INT64], "bbsss", 3),
    ("r3_zero_bits_by", [INT64, "const", FLOAT64, "allna", INT64], "bbbbs", 3),
    # 8 rounds of one 64-bit column each
    ("r8_sort", [INT64, FLOAT64, TIME64, INT64, FLOAT64, TIME64, INT64, FLOAT64], "sSsSsSsS", 8),
    ("r8_split1", [INT64, FLOAT64, TIME64, INT64, FLOAT64, TIME64, INT64, FLOAT64], "bsssssss", 8),
    ("r8_split4", [INT64, FLOAT64, TIME64, INT64, FLOAT64, TIME64, INT64, FLOAT64], "bBbBssss", 8),
    ("r8_all_by", [INT64, FLOAT64, TIME64, INT64, FLOAT64, TIME64, INT64, FLOAT64], "bbbbbbbb", 8),
    ("r8_by_sort_by", [INT64, FLOAT64, TIME64, INT64, FLOAT64, TIME64, INT64, FLOAT64], "bsbsbsbs", 8),
]


def build_round_case(rng, sts, n):
    cols, kst = [], []
    for st in sts:
        if st == "const":
            cols.append(np.full(n, 12345, np.int32)); kst.append(INT32)
        elif st == "allna":
            cols.append(np.full(n, np.nan)); kst.append(FLOAT64)
        else:
            cols.append(wide_col(rng, st, n) if WIDTH[st] == 64 else pool(rng, st, n, k=3)); kst.append(st)
    for j, st in enumerate(kst):                   # whole range: every column needs all its bits
        if sts[j] not in ("const", "allna"):
            span_whole(cols[j], st, n // 3)
    return cols, kst


def flags_of(spec):
    return [{"b": 0, "B": DESCENDING, "s": SORT_ONLY, "S": SORT_ONLY | DESCENDING}[c] for c in spec]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ROUND_CASES, ids=[c[0] for c in ROUND_CASES])
@pytest.mark.parametrize("w", [8, 4, 6, 7])
def test_several_rounds(plan, radix_bits, case, w):
    name, sts, spec, want_rounds = case
    radix_bits(w)
    rng = np.random.default_rng(len(name) * 100 + w)
    flags = flags_of(spec)
    sizes = (4097, 65_537) if w == 8 else (4096,)
    for n in sizes:
        cols, kst = build_round_case(rng, sts, n)
        for na_pos in (FIRST, LAST, REMOVE):
            if na_pos == REMOVE and not flags[0] & SORT_ONLY:
                continue
            p = run_case(plan, cols, kst, flags, na_pos, f"{name} n={n} na={na_pos} w={w}", also64=(n < 5000))
            assert p["nrounds"] == want_rounds and len(p["rounds"]) == want_rounds, p
            expect_passes(p, plan.stats, width=w)


@pytest.mark.gpu
def test_by_sort_by_takes_groups_from_the_leading_by_columns(plan):
    """[by, sort, by] over three 64-bit columns: the groups are those of column 0 alone (sort.cc:1478-1480), not of
    (column 0, column 2) -- the third column only orders the rows."""
    from datatable_b200 import engine
    rng = np.random.default_rng(5)
    n = 10_000
    cols = [wide_col(rng, INT64, n), wide_col(rng, FLOAT64, n), wide_col(rng, INT64, n)]
    flags = [0, SORT_ONLY, 0]
    for device in (True, False):
        p = run_case(plan, cols, [INT64, FLOAT64, INT64], flags, FIRST, f"device={device}", device=device)
        assert p["nrounds"] == 3
    order, offsets, ng = engine.group(dev(cols, [INT64, FLOAT64, INT64]), flags, FIRST)
    assert ng == len(np.unique(cols[0])), "one group per distinct value of column 0 (NA included)"
    g = engine.Groupby(dev(cols, [INT64, FLOAT64, INT64]), flags, FIRST)
    assert g.ngroups == ng and np.array_equal(to_np(g.offsets()), to_np(offsets))


# ---------------------------------------------------------------------------------------------------------------
# sizes around the pass tile (4096), the count chunk (65 536) and 16 chunks; a skewed column
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [4095, 4096, 4097, 65_535, 65_536, 65_537, 1_048_577])
def test_sizes(plan, n):
    rng = np.random.default_rng(n)
    shapes = [
        ([INT32], "b", 1), ([FLOAT64], "S", 1), ([INT64], "s", 1),
        ([INT16, FLOAT32], "bs", 1), ([INT64, FLOAT64], "bs", 2), ([FLOAT64, INT32, INT32, INT64], "bbss", 3),
    ]
    for sts, spec, want_rounds in shapes:
        if len(sts) == 1:
            cols = [full_range(rng, sts[0], n, 0.05)]
        else:
            cols, _ = build_round_case(rng, sts, n)
            cols[-1] = full_range(rng, sts[-1], n, 0.02)         # the last column is all over the place
        for na_pos in (FIRST, LAST):
            p = run_case(plan, cols, sts, flags_of(spec), na_pos, f"{sts} n={n}", device=True, also64=(n < 100_000))
            assert p["nrounds"] == want_rounds, p
            expect_passes(p, plan.stats)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [65_537, 1_048_577])
def test_skewed_column(plan, n):
    """One value in 99.99 % of the rows: its group runs across many tiles and chunks."""
    rng = np.random.default_rng(n + 1)
    k = np.full(n, 7, np.int32)
    m = rng.random(n) < 1e-4
    m[::10007] = True
    k[m] = full_range(rng, INT32, int(m.sum()), 0.2)
    s = full_range(rng, FLOAT64, n, 0.01)
    for flags in ([0], [DESCENDING | SORT_ONLY]):
        run_case(plan, [k], [INT32], flags, FIRST, f"skew {flags}")
    for spec in ("bs", "bS", "ss"):
        run_case(plan, [k, s], [INT32, FLOAT64], flags_of(spec), LAST, f"skew {spec}")


# ---------------------------------------------------------------------------------------------------------------
# the count-table path of the handle
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("sts,spec", [
    ((INT16,), "b"), ((INT8,), "B"), ((BOOL,), "b"), ((FLOAT32,), "b"),
    ((INT8, INT8), "bB"), ((BOOL, INT16, BOOL), "bbb"), ((INT8, INT8, BOOL), "bbs"), ((DATE32,), "b"),
])
def test_count_table_handle(plan, sts, spec):
    """engine.Groupby on device keys whose group-key domain is at most 2^22: the last pass counts the rows per group
    key and the offsets come from a scan over that table."""
    from datatable_b200 import engine
    rng = np.random.default_rng(len(spec) * 31 + sts[0])
    for n in (4097, 65_537):
        cols = []
        for st in sts:
            if st == FLOAT32:      # images 22 bits apart: a 6-bit key after the constant low bits are dropped
                c = np.array([1.0, 1.5, 2.0, 2.0**24, np.nan], np.float32)[rng.integers(0, 5, n)]
            elif st == DATE32:
                c = rng.integers(-3000, 3000, n).astype(np.int32)
                c[rng.random(n) < 0.02] = NA_INT[DATE32]
            else:
                c = pool(rng, st, n)
            cols.append(c)
        flags = flags_of(spec)
        for na_pos in (FIRST, LAST):
            want = ref_group(cols, list(sts), flags, na_pos)
            d = dev(cols, list(sts))
            g = plan(lambda: engine.Groupby(d, flags, na_pos))
            p = plan.plan
            assert p["nrounds"] == 1 and p["rounds"][-1]["count_table"] == 1, p
            assert g.ngroups == want[2]
            assert np.array_equal(to_np(g.order()), want[0]), f"{sts} n={n}: handle RowIndex"
            assert np.array_equal(to_np(g.offsets()), want[1]), f"{sts} n={n}: handle offsets"
            assert np.array_equal(to_np(g.first_rows()), want[0][want[1][:-1]]), f"{sts} n={n}: first rows"
            got = engine.group(d, flags, na_pos)
            assert_group_equal(got, want, f"{sts} n={n}: engine.group")


# ---------------------------------------------------------------------------------------------------------------
# degenerate inputs
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_degenerate_inputs(plan):
    from datatable_b200 import engine, _lib
    rng = np.random.default_rng(3)
    for n in (1, 2):
        for sts in ([INT32], [FLOAT64, INT64], [INT64, FLOAT64, TIME64]):
            cols = [pool(rng, st, 16)[:n] for st in sts]
            for spec in ("b" * len(sts), "s" * len(sts), "b" + "s" * (len(sts) - 1)):
                for na_pos in (FIRST, LAST):
                    run_case(plan, cols, sts, flags_of(spec), na_pos, f"n={n} {sts} {spec}")
    # one row returns before any NA is removed (sort.cc:1435-1439): an NA row stays
    for st in (INT32, FLOAT64):
        one = hard_values(st)[1][:1]
        run_case(plan, [one], [st], [SORT_ONLY], REMOVE, f"one NA row {st}")
        run_case(plan, [one, one], [st, st], [SORT_ONLY, SORT_ONLY], REMOVE, f"one NA row {st} x2")
    n = 70_000
    const = [np.full(n, 3, np.int32), np.full(n, -0.0), np.full(n, NA_INT[INT64], np.int64)]
    for spec in ("bbb", "sss", "bss"):
        run_case(plan, const, [INT32, FLOAT64, INT64], flags_of(spec), FIRST, f"constant {spec}")
        assert plan.stats["key_bits"] == 0
    # constant by-columns, varying sort columns: one group in the sort columns' order
    vary = [full_range(rng, FLOAT64, n, 0.05), full_range(rng, INT64, n, 0.05)]
    for spec in ("bbss", "bBsS"):
        run_case(plan, const[:2] + vary, [INT32, FLOAT64, FLOAT64, INT64], flags_of(spec), LAST, f"constant by {spec}")
        assert plan.stats["key_bits"] > 64
    nine = [np.arange(5, dtype=np.int32)] * 9
    with pytest.raises(_lib.DtbValueError):
        engine.group(nine, [0] * 9, FIRST)
    with pytest.raises(_lib.DtbValueError):
        engine.Groupby(dev(nine, [INT32] * 9), [0] * 9, FIRST)


# ---------------------------------------------------------------------------------------------------------------
# dtb_sort_grouped
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("vst", [FLOAT64, INT64])
@pytest.mark.parametrize("groups", ["few", "singletons", "one"])
def test_sort_grouped(vst, groups):
    """(group id, value) with 64-bit values needs two rounds; each group must come out ordered by (NA rank, image)
    of its values, stably."""
    import torch
    from datatable_b200 import engine
    rng = np.random.default_rng(vst * 3 + len(groups))
    n = 65_537
    k = {"few": rng.integers(0, 300, n), "singletons": rng.permutation(n), "one": np.zeros(n)}[groups].astype(np.int32)
    if vst == FLOAT64:
        v = full_range(rng, FLOAT64, n, 0.05)
        zs = rng.random(n) < 0.05
        v[zs] = np.where(rng.random(int(zs.sum())) < 0.5, -0.0, 0.0)
    else:
        v = full_range(rng, INT64, n, 0.05)
    order, offsets, ng = engine.group(dev([k], [INT32]), [0], FIRST)
    got = engine.sort_grouped(torch.from_numpy(v).cuda(), order, offsets)
    o, f = to_np(order), to_np(offsets)
    gid = np.repeat(np.arange(ng), np.diff(f))
    na, img = key_image(v[o], vst)
    perm = np.lexsort((img, np.where(na, 0, 1), gid))
    assert np.array_equal(to_np(got), o[perm])


# ---------------------------------------------------------------------------------------------------------------
# past chunk_scan_kernel's 1024 chunks per round: checked by properties on the GPU
# ---------------------------------------------------------------------------------------------------------------
def _signed_image(t, is_float):
    """Order-preserving signed int64 image of an int64 / float64 tensor (floats: -0.0 below +0.0)."""
    import torch
    if not is_float:
        return t
    b = t.view(torch.int64)
    return torch.where(b < 0, b ^ 0x7FFFFFFFFFFFFFFF, b)


@pytest.mark.gpu
def test_past_1024_chunks_by_properties(plan):
    import torch
    from datatable_b200 import engine
    n = 67_108_864 + 4097
    rng = np.random.default_rng(7)
    k0 = torch.from_numpy(pool(rng, INT64, n, k=5)).cuda()
    k1 = rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True).view(np.float64)
    k1[:4] = [np.inf, -np.inf, -0.0, 0.0]
    k1 = torch.from_numpy(k1).cuda()
    flags = [0, SORT_ONLY]
    order, offsets, ng = plan(lambda: engine.group([engine.Col(k0, INT64), engine.Col(k1, FLOAT64)], flags, FIRST))
    assert plan.plan["nrounds"] == 2, plan.plan
    assert order.numel() == n
    # a permutation
    seen = torch.zeros(n, dtype=torch.int8, device="cuda")
    seen[order.long()] = 1
    assert bool(seen.all())
    del seen
    # keys sorted per column (NA first), ties in ascending row id
    o = order.long()
    r0 = (k0[o] != -2**63).to(torch.int8); i0 = k0[o]
    v1 = k1[o]
    r1 = (~torch.isnan(v1)).to(torch.int8); i1 = torch.where(r1.bool(), _signed_image(v1, True), 0)
    del v1
    eq0 = (r0[1:] == r0[:-1]) & (i0[1:] == i0[:-1])
    gt0 = (r0[:-1] > r0[1:]) | ((r0[:-1] == r0[1:]) & (i0[:-1] > i0[1:]))
    eq1 = (r1[1:] == r1[:-1]) & (i1[1:] == i1[:-1])
    gt1 = (r1[:-1] > r1[1:]) | ((r1[:-1] == r1[1:]) & (i1[:-1] > i1[1:]))
    assert not bool(gt0.any()), "column 0 out of order"
    assert not bool((eq0 & gt1).any()), "column 1 out of order inside a run of column 0"
    assert not bool((eq0 & eq1 & (o[:-1] > o[1:])).any()), "ties not in ascending row order"
    # the offsets sit exactly where column 0 (the by-column) changes
    heads = torch.nonzero(~eq0).flatten() + 1
    want = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), heads,
                      torch.full((1,), n, dtype=torch.int64, device="cuda")])
    assert ng == want.numel() - 1 and torch.equal(offsets.long(), want)


# ---------------------------------------------------------------------------------------------------------------
# groups with na_position = remove are refused
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["group", "group64", "groupby_create", "groupby_create_reduce"])
@pytest.mark.parametrize("device", [True, False])
def test_groups_with_remove_are_refused(entry, device):
    """The RowIndex drops the first nacount(last key) rows, but the Groupby would still span every row: no such
    pair exists, so every entry point refuses the combination.  (The calls read no RowIndex: the only reducer
    here is nrows.)"""
    from datatable_b200 import engine, _lib
    k = np.array([3, 1, NA_INT[INT32], 2, 1, NA_INT[INT32]], np.int32)
    s = np.array([np.nan, 1.0, 2.0, np.nan, 0.5, 3.0])
    cols = dev([k, s], [INT32, FLOAT64]) if device or entry.startswith("groupby") else host([k, s], [INT32, FLOAT64])
    for flags in ([0, SORT_ONLY], [0, 0], [DESCENDING, SORT_ONLY | DESCENDING]):
        with pytest.raises(_lib.DtbValueError, match="remove"):
            if entry == "group":
                engine.group(cols, flags, REMOVE)
            elif entry == "group64":
                engine.group64(cols, flags, REMOVE)
            elif entry == "groupby_create":
                engine.Groupby(cols, flags, REMOVE)
            else:
                engine.Groupby(cols, flags, REMOVE, reducers=[(_lib.OP_NROWS, None)])
    # sort only: remove keeps working
    o, f, ng = engine.group(cols, [SORT_ONLY, SORT_ONLY], REMOVE)
    assert f is None and np.array_equal(to_np(o), ref_group([k, s], [INT32, FLOAT64], [SORT_ONLY] * 2, REMOVE)[0])
