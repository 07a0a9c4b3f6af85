#!/usr/bin/env python
"""
Generates tests/golden/golden_v4.json and golden_v4_NN.npz (parts below 1 MB) by running the *reference itself*
(the unmodified build staged by oracle/build_ref.sh) on group() with more key columns than golden_v1 has:

    PYTHONPATH=oracle/_ref python tests/golden/make_golden_v4.py

golden_v1 stops at three key columns.  These cases have 4 to 8, most of them 64 bits wide after normalisation
(int64 columns that span the whole range, float64 columns with infinities), so that the engine has to sort them in
2, 3 or 8 stable rounds.  The by() / sort() split falls inside a round, on a round boundary, and before rounds that
hold only sort columns; directions are mixed; sort-only calls use na_position first, last and remove.  Every column
draws from a small pool of hard values (the neighbours of the NA sentinels, signed zeros, infinities, the largest
finite value, the smallest subnormals, NaNs with several payloads, float32 values around 2^24), so that the rows tie
on the leading columns and the later columns decide.

The layout is that of golden_v1 (make_golden.py): every case stores its key columns and the reference's RowIndex
(`order`) and, under by(), the Groupby offsets.  tests/test_gpu_group_plan.py reads them.
"""
import io
import json
import os

import numpy as np

import datatable as dt
from datatable import f, by

HERE = os.path.dirname(os.path.abspath(__file__))

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64 = 1, 2, 3, 4, 5, 6, 7
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63}


def bits64(bits):
    return np.array([bits], dtype=np.uint64).view(np.float64)[0]


def bits32(bits):
    return np.array([bits], dtype=np.uint32).view(np.float32)[0]


POOL = {
    BOOL: np.array([0, 1, NA[BOOL]], np.int8),
    INT8: np.array([-127, 127, 0, -1, NA[INT8]], np.int8),
    INT16: np.array([-2**15 + 1, 2**15 - 1, 0, 1, NA[INT16]], np.int16),
    INT32: np.array([-2**31 + 1, 2**31 - 1, 0, -1, 7, NA[INT32]], np.int32),
    INT64: np.array([-2**63 + 1, 2**63 - 1, 0, -1, 2**40, NA[INT64]], np.int64),
    FLOAT64: np.array([-0.0, 0.0, np.inf, -np.inf, np.finfo(np.float64).max, -np.finfo(np.float64).max,
                       5e-324, -5e-324, 1.0, np.nan, bits64(0x7FF0000000000001), bits64(0xFFF8000000000000),
                       bits64(0xFFFFFFFFFFFFFFFF)], np.float64),
    FLOAT32: np.array([-0.0, 0.0, np.inf, -np.inf, np.finfo(np.float32).max, -np.finfo(np.float32).max,
                       bits32(1), bits32(0x80000001), 2.0**24 - 1, 2.0**24, 2.0**24 + 2, np.nan, bits32(0x7F800001),
                       bits32(0xFFC00000), bits32(0xFFFFFFFF)], np.float32),
}

arrays = {}
manifest = []
rng = np.random.default_rng(20261015)


def frame_col(a, st):
    if st == BOOL:
        return dt.Frame([None if x == -128 else bool(x) for x in a.tolist()], stype=dt.bool8)
    return dt.Frame(np.ascontiguousarray(a))


def pool_col(st, n, npool=None):
    p = POOL[st] if npool is None else POOL[st][:npool]
    return p[rng.integers(0, len(p), n)]


def add_case(name, keys, kst, reverse, na_position="first", nby=None):
    n = len(keys[0])
    frames = []
    for i, (k, st) in enumerate(zip(keys, kst)):
        fr = frame_col(k, st); fr.names = [f"k{i}"]; frames.append(fr)
    fr = dt.Frame(np.arange(n, dtype=np.int32)); fr.names = ["idx"]; frames.append(fr)
    DT = dt.cbind(*frames)
    for i, k in enumerate(keys):
        arrays[f"{name}__k{i}"] = np.ascontiguousarray(k)
    kexpr = [f[f"k{i}"] for i in range(len(keys))]
    if nby is None:
        R = DT[:, f.idx, dt.sort(*kexpr, reverse=reverse, na_position=na_position)]
    else:
        mods = [by(*[(-kexpr[i] if reverse[i] else kexpr[i]) for i in range(nby)])]
        if nby < len(keys):
            mods.append(dt.sort(*kexpr[nby:], reverse=reverse[nby:], na_position=na_position))
        R = DT[(slice(None), f.idx) + tuple(mods)]
        C = DT[(slice(None), {"cnt": dt.count()}) + tuple(mods)]
        cnt = C["cnt"].to_numpy().reshape(-1).astype(np.int64)
        arrays[f"{name}__offsets"] = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
    arrays[f"{name}__order"] = R["idx"].to_numpy().reshape(-1).astype(np.int32)
    manifest.append({"name": name, "n": n, "kst": list(kst), "vst": [], "reverse": list(reverse),
                     "na_position": na_position, "nby": nby, "reducers": []})


def directions(kst, mixed):
    # by() columns of stype bool are never reversed: the reference negates a by() column, and -bool is int
    return [bool(mixed and rng.integers(0, 2) and st != BOOL) for st in kst]


# (name, key stypes, by/sort splits to generate) -- the round structure the engine gives each set is in the
# comment; a split is the number of leading by() columns (None = sort only)
SETS = [
    # 2 rounds: {f64} {i64}
    ("w2", [INT64, FLOAT64], [None, 1, 2]),
    # 3 rounds: {i64} {i32, i32} {f64}; split 2 falls inside the middle round
    ("w3", [FLOAT64, INT32, INT32, INT64], [None, 1, 2, 3, 4]),
    # 3 rounds: {bool} {i64} {i8, i16, i32}; splits 1 and 2 inside the last round, 3 and 4 on boundaries
    ("w3b", [INT32, INT16, INT8, INT64, BOOL], [None, 1, 2, 3, 4, 5]),
    # 8 rounds of one 64-bit column each; split 1 leaves seven rounds of sort columns only
    ("w8", [INT64, FLOAT64, INT64, FLOAT64, INT64, FLOAT64, INT64, FLOAT64], [None, 1, 4, 7, 8]),
    # float32 / int16 / int8 / bool between wide columns: 4 to 6 keys of every stype
    ("mix", [FLOAT32, INT64, INT16, FLOAT64, INT8, BOOL], [None, 2, 3, 6]),
]

for sname, kst, splits in SETS:
    n = 2000 if len(kst) >= 8 else 3000
    # few values per column: the leading columns tie often enough for the last ones to matter
    keys = [pool_col(st, n, npool=None if j % 2 else 4) for j, st in enumerate(kst)]
    for nby in splits:
        for mixed in (False, True):
            rev = directions(kst, mixed)
            # without a sort() clause na_position has nothing to apply to: by() alone puts NA first
            naps = ("first", "last", "remove") if nby is None else ("first", "last") if nby < len(kst) else ("first",)
            for nap in naps:
                add_case(f"{sname}_by{nby}_{'mix' if mixed else 'asc'}_{nap}", keys, kst, rev, nap, nby)

# a constant column and an all-NA column between wide ones (0-bit columns inside the rounds)
n = 3000
kz = [pool_col(INT64, n), np.full(n, 5, np.int32), pool_col(FLOAT64, n), np.full(n, np.nan), pool_col(INT64, n)]
for nby in (None, 1, 2, 3, 5):
    for nap in (("first", "last", "remove") if nby is None else ("first", "last") if nby < 5 else ("first",)):
        add_case(f"zero_by{nby}_{nap}", kz, [INT64, INT32, FLOAT64, FLOAT64, INT64], [False, True, False, True, True],
                 nap, nby)


def save_parts(arrays, prefix, max_bytes=900_000):
    """prefix_00.npz, prefix_01.npz, ...: every case's arrays in one part, each part compressed and below
    max_bytes (as make_golden.save_parts does for golden_v1)."""
    cases = {}
    for key, a in arrays.items():
        cases.setdefault(key.split("__")[0], {})[key] = a
    parts, cur = [], {}
    for case in cases.values():
        trial = dict(cur, **case)
        buf = io.BytesIO(); np.savez_compressed(buf, **trial)
        if cur and buf.tell() > max_bytes:
            parts.append(cur); cur = dict(case)
        else:
            cur = trial
    parts.append(cur)
    for i, part in enumerate(parts):
        np.savez_compressed(f"{prefix}_{i:02d}.npz", **part)


save_parts(arrays, os.path.join(HERE, "golden_v4"))
with open(os.path.join(HERE, "golden_v4.json"), "w") as fh:
    json.dump({"generator": "tests/golden/make_golden_v4.py", "datatable_version": dt.__version__,
               "cases": manifest}, fh, indent=0)
print(f"{len(manifest)} cases, {sum(a.nbytes for a in arrays.values()) / 1e6:.2f} MB raw")
