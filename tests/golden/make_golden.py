#!/usr/bin/env python
"""
Generates tests/golden/golden_v1.json and golden_v1_NN.npz (parts below 1 MB) by running the *reference itself*.

Usage (in the build container, where the reference was built from
the reference's source tree with its own backend into a scratch copy):

    PYTHONPATH=/tmp/dtref/src python tests/golden/make_golden.py

The reference cannot travel to the GPU box, so the vectors are committed.
Each case stores its inputs (so the test does not depend on any RNG stream)
and the reference's outputs:

    order    int32[n']   RowIndex produced by group() (sort.cc:1411-1495)
    offsets  int32[ng+1] Groupby offsets              (groupby.h:41-47)
    red_i                reducer outputs              (column/{sumprod,mean,minmax,count}.h)

The literal cases restate the reference's own known-answer tests
(tests/ijby/test-sort.py, tests/test-groups.py, tests/test-reduce.py); the
expected values are *recomputed by the reference here*, not typed in.
"""
import io
import json
import os
import sys

import numpy as np

import datatable as dt
from datatable import f, by

HERE = os.path.dirname(os.path.abspath(__file__))

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64 = 1, 2, 3, 4, 5, 6, 7
NP2ST = {np.dtype(np.int8): INT8, np.dtype(np.int16): INT16, np.dtype(np.int32): INT32,
         np.dtype(np.int64): INT64, np.dtype(np.float32): FLOAT32, np.dtype(np.float64): FLOAT64}
NA = {INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63}
REDUCERS = {"sum": dt.sum, "mean": dt.mean, "min": dt.min, "max": dt.max, "count": dt.count}

arrays = {}
manifest = []


def frame_col(a, st):
    """dt column from a numpy array (bool columns arrive as int8 with -128 = NA)."""
    if st == BOOL:
        return dt.Frame([None if x == -128 else bool(x) for x in a.tolist()], stype=dt.bool8)
    return dt.Frame(np.ascontiguousarray(a))


def to_np(frame_col_, st_out=None):
    a = frame_col_.to_numpy()
    a = a.reshape(-1)
    if np.ma.isMaskedArray(a):
        if a.dtype == np.bool_:
            a = a.astype(np.int8)
        a = np.ma.filled(a, NA.get(NP2ST.get(a.dtype, 0), 0))
    if a.dtype == np.bool_:
        a = a.astype(np.int8)
    return np.ascontiguousarray(a)


def build_frame(keys, kst, vals, vst):
    n = len(keys[0]) if keys else len(vals[0])
    frames = []
    for i, (k, st) in enumerate(zip(keys, kst)):
        fr = frame_col(k, st); fr.names = [f"k{i}"]; frames.append(fr)
    for i, (v, st) in enumerate(zip(vals, vst)):
        fr = frame_col(v, st); fr.names = [f"v{i}"]; frames.append(fr)
    fr = dt.Frame(np.arange(n, dtype=np.int32)); fr.names = ["idx"]; frames.append(fr)
    return dt.cbind(*frames)


def add_case(name, keys, kst=None, reverse=None, na_position="first", nby=None,
             vals=(), vst=None, reducers=()):
    """
    keys      : list of numpy arrays (key columns, by-columns first)
    nby       : number of leading by() columns (None = pure sort; the rest are sort() columns)
    reducers  : list of (opname, value index)
    """
    keys = [np.ascontiguousarray(k) for k in keys]
    vals = [np.ascontiguousarray(v) for v in vals]
    kst = list(kst) if kst else [NP2ST[k.dtype] for k in keys]
    vst = list(vst) if vst else [NP2ST[v.dtype] for v in vals]
    nk = len(keys)
    n = len(keys[0])
    reverse = list(reverse) if reverse is not None else [False] * nk
    DT = build_frame(keys, kst, vals, vst)
    meta = {"name": name, "n": n, "kst": kst, "vst": vst, "reverse": reverse,
            "na_position": na_position, "nby": nby, "reducers": [list(r) for r in reducers]}
    for i, k in enumerate(keys):
        arrays[f"{name}__k{i}"] = k
    for i, v in enumerate(vals):
        arrays[f"{name}__v{i}"] = v

    kexpr = [f[f"k{i}"] for i in range(nk)]
    if nby is None:
        R = DT[:, f.idx, dt.sort(*kexpr, reverse=reverse, na_position=na_position)]
        arrays[f"{name}__order"] = to_np(R["idx"]).astype(np.int32)
    else:
        byx = [(-kexpr[i] if reverse[i] else kexpr[i]) for i in range(nby)]
        sortx = kexpr[nby:]
        mods = [by(*byx)]
        if sortx:
            mods.append(dt.sort(*sortx, reverse=reverse[nby:], na_position=na_position))
        R = DT[(slice(None), f.idx) + tuple(mods)]
        arrays[f"{name}__order"] = to_np(R["idx"]).astype(np.int32)
        C = DT[(slice(None), {"cnt": dt.count()}) + tuple(mods)]
        cnt = to_np(C["cnt"]).astype(np.int64)
        arrays[f"{name}__offsets"] = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int32)
        for j, (op, vi) in enumerate(reducers):
            if op == "nrows":
                out = cnt
            else:
                Rr = DT[(slice(None), {"r": REDUCERS[op](f[f"v{vi}"])}) + tuple(mods)]
                out = to_np(Rr["r"])
            arrays[f"{name}__red{j}"] = out
    manifest.append(meta)


# ---------------------------------------------------------------------------
def save_parts(arrays, prefix, max_bytes=900_000):
    """Writes the arrays as prefix_00.npz, prefix_01.npz, ... (every case's arrays in one part), each part
    compressed and below max_bytes, so that no stored file reaches 1 MB."""
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


# Literal cases restating the reference's own tests
# ---------------------------------------------------------------------------
I4 = np.int32
# tests/ijby/test-sort.py:132-178 (int32 small / stability / with NAs)
add_case("i4_small", [np.array([17, 2, 96, 245, 847569, 34, -45, 0x7FFFFFFF, 1], I4)])
add_case("i4_small_stable", [np.array([5, 3, 5, -2**31, 1000000, -2**31, 3, -5, 5, 3], I4)])
add_case("i4_na_only", [np.array([-2**31] * 5, I4)])
add_case("i4_const", [np.array([7] * 70, I4)])
# tests/ijby/test-sort.py:208-237 (u2 range boundaries, unsigned wrap)
add_case("i4_u2range", [np.array([0, 65535, 65534, 1, 65536, 2, -2**31, 65535, 0], I4)])
add_case("i4_unsigned", [np.array([-2**31 + 1, 2**31 - 1, 0, -1, 1, -2**31 + 1, 2**31 - 1], I4)])
add_case("i4_large_range", [np.array([2**31 - 1, -2**31 + 1, 0, 5, -2**31], I4)])
# tests/ijby/test-sort.py:259-305 (int8), :392-460 (int16), :468-514 (int64)
add_case("i1_small", [np.array([17, 2, 96, -128, 0, -17, 127, -127, 5, 5], np.int8)])
add_case("i2_small", [np.array([0, -10, 100, -1000, 10000, 2, 999, -32768, 32767, -32767], np.int16)])
add_case("i8_small", [np.array([10**7, 10**12, -10**12, 0, 1, -2**63, 2**62, -2**62, 10**18], np.int64)])
add_case("i8_bigrange", [np.array([2**63 - 1, -2**63 + 1, 0, -2**63, 3, 2**63 - 1], np.int64)])
# bool: sort.cc:690-720
add_case("b1_small", [np.array([1, 0, -128, 1, 0, 0, -128, 1], np.int8)], kst=[BOOL])
add_case("b1_desc", [np.array([1, 0, -128, 1, 0, 0, -128, 1], np.int8)], kst=[BOOL], reverse=[True])
add_case("b1_nalast", [np.array([1, 0, -128, 1, 0, 0, -128, 1], np.int8)], kst=[BOOL], na_position="last")
# tests/ijby/test-sort.py:520-620 (floats: NaN first, -0.0 < +0.0, inf)
fspecial = [0.0, -0.0, np.nan, 1.5, -0.0, 0.0, np.nan, -np.inf, np.inf, 1e-310, -1e-310,
            2.5, -2.5, 1e308, -1e308]
add_case("f8_special", [np.array(fspecial, np.float64)])
add_case("f8_special_desc", [np.array(fspecial, np.float64)], reverse=[True])
add_case("f8_special_nalast", [np.array(fspecial, np.float64)], na_position="last")
add_case("f8_special_desc_nalast", [np.array(fspecial, np.float64)], reverse=[True], na_position="last")
add_case("f8_special_remove", [np.array(fspecial, np.float64)], na_position="remove")
f4special = np.array([0.0, -0.0, np.nan, 1.5, -0.0, 0.0, np.nan, -np.inf, np.inf, 1e-40, -1e-40,
                      2.5, -2.5, 3e38, -3e38], np.float32)
add_case("f4_special", [f4special])
add_case("f4_special_desc", [f4special], reverse=[True])
# SURVEY 8(c) direction / NA placement matrix on x=[3,1,NA,2,1,NA]
xna = np.array([3, 1, -2**31, 2, 1, -2**31], I4)
for rev in (False, True):
    for nap in ("first", "last", "remove"):
        add_case(f"i4_dirna_{int(rev)}_{nap}", [xna], reverse=[rev], na_position=nap)
# tests/test-groups.py:39-52 (group order: NA first, ascending), :72-95 (stability)
add_case("grp_i4_basic", [np.array([3, 1, -2**31, 2, 1, -2**31, 3, 3], I4)], nby=1,
         vals=[np.arange(8, dtype=np.float64)], reducers=[("sum", 0), ("nrows", 0)])
add_case("grp_f8_zero_nan", [np.array([0.0, -0.0, np.nan, 1.5, -0.0, 0.0, np.nan, -np.inf, np.inf])],
         nby=1, vals=[np.arange(9, dtype=np.int32)], reducers=[("count", 0), ("sum", 0), ("min", 0)])
add_case("grp_desc", [np.array([3, 1, -2**31, 2, 1, -2**31, 3, 3], I4)], nby=1, reverse=[True],
         vals=[np.arange(8, dtype=np.float64)], reducers=[("sum", 0)])

# ---------------------------------------------------------------------------
# Seeded random cases
# ---------------------------------------------------------------------------
rng = np.random.default_rng(20260922)


def with_na(a, frac, st):
    a = a.copy()
    m = rng.random(len(a)) < frac
    if st in NA:
        a[m] = NA[st]
    elif st == BOOL:
        a[m] = -128
    else:
        a[m] = np.nan
    return a


def rnd_key(st, n, spread):
    if st == BOOL:
        return rng.integers(0, 2, n).astype(np.int8)
    if st in (FLOAT32, FLOAT64):
        dtp = np.float32 if st == FLOAT32 else np.float64
        if spread == "few":
            return rng.integers(-5, 6, n).astype(dtp) / 2
        if spread == "unit":
            return rng.random(n).astype(dtp)
        a = rng.standard_normal(n) * 10.0 ** rng.integers(-20, 20, n)
        return a.astype(dtp)
    dtp = {INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64}[st]
    info = np.iinfo(dtp)
    if spread == "few":
        lo, hi = -7, 8
    elif spread == "mid":
        lo, hi = max(info.min + 1, -1000), min(info.max, 30000)
    else:
        lo, hi = info.min + 1, info.max
    return rng.integers(lo, hi, n, dtype=np.int64, endpoint=True).astype(dtp)


cid = 0
for st in (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64):
    for spread in ("few", "mid", "full"):
        if st == BOOL and spread != "few":
            continue
        if st in (FLOAT32, FLOAT64):
            spread = {"few": "few", "mid": "unit", "full": "wide"}[spread]
        for n in (2, 63, 65, 1000, 5003):
            for rev in (False, True):
                nap = ("first", "last", "remove")[cid % 3]
                k = with_na(rnd_key(st, n, spread), 0.1 if cid % 2 else 0.0, st)
                add_case(f"rs{cid:03d}", [k], kst=[st], reverse=[rev], na_position=nap)
                cid += 1

# single-key groupby with every reducer over every value stype
vtypes = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
for st in (INT8, INT32, INT64, FLOAT64, FLOAT32, BOOL, INT16):
    for n, spread in ((257, "few"), (4000, "mid"), (6000, "few")):
        if st == BOOL:
            spread = "few"
        if st in (FLOAT32, FLOAT64) and spread == "mid":
            spread = "unit"
        k = with_na(rnd_key(st, n, spread), 0.05, st)
        vals, vst = [], []
        for vt in vtypes:
            v = rnd_key(vt, n, "few" if vt == BOOL else ("wide" if vt in (FLOAT32, FLOAT64) and cid % 2 else
                                                        ("unit" if vt in (FLOAT32, FLOAT64) else "mid")))
            vals.append(with_na(v, 0.2, vt)); vst.append(vt)
        reds = [(op, vi) for vi in range(len(vtypes)) for op in ("sum", "mean", "min", "max", "count")]
        reds.append(("nrows", 0))
        add_case(f"rg{cid:03d}", [k], kst=[st], nby=1, vals=vals, vst=vst, reducers=reds)
        cid += 1

# multi-key sort (tests/ijby/test-sort.py:828-940) and multi-key by (tests/test-groups.py:386-412)
for (st0, st1, st2) in ((INT64, INT32, None), (INT8, FLOAT64, None), (BOOL, INT16, FLOAT32),
                        (INT32, INT32, INT32), (FLOAT64, INT64, None)):
    for n in (100, 3001):
        sts = [s for s in (st0, st1, st2) if s is not None]
        keys = [with_na(rnd_key(s, n, "few"), 0.1, s) for s in sts]
        revs = [bool(rng.integers(0, 2)) for _ in sts]
        add_case(f"ms{cid:03d}", keys, kst=sts, reverse=revs, na_position=("first", "last")[cid % 2])
        cid += 1
        v = with_na(rng.standard_normal(n), 0.1, FLOAT64)
        add_case(f"mg{cid:03d}", keys, kst=sts, nby=len(sts), vals=[v],
                 reducers=[("sum", 0), ("mean", 0), ("min", 0), ("max", 0), ("count", 0), ("nrows", 0)])
        cid += 1
        if len(sts) >= 2:
            # by(first cols) + sort(last col): groups frozen at the by->sort transition (sort.cc:1478-1480)
            add_case(f"bs{cid:03d}", keys, kst=sts, nby=len(sts) - 1, reverse=[False] * (len(sts) - 1) + [revs[-1]],
                     vals=[v], reducers=[("sum", 0), ("count", 0)])
            cid += 1

# C4-shaped: (int64 with constant low 33 bits, int32) keys
n = 4096
k1 = (rng.integers(0, 50, n).astype(np.int64) << 33)
k2 = rng.integers(0, 40, n).astype(np.int32)
vs = [with_na(rng.standard_normal(n), 0.01, FLOAT64) for _ in range(3)]
add_case("c4_shape", [k1, k2], nby=2, vals=vs,
         reducers=[(op, vi) for vi in range(3) for op in ("mean", "min", "max", "count")])
# C2-shaped
n = 20000
add_case("c2_shape", [rng.integers(0, 1000, n).astype(np.int32)], nby=1, vals=[rng.random(n)],
         reducers=[("sum", 0)])

save_parts(arrays, os.path.join(HERE, "golden_v1"))
with open(os.path.join(HERE, "golden_v1.json"), "w") as fh:
    json.dump({"reference": "h2oai/datatable @ 3611640 (1.2.0a), sort.new=False",
               "datatable_version": dt.__version__, "cases": manifest}, fh, indent=0)
print(f"{len(manifest)} cases, {sum(a.nbytes for a in arrays.values())/1e6:.2f} MB raw")
