#!/usr/bin/env python
"""
Generates tests/golden/golden_v10.{npz,json} by running the *reference itself* (the unmodified build staged by
oracle/build_ref.sh) on DT[i, j, join(J), by(), sort()] -- group, sort and reduce over the joined frame's columns:

    PYTHONPATH=oracle/_ref python tests/golden/make_golden_v10.py

EvalContext::evaluate (eval_context.cc:144-164): natural_join first, then group / sort (by() and sort() may name g.
columns), then `i`, then j; a g. column is J's column seen through (i / sort RowIndex) x (join RowIndex), and j = :
is X's columns then J's non-key columns without the group columns (fexpr_literal_sliceall.cc:55-66).

    J key stypes   every one (bool .. float64, date32, time64), and int X against float J and the reverse
    J key layouts  dense (with a leading NA key), dense with one gap, sparse, 2 and 3 key columns
    X keys         NA, unmatched, fractions and values outside J's type
    empty          X of 0 rows, J of 0 rows
    queries        by(f.k) with every reducer over g. columns and cov / corr of an f. and a g. column; by(g.x) and
                   by(f.a, g.b) over f. columns; by(g.x) + sort(f.y); sort(-g.x); integer and slice i with and
                   without by(); j = : under by(g.x); [f.a, g.b]; cumsum / shift / fillna / cumcount over g. columns
                   under by(); g. without a join and a missing g. column (the reference's errors)

median and qcut of a g. column crash the reference (both sort the joined view inside its groups), so they have no
golden; tests/test_gpu_join_groupby.py checks them against the same functions over the joined column made plain.

Every case stores X and J (J unsorted: the key is set on both sides), the query as source text over X, J, dt, f, g,
join, by, sort, and the reference's result names, stypes and columns, or its error type and text.  Cases whose j is
one list of reducers under by() also store `restate` (by keys, reducers) for the numpy restatement of
tests/test_oracle_golden_v10.py.  The reference cannot travel to the GPU box, so the vectors are committed.
"""
import json
import os

import numpy as np

import datatable as dt
from datatable import f, g, join, by, sort

HERE = os.path.dirname(os.path.abspath(__file__))
BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64 = 1, 2, 3, 4, 5, 6, 7, 17, 18
FLOATS = (FLOAT32, FLOAT64)
NPT = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
       FLOAT32: np.float32, FLOAT64: np.float64, DATE32: np.int32, TIME64: np.int64}
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
DTST = {BOOL: dt.bool8, INT8: dt.int8, INT16: dt.int16, INT32: dt.int32, INT64: dt.int64,
        FLOAT32: dt.float32, FLOAT64: dt.float64, DATE32: dt.int32, TIME64: dt.int64}
ST_OF = {dt.bool8: BOOL, dt.int8: INT8, dt.int16: INT16, dt.int32: INT32, dt.int64: INT64, dt.float32: FLOAT32,
         dt.float64: FLOAT64, dt.stype.date32: DATE32, dt.stype.time64: TIME64}
TAG = {BOOL: "bool", INT8: "i8", INT16: "i16", INT32: "i32", INT64: "i64", FLOAT32: "f32", FLOAT64: "f64",
       DATE32: "date32", TIME64: "time64"}
arrays, manifest = {}, []
rng = np.random.default_rng(20261017)


def column(a, st, name):
    """single-column reference Frame; floats keep their bits, integer NA sentinels become None"""
    a = np.ascontiguousarray(a, dtype=NPT[st])
    if st in FLOATS:
        return dt.Frame({name: a})
    fr = dt.Frame({name: [None if x == NA[st] else (bool(x) if st == BOOL else int(x)) for x in a.tolist()]},
                  stypes={name: DTST[st]})
    if st == DATE32:
        fr[name] = fr[:, dt.as_type(f[name], dt.Type.date32)]
    elif st == TIME64:
        fr[name] = fr[:, dt.as_type(f[name], dt.Type.time64)]
    return fr


def frame(cols):
    if not cols:
        return dt.Frame()
    return dt.cbind(*[column(a, st, nm) for nm, (a, st) in cols.items()])


def to_np(fr, i):
    """column i of a reference Frame as its stype's storage (NA as the sentinel) and its stype"""
    col = fr[:, i]
    st = ST_OF[col.stypes[0]]
    if st in FLOATS:
        return (col.to_numpy().reshape(-1).astype(NPT[st]) if col.nrows else np.zeros(0, NPT[st])), st
    if st in (DATE32, TIME64):
        col = col[:, dt.as_type(f[0], DTST[st])]
    return np.array([NA[st] if x is None else int(x) for x in col.to_list()[0]], dtype=NPT[st]), st


def case(name, X, J, jkey, query, restate=None):
    """X, J: {name: (array, stype)}; query: source text over X, J, dt, f, g, join, by, sort"""
    c = {"name": name, "x": {nm: st for nm, (_, st) in X.items()}, "j": {nm: st for nm, (_, st) in J.items()},
         "jkey": list(jkey), "query": query}
    if restate is not None:
        c["restate"] = restate
    for nm, (a, st) in X.items():
        arrays[f"{name}.x.{nm}"] = np.ascontiguousarray(a, NPT[st])
    for nm, (a, st) in J.items():
        arrays[f"{name}.j.{nm}"] = np.ascontiguousarray(a, NPT[st])
    XF, JF = frame(X), frame(J)
    JF.key = list(jkey)
    try:
        R = eval(query, {"X": XF, "J": JF, "dt": dt, "f": f, "g": g, "join": join, "by": by, "sort": sort})
    except Exception as e:                                      # noqa: BLE001
        c["error"] = [type(e).__name__, str(e)]
        manifest.append(c)
        return
    c["names"], c["stypes"] = list(R.names), []
    for i in range(R.ncols):
        v, st = to_np(R, i)
        arrays[f"{name}.r{i}"] = v
        c["stypes"].append(st)
    c["nrows"] = R.nrows
    manifest.append(c)


def na(st):
    return np.nan if st in FLOATS else NA[st]


def with_na(a, st, p):
    a = a.astype(NPT[st])
    a[rng.random(len(a)) < p] = na(st)
    return a


def values(st, n, lo=-50, hi=50):
    if st == BOOL:
        return rng.integers(0, 2, n).astype(np.int8)
    if st in FLOATS:
        return (rng.integers(lo * 4, hi * 4, n) / 4).astype(NPT[st])
    return rng.integers(lo, hi, n).astype(NPT[st])


def jpayload(nj):
    """J's non-key columns: region (int32, few values, NA), price (float64, NA), w (float32), flag (bool)"""
    return {"region": (with_na(rng.integers(0, 4, nj), INT32, 0.15), INT32),
            "price": (with_na(values(FLOAT64, nj), FLOAT64, 0.15), FLOAT64),
            "w": (with_na(values(FLOAT32, nj), FLOAT32, 0.1), FLOAT32),
            "flag": (with_na(values(BOOL, nj), BOOL, 0.1), BOOL)}


def xpayload(nx):
    return {"qty": (with_na(values(INT32, nx, 0, 20), INT32, 0.05), INT32),
            "a": (with_na(rng.integers(0, 3, nx), INT16, 0.05), INT16),
            "v": (with_na(values(FLOAT64, nx), FLOAT64, 0.1), FLOAT64)}


SUMS = "X[:, {'s': dt.sum(g.price), 'n': dt.count(), 'c': dt.count(g.region), 'm': dt.mean(g.w), " \
       "'lo': dt.min(g.region), 'hi': dt.max(g.price)}, join(J), by(f.k)]"
SUMS_RESTATE = {"by": ["f.k"], "red": [["sum", "g.price"], ["count", None], ["count", "g.region"], ["mean", "g.w"],
                                       ["min", "g.region"], ["max", "g.price"]]}
BYG = "X[:, {'s': dt.sum(f.qty), 'n': dt.count(), 'm': dt.mean(f.v)}, join(J), by(g.region)]"
BYG_RESTATE = {"by": ["g.region"], "red": [["sum", "f.qty"], ["count", None], ["mean", "f.v"]]}


def keyed(name, jk, jst, xk, xst, queries=(SUMS, BYG), restates=(SUMS_RESTATE, BYG_RESTATE)):
    """one key column k: J's keys jk (shuffled here; the key sorts them), X's keys xk"""
    jk = np.asarray(jk)[rng.permutation(len(jk))]
    J = {"k": (jk, jst), **jpayload(len(jk))}
    X = {"k": (xk, xst), **xpayload(len(xk))}
    for qi, (q, r) in enumerate(zip(queries, restates)):
        case(f"{name}.q{qi}", X, J, ["k"], q, r)


def draw(pool, n, st, extra=()):
    return np.concatenate([rng.choice(np.asarray(pool), n), np.asarray(extra)]).astype(NPT[st])


# ---- J key stypes: dense keys with a leading NA key (the direct-address path), X of the same stype -------------
for st in (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64):
    if st == BOOL:
        jk = np.array([NA[BOOL], 0, 1], np.int8)
        xk = draw([0, 1, NA[BOOL]], 120, st)
    else:
        base = {INT64: 2**40, TIME64: 10**12, DATE32: 18000}.get(st, -5)
        jk = np.concatenate([[na(st)], base + np.arange(40)]).astype(NPT[st])
        xk = draw(np.concatenate([base + np.arange(-3, 44), [na(st)]]), 160, st)
    keyed(f"jst.{TAG[st]}", jk, st, xk, st)
# dense keys without an NA key
keyed("dense.nona", np.arange(100, 160, dtype=np.int32), INT32, draw(np.arange(95, 165), 200, INT32, [NA[INT32]]),
      INT32)
# one gap in the dense range: the binary search; one-row J; an all-NA J key
keyed("gap.i32", np.concatenate([[NA[INT32]], np.arange(0, 20), np.arange(21, 40)]).astype(np.int32), INT32,
      draw(np.concatenate([np.arange(-2, 42), [NA[INT32]]]), 200, INT32), INT32)
keyed("gap.i64", np.concatenate([np.arange(0, 30), [31]]).astype(np.int64), INT64,
      draw(np.arange(-2, 34), 150, INT64, [NA[INT64]]), INT64)
keyed("one.i32", np.array([7], np.int32), INT32, draw([6, 7, 8, NA[INT32]], 40, INT32), INT32)
keyed("onena.i32", np.array([NA[INT32]], np.int32), INT32, draw([6, 7, NA[INT32]], 40, INT32), INT32)
# sparse keys
sp = np.unique(rng.integers(-10**6, 10**6, 300)).astype(np.int32)
keyed("sparse.i32", sp, INT32, np.concatenate([rng.choice(sp, 300), rng.integers(-10**6, 10**6, 100),
                                                [NA[INT32]] * 5]).astype(np.int32), INT32)
sp64 = np.unique(rng.integers(-2**62, 2**62, 200, dtype=np.int64))
keyed("sparse.i64", sp64, INT64, np.concatenate([rng.choice(sp64, 200), sp64[:20] + 1, [NA[INT64]]]), INT64)
spf = np.concatenate([[np.nan], np.unique(rng.integers(-400, 400, 120)) / 4])
keyed("sparse.f64", spf, FLOAT64, np.concatenate([rng.choice(spf, 200), [0.125, 1e9, -np.inf]]), FLOAT64)
# mixed key stypes: int X against float J, float X against int J (fractions, inf, values outside J's type)
keyed("mixed.i32_f64", np.concatenate([[np.nan], np.arange(-10, 30), [0.5, 40.25]]), FLOAT64,
      draw(np.concatenate([np.arange(-12, 45), [NA[INT32]]]), 200, INT32), INT32)
keyed("mixed.f64_i32", np.concatenate([[NA[INT32]], np.arange(-10, 30)]).astype(np.int32), INT32,
      draw(np.concatenate([np.arange(-12, 33), [0.5, -3.25, np.inf, -np.inf, 2.0**40, np.nan]]), 220, FLOAT64),
      FLOAT64)
keyed("mixed.f32_i16", np.concatenate([[NA[INT16]], np.arange(-5, 25)]).astype(np.int16), INT16,
      draw(np.concatenate([np.arange(-7, 27), [2.0**15, -2.0**15 - 1, 1.5, np.nan]]), 200, FLOAT32), FLOAT32)
keyed("mixed.i64_i16", np.concatenate([[NA[INT16]], np.arange(-5, 25)]).astype(np.int16), INT16,
      draw(np.concatenate([np.arange(-7, 27), [2**15, 2**40, -2**15, NA[INT64]]]), 200, INT64), INT64)
keyed("mixed.i8_i64", np.arange(-20, 20, dtype=np.int64), INT64,
      draw(np.concatenate([np.arange(-25, 25), [NA[INT8]]]), 150, INT8), INT8)
# empty X, empty J
keyed("empty.x", np.arange(10, dtype=np.int32), INT32, np.zeros(0, np.int32), INT32)
keyed("empty.j", np.zeros(0, np.int32), INT32, draw([1, 2, NA[INT32]], 50, INT32), INT32)


# ---- multi-key joins: J = a subset of a product with NA in every column ------------------------------------------
def multi(name, jsts, xsts):
    sets = [np.concatenate([[na(st)], np.arange(4)]).astype(NPT[st]) for st in jsts]
    grids = np.meshgrid(*[np.arange(len(s)) for s in sets], indexing="ij")
    jk = [s[gr.reshape(-1)] for s, gr in zip(sets, grids)]
    keep = rng.random(len(jk[0])) < 0.7
    perm = rng.permutation(int(keep.sum()))
    jk = [a[keep][perm] for a in jk]
    keys = [f"k{i}" for i in range(len(jsts))]
    J = {**{nm: (a, st) for nm, a, st in zip(keys, jk, jsts)}, **jpayload(len(jk[0]))}
    X = {**{nm: (draw(np.concatenate([np.arange(-1, 6), [na(st)]]), 250, st), st) for nm, st in zip(keys, xsts)},
         **xpayload(250)}
    q = SUMS.replace("by(f.k)", f"by({', '.join('f.' + k for k in keys)})")
    case(f"{name}.q0", X, J, keys, q, {**SUMS_RESTATE, "by": [f"f.{k}" for k in keys]})
    case(f"{name}.q1", X, J, keys, BYG, BYG_RESTATE)


multi("multi.i32_i64", (INT32, INT64), (INT32, INT64))
multi("multi.i16_f64_i8", (INT16, FLOAT64, INT8), (INT32, FLOAT64, INT8))


# ---- the query shapes over one X / J pair: dense J with an NA key, X with NA and unmatched keys --------------------
JK = np.concatenate([[NA[INT32]], np.arange(0, 60)]).astype(np.int32)
J0 = {"k": (JK[rng.permutation(len(JK))], INT32), **jpayload(len(JK))}
X0 = {"k": (draw(np.concatenate([np.arange(-3, 64), [NA[INT32]]]), 300, INT32), INT32), **xpayload(300),
      "region": (with_na(rng.integers(0, 3, 300), INT32, 0.1), INT32)}    # X's own region: f.region is not g.region
JOINED = {
    "reducers": ("X[:, [dt.sum(g.price), dt.prod(g.w), dt.mean(g.price), dt.min(g.w), dt.max(g.region), "
                 "dt.count(g.price), dt.countna(g.price), dt.first(g.price), dt.last(g.region), dt.sd(g.price), "
                 "dt.nunique(g.region)], join(J), by(f.k)]"),      # median of a g. column crashes the reference
    "reducers_bool": "X[:, [dt.sum(g.flag), dt.min(g.flag), dt.max(g.flag), dt.mean(g.flag)], join(J), by(f.a)]",
    "covcorr": "X[:, [dt.cov(f.v, g.price), dt.corr(f.v, g.price), dt.corr(g.w, f.qty)], join(J), by(f.a)]",
    "byg": "X[:, {'s': dt.sum(f.qty), 'n': dt.count(), 'md': dt.median(f.v)}, join(J), by(g.region)]",
    "byfg": "X[:, [dt.mean(f.qty), dt.count(), dt.sum(g.price)], join(J), by(f.a, g.region)]",
    "byg_desc": "X[:, dt.sum(f.v), join(J), by(-g.region)]",
    "byg_sort": "X[:, :, join(J), by(g.region), sort(f.qty)]",
    "sort_g": "X[:, :, join(J), sort(-g.price)]",
    "sort_gf": "X[:, [f.k, g.price, f.qty], join(J), sort(g.region, -f.qty)]",
    "i_int_byg": "X[1, :, join(J), by(g.region)]",
    "i_slice_byg": "X[1:4, :, join(J), by(g.region)]",
    "i_slice_byg_red": "X[:3, dt.sum(g.price), join(J), by(g.region)]",
    "i_int": "X[7, :, join(J)]",
    "i_slice": "X[5:40:3, [f.qty, g.price, g.region], join(J)]",
    "i_neg": "X[-1, :, join(J)]",
    "all_byg": "X[:, :, join(J), by(g.region)]",
    "all": "X[:, :, join(J)]",
    "plain": "X[:, [f.a, g.price, g.k, f.k, g.region, f.region], join(J)]",
    "f_fallback": "X[:, [f.price, f.w], join(J)]",
    "cumsum": "X[:, [dt.cumsum(g.price), dt.cumsum(g.region)], join(J), by(f.a)]",
    "shift": "X[:, [dt.shift(g.price), dt.shift(g.region, -2)], join(J), by(f.a)]",
    "fillna": "X[:, [dt.fillna(g.price), dt.fillna(g.w, reverse=True)], join(J), by(f.a)]",
    "cumcount": "X[:, [dt.cumcount(), g.region], join(J), by(g.region)]",
    "err_nojoin": "X[:, g.price]",
    "err_missing": "X[:, g.nope, join(J)]",
}
for nm, q in JOINED.items():
    case(f"query.{nm}", X0, J0, ["k"], q,
         {"by": ["f.a", "g.region"], "red": [["mean", "f.qty"], ["count", None], ["sum", "g.price"]]}
         if nm == "byfg" else None)

np.savez_compressed(os.path.join(HERE, "golden_v10.npz"), **arrays)
with open(os.path.join(HERE, "golden_v10.json"), "w") as fh:
    json.dump({"generator": "tests/golden/make_golden_v10.py",
               "datatable_version": dt.__version__.split("+")[0],
               "cases": manifest}, fh, indent=0)
print(f"{len(manifest)} cases, {sum(1 for c in manifest if 'error' in c)} errors, "
      f"{sum(a.nbytes for a in arrays.values()) / 1e6:.2f} MB raw")
