#!/usr/bin/env python
"""
Generates tests/golden/golden_v13.{npz,json} by running the *reference itself* (the unmodified build staged by
oracle/build_ref.sh) on queries over zero rows:

    PYTHONPATH=oracle/_ref python tests/golden/make_golden_v13.py

    red.<st>.*        a 0-row frame without by(): every reducer, and all of them in one j (Groupby::single_group(0),
                      groupby.cc:60-68: one empty group, so one result row)
    by.<st>.*         a 0-row frame with by() / sort(): reducers, a plain column, every na_position
    row.<st>.*        row functions over 0 rows, with and without by(): cumsum .. cummax, shift, fillna, cumcount,
                      ngroup, qcut, cut(nbins=), cut(bins=).  The reference dies in fillna over 0 rows and raises
                      KeyError('stype.void') for qcut under by() over 0 rows: those cases record that, and the
                      tests hold the engine to the empty result instead
    sel.<i>.<j>       empty selections of a non-empty frame (an all-false and an all-NA mask, [], range(0), 5:5, a 0-row
                      selector frame) with a reducer, a row-function and a plain-column j; the mask taken from g.
    iby.*             an integer slice under by() that empties every group
    join.*, set.*     a join with a 0-row X and with a 0-row J; union / intersect / setdiff / symdiff / unique with an
                      empty operand; nunique, mode and nmodal of a 0-row frame

<st> runs over bool8, int8 .. int64, float32 and float64.  Every case stores its frames (X, J and the selector frames
S[...]), the query as source text over X, J, S, dt, f, g, join, by, sort, and the reference's result names, stypes,
row count and columns, or its error type and text.  Each query runs in a forked child, so that a query that kills
the process is recorded as `reference_crash` instead of ending the run.  The reference cannot travel to the GPU box,
so the vectors are committed.
"""
import json
import os

import numpy as np

import datatable as dt
from datatable import f, g, join, by, sort

HERE = os.path.dirname(os.path.abspath(__file__))
BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64 = 1, 2, 3, 4, 5, 6, 7
FLOATS = (FLOAT32, FLOAT64)
NPT = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32, INT64: np.int64,
       FLOAT32: np.float32, FLOAT64: np.float64}
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63}
DTST = {BOOL: dt.bool8, INT8: dt.int8, INT16: dt.int16, INT32: dt.int32, INT64: dt.int64,
        FLOAT32: dt.float32, FLOAT64: dt.float64}
ST_OF = {v: k for k, v in DTST.items()}
TAG = {BOOL: "bool8", INT8: "int8", INT16: "int16", INT32: "int32", INT64: "int64", FLOAT32: "float32",
       FLOAT64: "float64"}
arrays, manifest = {}, []
rng = np.random.default_rng(20261019)


def column(a, st, name):
    a = np.ascontiguousarray(a, dtype=NPT[st])
    if st in FLOATS:
        return dt.Frame({name: a}, stypes={name: DTST[st]})
    return dt.Frame({name: [None if x == NA[st] else (bool(x) if st == BOOL else int(x)) for x in a.tolist()]},
                    stypes={name: DTST[st]})


def frame(cols):
    return dt.cbind(*[column(a, st, nm) for nm, (a, st) in cols.items()])


def result_of(query, env):
    """("ok", names, stypes, nrows, columns as lists) or ("error", type, text); None when the child died."""
    rd, wr = os.pipe()
    pid = os.fork()
    if pid == 0:
        os.close(rd)
        try:
            R = eval(query, env)
            cols = [R[:, i].to_list()[0] for i in range(R.ncols)]
            out = ["ok", list(R.names), [TAG[ST_OF[s]] for s in R.stypes], R.nrows,
                   [[None if x is None else (float(x) if isinstance(x, float) else int(x)) for x in c] for c in cols]]
        except Exception as e:                                  # noqa: BLE001
            out = ["error", type(e).__name__, str(e)]
        os.write(wr, json.dumps(out).encode())
        os._exit(0)
    os.close(wr)
    data = b""
    while True:
        chunk = os.read(rd, 65536)
        if not chunk:
            break
        data += chunk
    os.close(rd)
    os.waitpid(pid, 0)
    return json.loads(data) if data else None


ST_TAG = {v: k for k, v in TAG.items()}


def case(name, X, query, S=None, J=None, jkey=()):
    """X, J, S[nm]: {column: (array, stype)}; query: source text"""
    S = S or {}
    c = {"name": name, "x": {nm: st for nm, (_, st) in X.items()}, "query": query,
         "s": {nm: {cn: st for cn, (_, st) in cols.items()} for nm, cols in S.items()},
         "j": {nm: st for nm, (_, st) in (J or {}).items()}, "jkey": list(jkey)}
    for nm, (a, st) in X.items():
        arrays[f"{name}.x.{nm}"] = np.ascontiguousarray(a, NPT[st])
    for nm, (a, st) in (J or {}).items():
        arrays[f"{name}.j.{nm}"] = np.ascontiguousarray(a, NPT[st])
    for snm, cols in S.items():
        for nm, (a, st) in cols.items():
            arrays[f"{name}.s.{snm}.{nm}"] = np.ascontiguousarray(a, NPT[st])
    env = {"X": frame(X), "S": {nm: frame(cols) for nm, cols in S.items()}, "dt": dt, "f": f, "g": g,
           "join": join, "by": by, "sort": sort, "np": np}
    if J is not None:
        env["J"] = frame(J)
        env["J"].key = list(jkey)
    r = result_of(query, env)
    if r is None:
        c["reference_crash"] = True
    elif r[0] == "error":
        c["error"] = r[1:]
    else:
        _, names, stypes, nrows, cols = r
        c["names"], c["stypes"], c["nrows"] = names, [ST_TAG[t] for t in stypes], nrows
        for i, (vals, st) in enumerate(zip(cols, c["stypes"])):
            na = np.nan if st in FLOATS else NA[st]
            arrays[f"{name}.r{i}"] = np.array([na if x is None else x for x in vals], dtype=NPT[st])
    manifest.append(c)


def with_na(a, st, p):
    a = np.asarray(a).astype(NPT[st])
    a[rng.random(len(a)) < p] = np.nan if st in FLOATS else NA[st]
    return a


def values(st, n):
    if st == BOOL:
        return rng.integers(0, 2, n)
    if st in FLOATS:
        return rng.integers(-40, 40, n) / 4
    return rng.integers(-50, 50, n)


ALL_ST = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)
REDUCERS = {"sum": "dt.sum(f.v)", "prod": "dt.prod(f.v)", "mean": "dt.mean(f.v)", "min": "dt.min(f.v)",
            "max": "dt.max(f.v)", "count": "dt.count(f.v)", "count0": "dt.count()", "countna": "dt.countna(f.v)",
            "first": "dt.first(f.v)", "last": "dt.last(f.v)", "sd": "dt.sd(f.v)", "median": "dt.median(f.v)",
            "nunique": "dt.nunique(f.v)", "cov": "dt.cov(f.v, f.w)", "corr": "dt.corr(f.v, f.w)"}
ROWFNS = {"cumsum": "dt.cumsum(f.v)", "cumprod": "dt.cumprod(f.v)", "cummin": "dt.cummin(f.v)",
          "cummax": "dt.cummax(f.v)", "shift": "dt.shift(f.v)", "shift_back": "dt.shift(f.v, -2)",
          "fillna": "dt.fillna(f.v, reverse=False)", "fillna_rev": "dt.fillna(f.v, reverse=True)",
          "cumcount": "dt.cumcount()", "ngroup": "dt.ngroup()", "qcut": "dt.qcut(f.v)",
          "cut_nbins": "dt.cut(f.v, nbins=4)", "cut_bins": "dt.cut(f.v, bins=[dt.Frame({'e': [-10.0, 0.0, 10.0]})])"}


def empty_frame(st):
    return {"v": (np.zeros(0), st), "w": (np.zeros(0), FLOAT64), "k": (np.zeros(0), INT32)}


# ---- a 0-row frame: reducers without by(), with by() and sort(), row functions -------------------------------------
for st in ALL_ST:
    t = TAG[st]
    E = empty_frame(st)
    for nm, q in REDUCERS.items():
        case(f"red.{t}.{nm}", E, f"X[:, {q}]")
    case(f"red.{t}.all", E, "X[:, [" + ", ".join(REDUCERS.values()) + "]]")
    case(f"by.{t}.reducers", E, "X[:, [dt.sum(f.v), dt.count(), dt.first(f.v), dt.min(f.v), dt.median(f.v), "
                                "dt.sd(f.v), dt.prod(f.v), dt.nunique(f.v)], by(f.k)]")
    case(f"by.{t}.col", E, "X[:, f.v, by(f.k)]")
    case(f"by.{t}.bykey", E, "X[:, dt.sum(f.w), by(f.v)]")
    for na in ("first", "last", "remove"):
        case(f"by.{t}.sort_{na}", E, f"X[:, :, sort(f.v, na_position='{na}')]")
    for nm, q in ROWFNS.items():
        case(f"row.{t}.{nm}", E, f"X[:, {q}]")
        case(f"row.{t}.{nm}_by", E, f"X[:, {q}, by(f.k)]")

# ---- empty selections of a non-empty frame -------------------------------------------------------------------------
N = 50
XN = {"k": (with_na(rng.integers(0, 4, N), INT32, 0.1), INT32),
      "v": (with_na(values(FLOAT64, N), FLOAT64, 0.1), FLOAT64),
      "q": (with_na(values(INT32, N), INT32, 0.1), INT32),
      "w": (with_na(values(FLOAT32, N), FLOAT32, 0.1), FLOAT32),
      "b": (with_na(values(BOOL, N), BOOL, 0.1), BOOL),
      "zero": (np.zeros(N, np.int8), BOOL),
      "nab": (np.full(N, NA[BOOL], np.int8), BOOL)}
S0 = {"s": {"C0": (np.zeros(0, np.int32), INT32)}}
SELECTORS = {"false": "f.zero", "allna": "f.nab", "list": "[]", "range": "range(0)", "slice": "5:5",
             "frame": "S['s']"}
JS = {"reducers": "[dt.sum(f.v), dt.count(), dt.first(f.q), dt.last(f.b), dt.median(f.q), dt.prod(f.q), dt.sd(f.w), "
                  "dt.min(f.w), dt.max(f.q), dt.mean(f.b), dt.countna(f.v), dt.nunique(f.q), dt.cov(f.v, f.q)]",
      "rowfns": "[dt.cumsum(f.v), dt.shift(f.q), dt.fillna(f.w, reverse=False), dt.cumcount(), dt.qcut(f.v), "
                "dt.cut(f.q)]",
      "cols": "[f.v, f.q, f.b]"}
for snm, sel in SELECTORS.items():
    for jnm, j in JS.items():
        case(f"sel.{snm}.{jnm}", XN, f"X[{sel}, {j}]", S=S0)
    case(f"sel.{snm}.all", XN, f"X[{sel}, :]", S=S0)

JKEYS = np.arange(0, 4, dtype=np.int32)
JN = {"k": (JKEYS.copy(), INT32), "active": (np.zeros(4, np.int8), BOOL),
      "price": (np.array([1.5, 2.5, np.nan, 4.0]), FLOAT64)}
case("sel.join_mask.reducers", XN, "X[g.active, [dt.sum(g.price), dt.count(), dt.first(f.v)], join(J)]", J=JN,
     jkey=["k"])
case("sel.join_mask.cols", XN, "X[g.active, [f.v, g.price], join(J)]", J=JN, jkey=["k"])
case("sel.join_mask.rowfns", XN, "X[g.active, dt.cumsum(g.price), join(J)]", J=JN, jkey=["k"])

# ---- an integer slice under by() that empties every group ----------------------------------------------------------
case("iby.first", XN, "X[100:, dt.first(f.v), by(f.k)]")
case("iby.reducers", XN, "X[100:, [dt.sum(f.v), dt.count(), dt.median(f.q)], by(f.k)]")
case("iby.int", XN, "X[100, dt.sum(f.v), by(f.k)]")
case("iby.sort", XN, "X[100:, :, sort(f.v)]")
case("iby.cols", XN, "X[100:, f.v, by(f.k)]")

# ---- joins and set operations with an empty operand; column statistics of a 0-row frame ---------------------------
XE = {"k": (np.zeros(0), INT32), "v": (np.zeros(0), FLOAT64)}
JE = {"k": (np.zeros(0), INT32), "price": (np.zeros(0), FLOAT64)}
case("join.x_empty", XE, "X[:, :, join(J)]", J=JN, jkey=["k"])
case("join.x_empty_sum", XE, "X[:, [dt.sum(g.price), dt.count()], join(J)]", J=JN, jkey=["k"])
case("join.j_empty", XN, "X[:, [f.k, g.price], join(J)]", J=JE, jkey=["k"])
case("join.j_empty_sum", XN, "X[:, [dt.sum(g.price), dt.count(g.price), dt.count()], join(J)]", J=JE, jkey=["k"])
for st in ALL_ST:
    t = TAG[st]
    SA = {"a": {"v": (with_na(values(st, 12), st, 0.2), st)}, "e": {"v": (np.zeros(0), st)}}
    for op in ("union", "intersect", "setdiff", "symdiff"):
        case(f"set.{t}.{op}_ae", XE, f"dt.{op}(S['a'], S['e'])", S=SA)
        case(f"set.{t}.{op}_ea", XE, f"dt.{op}(S['e'], S['a'])", S=SA)
        case(f"set.{t}.{op}_ee", XE, f"dt.{op}(S['e'], S['e'])", S=SA)
    case(f"set.{t}.unique", XE, "dt.unique(S['e'])", S=SA)
    for fn in ("nunique", "mode", "nmodal"):
        case(f"stat.{t}.{fn}", empty_frame(st), f"X.{fn}()")

np.savez_compressed(os.path.join(HERE, "golden_v13.npz"), **arrays)
with open(os.path.join(HERE, "golden_v13.json"), "w") as fh:
    json.dump({"generator": "tests/golden/make_golden_v13.py",
               "datatable_version": dt.__version__.split("+")[0],
               "cases": manifest}, fh, indent=0)
print(f"{len(manifest)} cases, {sum(1 for c in manifest if 'error' in c)} errors, "
      f"{sum(1 for c in manifest if 'reference_crash' in c)} crashes, "
      f"{sum(a.nbytes for a in arrays.values()) / 1e6:.2f} MB raw")
