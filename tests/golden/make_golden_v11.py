#!/usr/bin/env python
"""
Generates tests/golden/golden_v11.{npz,json} by running the *reference itself* (the unmodified build staged by
oracle/build_ref.sh) on DT[i, j] with `i` a boolean or integer column, a list or a range:

    PYTHONPATH=oracle/_ref python tests/golden/make_golden_v11.py

    f.b, g.b          FExpr_Func::evaluate_i (expr/fexpr_func.cc:61-73): the rows whose bool8 value is true; g.b
                      through a join with unmatched rows
    Frame / numpy     FExpr_Frame::evaluate_i (expr/fexpr_frame.cc:159-198): bool8 (with NA, all true, all false,
                      one row, no rows) and int8 .. int64 selectors (NA, repeats, unsorted), and their errors
    list / tuple      FExpr_List::evaluate_i (expr/fexpr_list.cc:225-316): ints, bools, None, slices, frames, f.b
    range             FExpr_Literal_Range::evaluate_i (expr/fexpr_literal_range.cc:87-96)
    j                 every j kind on a selection that holds NA rows, but median and qcut: both crash the reference
                      there, so they are pinned on a boolean selection
    refusals          every form under by() and under sort()

Every case stores the frames (X, J and the selector frames S[...] / arrays A[...]), the query as source text over
X, J, S, A, dt, f, g, join, by, sort, and the reference's result names, stypes and columns, or its error type and
text.  Cases that select plain columns also store `restate`: the selector as source text for tests/rows_reference.py
and the result's columns of X.  The reference cannot travel to the GPU box, so the vectors are committed.
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
arrays, manifest = {}, []
rng = np.random.default_rng(20261017)


def column(a, st, name):
    a = np.ascontiguousarray(a, dtype=NPT[st])
    if st in FLOATS:
        return dt.Frame({name: a})
    return dt.Frame({name: [None if x == NA[st] else (bool(x) if st == BOOL else int(x)) for x in a.tolist()]},
                    stypes={name: DTST[st]})


def frame(cols):
    if not cols:
        return dt.Frame()
    return dt.cbind(*[column(a, st, nm) for nm, (a, st) in cols.items()])


def to_np(fr, i):
    col = fr[:, i]
    st = ST_OF[col.stypes[0]]
    if st in FLOATS:
        return (col.to_numpy().reshape(-1).astype(NPT[st]) if col.nrows else np.zeros(0, NPT[st])), st
    return np.array([NA[st] if x is None else int(x) for x in col.to_list()[0]], dtype=NPT[st]), st


def with_na(a, st, p):
    a = np.asarray(a).astype(NPT[st])
    a[rng.random(len(a)) < p] = np.nan if st in FLOATS else NA[st]
    return a


def xframe(n, pna=0.1):
    return {"k": (with_na(rng.integers(0, 4, n), INT32, pna), INT32),
            "v": (with_na(rng.integers(-200, 200, n) / 4, FLOAT64, pna), FLOAT64),
            "q": (with_na(rng.integers(-20, 20, n), INT32, pna), INT32),
            "w": (with_na(rng.integers(-40, 40, n) / 2, FLOAT32, pna), FLOAT32),
            "b": (with_na(rng.integers(0, 2, n), BOOL, pna), BOOL),
            "one": (np.ones(n, np.int8), BOOL),
            "zero": (np.zeros(n, np.int8), BOOL)}


def case(name, X, query, S=None, A=None, J=None, jkey=(), restate=None):
    """X, J, S[nm]: {column: (array, stype)}; A[nm]: numpy arrays; query: source text"""
    S, A = S or {}, A or {}
    c = {"name": name, "x": {nm: st for nm, (_, st) in X.items()}, "query": query,
         "s": {nm: {cn: st for cn, (_, st) in cols.items()} for nm, cols in S.items()}, "a": sorted(A),
         "j": {nm: st for nm, (_, st) in (J or {}).items()}, "jkey": list(jkey)}
    if restate is not None:
        c["restate"] = restate
    for nm, (a, st) in X.items():
        arrays[f"{name}.x.{nm}"] = np.ascontiguousarray(a, NPT[st])
    for nm, (a, st) in (J or {}).items():
        arrays[f"{name}.j.{nm}"] = np.ascontiguousarray(a, NPT[st])
    for snm, cols in S.items():
        for nm, (a, st) in cols.items():
            arrays[f"{name}.s.{snm}.{nm}"] = np.ascontiguousarray(a, NPT[st])
    for nm, a in A.items():
        arrays[f"{name}.a.{nm}"] = a
    env = {"X": frame(X), "S": {nm: frame(cols) for nm, cols in S.items()}, "A": A, "dt": dt, "f": f, "g": g,
           "join": join, "by": by, "sort": sort, "np": np}
    if name == "err.frame_keyed":
        env["S"]["s"].key = "C0"
    if J is not None:
        env["J"] = frame(J)
        env["J"].key = list(jkey)
    if name.startswith("err."):
        err = error_of(query, env)
        if err is None:
            c["reference_crash"] = True
        else:
            c["error"] = err
        manifest.append(c)
        return
    R = eval(query, env)
    c["names"], c["stypes"] = list(R.names), []
    for i in range(R.ncols):
        v, st = to_np(R, i)
        arrays[f"{name}.r{i}"] = v
        c["stypes"].append(st)
    c["nrows"] = R.nrows
    manifest.append(c)


def error_of(query, env):
    """[type, text] of the error the query raises, or None when the process dies in the query: then the case records
    `reference_crash`, and the tests check the text the reference's source writes (tests/rows_reference.py,
    SOURCE_ERRORS).  The query runs in a forked child, so that only the child dies."""
    rd, wr = os.pipe()
    pid = os.fork()
    if pid == 0:
        os.close(rd)
        try:
            eval(query, env)
            out = ["", "no error"]
        except Exception as e:                                  # noqa: BLE001
            out = [type(e).__name__, str(e)]
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
    if not data:                                                # the child died inside the query
        return None
    out = json.loads(data)
    assert out[0], query
    return out


N = 300
X0 = xframe(N)


def sel_frame(st, vals):
    return {"C0": (np.asarray(vals).astype(NPT[st]), st)}


# ---- boolean columns of X: NA, all true, all false; one row; no rows ---------------------------------------------
for col in ("b", "one", "zero"):
    case(f"mask.{col}", X0, f"X[f.{col}, :]", restate={"sel": f"M('{col}')", "cols": None})
case("mask.cols", X0, "X[f.b, [f.v, f.k]]", restate={"sel": "M('b')", "cols": ["v", "k"]})
X1 = xframe(1, 0)
case("mask.onerow", X1, "X[f.b, :]", restate={"sel": "M('b')", "cols": None})
X1n = {k: (a.copy(), st) for k, (a, st) in X1.items()}
X1n["b"] = (np.array([NA[BOOL]], np.int8), BOOL)
case("mask.onerow_na", X1n, "X[f.b, :]", restate={"sel": "M('b')", "cols": None})
Xe = xframe(0)
case("mask.norows", Xe, "X[f.b, :]", restate={"sel": "M('b')", "cols": None})
case("mask.norows_sum", Xe, "X[f.b, dt.sum(f.v)]")
case("err.mask_type", X0, "X[f.q, :]")
case("err.mask_float", X0, "X[f.v, :]")

# ---- selector frames: bool8 and every integer stype -----------------------------------------------------------------
sb = with_na(rng.integers(0, 2, N), BOOL, 0.2)
case("frame.bool", X0, "X[S['s'], :]", S={"s": sel_frame(BOOL, sb)}, restate={"sel": "F('s')", "cols": None})
case("frame.bool_true", X0, "X[S['s'], :]", S={"s": sel_frame(BOOL, np.ones(N))}, restate={"sel": "F('s')", "cols": None})
case("frame.bool_false", X0, "X[S['s'], :]", S={"s": sel_frame(BOOL, np.zeros(N))},
     restate={"sel": "F('s')", "cols": None})
for st, tag in ((INT8, "i8"), (INT16, "i16"), (INT32, "i32"), (INT64, "i64")):
    hi = 127 if st == INT8 else N
    idx = with_na(rng.integers(0, hi, 80), st, 0.1)
    idx[:3] = idx[5]                                              # repeats
    case(f"frame.{tag}", X0, "X[S['s'], :]", S={"s": sel_frame(st, idx)}, restate={"sel": "F('s')", "cols": None})
    if st != INT8:
        case(f"err.frame_{tag}_neg", X0, "X[S['s'], :]", S={"s": sel_frame(st, np.concatenate([idx[:5], [-3]]))})
        case(f"err.frame_{tag}_big", X0, "X[S['s'], :]", S={"s": sel_frame(st, np.concatenate([idx[:5], [N + 7]]))})
case("err.frame_i8_big", X1, "X[S['s'], :]", S={"s": sel_frame(INT8, [0, 0, 5])})
case("frame.i32_allna", X0, "X[S['s'], :]", S={"s": sel_frame(INT32, [NA[INT32]] * 4)},
     restate={"sel": "F('s')", "cols": None})
case("frame.i32_empty", X0, "X[S['s'], :]", S={"s": sel_frame(INT32, np.zeros(0))},
     restate={"sel": "F('s')", "cols": None})
case("frame.i32_sum", X0, "X[S['s'], [dt.sum(f.v), dt.count(), dt.count(f.q)]]",
     S={"s": sel_frame(INT32, with_na(rng.integers(0, N, 50), INT32, 0.2))})
case("err.frame_len", X0, "X[S['s'], :]", S={"s": sel_frame(BOOL, np.ones(N - 1))})
case("err.frame_len1", X0, "X[S['s'], :]", S={"s": sel_frame(BOOL, np.ones(1))})
case("err.frame_float", X0, "X[S['s'], :]", S={"s": sel_frame(FLOAT64, np.ones(3))})
case("err.frame_2cols", X0, "X[S['s'], :]", S={"s": {"a": (np.ones(3, np.int32), INT32), "b": (np.ones(3, np.int32), INT32)}})
case("err.frame_keyed", X0, "X[S['s'], :]", S={"s": sel_frame(INT32, [1, 2])})
# ---- numpy arrays -------------------------------------------------------------------------------------------------
case("numpy.bool", X0, "X[A['m'], :]", A={"m": rng.random(N) < 0.3}, restate={"sel": "N('m')", "cols": None})
case("numpy.i64", X0, "X[A['m'], :]", A={"m": rng.integers(0, N, 40)}, restate={"sel": "N('m')", "cols": None})
case("numpy.i32", X0, "X[A['m'], [f.q]]", A={"m": rng.integers(0, N, 40).astype(np.int32)},
     restate={"sel": "N('m')", "cols": ["q"]})
case("err.numpy_2d", X0, "X[A['m'], :]", A={"m": np.ones((3, 2), np.int64)})
case("err.numpy_float", X0, "X[A['m'], :]", A={"m": np.ones(3)})

# ---- lists and ranges over a small frame ---------------------------------------------------------------------------
Xs = xframe(8, 0.2)
LISTS = {
    "ints": "[0, -1, None, 3, 3, 7]", "mixed": "[0, -1, None, slice(2, 4)]", "none_first": "[None, 1]",
    "tuple": "(1, 2)", "empty": "[]", "nones": "[None]", "all_then_int": "[slice(None), 1]",
    "slices": "[slice(6, 1, -2), slice(None, 3), range(1, 3)]", "bools": "[True, False, False, True] * 2",
    "frames": "[slice(1, 3), S['s'], f.b, 7, A['m']]", "range_item": "[range(1, 3)]",
    "bools_all": "[True] * 8",
}
BADLISTS = {
    "int_bool": "[1, True]", "bool_int": "[True, 1]", "bool_len": "[True, False]", "float": "[1.5]",
    "int_float": "[1, 1.5]", "slice_float": "[slice(1, 3), 1.5]", "int_frame": "[1, S['s']]",
    "slice_bool": "[slice(1, 3), True]", "index": "[1, 9]", "row": "[slice(1, 2), 9]", "nested": "[[1]]",
    "none_bool": "[None, True]", "bool_none": "[True, False, None, True] * 2", "bool_elem": "[True, 1, False, True, True, True, True, True]",
}
SX = {"s": sel_frame(INT16, [5, NA[INT16], 0])}
AX = {"m": np.array([True, False] * 4)}
for nm, q in LISTS.items():
    case(f"list.{nm}", Xs, f"X[{q}, :]", S=SX, A=AX,
         restate={"sel": q.replace("S['s']", "F('s')").replace("A['m']", "N('m')").replace("f.b", "M('b')"),
                  "cols": None})
for nm, q in BADLISTS.items():
    case(f"err.list_{nm}", Xs, f"X[{q}, :]", S=SX, A=AX)
RANGES = {"neg": "range(7, 0, -3)", "negneg": "range(-1, -8, -2)", "step": "range(0, 8, 3)", "empty": "range(3, 3)",
          "back": "range(4, 0, -2)"}
for nm, q in RANGES.items():
    case(f"range.{nm}", Xs, f"X[{q}, :]", restate={"sel": q, "cols": None})
case("range.sum", Xs, "X[range(7, 0, -3), dt.sum(f.v)]")
case("err.range", Xs, "X[range(10, 0, -3), :]")
case("err.range_mixed", Xs, "X[range(-2, 3), :]")
case("err.range1", X1, "X[range(0, 2), :]")
case("err.bool_literal", Xs, "X[True, :]")

# ---- every j kind on a selection with NA rows (an int32 selector with NA) -----------------------------------------
SNA = {"s": sel_frame(INT32, with_na(rng.integers(0, N, 60), INT32, 0.15))}
JK = {
    "all": "X[S['s'], :]",
    "cols": "X[S['s'], [f.v, f.b, f.k]]",
    "reducers": ("X[S['s'], [dt.sum(f.v), dt.mean(f.q), dt.min(f.w), dt.max(f.k), dt.count(f.v), dt.count(), "
                 "dt.countna(f.q), dt.first(f.v), dt.last(f.q), dt.sd(f.v), dt.prod(f.k), dt.nunique(f.k)]]"),
    "covcorr": "X[S['s'], [dt.cov(f.v, f.q), dt.corr(f.w, f.v)]]",
    "cumulative": "X[S['s'], [dt.cumsum(f.v), dt.cumprod(f.k), dt.cummin(f.q), dt.cummax(f.w)]]",
    "shift": "X[S['s'], [dt.shift(f.v), dt.shift(f.q, -2)]]",
    "fillna": "X[S['s'], [dt.fillna(f.v), dt.fillna(f.q, reverse=True)]]",
    "cumcount": "X[S['s'], [dt.cumcount(), dt.ngroup(), f.q]]",
    "mask_reducers": "X[f.b, [dt.sum(f.v), dt.count(), dt.median(f.q)]]",
    "mask_cumsum": "X[f.b, dt.cumsum(f.v)]",
    "mask_qcut": "X[f.b, dt.qcut(f.v, nquantiles=5)]",
}
for nm, q in JK.items():
    case(f"j.{nm}", X0, q, S=SNA,
         restate={"sel": "F('s')", "cols": ["v", "b", "k"]} if nm == "cols" else None)

# ---- refusals under by() / sort() ---------------------------------------------------------------------------------
for mod in ("by(f.k)", "sort(f.q)"):
    t = mod[:2]
    case(f"err.{t}_mask", X0, f"X[f.b, :, {mod}]")
    case(f"err.{t}_frame", X0, f"X[S['s'], :, {mod}]", S={"s": sel_frame(INT32, [1])})
    case(f"err.{t}_numpy", X0, f"X[A['m'], :, {mod}]", A={"m": np.array([1, 2])})
    case(f"err.{t}_list", X0, f"X[[1, 2], :, {mod}]")
    case(f"err.{t}_range", X0, f"X[range(0, 3), :, {mod}]")
case("err.by_mask_sum", X0, "X[f.b, dt.sum(f.v), by(f.k)]")

# ---- g.b through a join with unmatched rows -------------------------------------------------------------------------
JKEYS = np.arange(0, 3, dtype=np.int32)                            # X's k has 0..3 and NA: 3 and NA match nothing
J0 = {"k": (JKEYS[::-1].copy(), INT32), "active": (np.array([1, NA[BOOL], 1], np.int8), BOOL),
      "price": (np.array([1.5, 2.5, np.nan]), FLOAT64)}
for nm, q in {"all": "X[g.active, :, join(J)]", "cumsum": "X[g.active, dt.cumsum(f.v), join(J)]",
              "sum": "X[g.active, [dt.sum(g.price), dt.count()], join(J)]", "mask_f": "X[f.b, [f.v, g.price], join(J)]",
              "err.join_type": "X[g.price, :, join(J)]"}.items():
    case(nm if nm.startswith("err.") else f"join.{nm}", X0, q, J=J0, jkey=["k"])

np.savez_compressed(os.path.join(HERE, "golden_v11.npz"), **arrays)
with open(os.path.join(HERE, "golden_v11.json"), "w") as fh:
    json.dump({"generator": "tests/golden/make_golden_v11.py",
               "datatable_version": dt.__version__.split("+")[0],
               "cases": manifest}, fh, indent=0)
print(f"{len(manifest)} cases, {sum(1 for c in manifest if 'error' in c)} errors, "
      f"{sum(a.nbytes for a in arrays.values()) / 1e6:.2f} MB raw")
