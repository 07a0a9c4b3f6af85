"""
A numpy restatement of dt.time.year / month / day / day_of_week / hour / minute / second / nanosecond
(YearMonthDay_ColumnImpl, DayOfWeek_ColumnImpl, HourMinSec_ColumnImpl in expr/time/, and the time64 -> date32 cast
CastTime64ToDate32_ColumnImpl), and the golden_v14 query shapes it is checked against (tests/test_oracle_golden_v14.py)
and the engine with it (tests/test_gpu_time.py).  It shares no code with the engine.

Everything is computed in int64 and wrapped to int32 / int64 where the reference's add wraps, with C's truncating
division and remainder.  The day of the week of z >= -3 takes z + 3 as unsigned, as the reference's compiled code does.
"""
import json
import os

import numpy as np

BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64 = 1, 2, 3, 4, 5, 6, 7, 17, 18
NA = {BOOL: -128, INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, DATE32: -2**31, TIME64: -2**63}
NA_INT32 = -2**31
DAY_NS = 86400 * 10**9
PARTS = ["year", "month", "day", "day_of_week", "hour", "minute", "second", "nanosecond"]
CODE = {p: k + 1 for k, p in enumerate(PARTS)}           # DTB_TIME_YEAR .. DTB_TIME_NANOSECOND
CLOCK = {"hour": (3600 * 10**9, 24), "minute": (60 * 10**9, 60), "second": (10**9, 60), "nanosecond": (1, 10**9)}
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _w32(x):
    return ((x + 2**31) % 2**32) - 2**31


def _tdiv(a, b):
    q = np.abs(a) // b
    return np.where(a < 0, -q, q)


def _tmod(a, b):
    r = np.abs(a) % b
    return np.where(a < 0, -r, r)


def days_of_time64(v):
    """The time64 -> date32 cast: floor(v / DAY); v - (DAY - 1) wraps in int64 near INT64_MIN.  v: valid values."""
    v = np.asarray(v, dtype=np.int64)
    with np.errstate(over="ignore"):
        s = np.where(v < 0, v - np.int64(DAY_NS - 1), v)             # numpy int64 arrays wrap
    with np.errstate(over="ignore"):
        q = np.where(s < 0, (s + np.int64(DAY_NS - 1)) // DAY_NS, s // DAY_NS)     # C's truncating division
    return _w32(q)


def civil(z):
    """(year, month, day) of day numbers z (int32 values, as int64), with the int32 wrap-around of the conversion."""
    z = _w32(np.asarray(z, dtype=np.int64) + 719468)
    era = _tdiv(np.where(z >= 0, z, _w32(z - 146096)), 146097)
    doe = _w32(z - _w32(era * 146097))
    yoe = _tdiv(_w32(_w32(_w32(doe - _tdiv(doe, 1460)) + _tdiv(doe, 36524)) - _tdiv(doe, 146096)), 365)
    doy = _w32(doe - _w32(_w32(365 * yoe + _tdiv(yoe, 4)) - _tdiv(yoe, 100)))
    mp = _tdiv(_w32(5 * doy + 2), 153)
    m = _w32(mp + np.where(mp < 10, 3, -9))
    y = _w32(_w32(yoe + _w32(era * 400)) + (m <= 2))
    d = _w32(_w32(doy - _tdiv(_w32(153 * mp + 2), 5)) + 1)
    return y, m, d


def iso_weekday(z):
    z = np.asarray(z, dtype=np.int64)
    return np.where(z >= -3, ((z + 3) % 2**32) % 7 + 1, _tmod(z + 4, 7) + 7)


def time_part(part, v, st):
    """Part `part` (a name of PARTS) of column v of stype st (DATE32 / TIME64): int32, NA as INT32_MIN."""
    v = np.asarray(v).astype(np.int64)
    valid = v != NA[st]
    x = np.where(valid, v, 0)
    if part in CLOCK:
        scale, modulo = CLOCK[part]
        r = x % DAY_NS                                                   # the floor modulo
        res = (r // scale) % modulo
    else:
        z = days_of_time64(x) if st == TIME64 else x
        if part == "day_of_week":
            res = iso_weekday(z)
        else:
            res = civil(z)[("year", "month", "day").index(part)]
    return np.where(valid, res, NA_INT32).astype(np.int32)


def at_rows(v, st, rows):
    """Column v seen through a RowIndex: an index < 0 is an NA row."""
    v = np.asarray(v)
    if rows is None:
        return v
    rows = np.asarray(rows, dtype=np.int64)
    return np.where(rows >= 0, v[np.clip(rows, 0, max(len(v) - 1, 0))] if len(v) else NA[st], NA[st]).astype(v.dtype)


# ---- golden_v14 -----------------------------------------------------------------------------------------------------
def load_golden():
    cases = json.load(open(os.path.join(GOLDEN, "golden_v14.json")))["cases"]
    arr = dict(np.load(os.path.join(GOLDEN, "golden_v14.npz")))
    return cases, arr


def case_rows(case, arr, orc):
    """The RowIndex of a case without by() (None = every row in place), formed on the host; sort() by the C oracle."""
    name, mode, i = case["name"], case["mode"], case["i"]
    n = len(arr[name + "." + next(iter(case["stypes"]))])
    if mode in ("sort", "sortdesc"):
        flags = [orc.SORT_ONLY | (orc.DESCENDING if mode == "sortdesc" else 0)]
        order, _, _ = orc.group([arr[name + ".s"]], flags, orc.NA_FIRST)
        order = np.asarray(order, dtype=np.int64)
        if i is not None:
            start, stop, step = [i[1], i[1] + 1 if i[1] != -1 else None, 1] if i[0] == "int" else i[1]
            order = order[slice(start, stop, step)]
        return order
    if i is None:
        return None
    kind, p = i
    if kind == "slice":
        return np.arange(n)[slice(*p)]
    if kind == "int":
        return np.array([p % n])
    if kind == "bool":
        return np.flatnonzero(arr[name + "." + p] == 1)
    if kind == "frame":
        sel = arr[name + ".isel"].astype(np.int64)
        return np.where(sel == NA[INT32], -1, sel)
    if kind == "list":
        return np.array([k % n for k in p], dtype=np.int64)
    return np.array([k % n for k in range(*p)], dtype=np.int64)                # range


def joined(case, arr, col):
    """J's column `col` in X's row order (NA where X's key has no match)."""
    name = case["name"]
    k = arr[name + ".k"].astype(np.int64)
    jk = arr[name + ".J.k"].astype(np.int64)
    pos = {int(key): r for r, key in enumerate(jk)}
    idx = np.array([pos.get(int(key), -1) if key != NA[INT32] else -1 for key in k], dtype=np.int64)
    st = case["jstypes"][col]
    return at_rows(arr[name + ".J." + col], st, idx), st


def j_parts(case):
    """[(output index, part, source)] of the time-part outputs of a case without by(): source ("x", col) or ("J", col)."""
    p = case["part"]
    j = case["j"]
    if j in ("one", "dict", "cut", "qcut", "cumsum", "shift", "fillna", "cumcount", "ngroup"):
        return [(0, p, ("x", "d"))]
    if j in ("list", "tuple"):
        return [(0, p, ("x", "d")), (1, p, ("x", "t"))]
    if j == "plain":
        return [(1, p, ("x", "d"))]
    if j == "all":
        return [(k, p, ("x", c)) for k, c in enumerate(case["stypes"]) if case["stypes"][c] in (DATE32, TIME64)]
    if j == "joincol":
        return [(0, p, ("J", "d"))]
    if j == "joinlist":
        return [(0, p, ("x", "d")), (1, p, ("J", "d"))]
    if j == "parts":
        return [(k, q, ("x", "t")) for k, q in enumerate(PARTS)]
    raise KeyError(j)


def expected_parts(case, arr, orc):
    """[(output index, int32 values)] the restatement gives for the time-part outputs of a case without by()."""
    rows = case_rows(case, arr, orc)
    out = []
    for idx, part, (kind, c) in j_parts(case):
        if kind == "J":
            v, st = joined(case, arr, c)
        else:
            v, st = arr[case["name"] + "." + c], case["stypes"][c]
        out.append((idx, time_part(part, at_rows(v, st, rows), st)))
    return out


def frame_query(dtb, case, arr, device=False):
    """The case's query on the Frame of module dtb (datatable_b200)."""
    name = case["name"]
    f, g, T = dtb.f, dtb.g, dtb.time

    def mk(cols, stypes):
        fr = dtb.Frame(cols, stypes=stypes)
        return fr.to_device() if device else fr

    DT = mk({nm: arr[name + "." + nm] for nm in case["stypes"]}, case["stypes"])
    J = None
    if "jstypes" in case:
        J = mk({nm: arr[name + ".J." + nm] for nm in case["jstypes"]}, case["jstypes"])
        J.key = "k"
    return DT[query_args(dtb, case, arr, J, lambda p: mk({"C0": arr[name + ".isel"]}, {"C0": INT32}))]


def query_args(mod, case, arr, J, isel_frame):
    """(i, j, modifiers...) of the case for module mod (datatable or datatable_b200)."""
    f, g, T = mod.f, mod.g, mod.time
    P = getattr(T, case["part"])
    j = {"one": lambda: P(f.d), "list": lambda: P([f.d, f.t]), "tuple": lambda: P((f.d, f.t)),
         "all": lambda: P(f[:]), "dict": lambda: {"y": P(f.d)}, "plain": lambda: [f.d, P(f.d)],
         "cut": lambda: [P(f.d), mod.cut(f.v)], "qcut": lambda: [P(f.d), mod.qcut(f.v)],
         "cumsum": lambda: [P(f.d), mod.cumsum(f.v)], "shift": lambda: [P(f.d), mod.shift(f.v)],
         "fillna": lambda: [P(f.d), mod.fillna(f.v, reverse=True)], "cumcount": lambda: [P(f.d), mod.cumcount()],
         "ngroup": lambda: [P(f.d), mod.ngroup()], "joincol": lambda: P(g.d), "joinlist": lambda: [P(f.d), P(g.d)],
         "parts": lambda: [getattr(T, q)(f.t) for q in PARTS],
         "bysum": lambda: mod.sum(f.v), "bycount": lambda: mod.count(),
         "byall": lambda: slice(None), "bykeys": lambda: [f.v, P(f.t)]}[case["j"]]()
    i = case["i"]
    if i is None:
        rows = slice(None)
    else:
        kind, p = i
        rows = {"slice": lambda: slice(*p), "int": lambda: p, "bool": lambda: f[p], "frame": lambda: isel_frame(p),
                "list": lambda: list(p), "range": lambda: range(*p)}[kind]()
    K = getattr(T, case.get("kpart") or "year")
    mods = {"none": lambda: (), "sort": lambda: (mod.sort(f.s),), "sortdesc": lambda: (mod.sort(-f.s),),
            "by": lambda: (mod.by(f.s),), "bysort": lambda: (mod.by(f.s), mod.sort(f.v)),
            "join": lambda: (mod.join(J),), "bypart": lambda: (mod.by(K(f.d)),),
            "bypartneg": lambda: (mod.by(-K(f.d)),), "bykpart": lambda: (mod.by(f.s, K(f.d)),),
            "sortpart": lambda: (mod.sort(K(f.t), f.s),), "sortpartneg": lambda: (mod.sort(-K(f.t), f.s),),
            "bypart_t": lambda: (mod.by(K(f.t)),), "bypartjoin": lambda: (mod.by(K(g.d)), mod.join(J)),
            "bypartsort": lambda: (mod.by(K(f.d)), mod.sort(f.s))}[case["mode"]]()
    return (rows, j) + mods


_KEYED = {"by": (["s"], [0]), "bysort": (["s", "v"], [0, 4]), "bypart": (["K:d"], [0]), "bypartneg": (["K:d"], [2]),
          "bykpart": (["s", "K:d"], [0, 0]), "sortpart": (["K:t", "s"], [4, 4]), "sortpartneg": (["K:t", "s"], [6, 4]),
          "bypart_t": (["K:t"], [0]), "bypartsort": (["K:d", "s"], [0, 4])}


def keyed_outputs(case, arr, orc):
    """[(output index, int32 values)] the restatement gives for a case with by() or a time part in sort() and no `i`:
    the by() key columns (a time part's key the part of its column) and the time-part outputs of j, with the
    RowIndex and the groups formed by the C oracle over the keys."""
    name = case["name"]
    keys, flags = _KEYED[case["mode"]]
    cols = []
    for k in keys:
        if k.startswith("K:"):
            c = k[2:]
            cols.append(time_part(case["kpart"], arr[name + "." + c], case["stypes"][c]))
        else:
            cols.append(arr[name + "." + k])
    order, offsets, _ = orc.group(cols, flags, orc.NA_FIRST)
    order = np.asarray(order, dtype=np.int64)
    nby = 0 if case["mode"].startswith("sort") else len([f for f in flags if not f & 4])
    reduced = case["j"] in ("bysum", "bycount")
    rows = order[np.asarray(offsets, dtype=np.int64)[:-1]] if reduced else order
    out = [(i, np.asarray(cols[i])[rows].astype(np.int32)) for i in range(nby)
           if keys[i].startswith("K:") or case["stypes"][keys[i]] == INT32]
    if reduced or case["j"] == "byall":
        return out
    parts = [(1, case["part"], ("x", "t"))] if case["j"] == "bykeys" else j_parts(case)
    for idx, part, (_, c) in parts:
        out.append((nby + idx, time_part(part, arr[name + "." + c][order], case["stypes"][c])))
    return out
