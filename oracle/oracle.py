"""
NumPy/ctypes front-end of the CPU oracle (oracle/dt_oracle.c).

TEST INFRASTRUCTURE ONLY -- imported by tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs.  The product package
(datatable_b200/) never imports this module.

Parity status: pinned against the reference (see dt_oracle.c header and
tests/test_oracle_golden.py).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liborc.so")

# stype codes: the reference's src/datatable/include/datatable.h:32-42
BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64 = 1, 2, 3, 4, 5, 6, 7
# sort flags / NA position: the reference's src/core/sort.h:36-48
DESCENDING, SORT_ONLY = 2, 4
NA_FIRST, NA_LAST, NA_REMOVE = 1, 2, 3
SUM, MEAN, MIN, MAX, COUNT, COUNTNA, NROWS = 1, 2, 3, 4, 5, 6, 7
FIRST, LAST, SD, MEDIAN, NUNIQUE = 8, 9, 10, 11, 12
SET_UNION, SET_INTERSECT, SET_SETDIFF, SET_SYMDIFF = 0, 1, 2, 3

_NP2ST = {
    np.dtype(np.bool_): BOOL, np.dtype(np.int8): INT8, np.dtype(np.int16): INT16,
    np.dtype(np.int32): INT32, np.dtype(np.int64): INT64,
    np.dtype(np.float32): FLOAT32, np.dtype(np.float64): FLOAT64,
}
_ST2NP = {BOOL: np.int8, INT8: np.int8, INT16: np.int16, INT32: np.int32,
          INT64: np.int64, FLOAT32: np.float32, FLOAT64: np.float64}


def build(force=False):
    if force or not os.path.exists(_SO) or \
            os.path.getmtime(_SO) < os.path.getmtime(os.path.join(_HERE, "dt_oracle.c")):
        subprocess.check_call(["make", "-s", "-C", _HERE, "liborc.so"])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(build())
        _lib.orc_group.restype = ctypes.c_int
        _lib.orc_reduce.restype = ctypes.c_int
        _lib.orc_gather.restype = ctypes.c_int
    return _lib


def set_threads(t):
    """Host threads of the parallel regions (default 1).  Results do not depend on it; only
    bench.py's CPU legs raise it."""
    lib().orc_set_threads(int(t))


def get_threads():
    return int(lib().orc_get_threads())


def stype_of(a, stype=None):
    """stype code of a numpy array (bool columns may be passed as int8 + stype=BOOL)."""
    if stype is not None:
        return stype
    return _NP2ST[a.dtype]


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def group(cols, flags=None, na_pos=NA_FIRST, stypes=None):
    """Returns (order int32[n'], offsets int32[ng+1] or None, ngroups or None).

    `order` already has the NA rows removed when na_pos == NA_REMOVE.
    """
    cols = [np.ascontiguousarray(c) for c in cols]
    n = len(cols[0])
    nc = len(cols)
    flags = list(flags) if flags is not None else [0] * nc
    sts = [stype_of(c, None if stypes is None else stypes[i]) for i, c in enumerate(cols)]
    cp = (ctypes.c_void_p * nc)(*[c.ctypes.data for c in cols])
    st = (ctypes.c_int * nc)(*sts)
    fl = (ctypes.c_int * nc)(*flags)
    order = np.empty(n, dtype=np.int32)
    offsets = np.empty(n + 1, dtype=np.int32)
    ng = ctypes.c_int64(0)
    nskip = ctypes.c_int64(0)
    rc = lib().orc_group(cp, st, fl, ctypes.c_int(nc), ctypes.c_int(na_pos),
                         ctypes.c_int64(n), _ptr(order), _ptr(offsets),
                         ctypes.byref(ng), ctypes.byref(nskip))
    if rc != 0:
        raise NotImplementedError("oracle: unsupported stype")
    if nskip.value:
        order = order[nskip.value:].copy()
    if ng.value < 0:
        return order, None, None
    return order, offsets[:ng.value + 1].copy(), ng.value


def out_dtype(op, st):
    """Output numpy dtype of a reducer (see orc_reduce header)."""
    if op in (COUNT, COUNTNA, NROWS, NUNIQUE):
        return np.int64
    if op in (SD, MEDIAN):
        return np.float32 if st == FLOAT32 else np.float64
    if op == SUM:
        return {FLOAT32: np.float32, FLOAT64: np.float64}.get(st, np.int64)
    if op == MEAN:
        return np.float32 if st == FLOAT32 else np.float64
    return _ST2NP[st]


def reduce(op, v, order, offsets, stype=None):
    v = np.ascontiguousarray(v) if v is not None else np.zeros(1, np.int8)
    st = stype_of(v, stype)
    ng = len(offsets) - 1
    out = np.empty(ng, dtype=out_dtype(op, st))
    offsets = np.ascontiguousarray(offsets, dtype=np.int32)
    op_ = None if order is None else np.ascontiguousarray(order, dtype=np.int32)
    rc = lib().orc_reduce(ctypes.c_int(op), _ptr(v), ctypes.c_int(st),
                          _ptr(op_) if op_ is not None else ctypes.c_void_p(0),
                          _ptr(offsets), ctypes.c_int64(ng), _ptr(out))
    if rc != 0:
        raise NotImplementedError("oracle: unsupported reducer/stype")
    return out


def gather(src, idx, stype=None):
    src = np.ascontiguousarray(src)
    st = stype_of(src, stype)
    idx = np.ascontiguousarray(idx, dtype=np.int32)
    out = np.empty(len(idx), dtype=src.dtype)
    rc = lib().orc_gather(_ptr(src), ctypes.c_int(st), _ptr(idx),
                          ctypes.c_int64(len(idx)), _ptr(out))
    if rc != 0:
        raise NotImplementedError("oracle: unsupported stype")
    return out


# ---------------------------------------------------------------------------
# SURVEY.md 8(f) rows: restatements of the callers of group()
# ---------------------------------------------------------------------------
def sort_grouped(v, order, offsets, stype=None):
    """Column::sort_grouped (sort.cc:1499-1530): rows reordered inside every group by the value,
    ascending, NA first, stable; restated as a stable sort by (group id, value)."""
    v = np.ascontiguousarray(v)
    offsets = np.asarray(offsets, dtype=np.int64)
    n = int(offsets[-1])
    order = np.arange(n, dtype=np.int32) if order is None else np.asarray(order, dtype=np.int32)
    gid = np.repeat(np.arange(len(offsets) - 1, dtype=np.int32), np.diff(offsets))
    o2, _, _ = group([gid, v[order]], [SORT_ONLY, SORT_ONLY], NA_FIRST,
                     stypes=None if stype is None else [INT32, stype])
    return order[o2]


def set_select(mode, order, offsets, cum_sizes):
    """Group selection of union / intersect / setdiff / symdiff (set_funcs.cc:126-456): row index of the
    first row of every kept group.  Inside a group the RowIndex ascends, so the inputs a group touches
    are found from the row indices (input k holds rows cum_sizes[k-1] .. cum_sizes[k]-1)."""
    out = []
    K = len(cum_sizes)
    for g in range(len(offsets) - 1):
        rows = order[offsets[g]:offsets[g + 1]]
        present = np.unique(np.searchsorted(np.asarray(cum_sizes), rows, side="right"))
        if mode == SET_UNION or K < 2:
            keep = True
        elif mode == SET_INTERSECT:
            keep = len(present) == K
        elif mode == SET_SETDIFF:
            keep = len(present) == 1 and present[0] == 0
        else:
            keep = (rows[0] < cum_sizes[0]) == (rows[-1] < cum_sizes[0]) if K == 2 else len(present) % 2 == 1
        if keep:
            out.append(rows[0])
    return np.array(out, dtype=np.int32)


def largest_group(offsets, skip):
    """stats.cc:984-991: index and size of the first largest group among groups [skip, ng)."""
    sizes = np.diff(np.asarray(offsets, dtype=np.int64))[skip:]
    if len(sizes) == 0 or sizes.max() == 0:
        return -1, 0
    i = int(np.argmax(sizes))               # first maximum
    return i + skip, int(sizes[i])


def _na_mask(a, st):
    if st in (FLOAT32, FLOAT64):
        return np.isnan(a)
    return a == {BOOL: -128, INT8: -128, INT16: -2**15, INT32: -2**31, INT64: -2**63}[st]


def join_index(xcols, xst, jcols, jst):
    """natural_join (frame/join.cc:392-470): for every X row, binary search (join.cc:392-406) over the
    rows of J (sorted by its key, NA first) with the column comparators of FwCmp (join.cc:199-232)."""
    nx, nj = len(xcols[0]), len(jcols[0])
    xna = [_na_mask(c, s) for c, s in zip(xcols, xst)]
    jna = [_na_mask(c, s) for c, s in zip(jcols, jst)]
    out = np.full(nx, -2**31, dtype=np.int32)
    if nj == 0:
        return out
    int_range = {BOOL: (-128, 127), INT8: (-128, 127), INT16: (-2**15, 2**15 - 1), INT32: (-2**31, 2**31 - 1),
                 INT64: (-2**63, 2**63 - 1)}
    for r in range(nx):
        xv, bad = [], False
        for c in range(len(xcols)):
            if xna[c][r]:
                xv.append(None); continue
            x = xcols[c][r].item()
            if jst[c] in int_range:                               # set_xrow: values J's type cannot hold match nothing
                if isinstance(x, float) and (x != int(x) if np.isfinite(x) else True):
                    bad = True
                elif not (int_range[jst[c]][0] <= int(x) <= int_range[jst[c]][1]):
                    bad = True
                x = int(x) if not bad else x
            else:                                                 # static_cast<TJ>(newval): one rounding, from X's type
                x = float(xcols[c][r:r + 1].astype(np.float32 if jst[c] == FLOAT32 else np.float64)[0])
            xv.append(x)
        if bad:
            continue

        def cmp(row):
            for c in range(len(xcols)):
                jvalid, xvalid = not jna[c][row], xv[c] is not None
                if jvalid and xvalid:
                    jv = jcols[c][row].item()
                    if jv != xv[c]:
                        return 1 if jv > xv[c] else -1
                elif jvalid != xvalid:
                    return int(jvalid) - int(xvalid)
            return 0
        start, end = 0, nj - 1
        found = -1
        while start < end:
            mid = (start + end) >> 1
            t = cmp(mid)
            if t > 0:
                end = mid
            elif t < 0:
                start = mid + 1
            else:
                found = mid; break
        if found < 0 and cmp(start) == 0:
            found = start
        if found >= 0:
            out[r] = found
    return out


SLICE_NA = -2**63          # a missing slice member (py::oslice::NA)


def _i32(x):
    """static_cast<int32_t>(int64) as the reference does it (two's-complement truncation)."""
    x &= 0xFFFFFFFF
    return x - (1 << 32) if x & 0x80000000 else x


def slice_groups(offsets, start, stop, step):
    """FExpr_Literal_SliceInt::evaluate_iby (expr/fexpr_literal_sliceint.cc:82-170): the slice applied inside
    every group of the grouped frame.  Returns (positions into the RowIndex of group(), new offsets); groups
    that select nothing disappear.  None / SLICE_NA = missing member; step 0 = repeat row `start` `stop` times."""
    offsets = np.asarray(offsets, dtype=np.int64)
    nrows = int(offsets[-1]) if len(offsets) else 0
    NA = (None, SLICE_NA)
    istart, istop, istep = [SLICE_NA if x in NA else int(x) for x in (start, stop, step)]
    if istep == SLICE_NA:
        istep = 1                                               # :86
    rows, offs = [], [0]
    step32 = _i32(istep)
    for g in range(len(offsets) - 1):
        off0, off1 = int(offsets[g]), int(offsets[g + 1])
        n = off1 - off0
        if step32 > 0:                                          # :102-125
            s0 = 0 if istart == SLICE_NA else istart
            s1 = nrows if istop == SLICE_NA else istop
            a, b = _i32(s0), _i32(s1)
            if a < 0: a += n
            if a < 0: a = 0
            a += off0
            if b < 0: b += n
            b += off0
            if b > off1: b = off1
            if a < b:
                rows.extend(range(a, b, step32)); offs.append(len(rows))
        elif step32 < 0:                                        # :126-148
            a = n - 1 if (istart == SLICE_NA or istart >= n) else _i32(istart)
            if a < 0: a += n
            a += off0
            if istop == SLICE_NA:
                b = off0 - 1
            else:
                b = _i32(istop)
                if b < 0: b += n
                if b < 0: b = -1
                b += off0
            if a > b:
                rows.extend(range(a, b, step32)); offs.append(len(rows))
        else:                                                   # :149-165  step == 0: `stop` copies of row `start`
            a = _i32(istart)
            if a < 0: a += n
            if a < 0 or a >= n:
                continue
            rows.extend([a + off0] * istop); offs.append(len(rows))
    return np.array(rows, dtype=np.int32), np.array(offs, dtype=np.int32)


def int_groups(offsets, i):
    """FExpr_Literal_Int::evaluate_iby (expr/fexpr_literal_int.cc:146-192): the i-th row of every group (negative: from
    its end); groups that are too short disappear, every remaining group has one row."""
    offsets = np.asarray(offsets, dtype=np.int64)
    if _i32(i) != i:
        return np.zeros(0, np.int32), np.zeros(1, np.int32)
    rows = []
    for g in range(len(offsets) - 1):
        a, b = int(offsets[g]), int(offsets[g + 1])
        r = a + i if i >= 0 else b + i
        if (i >= 0 and r < b) or (i < 0 and r >= a):
            rows.append(r)
    return np.array(rows, dtype=np.int32), np.arange(len(rows) + 1, dtype=np.int32)
