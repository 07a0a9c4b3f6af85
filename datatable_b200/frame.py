"""
Host-side mirror of the reference's Python surface for the DT[i, j, by(), sort()] path:
Frame, f, by(), sort(), sum/mean/min/max/count.  Only what the hot path needs -- no fread,
no general expression engine (SURVEY.md 8: out of scope).

    reference                                   here
    ---------                                   ----
    dt.Frame                 src/datatable/frame.py:23 / src/core/frame/      Frame
    f.A, f["A"], -f.A        src/datatable/expr/                               f / ColRef
    by(...), sort(...)       src/core/expr/py_by.cc, py_sort.cc:40-110         by / sort
    dt.sum/mean/min/max/count  src/datatable/expr/reduce.py:49-153             sum_/mean/min_/max_/count
    DT[i, j, by, sort]       src/core/frame/__getitem__.cc:47-194,
                             src/core/expr/eval_context.cc:144-288, 473-520    Frame.__getitem__

Evaluation follows EvalContext: group() on the by/sort columns -> (RowIndex, Groupby);
reducers are evaluated over (value column, RowIndex, Groupby); plain columns are gathered
through the RowIndex; group keys are the first row of every group
(eval_context.cc:473-485).  All of it runs in libdtb200.so on the GPU.
"""
import builtins
import copy

import numpy as np

from . import _lib, engine
from ._lib import (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DATE32, TIME64, FLAG_DESCENDING,
                   FLAG_SORT_ONLY, NA_FIRST, NA_LAST, NA_REMOVE)

try:
    import torch
except Exception:  # pragma: no cover
    torch = None

_NA_POS = {"first": NA_FIRST, "last": NA_LAST, "remove": NA_REMOVE}
_NA_VALUE = {INT8: -2**7, INT16: -2**15, INT32: -2**31, INT64: -2**63, BOOL: -128}


# ---------------------------------------------------------------------------
# f-expressions (only column references, their negation, and reducers)
# ---------------------------------------------------------------------------
class ColRef:
    """A column of the query's frame X (f., frame 0) or of the joined frame J (g., frame 1)."""
    def __init__(self, name, negated=False, frame=0):
        self.name = name
        self.negated = negated
        self.frame = frame

    def __neg__(self):            # sort(-f.A) / by(-f.A): DESCENDING flag, not arithmetic (fexpr_list.cc:346-358)
        return ColRef(self.name, not self.negated, self.frame)

    def __repr__(self):
        return f"{'-' if self.negated else ''}{'g' if self.frame else 'f'}.{self.name}"


class _FNamespace:
    def __init__(self, frame=0):
        self._frame = frame

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return ColRef(name, frame=self._frame)

    def __getitem__(self, name):
        return ColRef(name, frame=self._frame)


f = _FNamespace(0)
g = _FNamespace(1)


class _JKey(str):
    """The name under which a query's stages read a column of the joined frame J: its text is J's column name (the
    result column is named after it), but it never equals the name of an X column, so f.v and g.v stay apart."""
    __slots__ = ()

    def __eq__(self, other):
        return isinstance(other, _JKey) and str.__eq__(self, other)

    def __ne__(self, other):
        return not self == other

    def __hash__(self):
        return hash(("g", str(self)))


class Reducer:
    def __init__(self, op, name, arg):
        self.op, self.opname, self.arg = op, name, arg


def sum(x): return Reducer(_lib.OP_SUM, "sum", x)          # noqa: A001  (mirrors dt.sum)
def prod(x): return Reducer(_lib.OP_PROD, "prod", x)
def mean(x): return Reducer(_lib.OP_MEAN, "mean", x)
def min(x): return Reducer(_lib.OP_MIN, "min", x)          # noqa: A001
def max(x): return Reducer(_lib.OP_MAX, "max", x)          # noqa: A001
def countna(x): return Reducer(_lib.OP_COUNTNA, "countna", x)
# within-group ordered reducers (src/core/expr/head_reduce_unary.cc:544-558; SURVEY.md 8f)
def first(x): return Reducer(_lib.OP_FIRST, "first", x)
def last(x): return Reducer(_lib.OP_LAST, "last", x)
def sd(x): return Reducer(_lib.OP_SD, "sd", x)
def median(x): return Reducer(_lib.OP_MEDIAN, "median", x)
def nunique(x): return Reducer(_lib.OP_NUNIQUE, "nunique", x) if isinstance(x, (ColRef, str)) else _frame_nunique(x)


class Reducer2(Reducer):
    """A reducer of two columns (cov / corr, expr/head_reduce_binary.cc): arg = x, arg2 = y."""
    def __init__(self, op, name, x, y):
        super().__init__(op, name, _as_ref(x))
        self.arg2 = _as_ref(y)


def _binary(op, name, x, y):
    """One reducer per pair; a list argument broadcasts: both lists of the same length, or one of them of length 1
    (head_reduce_binary.cc:236-259)."""
    xs = list(x) if isinstance(x, (list, tuple)) else [x]
    ys = list(y) if isinstance(y, (list, tuple)) else [y]
    if not isinstance(x, (list, tuple)) and not isinstance(y, (list, tuple)):
        return Reducer2(op, name, x, y)
    n1, n2 = len(xs), len(ys)
    if n1 != n2 and n1 != 1 and n2 != 1:
        raise ValueError(f"Cannot apply reducer function {name}: argument 1 has {n1} columns, while argument 2 has "
                         f"{n2} columns")
    n = n1 if n1 != 1 else n2
    return [Reducer2(op, name, xs[i if n1 > 1 else 0], ys[i if n2 > 1 else 0]) for i in range(n)]


def cov(x, y): return _binary(_lib.OP_COV, "cov", x, y)
def corr(x, y): return _binary(_lib.OP_CORR, "corr", x, y)


def count(x=None):
    return Reducer(_lib.OP_NROWS if x is None else _lib.OP_COUNT, "count", x)


class RowFn:
    """A function that returns one value per row and runs inside every group, the result in the grouped order (GtoALL):
    qcut, cut, cumsum, cumprod, cummin, cummax, shift, fillna, cumcount, ngroup.  `cols` as given (a column, a list or
    tuple of columns, or f[:]; None for a function of no column; a Frame for cut); when the query runs they are
    resolved and columns() makes one RowFnCol per column, with the function's checks of its other arguments (evaluate_n of the reference's FExpr)."""
    def __init__(self, cols):
        self.cols = cols


class RowFnCol:
    """One output column of a RowFn over column `name`: run(c, order, offsets) -> (values, stype), one value per
    position of the RowIndex `order`, computed inside every group of `offsets`.  name None: the function reads no
    column of the query's frame (c is None) and its output is named `label`, or unnamed (C0, C1, ...) without one."""
    def __init__(self, name, run, label=None):
        self.name, self.run, self.label = name, run, label


class Qcut(RowFn):
    """dt.qcut(cols, nquantiles=None) (expr/fexpr_qcut.cc:41-181): nquantiles is checked when the query runs
    (FExpr_Qcut::evaluate_n)."""
    def __init__(self, cols, nquantiles):
        super().__init__(cols)
        self.nquantiles = nquantiles

    def columns(self, DT, refs):
        nq = self.nquantiles
        if isinstance(nq, (list, tuple)):
            if len(nq) != len(refs):
                raise ValueError(f"When nquantiles is a list or a tuple, its length must be the same as the number of "
                                 f"input columns, i.e. {len(refs)}, instead got: {len(nq)}")
            qs = []
            for i, x in enumerate(nq):
                x = _to_int32_strict(x)
                if x <= 0:
                    raise ValueError(f"All elements in nquantiles must be positive, got nquantiles[{i}]: {x}")
                qs.append(x)
        else:
            q = 10
            if nq is not None:
                q = _to_int32_strict(nq)
                if q <= 0:
                    raise ValueError(f"Number of quantiles must be positive, instead got: {q}")
            qs = [q] * len(refs)
        return [RowFnCol(r.name, lambda c, order, offsets, q=q: (engine.qcut(c, order, offsets, q), INT32))
                for r, q in zip(refs, qs)]


def qcut(cols, nquantiles=None):
    return Qcut(cols, nquantiles)


_NUMERIC = (BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64)


class Cut(RowFn):
    """dt.cut(cols, nbins=None, bins=None, right_closed=True) (expr/fexpr_cut.cc:88-170): nbins (a list, one per
    column, or one value for all) or the float64 bin edges of every column, checked by cut(); the column count and
    the stypes are checked when the query runs.  Refused under by(), as the reference refuses it.  cols may be a
    Frame with the query's row count: its columns are binned as they are, in the Frame's own row order."""
    def __init__(self, cols, nbins, edges, right_closed):
        super().__init__(cols)
        self.nbins, self.edges, self.right_closed = nbins, edges, right_closed

    def columns(self, DT, refs):
        framearg = isinstance(self.cols, Frame)
        src = self.cols if framearg else DT
        ncols = len(refs)
        if self.edges is not None:
            if len(self.edges) != ncols:
                raise ValueError(f"Number of elements in bins must be equal to the number of columns in the "
                                 f"frame/expression, i.e. {ncols}, instead got: {len(self.edges)}")
        elif len(self.nbins) != ncols and len(self.nbins) != 1:
            raise ValueError(f"When nbins has more than one element, its length must be the same as the number of "
                             f"columns in the frame/expression, i.e. {ncols}, instead got: {len(self.nbins)}")
        out = []
        for i, r in enumerate(refs):
            st = src._stypes[r.name]
            if st not in _NUMERIC:
                sep = "" if self.edges is not None else " "       # the reference's two texts differ by this space
                raise TypeError(f"cut() can only be applied to numeric{sep}columns, instead column {i} has an stype: "
                                f"{_STYPE_NAMES.get(st, st)}")
            kw = (dict(nbins=10, edges=self.edges[i]) if self.edges is not None else
                  dict(nbins=self.nbins[i % len(self.nbins)]))
            if not framearg:
                out.append(RowFnCol(r.name, lambda c, order, offsets, kw=kw:
                                    (engine.cut(c, order, right_closed=self.right_closed, **kw), INT32)))
            else:
                out.append(RowFnCol(None, lambda c, order, offsets, nm=r.name, kw=kw:
                                    (self._frame_cut(DT, nm, order, kw), INT32), label=r.name))
        return out

    def _frame_cut(self, DT, name, order, kw):
        """FExpr_Frame::evaluate_n (expr/fexpr_frame.cc:77-95): the Frame must have the query's row count."""
        F = self.cols
        n = DT.nrows if order is None else len(order)
        if F.nrows != n:
            if F.nrows == 1:
                raise NotImplementedError("a 1-row Frame broadcast to the rows of a query is outside the GPU hot path")
            raise ValueError(f"Frame has {F.nrows} rows, and cannot be used in an expression where {n} are expected")
        return engine.cut(engine.Col(_dev(F._col(name)), F._stypes[name]), None, right_closed=self.right_closed, **kw)


def cut(*args, cols=None, nbins=None, bins=None, right_closed=True):
    """pyfn_cut (expr/fexpr_cut.cc:217-302): equal-width bins over the min / max of every column (nbins, default
    10), or bins between explicit edges (bins: a list or tuple of 1-column Frames of at least 2 strictly increasing
    numeric values), as int32 with NA as INT32_MIN.  The arguments are checked here, with the reference's texts."""
    if len(args) > 1:
        raise TypeError(f"Function datatable.cut() takes only one positional argument, but {len(args)} were given")
    if args:
        cols = args[0]
    elif cols is None:
        raise TypeError("Function datatable.cut() requires exactly 1 positional argument, but none were given")
    if right_closed is None:
        right_closed = True
    if not isinstance(right_closed, bool):
        raise TypeError(f"Argument right_closed in function datatable.cut() should be a boolean, instead got "
                        f"{type(right_closed)}")
    if bins is not None and nbins is not None:
        raise ValueError("bins and nbins cannot be both set at the same time")
    edges, nb = None, None
    if bins is not None:
        if not isinstance(bins, (list, tuple)):
            raise TypeError(f"bins parameter must be a list or a tuple, instead got {type(bins)}")
        edges = [_bin_edges(F, i) for i, F in enumerate(bins)]
    elif isinstance(nbins, (list, tuple)):
        nb = []
        for i, x in enumerate(nbins):
            x = _cut_int32(x)
            if x <= 0:
                raise ValueError(f"All elements in nbins must be positive, got nbins[{i}]: {x}")
            nb.append(x)
    else:
        x = 10 if nbins is None else _cut_int32(nbins)
        if x <= 0:
            raise ValueError(f"Number of bins must be positive, instead got: {x}")
        nb = [x]
    if not isinstance(cols, Frame):
        _column_args_only("cut", cols)
    return Cut(cols, nb, edges, right_closed)


def _cut_int32(x):
    """to_int32_strict as pyfn_cut raises it: the reference's text says "too large" on both sides of the range."""
    if isinstance(x, int) and not isinstance(x, bool) and x < -2**31:
        raise ValueError(f"Value is too large to fit in an int32: {x}")
    return _to_int32_strict(x)


def _bin_edges(F, i):
    """The edges of bins Frame number i as float64, read to the host once (FExpr_Cut::bins_to_vector,
    fexpr_cut.cc:172-210)."""
    if not isinstance(F, Frame):
        raise TypeError(f"Expected a Frame, instead got {type(F)}")
    if F.ncols != 1:
        raise ValueError(f"To bin a column cut() needs exactly one column with the bin edges, instead for the frame "
                         f"{i} got: {F.ncols}")
    if F.nrows < 2:
        raise ValueError(f"To bin data at least two edges are required, instead for the frame {i} got: {F.nrows}")
    st = F.stypes[0]
    if st not in _NUMERIC:
        raise TypeError(f"Bin edges must be provided as the numeric columns only, instead for the frame {i} the column "
                        f"stype is {_STYPE_NAMES.get(st, st)}")
    a = F.to_numpy(F.names[0])
    na = np.isnan(a) if st in (FLOAT32, FLOAT64) else a == _NA_VALUE[st]
    e = a.astype(np.float64)                       # int64 rounds to nearest, as cast_inplace(FLOAT64) does
    for k in range(len(e)):
        if na[k]:
            raise ValueError(f"Bin edges must be numeric values only, instead for the frame {i} got None at row {k}")
        if k and not e[k] > e[k - 1]:
            raise ValueError(f"Bin edges must be strictly increasing, instead for the frame {i} at rows {k - 1} and {k} "
                             f"the values are {e[k - 1]:g} and {e[k]:g}")
    return e


def _has_cut(j):
    """Whether j holds a cut() (in a list, tuple or dict)."""
    if isinstance(j, Cut):
        return True
    if isinstance(j, (list, tuple)):
        return builtins.any(_has_cut(x) for x in j)
    return isinstance(j, dict) and builtins.any(_has_cut(x) for x in j.values())


_STYPE_NAMES = {BOOL: "bool8", INT8: "int8", INT16: "int16", INT32: "int32", INT64: "int64", FLOAT32: "float32",
                FLOAT64: "float64", DATE32: "date32", TIME64: "time64"}


class Cumulative(RowFn):
    """dt.cumsum / cumprod / cummin / cummax(cols, reverse=False) (expr/fexpr_cumsumprod.cc, expr/fexpr_cumminmax.cc):
    reverse must be a bool when the function is called; the column types are checked when the query runs."""
    def __init__(self, op, fname, cols, reverse):
        if not isinstance(reverse, bool):
            raise TypeError(f"Argument reverse in function datatable.{fname}() should be a boolean, instead got "
                            f"{type(reverse)}")
        super().__init__(cols)
        self.op, self.fname, self.reverse = op, fname, reverse

    def __repr__(self):
        return f"{self.fname}({_cols_repr(self.cols)}, reverse={self.reverse})"

    def columns(self, DT, refs):
        out = []
        for r in refs:
            st = DT._stypes[r.name]
            out_st = engine.cumulative_out_stype(self.op, st)
            if not out_st:
                raise TypeError(f"Invalid column of type {_STYPE_NAMES.get(st, st)} in {self!r}")
            out.append(RowFnCol(r.name, lambda c, order, offsets, out_st=out_st:
                                (engine.cumulative(self.op, c, order, offsets, self.reverse), out_st)))
        return out


def cumsum(cols, reverse=False): return Cumulative(_lib.OP_SUM, "cumsum", cols, reverse)
def cumprod(cols, reverse=False): return Cumulative(_lib.OP_PROD, "cumprod", cols, reverse)
def cummin(cols, reverse=False): return Cumulative(_lib.OP_MIN, "cummin", cols, reverse)
def cummax(cols, reverse=False): return Cumulative(_lib.OP_MAX, "cummax", cols, reverse)


def _column_args_only(fname, cols):
    """shift / fillna take column references; an expression or a reducer as the argument is not on the GPU path."""
    for c in _flatten([cols]):
        if not isinstance(c, (ColRef, str)):
            raise NotImplementedError(f"{fname}() of an expression ({c!r}) is outside the GPU hot path")


def _fixed_width(DT, name, fname):
    st = DT._stypes[name]
    if st not in _STYPE_NAMES:
        raise NotImplementedError(f"{fname}() of a column of stype {st} is outside the GPU hot path")
    return st


class Shift(RowFn):
    """dt.shift(cols, n=1) (expr/head_func_shift.cc:40-179): the value n rows earlier in the group (n < 0: -n rows
    later), NA where that row is outside the group; without by() the selected rows are one group."""
    def __init__(self, cols, n):
        _column_args_only("shift", cols)
        super().__init__(cols)
        self.n = n

    def columns(self, DT, refs):
        return [RowFnCol(r.name, lambda c, order, offsets, st=_fixed_width(DT, r.name, "shift"):
                         (engine.shift(c, order, offsets, self.n), st)) for r in refs]


def shift(cols=None, n=1):
    """pyfn_shift (expr/head_func_shift.cc:156-179): n is checked first, then cols; shift(frame, n) is
    frame[:, shift(f[:], n)]."""
    if n is None:
        n = 1
    if not isinstance(n, int) or isinstance(n, bool):
        raise TypeError(f"Argument n in function datatable.shift() should be an integer, instead got {type(n)}")
    if not -2**31 <= n < 2**31:
        raise ValueError(f"Value is too large to fit in an int32: {n}")       # the reference's text on both sides
    if cols is None:
        raise TypeError("Function shift() requires 1 positional argument, but none were given")
    if isinstance(cols, Frame):
        return cols[:, Shift(f[:], n)]
    if not isinstance(cols, (ColRef, Reducer, RowFn)):
        raise TypeError(f"The first argument to shift() must be a column expression or a Frame, instead got "
                        f"{type(cols)}")
    return Shift(cols, n)


class FillNA(RowFn):
    """dt.fillna(cols, reverse=False) without a value (expr/fexpr_fillna.cc:66-118, 157-181): the latest valid value of
    the group so far (reverse: the earliest at or after the row), NA before the first; without by() the selected
    rows are one group."""
    def __init__(self, cols, reverse):
        _column_args_only("fillna", cols)
        super().__init__(cols)
        self.reverse = reverse

    def columns(self, DT, refs):
        return [RowFnCol(r.name, lambda c, order, offsets, st=_fixed_width(DT, r.name, "fillna"):
                         (engine.fillna(c, order, offsets, self.reverse), st)) for r in refs]


def fillna(cols, value=None, reverse=None):
    """pyfn_fillna (expr/fexpr_fillna.cc:209-226).  fillna(cols, value=) is an elementwise if-else with the reference's
    type promotion, which belongs to an expression engine: NotImplementedError."""
    if value is not None and reverse is not None:
        raise ValueError("Parameters value and reverse in function datatable.fillna() cannot be both set at the same "
                         "time")
    if reverse is not None and not isinstance(reverse, bool):
        raise TypeError(f"Expected a boolean, instead got {type(reverse)}")
    if value is not None:
        raise NotImplementedError("fillna(cols, value=) is outside the GPU hot path")
    return FillNA(cols, bool(reverse))


class GroupIndex(RowFn):
    """dt.cumcount(reverse=False) / dt.ngroup(reverse=False) (expr/fexpr_cumcountngroup.cc:40-116): int64, no input
    column, an unnamed output (C0, C1, ...).  Without by() the selected rows are one group: 0 .. n-1 and 0."""
    def __init__(self, kind, fname, reverse):
        if reverse is None:
            reverse = False
        if not isinstance(reverse, bool):
            raise TypeError(f"Argument reverse in function datatable.{fname}() should be a boolean, instead got "
                            f"{type(reverse)}")
        super().__init__(None)
        self.kind, self.reverse = kind, reverse

    def columns(self, DT, refs):
        return [RowFnCol(None, lambda c, order, offsets: (engine.group_index(self.kind, offsets, self.reverse), INT64))]


def cumcount(reverse=False): return GroupIndex(_lib.GROUP_CUMCOUNT, "cumcount", reverse)
def ngroup(reverse=False): return GroupIndex(_lib.GROUP_NGROUP, "ngroup", reverse)


def _cols_repr(cols):
    if isinstance(cols, (list, tuple)):
        return "[" + ", ".join(_cols_repr(c) for c in cols) + "]"
    if isinstance(cols, ColRef) and isinstance(cols.name, slice):
        return "f[:]"
    return repr(cols) if isinstance(cols, ColRef) else f"f.{cols}"


def _to_int32_strict(x):
    """py::robj::to_int32_strict: an int (not a bool) that fits in an int32."""
    if not isinstance(x, int) or isinstance(x, bool):
        raise TypeError(f"Expected an integer, instead got {type(x)}")
    if x > 2**31 - 1:
        raise ValueError(f"Value is too large to fit in an int32: {x}")
    if x < -2**31:
        raise ValueError(f"Value is too small to fit in an int32: {x}")
    return x


def _rowfn_cols(DT, e, bynames):
    """The columns of RowFn e (FExpr::evaluate_n of its argument): one RowFnCol per input column.  f[:] under by()
    leaves out the by() columns."""
    if e.cols is None:
        return e.columns(DT, [])
    if isinstance(e, Cut) and isinstance(e.cols, Frame):    # FExpr_Frame::evaluate_n: the Frame's own columns
        return e.columns(DT, [ColRef(nm) for nm in e.cols.names])
    refs = []
    for c in _flatten([e.cols]):
        if isinstance(c, ColRef) and isinstance(c.name, slice):
            if c.name != slice(None):
                raise NotImplementedError("column slices other than f[:] are outside the GPU hot path")
            refs += [ColRef(nm) for nm in DT.names if nm not in bynames and not isinstance(nm, _JKey)]
        else:
            refs.append(_bind(DT, _as_ref(c)))
    return e.columns(DT, refs)


class by:
    def __init__(self, *cols):
        self.cols = [_as_ref(c) for c in _flatten(cols)]


class join:
    """join(J): natural join with the keyed frame J (src/core/expr/py_join.cc; frame/join.cc:392-470)."""

    def __init__(self, frame):
        if not isinstance(frame, Frame):
            raise TypeError("The argument to join() must be a Frame")
        if not frame.key:
            raise ValueError("The join frame is not keyed")
        self.frame = frame


class sort:
    """sort(*cols, reverse=False, na_position="first") -- py_sort.cc:40-110."""

    def __init__(self, *cols, reverse=False, na_position="first"):
        self.cols = [_as_ref(c) for c in _flatten(cols)]
        n = len(self.cols)
        if isinstance(reverse, (list, tuple)):
            if len(reverse) != n:
                raise ValueError(f"number of elements (nflags={len(reverse)}) in the reverse flag list "
                                 f"does not match the number of sort columns ({n})")
            self.reverse = [bool(r) for r in reverse]
        elif isinstance(reverse, bool):
            self.reverse = [reverse] * n
        else:
            raise TypeError("reverse should be a boolean or a list of booleans")
        if na_position not in _NA_POS:
            raise ValueError(f"na position value `{na_position}` is not supported")
        self.na_position = na_position


def _flatten(cols):
    out = []
    for c in cols:
        if isinstance(c, (list, tuple)):
            out.extend(_flatten(c))
        else:
            out.append(c)
    return out


def _as_ref(c):
    if isinstance(c, ColRef):
        return c
    if isinstance(c, str):
        return ColRef(c)
    raise TypeError(f"Unsupported key expression {c!r}: only column references are on the GPU path")


# ---------------------------------------------------------------------------
# Frame
# ---------------------------------------------------------------------------
class Frame:
    """Column store: every column is a numpy array (host) or a torch CUDA tensor (HBM) plus an stype.
    Bool columns with NAs are int8 with -128 (the reference's bool8 layout)."""
    _joined = None            # the keyed frame J of a query's view of X joined to J (_join_view)

    def __init__(self, data=None, stypes=None, **kwargs):
        self._cols = {}
        self._stypes = {}
        self._key = ()
        if data is None:
            data = kwargs
        if isinstance(data, Frame):
            self._cols, self._stypes = dict(data._cols), dict(data._stypes)
            return
        if not isinstance(data, dict):
            data = {"C0": data}
        n = None
        for name, col in data.items():
            st = None if stypes is None else stypes.get(name)
            if isinstance(col, (list, tuple)):
                col, st2 = _from_list(col)
                st = st or st2
            c = engine.Col(col, st)
            if n is None:
                n = c.nrows
            elif c.nrows != n:
                raise ValueError("columns have different numbers of rows")
            self._cols[name] = c.data
            self._stypes[name] = c.stype
        self._nrows = n or 0

    # -- metadata ---------------------------------------------------------------
    @property
    def names(self): return tuple(self._cols.keys())
    @property
    def nrows(self): return self._nrows
    @property
    def ncols(self): return len(self._cols)
    @property
    def shape(self): return (self.nrows, self.ncols)
    @property
    def stypes(self): return tuple(self._stypes[n] for n in self._cols)

    def _col(self, name):
        if name not in self._cols:
            raise KeyError(f"Column `{name}` does not exist in the Frame")
        return engine.Col(self._cols[name], self._stypes[name])

    def column(self, name):
        """Raw storage of a column (numpy array or CUDA tensor)."""
        return self._cols[name]

    def to_numpy(self, name=None):
        if name is None:
            return {n: self.to_numpy(n) for n in self._cols}
        c = self._cols[name]
        return c.cpu().numpy() if engine.is_tensor(c) else c

    def to_list(self):
        out = []
        for n in self._cols:
            a = self.to_numpy(n)
            st = self._stypes[n]
            if st in (FLOAT32, FLOAT64):
                out.append([None if np.isnan(x) else float(x) for x in a.tolist()])
            elif st == BOOL:
                out.append([None if x == -128 else bool(x) for x in a.tolist()])
            else:
                na = _NA_VALUE[st]
                out.append([None if x == na else int(x) for x in a.tolist()])
        return out

    def to_dict(self):
        return dict(zip(self.names, self.to_list()))

    # -- Arrow ingest / export (the reference reads Arrow through Frame(pa.Table), frame/__init__.cc; here the
    #    fixed-width columns become the NA-sentinel buffers the engine consumes, SURVEY.md 8f rank 4) -----------
    @classmethod
    def from_arrow(cls, table):
        """pyarrow.Table / RecordBatch -> Frame: bool/int8-64/float32-64 columns, nulls -> the reference's NA
        sentinels (bool8 = int8 with -128).  Zero-copy for null-free numeric columns."""
        import pyarrow as pa
        cols, sts = {}, {}
        for name, col in zip(table.column_names, table.columns):
            arr = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
            t = arr.type
            if pa.types.is_boolean(t):
                a = np.asarray(arr.cast(pa.int8()).fill_null(-128).to_numpy(zero_copy_only=False), dtype=np.int8)
                st = BOOL
            elif pa.types.is_integer(t) and t.bit_width <= 64 and pa.types.is_signed_integer(t):
                st = {8: INT8, 16: INT16, 32: INT32, 64: INT64}[t.bit_width]
                a = arr.fill_null(_NA_VALUE[st]).to_numpy(zero_copy_only=False) if arr.null_count else arr.to_numpy()
            elif pa.types.is_floating(t) and t.bit_width in (32, 64):
                st = FLOAT32 if t.bit_width == 32 else FLOAT64
                a = arr.to_numpy(zero_copy_only=False)          # nulls become NaN == NA
            else:
                raise _lib.DtbNotImplError(f"Arrow column `{name}` of type {t} is outside the GPU hot path")
            cols[name], sts[name] = np.ascontiguousarray(a), st
        return cls(cols, stypes=sts)

    def to_jay(self, path):
        """Frame -> Jay file the reference opens with dt.fread (src/core/jay/save_jay.cc); see datatable_b200/jay.py."""
        from .jay import save_jay
        save_jay(self, path)

    def to_arrow(self):
        """Frame -> pyarrow.Table with NA sentinels turned back into nulls."""
        import pyarrow as pa
        out = {}
        for n in self._cols:
            a, st = self.to_numpy(n), self._stypes[n]
            if st in (FLOAT32, FLOAT64):
                out[n] = pa.array(a, mask=np.isnan(a))
            elif st == BOOL:
                out[n] = pa.array(a.astype(np.bool_), mask=(a == -128))
            else:
                out[n] = pa.array(a, mask=(a == _NA_VALUE[st]))
        return pa.table(out)

    def to_device(self):
        """Copy every column into HBM (the analogue of a device-backed Buffer, SURVEY.md 8f rank 4)."""
        return _result([(n, _dev(self._col(n)), self._stypes[n]) for n in self._cols], self._nrows)

    # -- DT.key (frame/key.cc:118-180): sort by the key columns, require unique rows, key columns first
    @property
    def key(self):
        return tuple(self._key)

    @key.setter
    def key(self, val):
        names = [val] if isinstance(val, str) else list(val or [])
        if not names:
            self._key = ()
            return
        for nm in names:
            if not isinstance(nm, str):
                raise TypeError("Key should be a list/tuple of column names")
            if nm not in self._cols:
                raise KeyError(f"Column `{nm}` does not exist in the Frame")
        if len(set(names)) != len(names):
            raise ValueError("A column is specified multiple times within the key")
        if self._nrows:
            order, offsets, ng = engine.group([self._col(nm) for nm in names], [0] * len(names), NA_FIRST)
            if ng < self._nrows:
                raise ValueError("Cannot set a key: the values are not unique")
        rest = [nm for nm in self._cols if nm not in names]
        cols, sts = {}, {}
        for nm in names + rest:
            c = self._col(nm)
            if self._nrows:
                o = order if (engine.is_tensor(c.data) and c.data.is_cuda) == engine.is_tensor(order) else (
                    order.cpu().numpy() if engine.is_tensor(order) else torch.from_numpy(order).cuda())
                cols[nm] = engine.gather(c, o)
            else:
                cols[nm] = c.data
            sts[nm] = c.stype
        self._cols, self._stypes = cols, sts
        self._key = tuple(names)

    # -- column statistics that go through group() (stats.cc:955-1003) ---------------------------
    def nunique(self):
        return _frame_nunique(self)

    def mode(self):
        return _frame_mode(self)[0]

    def nmodal(self):
        return _frame_mode(self)[1]

    # -- DT.sort(cols) (sort.cc:1544-1574) ------------------------------------------
    def sort(self, *cols):
        return self[:, :, sort(*cols)]

    # -- DT[i, j, by, sort] -------------------------------------------------------------
    def __getitem__(self, item):
        if not isinstance(item, tuple):
            item = (slice(None), item)
        if len(item) < 2:
            raise ValueError("Frame[...] needs at least i and j")
        i, j = item[0], item[1]
        by_, sort_, join_ = None, None, None
        for m in item[2:]:
            if isinstance(m, by):
                by_ = m
            elif isinstance(m, sort):
                sort_ = m
            elif isinstance(m, join):
                join_ = m
            else:
                raise TypeError(f"Unsupported modifier {m!r}")
        isel = None
        if i is None:                                    # FExpr_Literal_None: every row (fexpr_literal_none.cc:88-96)
            i = slice(None)
        if not (isinstance(i, slice) and i == slice(None)):
            ok = (isinstance(i, int) and not isinstance(i, bool)) or (
                isinstance(i, slice) and all(x is None or (isinstance(x, int) and not isinstance(x, bool)) for x in (i.start, i.stop, i.step)))
            if not ok and not isinstance(i, _ROW_SELECTORS):
                raise NotImplementedError("row filters other than an integer or an integer slice are outside the GPU hot path")
            isel = i
        # EvalContext::evaluate (eval_context.cc:144-172) for the hot-path shapes: the join first (J's columns the
        # query reads are looked up once, X-aligned, by _Upload), then group / sort, then `i`, then j
        DT = self if join_ is None else _join_view(self, join_.frame)
        names, exprs, by_, sort_, isel = _resolve(DT, j, by_, sort_, isel)
        masks = isel.mask_columns() if isinstance(isel, _Rows) else []
        up = _Upload(DT, masks + [r.name for m in (by_, sort_) if m is not None for r in m.cols], exprs)
        order, groups, ngroups, late = _group(DT, up, by_, sort_, isel, exprs)
        keys = by_.cols if by_ is not None else []
        if any(isinstance(e, Reducer) for e in exprs):
            if by_ is None:                     # one group over the selected rows (Groupby::single_group, groupby.cc:60-68)
                groups, ngroups = _one_group(self.nrows if order is None else len(order)), 1
            return _result(_reducer_cols(up, names, exprs, keys, order, groups, late), ngroups, _on_host(self))
        return _result(_row_cols(up, j_is_all(j), names, exprs, keys, order, groups),
                       self.nrows if order is None else len(order), _on_host(self))


def _from_list(lst):
    """Python list -> (array, stype) with None as NA (bool8 / int32 / int64 / float64 like the reference)."""
    vals = [x for x in lst if x is not None]
    if vals and all(isinstance(x, bool) for x in vals):
        return np.array([-128 if x is None else int(x) for x in lst], dtype=np.int8), BOOL
    if all(isinstance(x, int) for x in vals):
        big = any(abs(x) > 2**31 - 1 for x in vals)
        dt_, na = (np.int64, -2**63) if big else (np.int32, -2**31)
        return np.array([na if x is None else x for x in lst], dtype=dt_), (INT64 if big else INT32)
    return np.array([np.nan if x is None else float(x) for x in lst], dtype=np.float64), FLOAT64


_COPY_STREAMS = {}


def _copy_stream():
    """One upload stream per device for the life of the process.  torch's caching allocator keeps freed blocks per
    stream: a fresh stream per query (the first version) could never reuse the previous query's staging buffers and
    cudaMalloc'ed every uploaded column again (12 GB per C2 query until the device was full)."""
    dev = torch.cuda.current_device()
    if dev not in _COPY_STREAMS:
        _COPY_STREAMS[dev] = torch.cuda.Stream()
    return _COPY_STREAMS[dev]


_PIECE_BYTES = 1 << 30        # host value columns of >= 2 GB are uploaded (and reduced) in 1 GB pieces


def _on_host(*frames):
    """Whether a query's results go back to the host: none of the frames' columns is in HBM."""
    return not any(engine.is_tensor(c) and c.is_cuda for fr in frames for c in fr._cols.values())


def _dev(c):
    """The data of column c in HBM: c's own tensor when it is there, else a copy."""
    t = c.data if engine.is_tensor(c.data) else torch.from_numpy(np.ascontiguousarray(c.data))
    return t if t.is_cuda else t.cuda()


def _result(cols, nrows, host=False):
    """A result frame of the columns (name, data, stype), taken one at a time: a repeated name becomes name.0, name.1,
    ... (frame/names.cc: _deduplicate), and for a host frame a column in HBM comes back to the host as soon as it is
    taken, before the next one is computed."""
    out = Frame()
    for name, data, st in cols:
        name = str(name)                                   # a column of J is named after J's column
        base, k = name, 0
        while name in out._cols:
            name = f"{base}.{k}"
            k += 1
        if host and engine.is_tensor(data) and data.is_cuda:
            data = data.cpu().numpy()
        out._cols[name] = data
        out._stypes[name] = st
    out._nrows = nrows
    return out


def _resolve(DT, j, by_, sort_, isel=None):
    """(names, expressions of j, by_, sort_, isel) with every column reference bound to the column it names (_bind),
    and `i` other than an integer or an integer slice resolved into _Rows (_resolve_i).  Every check of the query's
    arguments runs here, before the device is touched."""
    if by_ is not None and sort_ is not None and sort_.na_position == "remove":
        # the rows dropped from the front of the RowIndex would still be counted by the groups
        raise ValueError("na_position = \"remove\" in sort() is not supported together with by()")
    if by_ is not None and _has_cut(j):                # FExpr_Cut::evaluate_n checks ctx.has_groupby() first
        raise NotImplementedError("cut() cannot be used in a groupby context")
    if by_ is not None:
        by_ = copy.copy(by_)
        by_.cols = [_bind(DT, r) for r in by_.cols]
    if sort_ is not None:
        sort_ = copy.copy(sort_)
        sort_.cols = [_bind(DT, r) for r in sort_.cols]
    if isinstance(isel, _ROW_SELECTORS):
        isel = _resolve_i(DT, isel, by_ is not None or sort_ is not None)
    names, exprs = _resolve_j(DT, j, [r.name for r in by_.cols] if by_ is not None else ())
    if torch is None or not torch.cuda.is_available():
        raise _lib.DtbCudaError("no usable CUDA device: datatable_b200 has no CPU fallback")
    return names, exprs, by_, sort_, isel


# ---------------------------------------------------------------------------
# `i` as a boolean or integer column, a list or a range (evaluate_i without by() / sort())
# ---------------------------------------------------------------------------
class _Rows:
    """A resolved `i`: the pieces whose RowIndices are concatenated, in order (RowIndex::concat of FExpr_List's
    _evaluate_i_other, fexpr_list.cc:225-243; one piece for every other form).  A piece is
        ("rows", int32 ndarray)   positions built on the host (ints, bools, slices, ranges)
        ("mask", name)            a bool8 column of the queried frame, X's own or J's (_JKey), read from HBM
        ("mask", Col)             a bool8 selector Frame's column
        ("ints", Col)             an integer selector Frame's column, checked against the rows once its min / max
                                  are known (fexpr_frame.cc:183-195)"""

    def __init__(self, pieces):
        self.pieces = pieces

    def mask_columns(self):
        """The queried frame's columns that select rows: uploaded first, as group keys are."""
        return [x for kind, x in self.pieces if kind == "mask" and not isinstance(x, engine.Col)]


_ROW_SELECTORS = (Frame, ColRef, list, tuple, range, np.ndarray)


def _i_kind(x):
    """The reference's name of the kind of expression x is (_name_type, fexpr_list.cc:117-132)."""
    if x is None:
        return "None"
    if isinstance(x, (bool, np.bool_)):
        return "bool"
    if isinstance(x, (int, np.integer)):
        return "integer"
    if isinstance(x, (float, np.floating)):
        return "float"
    if isinstance(x, str):
        return "string"
    if isinstance(x, ColRef):
        return "expression"
    if isinstance(x, range):
        return "integer slice"
    if isinstance(x, slice):
        if x == slice(None):
            return "slice"
        return "integer slice" if _int_slice(x) else "string-slice"
    return "?"                                   # a Frame, a numpy array, a nested list


def _int_slice(s):
    return all(v is None or (isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_)))
               for v in (s.start, s.stop, s.step))


def _rows_s(n):
    return f"{n} row{'' if n == 1 else 's'}"


def _resolve_i(DT, i, grouped):
    """_Rows of `i` over the rows of DT (FExpr_*::evaluate_i); under by() / sort() the reference's refusal
    (FExpr_*::evaluate_iby)."""
    if isinstance(i, (Frame, np.ndarray)):
        if grouped:
            raise TypeError("A Frame cannot be used as an i-selector in the presence of a groupby")
        return _Rows([_frame_piece(DT, i)])
    if isinstance(i, ColRef):
        if grouped:
            raise NotImplementedError("FExpr_Func::evaluate_iby() not implemented yet")
        return _Rows([_mask_piece(DT, i)])
    if isinstance(i, range):
        if grouped:
            raise NotImplementedError("A range selector cannot yet be used in i in the presence of by clause")
        return _Rows([_range_piece(DT.nrows, i)])
    if grouped:
        raise NotImplementedError("FExpr_List::evaluate_iby() not implemented yet")
    return _Rows(_list_pieces(DT, list(i)))


def _mask_piece(DT, ref):
    """f.b / g.b (FExpr_Func::evaluate_i, fexpr_func.cc:61-73): a bool8 column of X or, through the join, of J."""
    if ref.negated or isinstance(ref.name, slice):
        raise NotImplementedError(f"{ref!r} as a row filter is outside the GPU hot path")
    ref = _bind(DT, ref)
    if ref.name not in DT._stypes:
        raise KeyError(f"Column `{ref.name}` does not exist in the Frame")
    st = DT._stypes[ref.name]
    if st != BOOL:
        raise TypeError(f"Filter expression must be boolean, instead it was of type {_STYPE_NAMES.get(st, st)}")
    return ("mask", ref.name)


def _frame_piece(DT, sel):
    """A single-column Frame or a numpy array (FExpr_Frame::evaluate_i, fexpr_frame.cc:159-198): a bool8 column
    selects its rows whose value is true, an integer column lists rows."""
    if isinstance(sel, np.ndarray):
        if sel.ndim == 2:
            if sel.shape[1] != 1:
                raise ValueError(f"Only a single-column Frame may be used as `i` selector, instead got a Frame with "
                                 f"{sel.shape[1]} columns")
            sel = sel[:, 0]
        elif sel.ndim != 1:
            raise NotImplementedError(f"a {sel.ndim}-dimensional array as a row filter is outside the GPU hot path")
        sel = Frame({"C0": sel})
    if sel.ncols != 1:
        raise ValueError(f"Only a single-column Frame may be used as `i` selector, instead got a Frame with "
                         f"{sel.ncols} columns")
    if sel.key:
        raise NotImplementedError("A keyed frame cannot be used as an i selector")
    c = sel._col(sel.names[0])
    if c.stype == BOOL:
        if c.nrows != DT.nrows:
            raise ValueError(f"A boolean column used as `i` selector has {_rows_s(c.nrows)}, but applied to a Frame "
                             f"with {_rows_s(DT.nrows)}")
        return ("mask", c)
    if c.stype not in (INT8, INT16, INT32, INT64):
        raise TypeError(f"A Frame which is used as an `i` selector should be either boolean or integer, instead got "
                        f"`{_STYPE_NAMES.get(c.stype, c.stype)}`")
    return ("ints", c)


def _range_piece(n, r):
    """range(a, b, s) (FExpr_Literal_Range::evaluate_i, fexpr_literal_range.cc:87-96; orange::normalize)."""
    count = len(r)
    if count == 0:
        return ("rows", np.zeros(0, np.int32))
    a, z = r.start, r.start + (count - 1) * r.step
    if not (-n <= a < n and -n <= z < n) or (a >= 0) != (z >= 0):
        raise ValueError(f"{r!r} cannot be applied to a Frame with {_rows_s(n)}")
    if a < 0:
        a += n
    return ("rows", np.arange(a, a + count * r.step, r.step, dtype=np.int32)[:count])


def _slice_piece(n, s):
    """An integer slice (FExpr_Literal_SliceInt::evaluate_i, fexpr_literal_sliceint.cc:57-62) or f[:]'s every row."""
    if s.step == 0:
        raise NotImplementedError("repeat slices (step 0) without by() are outside the GPU hot path")
    return ("rows", np.arange(*s.indices(n), dtype=np.int32))


def _list_pieces(DT, items):
    """A list or tuple (FExpr_List::evaluate_i, fexpr_list.cc:225-316)."""
    n = DT.nrows
    if not items:
        return [("rows", np.zeros(0, np.int32))]
    kind0 = _i_kind(items[0])
    if kind0 == "bool":                                           # _evaluate_i_bools
        if len(items) != n:
            raise ValueError(f"The length of boolean list in i selector does not match the number of rows in the "
                             f"Frame: {len(items)} vs {n}")
        for k, x in enumerate(items):
            if _i_kind(x) != "bool":
                raise TypeError(f"Element {k} in the i-selector list is {_i_kind(x)}, whereas the previous elements "
                                f"were boolean")
        return [("rows", np.flatnonzero(np.array(items, dtype=bool)).astype(np.int32))]
    if kind0 == "integer":                                        # _evaluate_i_ints
        rows = []
        for k, x in enumerate(items):
            kind = _i_kind(x)
            if kind == "integer":
                x = int(x)
                if not -n <= x < n:
                    raise ValueError(f"Index {x} is invalid for a Frame with {n} rows")
                rows.append(x % n)
            elif kind in ("slice", "integer slice"):
                return _other_pieces(DT, items)
            elif kind != "None":
                raise TypeError(f"Invalid item of type {kind} at index {k} in the i-selector list")
        return [("rows", np.array(rows, dtype=np.int32))]
    return _other_pieces(DT, items)


def _other_pieces(DT, items):
    """_evaluate_i_other (fexpr_list.cc:225-243): every item's own RowIndex, None skipped."""
    n = DT.nrows
    pieces = []
    for k, x in enumerate(items):
        kind = _i_kind(x)
        if kind == "None":
            continue
        if isinstance(x, (Frame, np.ndarray)):
            pieces.append(_frame_piece(DT, x))
        elif kind == "integer":
            x = int(x)
            if not -n <= x < n:
                raise ValueError(f"Row `{x}` is invalid for a frame with {_rows_s(n)}")
            pieces.append(("rows", np.array([x % n], dtype=np.int32)))
        elif kind == "expression":
            pieces.append(_mask_piece(DT, x))
        elif isinstance(x, range):
            pieces.append(_range_piece(n, x))
        elif kind in ("slice", "integer slice"):
            pieces.append(_slice_piece(n, x))
        else:
            raise TypeError(f"Invalid expression of type {kind} at index {k} in the i-selector list")
    return pieces or [("rows", np.zeros(0, np.int32))]


def _selected_rows(DT, up, sel):
    """The int32 RowIndex in HBM of the resolved `i` sel (_Rows): the compaction of every boolean piece
    (dtb_mask_rows), every integer piece checked and made int32 (dtb_int_rows), the host-built pieces uploaded, and
    the pieces concatenated in order."""
    n = DT.nrows
    parts = []
    for kind, x in sel.pieces:
        if kind == "rows":
            parts.append(x)
        elif kind == "mask":
            parts.append(engine.mask_rows((up.col(x) if isinstance(x, str) else engine.Col(_dev(x), BOOL)).data))
        else:
            rows, lo, hi, nna = engine.int_rows(_dev(x), x.stype)
            if nna < x.nrows:                                     # fexpr_frame.cc:183-195
                if lo < 0:
                    raise ValueError(f"An integer column used as an `i` selector contains an invalid negative index: "
                                     f"{lo}")
                if hi >= n:
                    raise ValueError(f"An integer column used as an `i` selector contains index {hi} which is not "
                                     f"valid for a Frame with {_rows_s(n)}")
            parts.append(rows)
    if len(parts) == 1 and engine.is_tensor(parts[0]):
        return parts[0]
    if all(isinstance(p, np.ndarray) for p in parts):
        return torch.from_numpy(np.concatenate(parts) if len(parts) != 1 else parts[0]).cuda()
    out = torch.empty(builtins.sum(len(p) for p in parts), dtype=torch.int32, device="cuda")
    a = 0
    for p in parts:
        out[a:a + len(p)].copy_(torch.from_numpy(p) if isinstance(p, np.ndarray) else p)
        a += len(p)
    return out


def _join_view(X, J):
    """X joined to the keyed frame J (natural_join, frame/join.cc:392-470): a frame of X's columns that also knows
    every column of J by its _JKey and stype.  _Upload adds the columns of J the query reads, in X's row order."""
    for nm in J.key:
        if nm not in X._cols:
            raise ValueError(f"Key column `{nm}` does not exist in the left Frame")
    V = Frame()
    V._cols, V._stypes, V._nrows = dict(X._cols), dict(X._stypes), X.nrows
    V._stypes.update((_JKey(nm), st) for nm, st in J._stypes.items())
    V._joined = J
    return V


def _bind(DT, ref):
    """The column ColRef `ref` names (FExpr_ColumnAsAttr::evaluate_n, fexpr_column_asattr.cc:38-48), as the ColRef
    of its key in DT: g.x is J's column x (_JKey); f.x is X's column x or, where X has no x and J has a non-key
    column x, J's x.  The reference raises KeyError for the latter; here DT[:, f.v, join(J)] keeps reading J's v."""
    if isinstance(ref.name, slice):
        if ref.frame:
            raise NotImplementedError("column slices of the join frame are outside the GPU hot path")
        return ref
    J = DT._joined
    if ref.frame:
        if J is None:
            raise ValueError("Column expression references a non-existing join frame")
        if ref.name not in J._cols:
            raise KeyError(f"Column `{ref.name}` does not exist in the Frame")
        return ColRef(_JKey(ref.name), ref.negated)
    if J is not None and ref.name not in DT._cols and ref.name in J._cols and ref.name not in J.key:
        return ColRef(_JKey(ref.name), ref.negated)
    return ref


def _bind_expr(DT, e):
    """Expression e of j with its column references bound (_bind); row functions bind theirs in _rowfn_cols."""
    if isinstance(e, ColRef):
        return _bind(DT, e)
    if isinstance(e, Reducer) and isinstance(e.arg, ColRef):
        e = copy.copy(e)
        e.arg = _bind(DT, e.arg)
        if isinstance(e, Reducer2):
            e.arg2 = _bind(DT, e.arg2)
    return e


class _Upload:
    """The columns a query reads, in HBM.  Host columns are uploaded once (pinned memory -> DMA), the whole query then
    runs on HBM-resident buffers, and only the result frame travels back.  Every upload the query needs starts here,
    on a copy stream, key columns first, so that the PCIe transfer of the value columns overlaps the sort of the keys;
    col(name) waits for a column (stream event) only where it is first used.
    A joined query (DT from _join_view) uploads X's join key columns right after its group keys; once they have
    arrived, one join_gather reads every column of J the query uses, in X's row order, and from then on those
    columns are read like X's own."""

    def __init__(self, DT, keynames, exprs):
        self.frame = DT
        self._cache = {}
        self._pending = {}        # name -> (Col in HBM, event of its upload)
        self._pieces = {}         # large value columns travel in pieces, each with its own event (see _late_reduce)
        needed = list(keynames)
        for e in exprs:
            nm = e.arg.name if isinstance(e, Reducer) and e.arg is not None else getattr(e, "name", None)
            if nm is not None:
                needed.append(nm)
            if isinstance(e, Reducer2):
                needed.append(e.arg2.name)
        needed = list(dict.fromkeys(needed))
        jneeded = [nm for nm in needed if isinstance(nm, _JKey)]
        joinkeys = list(DT._joined.key) if jneeded else []
        keynames = [nm for nm in keynames if not isinstance(nm, _JKey)] + joinkeys
        copy_stream = None
        for nm in dict.fromkeys(keynames + [nm for nm in needed if not isinstance(nm, _JKey)]):
            c = DT._col(nm)
            t = c.data if engine.is_tensor(c.data) else torch.from_numpy(c.data)
            if t.is_cuda:
                continue
            if copy_stream is None:
                copy_stream = _copy_stream()
                copy_stream.wait_stream(torch.cuda.current_stream())    # buffers freed by earlier queries are reused in order
            with torch.cuda.stream(copy_stream):
                if nm not in keynames and t.dim() == 1 and t.numel() * t.element_size() >= _PIECE_BYTES * 2:
                    d = torch.empty_like(t, device="cuda")
                    step = builtins.max(1, _PIECE_BYTES // t.element_size())
                    pcs = []
                    for a in range(0, t.numel(), step):
                        b = builtins.min(a + step, t.numel())
                        d[a:b].copy_(t[a:b], non_blocking=True)
                        pev = torch.cuda.Event(); pev.record(copy_stream)
                        pcs.append((a, b, pev))
                    self._pieces[nm] = pcs
                    ev = pcs[-1][2]
                else:
                    d = t.cuda(non_blocking=True)                       # pinned host memory -> async DMA
                    ev = torch.cuda.Event(); ev.record(copy_stream)
            self._pending[nm] = (engine.Col(d, c.stype), ev)
        if jneeded:
            J = DT._joined
            jcol = lambda nm: engine.Col(_dev(J._col(nm)), J._stypes[nm])     # noqa: E731
            vals = engine.join_gather([self.col(nm) for nm in joinkeys], [jcol(nm) for nm in joinkeys],
                                      [jcol(str(nm)) for nm in jneeded])
            for nm, v in zip(jneeded, vals):
                DT._cols[nm] = v
                self._cache[nm] = engine.Col(v, DT._stypes[nm])

    def col(self, name):
        if name not in self._cache:
            if name in self._pending:
                c, ev = self._pending[name]
                torch.cuda.current_stream().wait_event(ev)
                c.data.record_stream(torch.cuda.current_stream())
            else:
                c = self.frame._col(name)
                c = engine.Col(_dev(c), c.stype)
            self._cache[name] = c
        return self._cache[name]

    def arriving(self, name):
        """Whether the column is still on its way: its upload was started and nothing has waited for it yet."""
        return name in self._pending and name not in self._cache

    def pieces(self, name):
        """[(rows, row0, event), ...] of a column that is still arriving in pieces, else None."""
        if name not in self._pieces or not self.arriving(name):
            return None
        c = self._pending[name][0]
        c.data.record_stream(torch.cuda.current_stream())
        return [(c.data[a:b], a, ev) for a, b, ev in self._pieces[name]]


def _one_group(n, none_if_empty=False):
    """Offsets of one group over n rows (Groupby::single_group, groupby.cc:60-68); none_if_empty: no group when n is
    0.  A blocking copy to the device: made only where a query needs it."""
    return torch.tensor([0, n] if n or not none_if_empty else [0], dtype=torch.int32, device="cuda")


def _group(DT, up, by_, sort_, isel, exprs):
    """compute_groupby_and_sort (eval_context.cc:249-288) and `i`: (order, groups, ngroups, late).
    order: the RowIndex of the selected rows, None for every row in place.  groups: the Groupby offsets, the Groupby
    handle for by() with reducers, or None without by() / sort().  late: the handle was made without the reducers
    (see _groupby_handle).  isel, an integer or integer slice for `i`, is applied inside every group under by() /
    sort() (iexpr_->evaluate_iby, eval_context.cc:154-158), to the rows otherwise (evaluate_i, :159-163); the other
    forms of `i` (_Rows) only exist without by() / sort()."""
    keycols, flags = [], []
    na_pos = NA_FIRST
    if by_ is not None:
        for ref in by_.cols:
            keycols.append(up.col(ref.name))
            flags.append(FLAG_DESCENDING if ref.negated else 0)
    if sort_ is not None:
        na_pos = _NA_POS[sort_.na_position]
        for ref, rev in zip(sort_.cols, sort_.reverse):
            keycols.append(up.col(ref.name))
            desc = (not rev) if ref.negated else rev                 # fexpr_list.cc:346-358
            flags.append((FLAG_DESCENDING if desc else 0) | FLAG_SORT_ONLY)
    if keycols and isel is not None:
        # i under by() / sort(): group() first, then the slice inside every group; its positions are composed with
        # the RowIndex (apply_rowindex) and the Groupby is replaced (replace_groupby)
        order, offsets, _ = engine.group(keycols, flags, na_pos)
        if offsets is None:                                            # sort() alone: Groupby::single_group
            offsets = _one_group(len(order))
        if isinstance(isel, int):
            st_, sp_, se_ = isel, (isel + 1 if isel != -1 else None), 1     # fexpr_literal_int.cc:146-192 == the slice [i, i+1)
            if not -2**31 <= isel < 2**31:
                st_, sp_, se_ = 0, 0, 1
        else:
            st_, sp_, se_ = isel.start, isel.stop, isel.step
        sel, offsets = engine.slice_groups(offsets, st_, sp_, se_)
        return engine.gather(order, sel), offsets, len(offsets) - 1, False
    if isinstance(isel, _Rows):
        return _selected_rows(DT, up, isel), None, None, False
    if isel is not None:
        # no by() / sort(): evaluate_i -- a plain row slice (python slice semantics; step 0 = repeat is not taken here)
        n_ = DT.nrows
        if isinstance(isel, int):
            if not -n_ <= isel < n_:
                raise ValueError(f"Row `{isel}` is invalid for a frame with {n_} row{'s' if n_ != 1 else ''}")
            rng_ = range(isel % n_, isel % n_ + 1)
        else:
            if isel.step == 0:
                raise NotImplementedError("repeat slices (step 0) without by() are outside the GPU hot path")
            rng_ = range(*isel.indices(n_))
        return torch.arange(rng_.start, rng_.stop, rng_.step, dtype=torch.int32, device="cuda"), None, None, False
    if not keycols:
        return None, None, None, False
    if by_ is not None and any(isinstance(e, Reducer) for e in exprs):
        gb, late = _groupby_handle(up, keycols, flags, na_pos, exprs)
        return None, gb, gb.ngroups, late
    order, offsets, ngroups = engine.group(keycols, flags, na_pos)
    return order, offsets, ngroups, False


def _fused(exprs):
    """The reducers of j that a Groupby handle evaluates by itself: all but cov / corr and median / nunique (which
    read the rows sorted inside their group), in the order of j."""
    return [e for e in exprs if isinstance(e, Reducer) and e.op not in _SORTED_OPS and not isinstance(e, Reducer2)]


def _groupby_handle(up, keycols, flags, na_pos, exprs):
    """group() for by() with reducers: (Groupby handle, late).  The RowIndex and the Groupby stay in HBM behind the
    handle.  The reducers of j are known before group() runs: they are handed over so that the engine can overlap
    them with the sort (dtb_groupby_create_reduce).
    Host frame whose value columns are still on their way over PCIe (late): group() first (the sort runs under the
    upload), the reducers afterwards through the handle, each waiting only for its own column.  Handing the reducers
    to group() would make the stream wait for every value column before the sort starts.  Columns with several
    reducers keep the fused call (bucketed multi-reducer)."""
    fused = _fused(exprs)
    arriving = [e.arg.name for e in fused if e.arg is not None and up.arriving(e.arg.name)]
    per_col = {nm: builtins.sum(2 if e.op == _lib.OP_MEAN else 1 for e in fused if e.arg is not None and e.arg.name == nm)
               for nm in arriving}
    if arriving and all(c < 2 for c in per_col.values()):
        return engine.Groupby(keycols, flags, na_pos), True
    reds = [(e.op, None if e.arg is None else up.col(e.arg.name)) for e in fused]
    return engine.Groupby(keycols, flags, na_pos, reducers=reds), False


def _late_reduce(up, gb, e):
    """Reducer e of a late handle.  A column still arriving in pieces is folded piece by piece, every piece as soon
    as it has arrived (dtb_groupby_reduce_add): after the last byte only the last piece's share of the reducer is
    left."""
    nm = None if e.arg is None else e.arg.name
    pieces = up.pieces(nm)
    res = None if pieces is None else gb.reduce_pieces(e.op, up.frame._stypes[nm], pieces)
    return res if res is not None else gb.reduce(e.op, None if nm is None else up.col(nm))


def _reducer_cols(up, names, exprs, keys, order, groups, late):
    """One row per group: the by() keys `keys` from the first row of every group (get_group_rowindex,
    eval_context.cc:124-135), then every reducer of j, over the Groupby handle `groups` or over (order, offsets
    `groups`).  Yields (name, data, stype) one column at a time: the keys of a late handle reach the host while the
    value columns are still arriving, before the reducers fold them."""
    gb = groups if isinstance(groups, engine.Groupby) else None
    if keys:
        first = gb.first_rows() if gb is not None else engine.gather(order, groups[:-1])
        for ref in keys:
            c = up.col(ref.name)
            yield ref.name, engine.gather(c, first), c.stype
    bynames = [r.name for r in keys]
    if late:
        late_results = iter([_late_reduce(up, gb, e) for e in _fused(exprs)])
    ifused = 0
    npos = gb.norder if gb is not None else (up.frame.nrows if order is None else len(order))
    for name, e in zip(names, exprs):
        if not isinstance(e, Reducer):
            raise NotImplementedError("mixing reducers and plain columns under by() is outside the hot path")
        if e.op == _lib.OP_MEDIAN and npos == 0 and _red_stype(up.col, e):
            # over zero rows the reference's median is an NA column of its argument's own stype, not of the median's
            # (compute_median, head_reduce_unary.cc:493-496)
            st = up.col(e.arg.name).stype
            ng = gb.ngroups if gb is not None else int(groups.shape[0]) - 1
            yield name, torch.full((ng,), float("nan") if st in (FLOAT32, FLOAT64) else _NA_VALUE[st],
                                   dtype=engine._torch_dtype(st), device="cuda"), st
            continue
        if gb is None:
            data = _reduce(up.col, e, order, groups, bynames)
        elif isinstance(e, Reducer2):
            data = _reduce2_grouped(up.col, e, bynames, gb.ngroups, lambda x, y: gb.reduce2(e.op, x, y))
        elif e.op in _SORTED_OPS:
            c = up.col(e.arg.name)                      # Median_ColumnImpl::pre_materialize_hook: sort_grouped first
            data = gb.reduce_ordered(e.op, c, gb.sort_grouped(c))
        else:
            data = next(late_results) if late else gb.reduced(ifused)
            ifused += 1
        yield name, data, _red_stype(up.col, e)
    if gb is not None:
        gb.close()


def _row_cols(up, j_all, names, exprs, keys, order, offsets):
    """One row per position of `order` (None: every row in place).  Under by() the key columns come first, and j = :
    leaves them out of the rest; row functions run inside every group of `offsets`, without by() inside one group of
    the selected rows in their order.  Yields (name, data, stype) one column at a time."""
    for ref in keys:
        c = up.col(ref.name)
        yield ref.name, engine.gather(c, order), c.stype
    bynames = [r.name for r in keys]
    for name, e in zip(names, exprs):
        if e.name in bynames and j_all:
            continue
        if isinstance(e, RowFnCol):                    # in the grouped order (GtoALL)
            offs = offsets if keys else _one_group(up.frame.nrows if order is None else len(order), none_if_empty=True)
            yield (name, *e.run(None if e.name is None else up.col(e.name), order, offs))
        elif order is None:
            c = up.frame._col(e.name)
            yield name, c.data, c.stype
        else:
            c = up.col(e.name)
            yield name, engine.gather(c, order), c.stype


def j_is_all(j):
    return isinstance(j, slice) and j == slice(None)


def _resolve_j(DT, j, bynames=()):
    if j_is_all(j):
        # every column of X, then J's non-key columns (FExpr_Literal_SliceAll::evaluate_j, fexpr_literal_sliceall.cc:55-66)
        J = DT._joined
        ks = [n for n in DT.names if not isinstance(n, _JKey)] + ([] if J is None else
                                                                  [_JKey(n) for n in J.names if n not in J.key])
        return list(ks), [ColRef(n) for n in ks]
    if isinstance(j, dict):
        names, es = [], []
        for k, v in j.items():
            vs = v if isinstance(v, list) else [v]              # a broadcast cov / corr: k, k.0, k.1, ... (see add)
            for x in vs:
                if isinstance(x, RowFn):                        # several columns: k.x, k.y, ...
                    qc = _rowfn_cols(DT, x, bynames)
                    names += [k] if len(qc) == 1 else [f"{k}.{c.label or c.name}" for c in qc]
                    es += qc
                else:
                    names.append(k)
                    es.append(_bind_expr(DT, _as_expr(x)))
        return names, es
    if isinstance(j, (list, tuple)):
        es = [_bind_expr(DT, _as_expr(x)) for v in j for x in (v if isinstance(v, list) else [v])]
    else:
        es = [_bind_expr(DT, _as_expr(x)) for x in (j if isinstance(j, list) else [j])]
    es = [c for e in es for c in (_rowfn_cols(DT, e, bynames) if isinstance(e, RowFn) else [e])]
    names = []
    nbin = 0
    for e in es:
        if isinstance(e, Reducer2) or (isinstance(e, RowFnCol) and e.name is None and e.label is None):
            names.append(f"C{nbin}")                                  # unnamed columns (cov, corr, cumcount, ngroup): C0, C1, ...
            nbin += 1
        elif isinstance(e, Reducer):
            names.append("count" if e.arg is None else e.arg.name)     # reducers keep the column's name
        else:
            names.append(e.label if isinstance(e, RowFnCol) and e.label is not None else e.name)
    return names, es


def _as_expr(v):
    if isinstance(v, (Reducer, ColRef, RowFn)):
        return v
    if isinstance(v, str):
        return ColRef(v)
    raise TypeError(f"Unsupported j expression {v!r}")


def _red_stype(dcol, e):
    """Output stype of a reducer column (bool8 min/max stay bool8, fexpr_minmax.cc:50-72)."""
    if e.op == _lib.OP_NROWS or e.arg is None:
        return INT64
    if isinstance(e, Reducer2):
        return engine.reduce2_out_stype(e.op, dcol(e.arg.name).stype, dcol(e.arg2.name).stype)
    return engine.reduce_out_stype(e.op, dcol(e.arg.name).stype)


_SORTED_OPS = (_lib.OP_MEDIAN, _lib.OP_NUNIQUE)


def _reduce2_grouped(dcol, e, bynames, ngroups, run):
    """cov / corr: an all-NA column when either argument is a by() column (make_na_result, head_reduce_binary.cc:48-52,
    240-251), else run(x, y)."""
    if e.arg.name in bynames or e.arg2.name in bynames:
        st = engine.reduce2_out_stype(e.op, dcol(e.arg.name).stype, dcol(e.arg2.name).stype)
        if not st:
            raise _lib.DtbValueError(f"Invalid columns in reducer {e.opname}")
        return torch.full((ngroups,), float("nan"), dtype=torch.float32 if st == FLOAT32 else torch.float64, device="cuda")
    return run(dcol(e.arg.name), dcol(e.arg2.name))


def _reduce(dcol, e, order, offsets, bynames=()):
    if isinstance(e, Reducer2):
        return _reduce2_grouped(dcol, e, bynames, int(offsets.shape[0]) - 1,
                                lambda x, y: engine.reduce2(e.op, x, y, order, offsets))
    if e.op == _lib.OP_NROWS:
        return engine.reduce(e.op, None, order, offsets)
    c = dcol(e.arg.name)
    if e.op in _SORTED_OPS:
        order = engine.sort_grouped(c, order, offsets)
    return engine.reduce(e.op, c, order, offsets)


# ---------------------------------------------------------------------------
# Callers of group() beyond DT[i, j, by, sort] (SURVEY.md 8f): set operations, column statistics, join
# ---------------------------------------------------------------------------
_NUM_ORDER = [BOOL, INT8, INT16, INT32, INT64, FLOAT32, FLOAT64]
_TORCH_OF = {BOOL: "int8", INT8: "int8", INT16: "int16", INT32: "int32", INT64: "int64", FLOAT32: "float32", FLOAT64: "float64"}


def _promote(cols):
    """Common stype of rbind-ed columns with NA mapped: the highest input stype, as Type::common gives for numeric
    types (types/typeimpl_numeric.cc:36-41), so float32 beats every integer type.  Each value is cast once, on the
    device (int64 -> float32 rounds once, as the reference's cast does)."""
    sts = {c.stype for c in cols}
    if len(sts) == 1:
        return [_dev(c) for c in cols], cols[0].stype
    tgt = builtins.max(sts, key=_NUM_ORDER.index)
    isf = tgt in (FLOAT32, FLOAT64)
    out = []
    for c in cols:
        t = _dev(c)
        if c.stype != tgt:
            if c.stype in (FLOAT32, FLOAT64):
                t = t.to(getattr(torch, _TORCH_OF[tgt]))
            else:
                na = t == _NA_VALUE[c.stype]
                t = t.to(getattr(torch, _TORCH_OF[tgt]))
                t = torch.where(na, torch.full_like(t, float("nan") if isf else _NA_VALUE[tgt]), t)
        out.append(t)
    return out, tgt


def _set_op(mode, frames):
    frames = [fr for fr in _flatten(frames)]
    for fr in frames:
        if not isinstance(fr, Frame):
            raise TypeError("set functions expect a list or sequence of Frames")
        if fr.ncols > 1:
            raise ValueError(f"Only single-column Frames are allowed, but received a Frame with {fr.ncols} columns")
    frames = [fr for fr in frames if fr.ncols == 1]
    if not frames:
        return Frame()
    name = frames[0].names[0]
    tens, st = _promote([fr._col(fr.names[0]) for fr in frames])
    if len(frames) <= 1:
        mode = _lib.SET_UNION                                  # set_funcs.cc:302-305, 356-359, 438-441
    cat = tens[0] if len(tens) == 1 else torch.cat(tens)
    cd = engine.Col(cat, st)
    if cat.numel() == 0:
        vals = cat
    else:
        order, offsets, ng = engine.group([cd], [0], NA_FIRST)
        rows = engine.set_select(mode, order, offsets, np.cumsum([t.numel() for t in tens]))
        vals = engine.gather(cd, rows)
    return _result([(name, vals, st)], int(vals.shape[0]), _on_host(*frames))


def union(*frames): return _set_op(_lib.SET_UNION, frames)
def intersect(*frames): return _set_op(_lib.SET_INTERSECT, frames)
def setdiff(*frames): return _set_op(_lib.SET_SETDIFF, frames)
def symdiff(*frames): return _set_op(_lib.SET_SYMDIFF, frames)


def unique(frame):
    """dt.unique(frame): the sorted unique values (NA first) -- the union of the frame's columns
    (set_funcs.cc:183-196).  The result keeps the name of a single column; of several it is named C0, the default
    name of a column whose name the reference leaves empty."""
    return _set_op(_lib.SET_UNION, [_result([(nm if frame.ncols == 1 else "C0", frame._cols[nm], frame._stypes[nm])],
                                            frame.nrows) for nm in frame.names])


def _column_groups(frame, name):
    c = frame._col(name)
    cd = engine.Col(_dev(c), c.stype)
    if cd.nrows == 0:
        return cd, None, None, 0, False
    order, offsets, ng = engine.group([cd], [0], NA_FIRST)
    # the NA rows sort first: the column has NAs iff the first sorted row is NA (stats.cc:966-975)
    first = engine.gather(cd, order[:1]).cpu().numpy()
    has_na = bool(np.isnan(first[0])) if c.stype in (FLOAT32, FLOAT64) else bool(first[0] == _NA_VALUE[c.stype])
    return cd, order, offsets, ng, has_na


def _frame_nunique(frame):
    """Frame.nunique(): distinct non-NA values per column (stats.cc:955-979 via group())."""
    cols = []
    for name in frame.names:
        cd, order, offsets, ng, has_na = _column_groups(frame, name)
        cols.append((name, np.array([ng - int(has_na)], dtype=np.int64), INT64))
    return _result(cols, 1)


def _frame_mode(frame):
    """(Frame.mode(), Frame.nmodal()): value and size of the first largest non-NA group (stats.cc:981-1003)."""
    mode, nmodal = [], []
    for name in frame.names:
        cd, order, offsets, ng, has_na = _column_groups(frame, name)
        idx, size = (-1, 0) if order is None else engine.largest_group(offsets, int(has_na))
        if size:
            val = engine.gather(cd, engine.gather(engine.Col(order, INT32), offsets[idx:idx + 1])).cpu().numpy()
        else:
            val = np.array([np.nan if cd.stype in (FLOAT32, FLOAT64) else _NA_VALUE[cd.stype]],
                           dtype=getattr(np, _TORCH_OF[cd.stype]))
        mode.append((name, val, cd.stype))
        nmodal.append((name, np.array([size], dtype=np.int64), INT64))
    return _result(mode, 1), _result(nmodal, 1)
