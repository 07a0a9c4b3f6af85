"""
datatable_b200 -- H100-native groupby/sort engine behind h2oai/datatable's
DT[i, j, by(), sort()] hot path.  See DESIGN.md / INTEGRATION.md.

Importing this package loads libdtb200.so (sm_90a CUDA); it raises if the
library has not been built.  There is no CPU fallback.
"""
from . import _lib
from ._lib import (DtbError, DtbValueError, DtbNotImplError, DtbCudaError, DtbMemoryError)
from . import engine
from .frame import (Frame, f, g, by, sort, join, sum, prod, cov, corr, mean, min, max, count, countna, first, last, sd, median,   # noqa: A004
                    qcut, cut, cumsum, cumprod, cummin, cummax, shift, fillna, cumcount, ngroup, unique, nunique, union, intersect, setdiff, symdiff)
from .jay import open_jay, save_jay
from . import time

__all__ = ["engine", "Frame", "f", "g", "by", "sort", "sum", "prod", "cov", "corr", "mean", "min", "max", "count", "countna", "first", "last", "sd", "median", "qcut", "cut", "cumsum", "cumprod", "cummin", "cummax", "shift", "fillna", "cumcount", "ngroup", "join", "time", "unique", "nunique", "union", "intersect", "setdiff", "symdiff", "open_jay", "save_jay", "DtbError", "DtbValueError", "DtbNotImplError", "DtbCudaError", "DtbMemoryError"]
