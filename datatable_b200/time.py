"""
datatable_b200.time -- the calendar and clock parts of date32 / time64 columns, as datatable.time provides them
(src/core/expr/time/): year, month, day, day_of_week (ISO: Monday = 1 .. Sunday = 7) of a date32 or time64 column,
hour, minute, second, nanosecond of a time64 column.  Each is an int32 column computed on the GPU (dtb_time_part).

The argument is a column, a list or tuple of columns, f[:] or a joined frame's g. columns.  In j a part is a row
function, with or without by(); in by() and sort() it is a derived key (-year(f.d): descending), computed once over the
frame and grouped like a stored column.
"""
from . import _lib
from .frame import TimePart

__all__ = ["year", "month", "day", "day_of_week", "hour", "minute", "second", "nanosecond"]


def _part(part, fname, argname, args, kwargs):
    """The reference's argument checks (py::XArgs: one positional-only argument)."""
    for k in kwargs:
        if k == argname and args:
            raise TypeError(f"Function datatable.{fname}() got multiple values for argument {k}")
        if k == argname:
            raise TypeError(f"Function datatable.{fname}() got argument {k} as a keyword, but it should be "
                            f"positional-only")
        raise TypeError(f"Function datatable.{fname}() got an unexpected keyword argument {k}")
    if len(args) > 1:
        raise TypeError(f"Function datatable.{fname}() takes only one positional argument, but {len(args)} were given")
    if not args:
        raise TypeError(f"Function datatable.{fname}() requires exactly 1 positional argument, but none were given")
    return TimePart(part, fname, args[0])


def year(*args, **kwargs): return _part(_lib.TIME_YEAR, "year", "date", args, kwargs)
def month(*args, **kwargs): return _part(_lib.TIME_MONTH, "month", "date", args, kwargs)
def day(*args, **kwargs): return _part(_lib.TIME_DAY, "day", "date", args, kwargs)
def day_of_week(*args, **kwargs): return _part(_lib.TIME_DAY_OF_WEEK, "day_of_week", "date", args, kwargs)
def hour(*args, **kwargs): return _part(_lib.TIME_HOUR, "hour", "time", args, kwargs)
def minute(*args, **kwargs): return _part(_lib.TIME_MINUTE, "minute", "time", args, kwargs)
def second(*args, **kwargs): return _part(_lib.TIME_SECOND, "second", "time", args, kwargs)
def nanosecond(*args, **kwargs): return _part(_lib.TIME_NANOSECOND, "nanosecond", "time", args, kwargs)
