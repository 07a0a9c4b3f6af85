"""A numpy restatement of the reference's `i` node without by() / sort() (FExpr_*::evaluate_i) for the forms
datatable_b200 runs on the GPU: a boolean or integer column, a list, a range.  Selectors are given as
("mask", int8 bool8 array) / ("ints", integer array, its NA value), Python ints, None, slices, ranges and lists of
them.  rows(sel, n) returns the int64 RowIndex, -1 for an NA row.

    bool8 column      ArrayRowIndexImpl::init_from_boolean_column (rowindex_array.cc:130-170): rows whose value is
                      valid and non-zero, ascending
    integer column    RowIndex(const Column&) (rowindex_array.cc:63-128): the values in their order, NA -> NA row
    list              FExpr_List::evaluate_i (fexpr_list.cc:225-316): ints (negatives wrap), bools, or the
                      concatenation of every item's RowIndex
    range             FExpr_Literal_Range::evaluate_i (fexpr_literal_range.cc:87-96)
"""
import numpy as np


def mask_rows(m):
    m = np.asarray(m).view(np.int8) if np.asarray(m).dtype == np.bool_ else np.asarray(m, dtype=np.int8)
    return np.flatnonzero((m != 0) & (m != -128)).astype(np.int64)


def int_rows(a, na):
    a = np.asarray(a).astype(np.int64)
    return np.where(a == na, -1, a)


def range_rows(r, n):
    count = len(r)
    if count == 0:
        return np.zeros(0, np.int64)
    a, z = r.start, r.start + (count - 1) * r.step
    if not (-n <= a < n and -n <= z < n) or (a >= 0) != (z >= 0):
        raise ValueError(f"{r!r} cannot be applied to a Frame with {n} row{'' if n == 1 else 's'}")
    a += n if a < 0 else 0
    return a + r.step * np.arange(count, dtype=np.int64)


def rows(sel, n):
    if isinstance(sel, tuple) and sel and sel[0] == "mask":
        return mask_rows(sel[1])
    if isinstance(sel, tuple) and sel and sel[0] == "ints":
        return int_rows(sel[1], sel[2])
    if isinstance(sel, range):
        return range_rows(sel, n)
    if isinstance(sel, slice):
        return np.arange(*sel.indices(n), dtype=np.int64)
    if isinstance(sel, bool):
        raise TypeError("A boolean value cannot be used as a row selector")
    if isinstance(sel, int):
        if not -n <= sel < n:
            raise ValueError(f"Row `{sel}` is invalid for a frame with {n} row{'' if n == 1 else 's'}")
        return np.array([sel % n], np.int64)
    assert isinstance(sel, list)
    if not sel:
        return np.zeros(0, np.int64)
    if all(isinstance(x, bool) for x in sel):
        if len(sel) != n:
            raise ValueError(f"The length of boolean list in i selector does not match the number of rows in the "
                             f"Frame: {len(sel)} vs {n}")
        return np.flatnonzero(np.array(sel, bool)).astype(np.int64)
    if all(x is None or (isinstance(x, int) and not isinstance(x, bool)) for x in sel) and sel[0] is not None:
        for x in sel:
            if x is not None and not -n <= x < n:
                raise ValueError(f"Index {x} is invalid for a Frame with {n} rows")
        return np.array([x % n for x in sel if x is not None], np.int64)
    parts = [rows(x, n) for x in sel if x is not None]
    return np.concatenate(parts) if parts else np.zeros(0, np.int64)


def gather(col, ri, na):
    """col seen through the RowIndex ri (-1: NA)"""
    out = col[np.maximum(ri, 0)] if len(col) else np.full(len(ri), na, col.dtype)
    out = np.array(out, copy=True)
    out[ri < 0] = na
    return out


# The error of every golden_v11 case on which the reference's process died in the generator
# (`reference_crash`): (type, text) as the reference's source writes them (fexpr_frame.cc:160-194,
# fexpr_list.cc:225-316, fexpr_literal_int.cc:135-143, fexpr_literal_range.cc:87-96).
SOURCE_ERRORS = {
    "err.frame_len": ("ValueError", "A boolean column used as `i` selector has 299 rows, but applied to a Frame with "
                                    "300 rows"),
    "err.frame_len1": ("ValueError", "A boolean column used as `i` selector has 1 row, but applied to a Frame with "
                                     "300 rows"),
    "err.frame_2cols": ("ValueError", "Only a single-column Frame may be used as `i` selector, instead got a Frame "
                                      "with 2 columns"),
    "err.numpy_2d": ("ValueError", "Only a single-column Frame may be used as `i` selector, instead got a Frame with "
                                   "2 columns"),
    "err.list_int_bool": ("TypeError", "Invalid item of type bool at index 1 in the i-selector list"),
    "err.list_bool_int": ("ValueError", "The length of boolean list in i selector does not match the number of rows "
                                        "in the Frame: 2 vs 8"),
    "err.list_bool_len": ("ValueError", "The length of boolean list in i selector does not match the number of rows "
                                        "in the Frame: 2 vs 8"),
    "err.list_float": ("TypeError", "Invalid expression of type float at index 0 in the i-selector list"),
    "err.list_int_float": ("TypeError", "Invalid item of type float at index 1 in the i-selector list"),
    "err.list_slice_float": ("TypeError", "Invalid expression of type float at index 1 in the i-selector list"),
    "err.list_int_frame": ("TypeError", "Invalid item of type ? at index 1 in the i-selector list"),
    "err.list_slice_bool": ("TypeError", "Invalid expression of type bool at index 1 in the i-selector list"),
    "err.list_index": ("ValueError", "Index 9 is invalid for a Frame with 8 rows"),
    "err.list_row": ("ValueError", "Row `9` is invalid for a frame with 8 rows"),
    "err.list_nested": ("TypeError", "Invalid expression of type ? at index 0 in the i-selector list"),
    "err.list_none_bool": ("TypeError", "Invalid expression of type bool at index 1 in the i-selector list"),
    "err.list_bool_none": ("TypeError", "Element 2 in the i-selector list is None, whereas the previous elements "
                                        "were boolean"),
    "err.list_bool_elem": ("TypeError", "Element 1 in the i-selector list is integer, whereas the previous elements "
                                        "were boolean"),
    "err.range": ("ValueError", "range(10, 0, -3) cannot be applied to a Frame with 8 rows"),
    "err.range_mixed": ("ValueError", "range(-2, 3) cannot be applied to a Frame with 8 rows"),
    "err.range1": ("ValueError", "range(0, 2) cannot be applied to a Frame with 1 row"),
    # the integer selector's checks read its min / max: raised once the device has computed them
    "err.frame_i16_neg": ("ValueError", "An integer column used as an `i` selector contains an invalid negative "
                                        "index: -3"),
    "err.frame_i32_neg": ("ValueError", "An integer column used as an `i` selector contains an invalid negative "
                                        "index: -3"),
    "err.frame_i64_neg": ("ValueError", "An integer column used as an `i` selector contains an invalid negative "
                                        "index: -3"),
    "err.frame_i16_big": ("ValueError", "An integer column used as an `i` selector contains index 307 which is not "
                                        "valid for a Frame with 300 rows"),
    "err.frame_i32_big": ("ValueError", "An integer column used as an `i` selector contains index 307 which is not "
                                        "valid for a Frame with 300 rows"),
    "err.frame_i64_big": ("ValueError", "An integer column used as an `i` selector contains index 307 which is not "
                                        "valid for a Frame with 300 rows"),
    "err.frame_i8_big": ("ValueError", "An integer column used as an `i` selector contains index 5 which is not valid "
                                       "for a Frame with 1 row"),
}
DATA_ERRORS = {k for k in SOURCE_ERRORS if k.startswith("err.frame_i")}
