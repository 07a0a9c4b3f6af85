"""The argument contract of the per-group entry points (include/dtb200.h, "Per-group functions").

CPU: every entry point that takes raw offsets, and dtb_gather, returns the code and the message of the first failing
check, in the documented order, before any CUDA call -- so the same with or without a device.
GPU: what needs the offsets' values or a handle: offsets that are not a Groupby, out = NULL past the host checks, and
positions beyond the value column without an order.
"""
import ctypes

import numpy as np
import pytest

from datatable_b200 import _lib

L = _lib.lib
STR32 = 21
V = np.array([1.0, 2.0, 3.0])
Y = np.array([4.0, 5.0, 7.0])
OFFS = np.array([0, 3], dtype=np.int32)
OUT = np.zeros(8, dtype=np.int64)                      # room for the output of every entry point


def _ptr(a):
    return a.ctypes.data


def _col(a, data_key="data"):
    return _lib.dtb_col(ctypes.c_void_p(a[data_key]), a["stype"], 0)


# entry point -> (its own argument when valid, call(args)); args: op, stype, nrows, data, y, order, offsets, ngroups, out
ENTRIES = {
    "dtb_reduce": (_lib.OP_SUM, lambda a: L.dtb_reduce(a["op"], _col(a), a["nrows"], a["order"], 0, a["offsets"],
                                                       a["ngroups"], None, a["out"])),
    "dtb_reduce2": (_lib.OP_COV, lambda a: L.dtb_reduce2(a["op"], _col(a), _col(dict(a, stype=_lib.FLOAT64), "y"),
                                                         a["nrows"], a["order"], 0, a["offsets"], a["ngroups"], None,
                                                         a["out"])),
    "dtb_cumulative": (_lib.OP_SUM, lambda a: L.dtb_cumulative(a["op"], 0, _col(a), a["nrows"], a["order"], 0,
                                                               a["offsets"], a["ngroups"], None, a["out"])),
    "dtb_shift": (None, lambda a: L.dtb_shift(_col(a), a["nrows"], a["order"], 0, a["offsets"], a["ngroups"], 1, None,
                                              a["out"])),
    "dtb_fillna": (None, lambda a: L.dtb_fillna(0, _col(a), a["nrows"], a["order"], 0, a["offsets"], a["ngroups"], None,
                                                a["out"])),
    "dtb_group_index": (_lib.GROUP_CUMCOUNT, lambda a: L.dtb_group_index(a["op"], 0, a["offsets"], a["ngroups"], None,
                                                                         a["out"])),
    "dtb_qcut": (10, lambda a: L.dtb_qcut(_col(a), a["nrows"], a["order"], a["offsets"], a["ngroups"], a["op"], None,
                                          a["out"])),
    "dtb_sort_grouped": (None, lambda a: L.dtb_sort_grouped(_col(a), a["nrows"], a["order"], a["offsets"], a["ngroups"],
                                                            None, a["out"])),
}
ROW_FNS = ("dtb_cumulative", "dtb_shift", "dtb_fillna", "dtb_qcut")
VALUE_FREE = ("dtb_group_index",)


def _common(code, msg):
    return {e: (code, msg) for e in ENTRIES}


def _valued(code, msg):
    return {e: (code, msg) for e in ENTRIES if e not in VALUE_FREE}


# The checks in their order: (name, bad arguments, {entry point: (code, message)}).  An entry point a check does not
# apply to is absent from its table.
CHECKS = [
    ("own argument", {}, {
        "dtb_reduce": ({"op": 99}, _lib.EINVAL, "unknown reducer 99"),
        "dtb_reduce2": ({"op": _lib.OP_SUM}, _lib.EINVAL, "dtb_reduce2 takes DTB_OP_COV or DTB_OP_CORR"),
        "dtb_cumulative": ({"op": _lib.OP_MEAN}, _lib.EINVAL,
                           "dtb_cumulative takes DTB_OP_SUM, DTB_OP_PROD, DTB_OP_MIN or DTB_OP_MAX"),
        "dtb_group_index": ({"op": 3}, _lib.EINVAL, "dtb_group_index takes DTB_GROUP_CUMCOUNT or DTB_GROUP_NGROUP"),
        "dtb_qcut": ({"op": 0}, _lib.EINVAL, "Number of quantiles must be positive, instead got: 0"),
    }),
    ("no fixed width", {"stype": STR32}, {
        "dtb_reduce": (_lib.ENOTIMPL, "Invalid column of stype 21 in reducer 1"),
        "dtb_reduce2": (_lib.ENOTIMPL, "Invalid columns of stypes 21, 7 in reducer 14"),
        "dtb_cumulative": (_lib.ENOTIMPL, "cumulative functions cannot be applied to columns of stype 21"),
        "dtb_shift": (_lib.ENOTIMPL, "shift cannot be applied to columns of stype 21"),
        "dtb_fillna": (_lib.ENOTIMPL, "fillna cannot be applied to columns of stype 21"),
        "dtb_qcut": (_lib.ENOTIMPL, "qcut() cannot be applied to columns of stype 21"),
        "dtb_sort_grouped": (_lib.ENOTIMPL, "Unable to sort Column of stype 21"),
    }),
    ("stype the op refuses", {"stype": _lib.DATE32}, {
        "dtb_reduce": (_lib.EINVAL, "Invalid column of stype 17 in reducer 1"),
        "dtb_reduce2": (_lib.EINVAL, "Invalid columns of stypes 17, 7 in reducer 14"),
        "dtb_cumulative": (_lib.EINVAL, "Invalid column of stype 17 in cumulative function 1"),
    }),
    ("ngroups < 0", {"ngroups": -1}, _common(_lib.EINVAL, "ngroups must be non-negative")),
    ("offsets NULL", {"offsets": None}, _common(_lib.EINVAL, "offsets is NULL")),
    ("nrows_value < 0", {"nrows": -1}, _valued(_lib.EINVAL, "nrows_value must be non-negative")),
    ("value data NULL", {"data": None}, _valued(_lib.EINVAL, "value column data is NULL")),
    ("out NULL", {"out": None}, _common(_lib.EINVAL, "out is NULL")),
]


def _base(entry):
    return dict(op=ENTRIES[entry][0], stype=_lib.FLOAT64, nrows=3, data=_ptr(V), y=_ptr(Y), order=None,
                offsets=_ptr(OFFS), ngroups=1, out=_ptr(OUT))


def _bad(entry, i):
    """The bad arguments of check i for `entry`, or None when the check does not apply to it."""
    name, bad, table = CHECKS[i]
    if entry not in table:
        return None
    return table[entry][0] if name == "own argument" else bad


def _expected(entry, i):
    return tuple(CHECKS[i][2][entry][-2:])


def _call(entry, args):
    rc = ENTRIES[entry][1](args)
    return rc, L.dtb_last_error().decode()


def _run(entry, bad):
    return _call(entry, dict(_base(entry), **bad))


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_each_bad_argument_alone(entry):
    for i, (name, _, _) in enumerate(CHECKS):
        bad = _bad(entry, i)
        if bad is not None:
            assert _run(entry, bad) == _expected(entry, i), (entry, name)


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_first_failing_check_wins(entry):
    """Check i and every later check fail at once: the call reports check i."""
    for i, (name, _, _) in enumerate(CHECKS):
        if _bad(entry, i) is None:
            continue
        bad = {}
        for j in reversed(range(i, len(CHECKS))):
            later = _bad(entry, j)
            if later is not None:
                bad.update(later)
        assert _run(entry, bad) == _expected(entry, i), (entry, name, bad)


def test_gather_checks_before_any_gpu_work():
    order = np.array([0, 2], dtype=np.int32)
    out = np.zeros(2, dtype=np.float64)

    def call(stype=_lib.FLOAT64, nrows_src=3, order=_ptr(order), n=2, out=_ptr(out)):
        return (L.dtb_gather(_lib.dtb_col(ctypes.c_void_p(_ptr(V)), stype, 0), nrows_src, order, 0, n, None, out),
                L.dtb_last_error().decode())

    assert call(stype=STR32) == (_lib.ENOTIMPL, "Unable to gather Column of stype 21")
    assert call(stype=STR32, n=-1) == (_lib.ENOTIMPL, "Unable to gather Column of stype 21")
    assert call(n=-1) == (_lib.EINVAL, "negative size")
    assert call(nrows_src=-1, order=None) == (_lib.EINVAL, "negative size")
    assert call(order=None) == (_lib.EINVAL, "order/out is NULL")
    assert call(out=None) == (_lib.EINVAL, "order/out is NULL")


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch():
    import torch
    torch.cuda.set_device(0)
    return torch


def _args(torch, entry, device, offsets, **kw):
    """(valid arguments of `entry` over `offsets`, all in host or all in device memory; the buffers they point to).
    The output, the last buffer, has room for 8 elements of 8 bytes."""
    bufs = []

    def put(a):
        a = torch.from_numpy(np.ascontiguousarray(a)).cuda() if device else np.ascontiguousarray(a)
        bufs.append(a)
        return a.data_ptr() if device else a.ctypes.data

    offs = np.asarray(offsets, dtype=np.int32)
    a = dict(_base(entry), data=put(V), y=put(Y), offsets=put(offs), ngroups=len(offs) - 1,
             out=put(np.zeros(8, np.int64)))
    a.update(kw)
    return a, bufs


def _out(bufs, dtype, count):
    out = bufs[-1]
    return (out.cpu().numpy() if hasattr(out, "cpu") else out).view(dtype)[:count]


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("entry", list(ENTRIES))
def test_offsets_that_are_not_a_groupby(torch, entry, device):
    for offsets in ([0, 2, 2, 3], [1, 3]):                  # an empty group; offsets[0] != 0
        a, bufs = _args(torch, entry, device, offsets)
        rc, msg = _call(entry, a)
        assert rc == _lib.EINVAL and "not a Groupby" in msg, (entry, offsets, rc, msg)
    a, bufs = _args(torch, entry, device, [0, 1, 3])
    assert _call(entry, a)[0] == _lib.OK, (entry, L.dtb_last_error().decode())
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("entry", list(ENTRIES))
def test_out_null_with_valid_offsets(torch, entry, device):
    a, bufs = _args(torch, entry, device, [0, 1, 3], out=None)
    assert _call(entry, a) == (_lib.EINVAL, "out is NULL"), entry


@pytest.mark.gpu
def test_handle_entry_points(torch):
    from datatable_b200 import engine
    gb = engine.Groupby([torch.tensor([2, 1, 2], dtype=torch.int32, device="cuda")], [0], _lib.NA_FIRST)
    try:
        xd = torch.from_numpy(V).cuda()
        x = _lib.dtb_col(ctypes.c_void_p(xd.data_ptr()), _lib.FLOAT64, 0)
        last = lambda: L.dtb_last_error().decode()                      # noqa: E731
        assert (L.dtb_groupby_reduce(gb._h, _lib.OP_SUM, x, 3, None, None), last()) == (_lib.EINVAL, "out is NULL")
        assert (L.dtb_groupby_reduce2(gb._h, _lib.OP_COV, x, x, 3, None, None), last()) == (_lib.EINVAL, "out is NULL")
        assert (L.dtb_groupby_reduce(gb._h, 99, x, 3, None, None), last()) == (_lib.EINVAL, "unknown reducer 99")
        assert (L.dtb_groupby_reduce(gb._h, _lib.OP_SUM, x, -1, None, None), last()) == \
            (_lib.EINVAL, "nrows_value must be non-negative")
        assert gb.reduce(_lib.OP_SUM, xd).cpu().tolist() == [2.0, 4.0]
    finally:
        gb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_positions_beyond_the_column(torch, device):
    """Offsets covering 5 positions of a 3-row column, without an order: the row functions refuse it; the reducers
    and dtb_sort_grouped read positions 3 and 4 as NA."""
    for entry in ROW_FNS:
        a, bufs = _args(torch, entry, device, [0, 2, 5])
        assert _call(entry, a) == (_lib.EINVAL, "offsets cover more rows than the value column has"), entry
    for op, want in ((_lib.OP_SUM, [3.0, 3.0]), (_lib.OP_COUNT, [2, 1])):
        a, bufs = _args(torch, "dtb_reduce", device, [0, 2, 5], op=op)
        assert _call("dtb_reduce", a)[0] == _lib.OK, L.dtb_last_error().decode()
        torch.cuda.synchronize()
        assert _out(bufs, np.float64 if op == _lib.OP_SUM else np.int64, 2).tolist() == want
    a, bufs = _args(torch, "dtb_sort_grouped", device, [0, 2, 5])
    assert _call("dtb_sort_grouped", a)[0] == _lib.OK, L.dtb_last_error().decode()
    assert _out(bufs, np.int32, 5).tolist() == [0, 1, 3, 4, 2]           # NA first inside the group


def test_parsed_arguments_keep_their_copies_alive():
    """Strided offsets and order are copied to contiguous memory: the pointers handed to the library must stay valid
    while the parsed arguments live, even when the allocator is asked for blocks of the same size."""
    from datatable_b200 import engine
    offsets = np.array([0, -1, 2, -1, 5, -1], dtype=np.int32)[::2]
    order = np.array([4, -1, 3, -1, 2, -1, 1, -1, 0, -1], dtype=np.int32)[::2]
    g = engine._Grouped([], order, offsets)
    junk = [np.full(k, -7, dtype=np.int32) for k in (3, 5) for _ in range(64)]
    assert np.ctypeslib.as_array((ctypes.c_int32 * 3).from_address(g.offsets.value)).tolist() == [0, 2, 5]
    assert np.ctypeslib.as_array((ctypes.c_int32 * 5).from_address(g.order.value)).tolist() == [4, 3, 2, 1, 0]
    del junk


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_strided_inputs_give_what_contiguous_ones_give(torch, device):
    from datatable_b200 import engine
    rng = np.random.default_rng(5)
    n = 1000
    v = rng.integers(-50, 50, n).astype(np.float64)        # integer values: sums are exact in any order
    v[rng.random(n) < 0.1] = np.nan
    w = rng.integers(-50, 50, n).astype(np.float64)
    order = rng.permutation(n).astype(np.int32)
    offsets = np.concatenate([[0], np.sort(rng.choice(np.arange(1, n), 40, replace=False)), [n]]).astype(np.int32)

    def strided(a):                                        # every other element of a twice as long buffer
        b = np.zeros(2 * len(a), dtype=a.dtype)
        b[::2] = a
        return torch.from_numpy(b).cuda()[::2] if device else b[::2]

    def dense(a):
        return torch.from_numpy(a).cuda() if device else a.copy()

    calls = {
        "reduce": lambda p: engine.reduce(_lib.OP_SUM, p(v), p(order), p(offsets)),
        "reduce2": lambda p: engine.reduce2(_lib.OP_COV, p(v), p(w), p(order), p(offsets)),
        "sort_grouped": lambda p: engine.sort_grouped(p(v), p(order), p(offsets)),
        "qcut": lambda p: engine.qcut(p(v), p(order), p(offsets), 7),
        "cumulative": lambda p: engine.cumulative(_lib.OP_SUM, p(v), p(order), p(offsets)),
        "shift": lambda p: engine.shift(p(v), p(order), p(offsets), 2),
        "fillna": lambda p: engine.fillna(p(v), p(order), p(offsets)),
        "group_index": lambda p: engine.group_index(_lib.GROUP_CUMCOUNT, p(offsets), True),
    }
    for name, call in calls.items():
        got, want = call(strided), call(dense)
        got, want = [x.cpu().numpy() if hasattr(x, "cpu") else x for x in (got, want)]
        assert got.dtype == want.dtype, name
        if name == "reduce2":                              # folded in an unspecified order
            assert np.allclose(got, want, rtol=1e-12, atol=0, equal_nan=True), name
        else:
            assert np.array_equal(got, want, equal_nan=got.dtype.kind == "f"), name


@pytest.mark.gpu
def test_own_argument_errors_reset_the_call_statistics(torch):
    from datatable_b200 import engine
    vd = torch.from_numpy(V).cuda()
    od = torch.tensor([0, 3], dtype=torch.int32, device="cuda")
    engine.cumulative(_lib.OP_SUM, vd, None, od)
    assert _lib.last_call_stats()["kernels_launched"] > 0
    a = dict(_base("dtb_cumulative"), data=vd.data_ptr(), offsets=od.data_ptr(), op=_lib.OP_MEAN)
    assert _call("dtb_cumulative", a)[0] == _lib.EINVAL
    assert _lib.last_call_stats()["kernels_launched"] == 0
