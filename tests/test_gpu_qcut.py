"""GPU: dt.qcut (dtb_qcut, engine.qcut, the Frame's qcut()) against the reference's goldens (golden_v6) and, on large
seeded inputs, bit for bit against the numpy restatement in tests/qcut_reference.py.
"""
import ctypes

import numpy as np
import pytest

from oracle import oracle as orc
from qcut_reference import (FLOAT32, FLOAT64, INT32, INT64, NA, case_groups, j_columns, load_golden, qcut_column,
                            qcut_groups)

pytestmark = pytest.mark.gpu

ALL_CASES, ARR = load_golden()
CASES = [c for c in ALL_CASES if "error" not in c]


@pytest.fixture(scope="module")
def eng():
    import torch
    torch.cuda.set_device(0)
    from datatable_b200 import engine, _lib
    return engine, _lib, torch


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _assert_same(got, want, label=""):
    got = _np(got)
    if want.dtype.kind == "f":
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan), label
        assert np.array_equal(got[~nan], want[~nan]), label
    else:
        assert got.dtype == want.dtype, label
        assert np.array_equal(got, want), label


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_engine_qcut_golden(eng, case, device):
    engine, _lib, torch = eng
    order, offsets, grouped = case_groups(case, ARR, orc)
    if not grouped:
        n = int(offsets[-1]) if len(offsets) > 1 else 0
        offsets = np.array([0, n] if n else [0], dtype=np.int32)
    put = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if device else (lambda a: a)
    outputs = [(nm, spec) for nm, spec in zip(case["names"][-len(j_columns(case)):], j_columns(case))]
    for nm, (kind, src, q) in outputs:
        if kind != "qcut":
            continue
        v = ARR[case["name"] + "." + src]
        got = engine.qcut(put(v), None if order is None else put(np.asarray(order, np.int32)), put(offsets), q,
                          stype=case["stypes"][src])
        assert engine.is_tensor(got) == device
        _assert_same(got, ARR[case["name"] + ".out_" + nm], nm)


def _frame_query(dtb, case, fr):
    f, q, j = dtb.f, case["q"], case["j"]
    J = {"one": lambda: dtb.qcut(f.x, nquantiles=q),
         "list": lambda: dtb.qcut([f.x, f.y], nquantiles=q),
         "tuple": lambda: dtb.qcut((f.x, f.y), nquantiles=tuple(q)),
         "all": lambda: dtb.qcut(f[:], nquantiles=q),
         "dict": lambda: {"q": dtb.qcut(f.x, nquantiles=q)},
         "dictlist": lambda: {"q": dtb.qcut([f.x, f.y], nquantiles=q)},
         "plain": lambda: [f.x, dtb.qcut(f.x, nquantiles=q)],
         "bykey": lambda: dtb.qcut(f.ka, nquantiles=q)}[j]()
    i = case["i"]
    rows = slice(None) if i is None else (i if isinstance(i, int) else slice(*i))
    mods = {"none": (), "by": (dtb.by(f.ka),), "by2": (dtb.by(f.ka, f.kb),), "bysort": (dtb.by(f.ka), dtb.sort(f.s)),
            "sort": (dtb.sort(f.s),), "sortdesc": (dtb.sort(-f.s),)}[case["mode"]]
    return fr[(rows, J) + mods]


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_frame_qcut_golden(eng, case, device):
    import datatable_b200 as dtb
    fr = dtb.Frame({nm: ARR[case["name"] + "." + nm] for nm in case["stypes"]}, stypes=case["stypes"])
    if device:
        fr = fr.to_device()
    R = _frame_query(dtb, case, fr)
    assert list(R.names) == case["names"]
    assert R.nrows == case["nrows"]
    assert list(R.stypes) == [{"stype.int32": INT32, "stype.float64": FLOAT64}[st] for st in case["out_stypes"]]
    for nm in case["names"]:
        _assert_same(R.to_numpy(nm), ARR[case["name"] + ".out_" + nm], nm)


def test_frame_qcut_output_stype(eng):
    import datatable_b200 as dtb
    fr = dtb.Frame({"x": np.array([1.5, np.nan, -0.0, 0.0]), "g": np.array([1, 2, 1, 2], np.int32)})
    for R in (fr[:, dtb.qcut(dtb.f.x)], fr[:, dtb.qcut(dtb.f.x), dtb.by(dtb.f.g)], fr[1:, dtb.qcut(dtb.f.x)]):
        assert R.stypes[-1] == dtb._lib.INT32
    with pytest.raises(NotImplementedError):                      # a reducer next to qcut() is not taken
        fr[:, [dtb.sum(dtb.f.x), dtb.qcut(dtb.f.x)], dtb.by(dtb.f.g)]


# ---- large seeded cases against the restatement --------------------------------------------------------------------
def _run(engine, torch, v, st, keys, q):
    """group() of the keys on the GPU, then qcut per group on the GPU and in the restatement."""
    vd = torch.from_numpy(v).cuda()
    if keys is None:
        order, offsets = None, torch.tensor([0, len(v)], dtype=torch.int32, device="cuda")
    else:
        order, offsets, _ = engine.group([torch.from_numpy(keys).cuda()], [0])
    got = engine.qcut(vd, order, offsets, q, stype=st).cpu().numpy()
    o = None if order is None else order.cpu().numpy()
    return got, qcut_groups(v, st, o, offsets.cpu().numpy(), q)


def test_large_many_groups(eng):
    engine, _lib, torch = eng
    rng = np.random.default_rng(61)
    n = 10_000_000
    keys = rng.integers(0, 100_000, n).astype(np.int32)
    v = np.round(rng.standard_normal(n), 2)
    v[rng.random(n) < 0.05] = np.nan
    got, want = _run(engine, torch, v, FLOAT64, keys, 10)
    assert np.array_equal(got, want)
    vi = rng.integers(-40, 40, n).astype(np.int32)
    vi[rng.random(n) < 0.05] = NA[INT32]
    got, want = _run(engine, torch, vi, INT32, keys, 7)
    assert np.array_equal(got, want)


def test_composite_needs_two_sort_rounds(eng):
    """int64 keys over their whole range and float64 values with all 64 bits in use: the (group id, value) key is
    wider than 64 bits."""
    engine, _lib, torch = eng
    rng = np.random.default_rng(62)
    n = 2_000_000
    uniq = rng.integers(-2**63 + 1, 2**63 - 1, 1000, dtype=np.int64)
    keys = uniq[rng.integers(0, 1000, n)]
    v = rng.standard_normal(n) * np.exp2(rng.integers(-300, 300, n))
    rep = rng.random(n) < 0.3                                     # repeated values inside the groups
    v[rep] = v[rng.integers(0, 1000, int(rep.sum()))]
    v[rng.random(n) < 0.02] = np.nan
    got, want = _run(engine, torch, v, FLOAT64, keys, 13)
    assert np.array_equal(got, want)
    vi = rng.integers(-2**63 + 1, 2**63 - 1, n, dtype=np.int64)
    vi[::7] = vi[0]
    vi[rng.random(n) < 0.02] = NA[INT64]
    got, want = _run(engine, torch, vi, INT64, keys, 1000)
    assert np.array_equal(got, want)


def test_one_group_dominated_by_one_value(eng):
    engine, _lib, torch = eng
    rng = np.random.default_rng(63)
    n = 20_000_000
    v = np.full(n, 5.0)
    m = rng.random(n) < 0.1
    v[m] = rng.integers(-1000, 1000, int(m.sum())).astype(np.float64)
    v[rng.random(n) < 0.01] = np.nan
    got, want = _run(engine, torch, v, FLOAT64, None, 10)
    assert np.array_equal(got, want)
    assert np.array_equal(want, qcut_column(v, FLOAT64, 10))


def test_float_columns_dense_in_zeros_and_nans(eng):
    engine, _lib, torch = eng
    rng = np.random.default_rng(64)
    n = 1_000_000
    keys = rng.integers(0, 100, n).astype(np.int32)
    for st, T, ui, payload in ((FLOAT64, np.float64, np.uint64, 0x7FF0000000000ABC), (FLOAT32, np.float32, np.uint32, 0x7F800ABC)):
        pool = np.array([0.0, -0.0, np.nan, -np.nan, 2.5, -np.inf, np.finfo(T).smallest_subnormal], dtype=T)
        pool = np.concatenate([pool, np.array([payload], dtype=ui).view(T)])
        v = rng.choice(pool, n)
        got, want = _run(engine, torch, v, st, keys, 10)
        assert np.array_equal(got, want)


def test_no_groups(eng):
    engine, _lib, torch = eng
    empty = np.array([0], dtype=np.int32)
    assert len(engine.qcut(np.zeros(4), None, empty, 10)) == 0
    got = engine.qcut(torch.zeros(4, dtype=torch.float64, device="cuda"), None, torch.from_numpy(empty).cuda(), 10)
    assert got.is_cuda and got.numel() == 0


def test_profile_names_the_qcut_kernels(eng):
    engine, _lib, torch = eng
    engine.set_option("profile", 1)
    try:
        _lib.profile_records(reset=True)
        engine.qcut(torch.arange(1000, dtype=torch.float64, device="cuda"), None,
                    torch.tensor([0, 400, 1000], dtype=torch.int32, device="cuda"), 4)
        names = {nm for nm, _ in _lib.profile_records(reset=True)}
    finally:
        engine.set_option("profile", 0)
    assert {"qcut_coef", "qcut_emit"} <= names


def test_abi_error_codes(eng):
    engine, _lib, torch = eng
    lib = _lib.lib
    v = np.array([1.0, 2.0, 3.0])
    out = np.empty(3, dtype=np.int32)
    col = _lib.dtb_col(ctypes.c_void_p(v.ctypes.data), _lib.FLOAT64, 0)

    def call(offsets, ng, q=10, c=col, order=None):
        o = np.asarray(offsets, dtype=np.int32)
        return lib.dtb_qcut(c, 3, order, ctypes.c_void_p(o.ctypes.data), ng, q, None, ctypes.c_void_p(out.ctypes.data))

    assert call([0, 3], 1) == _lib.OK
    assert list(out) == [0, 4, 9]
    assert call([0, 3], 1, q=0) == _lib.EINVAL
    assert "Number of quantiles must be positive, instead got: 0" in lib.dtb_last_error().decode()
    assert call([0, 3], 1, q=-1) == _lib.EINVAL
    assert call([0, 3], -1) == _lib.EINVAL
    assert call([0, 2, 2, 3], 3) == _lib.EINVAL                # an empty group: not a Groupby
    assert call([1, 3], 1) == _lib.EINVAL                      # offsets[0] != 0
    bad = _lib.dtb_col(ctypes.c_void_p(v.ctypes.data), 21, 0)  # str32: no fixed width
    assert call([0, 3], 1, c=bad) == _lib.ENOTIMPL
    # device offsets are checked on the device
    od = torch.tensor([0, 2, 2, 3], dtype=torch.int32, device="cuda")
    vd = torch.from_numpy(v).cuda()
    outd = torch.empty(3, dtype=torch.int32, device="cuda")
    rc = lib.dtb_qcut(_lib.dtb_col(ctypes.c_void_p(vd.data_ptr()), _lib.FLOAT64, 0), 3, None,
                      ctypes.c_void_p(od.data_ptr()), 3, 10, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream),
                      ctypes.c_void_p(outd.data_ptr()))
    assert rc == _lib.EINVAL
