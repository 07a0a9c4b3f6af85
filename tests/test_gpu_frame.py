"""GPU: the Frame / f / by / sort surface, written the way the reference's own tests read
(tests/test-groups.py, tests/ijby/test-sort.py, tests/test-reduce.py)."""
import math
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def dtmod():
    import datatable_b200 as dt
    return dt


def test_groups_order_na_first():            # tests/test-groups.py:39-52
    dt = dtmod(); f, by = dt.f, dt.by
    DT = dt.Frame(A=[1, 2, 1, None, 2, 1], B=[0, 1, 2, 3, 4, 5])
    R = DT[:, dt.sum(f.B), by(f.A)]
    assert R.names == ("A", "B")
    assert R.to_list() == [[None, 1, 2], [3, 7, 5]]


def test_groups_stable_inside():             # tests/test-groups.py:72-95
    dt = dtmod(); f, by = dt.f, dt.by
    DT = dt.Frame(A=[2, 1, 2, 1, 2, 1, 1], B=[0, 1, 2, 3, 4, 5, 6])
    R = DT[:, f.B, by(f.A)]
    assert R.to_list() == [[1, 1, 1, 1, 2, 2, 2], [1, 3, 5, 6, 0, 2, 4]]


def test_count_251x4000():                   # tests/test-groups.py:318-323
    dt = dtmod(); f, by = dt.f, dt.by
    n = 4000
    DT = dt.Frame(A=np.tile(np.arange(251, dtype=np.int32), n))
    R = DT[:, dt.count(), by(f.A)]
    assert R.shape == (251, 2)
    assert R.to_list() == [list(range(251)), [n] * 251]


def test_multikey_sum_vs_python():           # tests/test-groups.py:386-412
    dt = dtmod(); f, by = dt.f, dt.by
    random.seed(12)
    n = 20000
    a = [random.randint(0, 9) for _ in range(n)]
    b = [random.choice([None, -3, 0, 7]) for _ in range(n)]
    v = [random.random() for _ in range(n)]
    DT = dt.Frame(A=a, B=b, V=v)
    R = DT[:, dt.sum(f.V), by(f.A, f.B)]
    exp = {}
    for x, y, z in zip(a, b, v):
        exp[(x, y)] = exp.get((x, y), 0.0) + z
    keys = sorted(exp, key=lambda t: (t[0], -1e9 if t[1] is None else t[1]))
    got = R.to_list()
    assert got[0] == [k[0] for k in keys]
    assert got[1] == [k[1] for k in keys]
    assert all(math.isclose(g, exp[k], rel_tol=1e-9) for g, k in zip(got[2], keys))


def test_by_and_sort():                      # tests/test-groups.py:448-457
    dt = dtmod(); f, by, sort = dt.f, dt.by, dt.sort
    DT = dt.Frame(A=[1, 2, 1, 2, 1, 2], B=[3.5, 1.0, None, 9.0, 0.5, -1.0])
    R = DT[:, f.B, by(f.A), sort(f.B)]
    assert R.to_list() == [[1, 1, 1, 2, 2, 2], [None, 0.5, 3.5, -1.0, 1.0, 9.0]]
    R = DT[:, f.B, by(f.A), sort(-f.B)]
    assert R.to_list() == [[1, 1, 1, 2, 2, 2], [None, 3.5, 0.5, 9.0, 1.0, -1.0]]


def test_sort_int32_small_stable():          # tests/ijby/test-sort.py:132-178
    dt = dtmod(); f = dt.f
    DT = dt.Frame(A=[5, 3, 5, None, 1000000, None, 3, -5, 5, 3], I=list(range(10)))
    R = DT.sort("A")
    assert R.to_list() == [[None, None, -5, 3, 3, 3, 5, 5, 5, 1000000], [3, 5, 7, 1, 6, 9, 0, 2, 8, 4]]


def test_sort_float_nan_zero():              # tests/ijby/test-sort.py:531-536, 586-594
    dt = dtmod(); f, sort = dt.f, dt.sort
    DT = dt.Frame(A=np.array([0.0, -0.0, np.nan, 1.5, -0.0, 0.0, -np.inf, np.inf]))
    R = DT[:, f.A, sort(f.A)]
    a = R.to_numpy("A")
    assert np.isnan(a[0])
    assert a[1] == -np.inf and a[-1] == np.inf
    assert np.signbit(a[2:6]).tolist() == [True, True, False, False]


def test_sort_na_position_reverse():         # tests/ijby/test-sort.py:1066-1092, SURVEY 8c
    dt = dtmod(); f, sort = dt.f, dt.sort
    DT = dt.Frame(x=[3, 1, None, 2, 1, None], i=list(range(6)))
    assert DT[:, f.i, sort(f.x)].to_list() == [[2, 5, 1, 4, 3, 0]]
    assert DT[:, f.i, sort(-f.x)].to_list() == [[2, 5, 0, 3, 1, 4]]
    assert DT[:, f.i, sort(f.x, na_position="last")].to_list() == [[1, 4, 3, 0, 2, 5]]
    assert DT[:, f.i, sort(f.x, reverse=True, na_position="last")].to_list() == [[0, 3, 1, 4, 2, 5]]
    assert DT[:, f.i, sort(f.x, na_position="remove")].to_list() == [[1, 4, 3, 0]]
    with pytest.raises(ValueError):
        sort(f.x, na_position="middle")


def test_multicolumn_sort_vs_python():       # tests/ijby/test-sort.py:909-940
    dt = dtmod(); f, sort = dt.f, dt.sort
    random.seed(3)
    n = 5000
    a = [random.randint(-3, 3) for _ in range(n)]
    b = [random.choice([0.5, -0.5, 2.25, 7.0]) for _ in range(n)]
    c = [random.randint(0, 1) == 1 for _ in range(n)]
    DT = dt.Frame(A=a, B=b, C=c, I=list(range(n)))
    R = DT[:, f.I, sort(f.A, f.B, f.C)]
    exp = sorted(range(n), key=lambda i: (a[i], b[i], c[i]))
    assert R.to_list() == [exp]
    R = DT[:, f.I, sort(f.A, f.B, f.C, reverse=[True, False, True])]
    exp = sorted(range(n), key=lambda i: (-a[i], b[i], -int(c[i])))
    assert R.to_list() == [exp]


def test_reducers_stypes_and_na():           # tests/test-reduce.py:262-400, 402-496, 499-555
    dt = dtmod(); f, by = dt.f, dt.by
    from datatable_b200._lib import INT8, INT32, INT64, FLOAT32, FLOAT64
    DT = dt.Frame(G=[1, 1, 2, 2, 3], I=np.array([5, -128, 7, 1, -128], np.int8),
                  F=np.array([1.5, np.nan, np.inf, -np.inf, np.nan], np.float32),
                  D=[None, 2.0, 4.0, None, None])
    R = DT[:, {"si": dt.sum(f.I), "mi": dt.mean(f.I), "lo": dt.min(f.I), "hi": dt.max(f.I),
               "c": dt.count(f.I), "n": dt.count(), "sf": dt.sum(f.F), "mf": dt.mean(f.F),
               "xf": dt.max(f.F), "md": dt.mean(f.D), "nd": dt.min(f.D)}, by(f.G)]
    assert R.stypes == (INT32, INT64, FLOAT64, INT8, INT8, INT64, INT64, FLOAT32, FLOAT32, FLOAT32, FLOAT64, FLOAT64)
    L = R.to_dict()
    assert L["si"] == [5, 8, 0]                 # all-NA group sums to 0, never NA
    assert L["mi"] == [5.0, 4.0, None]
    assert L["lo"] == [5, 1, None] and L["hi"] == [5, 7, None]
    assert L["c"] == [1, 2, 0] and L["n"] == [2, 2, 1]
    assert L["sf"][0] == 1.5 and L["sf"][2] == 0.0 and L["sf"][1] is None   # inf + -inf = nan
    assert L["mf"][0] == 1.5 and L["mf"][2] is None
    assert L["xf"] == [1.5, math.inf, None]
    assert L["md"] == [2.0, 4.0, None] and L["nd"] == [2.0, 4.0, None]


def test_reducers_without_by():              # tests/test-reduce.py:84-93
    dt = dtmod(); f = dt.f
    DT = dt.Frame(A=[1, None, 5, 10], B=[0.5, 1.5, None, 2.0])
    R = DT[:, [dt.sum(f.A), dt.max(f.B), dt.count(f.A), dt.count()]]
    assert R.to_list() == [[16], [2.0], [3], [4]]


def test_repeated_column_names_deduplicated():   # frame/names.cc: _deduplicate gives x, x.0, x.1, ...
    dt = dtmod(); f = dt.f
    DT = dt.Frame(x=[1, None, 3])
    for fr in (DT, DT.to_device()):
        R = fr[:, [f.x, f.x]]
        assert R.names == ("x", "x.0")
        assert R.to_list() == [[1, None, 3], [1, None, 3]]


def test_device_frame_stays_on_device():
    import torch
    dt = dtmod(); f, by = dt.f, dt.by
    n = 1_000_000
    g = torch.Generator(device="cuda"); g.manual_seed(1)
    DT = dt.Frame(k=torch.randint(0, 1000, (n,), generator=g, device="cuda", dtype=torch.int32),
                  v=torch.rand(n, generator=g, device="cuda", dtype=torch.float64))
    R = DT[:, dt.sum(f.v), by(f.k)]
    assert engine_is_cuda(R.column("v")) and R.nrows == 1000
    ref = torch.zeros(1000, dtype=torch.float64, device="cuda").index_add_(0, DT.column("k").long(), DT.column("v"))
    assert torch.allclose(R.column("v"), ref, rtol=1e-9)


def engine_is_cuda(x):
    import torch
    return isinstance(x, torch.Tensor) and x.is_cuda


def test_unique_and_nunique():               # tests/test-sets.py (unique), tests/test-dt-stats.py (nunique)
    dt = dtmod()
    DT = dt.Frame(A=[3, 1, None, 3, 2, None, 1, 7])
    assert dt.unique(DT).to_list() == [[None, 1, 2, 3, 7]]
    DF = dt.Frame(A=[3, 1, None, 3, 2, None, 1, 7], B=[0.5, float("nan"), 0.5, -0.0, 0.0, 1.5, 1.5, 0.5])
    assert dt.nunique(DF).to_list() == [[4], [4]]       # -0.0 and +0.0 are distinct keys (bit pattern order)
