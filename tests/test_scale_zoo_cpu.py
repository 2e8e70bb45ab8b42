"""CPU: L2O-Scale's problem zoo (open_l2o_b200.scale_zoo) — the problem sets against a table transcribed from
SC/problems/problem_sets.py, the synthetic datasets, every objective's torch restatement (fp64) against numpy formulas,
the l2o_zoo C ABI's argument checks, and scale_metarun's flags and problem assembly."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from open_l2o_b200 import _lib
from open_l2o_b200 import scale_metarun as smr
from open_l2o_b200 import scale_zoo as Z

PI4 = np.pi / 4.
FC = [((8, 2), (8, 5), 10), ((12, 2), (8, 5, 3), 200), ((5, 2), (4, 4, 4, 4), 100), ((11, 2), (4, 5, 6), 64),
      ((9, 2), (8,), 128), ((7, 2), (8, 5), 16), ((8, 2), (32, 64), 10), ((12, 2), (16, 8, 3), 200),
      ((5, 2), (8, 8, 8, 8), 100), ((11, 2), (10, 12, 12), 64), ((9, 2), (32,), 128), ((7, 2), (32, 64), 16)]
DATA = [(20, 1000, 100), (12, 200, 10), (56, 5000, 100), (64, 1000, 50), (13, 10000, 50), (20, 1000, 128),
        (12, 300, 16), (56, 5000, 128), (64, 1000, 64), (13, 10000, 32)]
SYM = [(20, 1000, 100), (12, 100, 10), (56, 5000, 100), (64, 1000, 50), (13, 10000, 50), (20, 1000, 128),
       (12, 100, 16), (56, 5000, 128), (64, 1000, 64), (13, 10000, 32)]
OPT = ["Ackley", "Beale", "Booth", "Branin", "LogSumExp", "Matyas", "Michalewicz", "Rosenbrock", "StyblinskiTang"]
NINE = ["Rosenbrock", "LogSumExp", "Ackley", "Beale", "Booth", "StyblinskiTang", "Matyas", "Branin", "Michalewicz"]


def q(n, **kw):
    return ("Quadratic", (n,), kw)


# flag -> [(class, args, kwargs, batch_size, dataset rows)] as problem_sets.py writes them; nested specs as tuples
TABLE = {
    "quadratic": [q(20) + (None, None), q(25) + (None, None), q(50) + (None, None), q(100) + (None, None)],
    "noisy_quadratic": [q(20, noise_stdev=0.5) + (None, None), q(25, noise_stdev=0.0) + (None, None),
                        q(50, noise_stdev=1.0) + (None, None), q(100, noise_stdev=2.0) + (None, None)],
    "large_quadratic": [q(784) + (None, None), q(1024) + (None, None), q(2048) + (None, None)],
    "bowl": [("Bowl", (0.1,), {"noise_stdev": 0.0}, None, None), ("Bowl", (1.0,), {"noise_stdev": 0.0}, None, None),
             ("Bowl", (5.0,), {"noise_stdev": 0.0}, None, None),
             ("Bowl", (5.0,), {"noise_stdev": 0.0, "angle": PI4}, None, None)],
    "noisy_bowl": [("Bowl", (0.1,), {"noise_stdev": 0.1}, None, None),
                   ("Bowl", (1.0,), {"noise_stdev": 0.1}, None, None),
                   ("Bowl", (5.0,), {"noise_stdev": 0.1}, None, None),
                   ("Bowl", (5.0,), {"noise_stdev": 0.1, "angle": PI4}, None, None)],
    "sparse_softmax": [("SparseSoftmaxRegression", (5, 2), {"noise_stdev": 0.0}, 23, 5)],
    "one_hot_sparse_softmax": [("OneHotSparseSoftmaxRegression", (5, 2), {"noise_stdev": 0.0}, 23, 5)],
    "softmax_2_class": [("SoftmaxRegression", (10, 2), {}, 100, 1000), ("SoftmaxRegression", (100, 2), {}, 50, 1000),
                        ("SoftmaxRegression", (200, 2), {}, 20, 1000), ("SoftmaxRegression", (256, 2), {}, 100, 1000)],
    "noisy_softmax_2_class": [("SoftmaxRegression", (10, 2), {"noise_stdev": 0.5}, 100, 1000),
                              ("SoftmaxRegression", (100, 2), {"noise_stdev": 0.1}, 50, 1000),
                              ("SoftmaxRegression", (200, 2), {"noise_stdev": 0.1}, 20, 1000),
                              ("SoftmaxRegression", (256, 2), {"noise_stdev": 0.5}, 100, 1000)],
    "optimization_test": [(c, (), {}, None, None) for c in OPT],
    "noisy_optimization_test": [(c, (), {"noise_stdev": 1.}, None, None) for c in OPT],
    "fully_connected_random_2_class": [("FullyConnected", a, {"hidden_sizes": h, "activation": torch.sigmoid}, b, 1000)
                                       for a, h, b in FC],
    "matmul": [("MatMulAlgorithm", (2, k), {}, None, None) for k in range(5, 9)]
              + [("MatMulAlgorithm", (3, k), {}, None, None) for k in range(19, 25)],
    "log_objective": [("LogObjective", (q(n),), {}, None, None) for n in (20, 50, 100)]
                     + [("LogObjective", (("Bowl", (c,), {}),), {}, None, None) for c in (0.1, 1.0, 5.0)],
    "rescale": [("Rescale", (("Norm", (18,), {"norm_power": p}),), {"scale": s}, None, None)
                for p, s in ((2.5, 0.123), (1.5, 8), (2., 50), (3., 200), (1., 1000))]
               + [("Rescale", (q(n),), {"scale": s}, None, None) for n, s in ((20, 0.1), (25, 10.), (50, 350.),
                                                                             (100, 132))],
    "norm": [("Norm", (27,), {"norm_power": 1.}, None, None), ("Norm", (25,), {"norm_power": 2.}, None, None),
             ("Norm", (22,), {"norm_power": 3.}, None, None)],
    "noisy_norm": [("Norm", (19,), {"noise_stdev": .1, "norm_power": 1.}, None, None),
                   ("Norm", (26,), {"noise_stdev": .1, "norm_power": 2.}, None, None),
                   ("Norm", (23,), {"noise_stdev": .1, "norm_power": 3.}, None, None)],
    "sum": [("SumTask", ([q(n) for n in (11, 3, 9, 7, 5, 13, 12)],), {}, None, None),
            ("SumTask", ([("Norm", (18,), {"norm_power": 3}), q(25), ("Rosenbrock", (), {})],), {}, None, None),
            ("SumTask", ([(c, (), {}) for c in NINE],), {}, None, None),
            ("SumTask", ([(c, (), {}) for c in NINE] + [q(5), q(13)],), {}, None, None),
            ("SumTask", ([q(11), q(3)],), {}, None, None),
            ("SumTask", ([("Rosenbrock", (), {}), ("LogSumExp", (), {}), ("Ackley", (), {})],), {}, None, None)],
    "noisy_sum": [("SumTask", ([q(n, noise_stdev=0.1) for n in (11, 3, 9, 7, 5, 13, 12)],), {}, None, None),
                  ("SumTask", ([(c, (), {}) for c in NINE] + [q(5), q(13, noise_stdev=0.5)],), {}, None, None)],
    "sparse_gradient": [("SparseProblem", (q(n),), {}, None, None) for n in (20, 50, 100)]
                       + [("SparseProblem", (("Bowl", (c,), {}),), {}, None, None) for c in (0.1, 1.0, 5.0)],
    "min_max_well": [("MinMaxWell", (n,), {}, None, None) for n in (20, 12, 56, 64, 13)],
    "sum_of_quadratics": [("SumOfQuadratics", (n,), {}, b, m) for n, m, b in SYM],
    "projection_quadratic": [("ProjectionQuadratic", (n,), {}, b, m) for n, m, b in SYM],
    "outward_snake": [("OutwardSnake", (n,), {}, b, m) for n, m, b in DATA],
    "dependency_chain": [("DependencyChain", (n,), {}, b, m) for n, m, b in DATA],
    "lasso": [("Lasso", (20,), {}, None, None)],
    "rastrigin": [("Rastrigin", (2,), {}, None, None)],
}
DOWNLOADS = ["mnist_conv", "cifar10_conv", "mnist_mlp"]


def _spec_tuple(s):
    """A Spec as (class name, args, kwargs) with nested specs converted the same way."""
    def conv(a):
        if isinstance(a, Z.Spec):
            return _spec_tuple(a)
        if isinstance(a, list):
            return [conv(b) for b in a]
        return a
    return (s.callable.__name__, tuple(conv(a) for a in s.args), dict(s.kwargs))


def _set(name):
    return dict(Z.INCLUDE_FLAGS)[name]()


@pytest.mark.parametrize("flag", sorted(TABLE))
def test_problem_set_matches_problem_sets_py(flag):
    got = _set(flag)
    want = TABLE[flag]
    assert len(got) == len(want)
    for (spec, dataset, batch), (cls, args, kwargs, bsz, rows) in zip(got, want):
        assert _spec_tuple(spec) == (cls, args, kwargs)
        assert batch == bsz
        assert (dataset is None) == (rows is None)
        if dataset is not None:
            assert dataset.data.shape[0] == rows == len(dataset.labels)


def test_every_include_flag_is_covered_and_downloads_raise():
    assert sorted(list(TABLE) + DOWNLOADS) == sorted(n for n, _ in Z.INCLUDE_FLAGS)
    for name in DOWNLOADS:
        with pytest.raises(NotImplementedError):
            _set(name)
    for fn in (Z.mnist, Z.cifar10, Z.adapter_rosenbrock_local, Z.adapter_rosenbrock_worker):
        with pytest.raises(NotImplementedError):
            fn()


def test_problems_and_data_order_and_mlp_sparse_pairing():
    lst = Z.problems_and_data(["rastrigin", "quadratic", "sparse_softmax"])
    names = [s.callable.__name__ for s, _, _ in lst]
    assert names == ["SparseSoftmaxRegression"] + ["Quadratic"] * 4 + ["Rastrigin"]
    with_mlp = Z.problems_and_data(["sparse_gradient", "fully_connected_random_2_class"])
    assert len(with_mlp) == 12 + 6 + 3
    assert [s.callable.__name__ for s, _, _ in with_mlp[-3:]] == ["SparseProblem"] * 3
    assert with_mlp[-3][1] is not None and with_mlp[-3][2] == 10
    with pytest.raises(ValueError):
        Z.problems_and_data(["no_such_set"])


# ---- datasets -------------------------------------------------------------------------------------------------------
def test_datasets_shapes_labels_and_seeds():
    d = Z.noisy_parity_class(50, random_seed=123)
    assert d.data.shape == (50, 5) and d.data.dtype == np.float32 and set(np.unique(d.data)) <= {0., 1.}
    assert d.labels.shape == (50,) and set(np.unique(d.labels)) <= {0, 1}
    assert np.array_equal(d.data, Z.noisy_parity_class(50, random_seed=123).data)
    r = Z.random(10, 200, random_seed=123, sep=2.0)
    assert r.data.shape == (200, 10) and set(np.unique(r.labels)) == {0, 1}
    assert np.array_equal(r.data, Z.random(10, 200, random_seed=123, sep=2.0).data)
    b = Z.random_binary(7, 30, random_seed=4)
    assert b.data.shape == (30, 7) and set(np.unique(b.data)) <= {0., 1.} and b.labels.shape == (30, 1)
    assert not b.labels.any() and np.array_equal(b.data, Z.random_binary(7, 30, random_seed=4).data)
    s = Z.random_symmetric(6, 40, random_seed=5)
    assert s.data.shape == (40, 6) and np.array_equal(s.data[:20], -s.data[20:]) and s.labels.shape == (40, 1)
    assert np.array_equal(s.data, Z.random_symmetric(6, 40, random_seed=5).data)
    m = Z.random_mlp(8, 100, random_seed=6)
    assert m.data.shape == (100, 8) and m.labels.shape == (100,) and set(np.unique(m.labels)) <= {0, 1}
    assert np.array_equal(m.labels, Z.random_mlp(8, 100, random_seed=6).labels)
    # the reference draws random_mlp's inputs then 6 layers of weights from np.random.seed(seed)
    rng = np.random.RandomState(6)
    x = rng.normal(size=(100, 8))
    assert np.array_equal(m.data, x.astype("float32"))


def test_batch_indices_cover_each_epoch():
    d = Z.Dataset(np.arange(10, dtype="float32")[:, None], np.zeros(10, dtype="int32"))
    bs = d.batch_indices(6, 3, np.random.RandomState(0))
    assert all(len(b) == 3 for b in bs)
    assert len(set(bs[0] + bs[1] + bs[2])) == 9


# ---- objectives (fp64 torch restatement) vs numpy -------------------------------------------------------------------
def _f(problem, x, data=None):
    ps = [torch.as_tensor(np.asarray(x, dtype=np.float64)).reshape(s) for s in problem.param_shapes] \
        if len(problem.param_shapes) == 1 else x
    d = None if data is None else torch.as_tensor(data, dtype=torch.float64)
    return float(problem.torch_objective(ps, d))


TWO_D = {
    "Rosenbrock": lambda x, y: (1 - x) ** 2 + 100 * (y - x * x) ** 2,
    "Saddle": lambda x, y: x * x - y * y,
    "LogSumExp": lambda x, y: np.log(np.exp(x + 3 * y - .1) + np.exp(x - 3 * y - .1) + np.exp(-x - .1) + 1),
    "Ackley": lambda x, y: (-20 * np.exp(-0.2 * np.sqrt(0.5 * (x * x + y * y)))
                            - np.exp(0.5 * (np.cos(2 * np.pi * x) + np.cos(2 * np.pi * y))) + np.e + 20),
    "Beale": lambda x, y: (1.5 - x + x * y) ** 2 + (2.25 - x + x * y ** 2) ** 2 + (2.625 - x + x * y ** 3) ** 2,
    "Booth": lambda x, y: (x + 2 * y - 7) ** 2 + (2 * x + y - 5) ** 2,
    "StyblinskiTang": lambda x, y: 0.5 * (x ** 4 - 16 * x ** 2 + 5 * x + y ** 4 - 16 * y ** 2 + 5 * y) + 80,
    "Matyas": lambda x, y: 0.26 * (x * x + y * y) - 0.48 * x * y,
    "Branin": lambda x, y: ((y - 5.1 / (4 * np.pi ** 2) * x * x + 5 / np.pi * x - 6) ** 2
                            + 10 * (1 - 1 / (8 * np.pi)) * np.cos(x) + 10),
    "Michalewicz": lambda x, y: 2 - (np.sin(x) * np.sin(x * x / np.pi) ** 10 + np.sin(y) * np.sin(2 * y * y / np.pi) ** 10),
}


@pytest.mark.parametrize("name", sorted(TWO_D))
def test_two_d_objectives(name):
    p = getattr(Z, name)(random_seed=0)
    for x, y in ((0.3, -1.2), (2.5, 0.7), (-1.1, 3.3)):
        assert _f(p, [x, y]) == pytest.approx(TWO_D[name](x, y), rel=1e-12, abs=1e-12)


def test_known_minima():
    assert _f(Z.Rosenbrock(), [1, 1]) == 0.0
    assert _f(Z.Booth(), [1, 3]) == 0.0
    assert _f(Z.Matyas(), [0, 0]) == 0.0
    assert _f(Z.Beale(), [3, 0.5]) == 0.0


def test_matrix_and_elementwise_objectives():
    rs = np.random.RandomState(1)
    for n in (3, 20):
        x = rs.randn(n)
        qd = Z.Quadratic(n, random_seed=7)
        r = qd.w.astype(np.float64) @ x - qd.y[:, 0]
        assert _f(qd, x) == pytest.approx(0.5 * (r ** 2).sum(), rel=1e-12)
        w = np.random.RandomState(7).randn(n, n).astype("float32")   # seed use: W then y from the problem's seed
        assert np.array_equal(qd.w, w)
        la = Z.Lasso(n, lambda_=0.7, random_seed=7)
        assert _f(la, x) == pytest.approx(0.5 * (r ** 2).sum() + 0.7 * np.abs(x).sum(), rel=1e-12)
        for pw in (1., 1.5, 3.):
            nm = Z.Norm(n, random_seed=7, norm_power=pw)
            assert _f(nm, x) == pytest.approx(((np.abs(r) + 1e-6) ** pw).sum() ** (1 / pw), rel=1e-12)
        ra = Z.Rastrigin(n, alpha=3, random_seed=7)
        rr = ra.a.astype(np.float64) @ x - ra.b[:, 0]
        want = (0.5 * rr ** 2).mean() - 3 * (ra.c[:, 0] @ np.cos(2 * np.pi * x)) + 3 * n * n
        assert _f(ra, x) == pytest.approx(want, rel=1e-12)
        assert _f(Z.IsotropicQuadratic([(n,)]), x) == pytest.approx((x ** 2).sum(), rel=1e-12)
        dc = Z.DependencyChain(n - 1)
        assert _f(dc, x) == pytest.approx(((x[0] ** 2 + x[1:] ** 2 / (x[:-1] ** 2 + 1e-6))).sum(), rel=1e-12)
        mm = Z.MinMaxWell(n)
        assert _f(mm, x) == pytest.approx((x ** 2).max() + 1 / (x ** 2).min() - 2 + 1e-12, rel=1e-12)
        d = rs.randn(7, n)
        assert _f(Z.ProjectionQuadratic(n), x, d) == pytest.approx(((x * d) ** 2).sum(), rel=1e-12)
        assert _f(Z.SumOfQuadratics(n), x, d) == pytest.approx(((x - d) ** 2).sum() - (d ** 2).sum() + 1e-12,
                                                               rel=1e-10)
        snake = 1 / (np.sqrt((x ** 2).sum()) + 1e-6) * d[:, 0].sum() + (((x[1:] - np.cos(x[:-1]) * np.pi) * d[:, 1:])
                                                                          ** 2).sum()
        assert _f(Z.OutwardSnake(n), x, d) == pytest.approx(snake, rel=1e-12)
    b = Z.Bowl(5.0, angle=PI4)
    m = np.sqrt(np.diag([5.0, 1.0])) @ np.array([[np.cos(PI4), -np.sin(PI4)], [np.sin(PI4), np.cos(PI4)]])
    assert _f(b, [0.4, -0.9]) == pytest.approx(0.5 * ((m @ [0.4, -0.9]) ** 2).sum(), rel=1e-6)


def test_wrappers_and_dataset_families():
    rs = np.random.RandomState(2)
    x = rs.randn(20)
    inner = Z.Quadratic(20, random_seed=3)
    f0 = _f(inner, x)
    assert _f(Z.Rescale(Z.Spec(Z.Quadratic, (20,), {"random_seed": 3}), scale=4.), x * 4.) == pytest.approx(f0)
    assert _f(Z.LogObjective(Z.Spec(Z.Quadratic, (20,), {"random_seed": 3})), x) == \
        pytest.approx(np.log(f0 + 1e-6) - np.log(1e-6))
    st = Z.SumTask([Z.Spec(Z.Quadratic, (20,), {"random_seed": 3}), Z.Spec(Z.Booth, (), {})])
    ps = [torch.as_tensor(x).reshape(20, 1), torch.tensor([1.0, 2.0], dtype=torch.float64)]
    assert float(st.torch_objective(ps)) == pytest.approx(f0 + TWO_D["Booth"](1.0, 2.0))
    sm = Z.SoftmaxRegression(4, 2)
    w, bias = torch.randn(4, 2, dtype=torch.float64), torch.randn(2, dtype=torch.float64)
    data, labels = torch.randn(9, 4, dtype=torch.float64), torch.randint(0, 2, (9,))
    z = (data @ w + bias)[:, 0].numpy()
    lab = labels.numpy()
    want = np.mean(np.maximum(z, 0) - z * lab + np.log1p(np.exp(-np.abs(z))))
    assert float(sm.torch_objective([w, bias], data, labels)) == pytest.approx(want, rel=1e-12)
    sp, oh = Z.SparseSoftmaxRegression(5, 2), Z.OneHotSparseSoftmaxRegression(5, 2)
    ps = [torch.randn(s, dtype=torch.float64) for s in sp.param_shapes]
    ids = torch.randint(0, 2, (6, 5)).double()
    assert float(sp.torch_objective(ps, ids, labels[:6])) == pytest.approx(float(oh.torch_objective(ps, ids, labels[:6])))
    fc = Z.FullyConnected(3, 2, hidden_sizes=(4,))
    assert fc.param_shapes == [(3, 4), (4,), (4, 2), (2,)]
    mm = Z.MatMulAlgorithm(2, 8)
    assert mm.param_shapes == [(4, 8), (4, 8)]
    init = mm.init_tensors(0, "cpu")
    assert torch.allclose(init[0].norm(dim=0), torch.ones(8))
    assert math.isfinite(float(mm.torch_objective([t.double() for t in init])))


def test_init_tensors_distributions():
    for cls, lo, hi in ((Z.Rosenbrock, -5., 10.), (Z.Ackley, -32.768, 32.768), (Z.Beale, -4.5, 4.5),
                        (Z.Booth, -10., 10.), (Z.Michalewicz, 0., np.pi)):
        t = cls().init_tensors(0, "cpu")[0]
        assert t.shape == (2,) and bool(((t >= lo) & (t <= hi)).all())
    b = Z.Branin().init_tensors(1, "cpu")[0]
    assert -5 <= float(b[0]) <= 10 and 0 <= float(b[1]) <= 15
    a, b2 = Z.Quadratic(5).init_tensors(3, "cpu"), Z.Quadratic(5).init_tensors(3, "cpu")
    assert torch.equal(a[0], b2[0]) and a[0].shape == (5, 1)


def test_kernel_objective_needs_cuda_tensors():
    p = Z.Booth()
    with pytest.raises(_lib.L2OError):
        p.objective([torch.zeros(2)])


# ---- C ABI -------------------------------------------------------------------------------------------------------------
def _args(**kw):
    a = _lib.ZooArgs()
    a.family, a.n, a.rows = kw.get("family", _lib.ZOO["QUADRATIC"]), kw.get("n", 4), kw.get("rows", 4)
    a.p0 = kw.get("p0", 2.0)
    fake = 256
    for name in ("x", "v", "A", "y", "c", "f", "out"):
        setattr(a, name, kw.get(name, fake))
    return a


@pytest.mark.skipif(not os.path.exists(_lib.LIB_PATH), reason="library not built")
def test_zoo_abi_argument_checks_without_gpu():
    L, Z_ = _lib.lib(), _lib.ZOO
    INV, UNS = _lib.L2O_E_INVALID, _lib.L2O_E_UNSUPPORTED
    assert L.l2o_zoo_value_grad(None, None) == INV and L.l2o_zoo_hvp(None, None) == INV
    bad = [dict(x=None), dict(out=None), dict(family=-1), dict(family=21), dict(n=0),
           dict(rows=5), dict(A=None), dict(y=None), dict(family=Z_["BOWL"], n=3, rows=3),
           dict(family=Z_["RASTRIGIN"], c=None), dict(family=Z_["NORM"], p0=0.0), dict(family=Z_["NORM"], p0=-1.0),
           dict(family=Z_["ROSENBROCK"], n=3), dict(family=Z_["PROJECTION_QUADRATIC"], rows=0),
           dict(family=Z_["OUTWARD_SNAKE"], n=1), dict(family=Z_["DEPENDENCY_CHAIN"], n=1),
           dict(family=Z_["SUM_OF_QUADRATICS"], A=None)]
    for kw in bad:
        a = _args(**kw)
        assert L.l2o_zoo_value_grad(C.byref(a), None) == INV, kw
        assert L.l2o_zoo_hvp(C.byref(a), None) == INV, kw
    a = _args(v=None)
    assert L.l2o_zoo_hvp(C.byref(a), None) == INV
    big = _lib.ZOO_MAX_N + 1
    for kw in (dict(n=big, rows=big), dict(family=Z_["ISOTROPIC_QUADRATIC"], n=big),
               dict(family=Z_["PROJECTION_QUADRATIC"], n=big, rows=3)):
        a = _args(**kw)
        assert L.l2o_zoo_value_grad(C.byref(a), None) == UNS, kw
        assert L.l2o_zoo_hvp(C.byref(a), None) == UNS, kw
    assert len(_lib.ZOO_FAMILIES) == 21


# ---- scale_metarun ---------------------------------------------------------------------------------------------------
def test_metarun_flags_and_defaults():
    f = smr.parse([])
    assert f.optimizer == "HierarchicalRNN" and f.num_problems == 1 and f.num_meta_iterations == 5
    assert f.meta_learning_rate == 1e-6 and f.gradient_clip_level == 1e4 and f.use_second_derivatives is True
    assert f.num_unroll_scale == 40 and f.min_num_unrolls == 10 and f.fix_unroll_length == 20 and not f.if_cl
    assert smr.included(f) == []
    f = smr.parse(["--optimizer", "TrainableAdam", "--include_quadratic_problems", "--include_bowl_problems=false",
                   "--nouse_second_derivatives", "--if_cl", "--include_softmax_2_class_problems=true",
                   "--num_problems", "3", "--meta_learning_rate", "0.01"])
    assert f.optimizer == "TrainableAdam" and f.use_second_derivatives is False and f.if_cl is True
    assert smr.included(f) == ["quadratic", "softmax_2_class"] and f.num_problems == 3 and f.meta_learning_rate == 0.01
    assert smr.optimizer_kwargs(f) == {}
    kw = smr.optimizer_kwargs(smr.parse(["--cell_cls", "LSTMCell", "--optimizer", "CoordinatewiseRNN"]))
    assert kw["cell_sizes"] == [10, 20, 20] and kw["cell_cls"] == "LSTMCell" and kw["init_lr_range"] == (1e-6, 1e-2)


def test_sample_numiter():
    rng = np.random.RandomState(0)
    v = [smr.sample_numiter(rng, 20, 10) for _ in range(200)]
    assert min(v) >= 10 and max(v) <= 30


def test_metarun_assembles_problems_for_a_stub_loop(tmp_path):
    seen = {}

    def stub(make_trainer, problems, num_problems, num_meta_iterations, num_unroll_func, num_partial_func, **kw):
        seen.update(problems=problems, num_problems=num_problems, kw=kw, unrolls=num_unroll_func(),
                    itrs=num_partial_func())
        return torch.zeros(1), []
    f = smr.parse(["--optimizer", "GlobalLearningRate", "--device", "cpu", "--train_dir", str(tmp_path),
                   "--include_quadratic_problems", "--include_optimization_test_problems",
                   "--include_softmax_2_class_problems", "--num_problems", "7"])
    smr.run(f, out=None, train_optimizer=stub)
    probs = seen["problems"]
    assert len(probs) == 4 + 4 + 9 and seen["num_problems"] == 7
    shapes = [[tuple(t.shape) for t in init()] for _, init in probs]
    assert shapes[:4] == [[(20, 1)], [(25, 1)], [(50, 1)], [(100, 1)]]
    assert shapes[4:8] == [[(10, 2), (2,)], [(100, 2), (2,)], [(200, 2), (2,)], [(256, 2), (2,)]]
    assert shapes[8:] == [[(2,)]] * 9
    # the softmax problems evaluate (torch ops) on a batch of batch_size rows
    obj, init = probs[4]
    assert math.isfinite(float(obj(init())))
    assert 10 <= seen["unrolls"] <= 30 and 10 <= seen["itrs"] <= 30
    assert seen["kw"]["save_path"].startswith(str(tmp_path))
    with pytest.raises(ValueError):
        smr.run(smr.parse(["--device", "cpu", "--train_dir", str(tmp_path)]), train_optimizer=stub)
