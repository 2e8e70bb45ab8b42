"""GPU: ``l2o_zoo_hess_form`` against fp64 triple autograd of the torch restatements, determinism, graph replay and
launch counts; the regularisers inside the five trainers' meta-gradients, kernel path against ``torch_objective``;
and scale_metarun with ``--reg_optimizer``."""
import math

import numpy as np
import pytest
import torch

from open_l2o_b200 import _lib
from open_l2o_b200 import scale_zoo as Z
from oracle import scale_reg_oracle as O
from tests.test_scale_zoo_gpu import CASES, DATA_CASES

pytestmark = pytest.mark.gpu
DEV = "cuda"
CONSTANT_HESSIAN = ("Quadratic", "Lasso", "Bowl", "IsotropicQuadratic", "ProjectionQuadratic", "SumOfQuadratics",
                    "Booth", "Matyas", "Saddle")


def _rel(a, b):
    a, b = a.double().cpu().reshape(-1), b.double().cpu().reshape(-1)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _reference(problem, x32, U, V, data=None):
    """fp64 autograd of the torch restatement: q = sum_k u_k^T H v_k and dq/dx."""
    x = x32.detach().double().cpu().requires_grad_(True)
    d = None if data is None else data.double().cpu()
    f = problem.torch_objective([x.view(problem.param_shapes[0])], d)
    (g,) = torch.autograd.grad(f, x, create_graph=True)
    q = 0.0
    for u, v in zip(U.double().cpu(), V.double().cpu()):
        (hv,) = torch.autograd.grad(g, x, grad_outputs=v, create_graph=True)
        q = q + (hv * u).sum()
    (dq,) = torch.autograd.grad(q, x)
    return q.detach(), dq


def _pairs(n, k, seed, same):
    g = torch.Generator().manual_seed(seed + 1000)
    U = torch.randn(k, n, generator=g)
    V = U if same else torch.randn(k, n, generator=g)
    return U.to(DEV), (U.to(DEV) if same else V.to(DEV))


def _check(problem, name, seed, data=None, tol=1e-5):
    x = problem.init_tensors(seed, DEV)[0].reshape(-1).contiguous()
    z = problem.kernel(x, data)
    for k in (1, 10):
        for same in (False, True):
            U, V = _pairs(x.numel(), k, seed, same)
            q, dq = z.hess_form(x, U, U if same else V)
            qr, dqr = _reference(problem, x, U, V, data)
            torch.cuda.synchronize()
            eq = abs(float(q) - float(qr)) / max(abs(float(qr)), 1e-30)
            assert eq <= tol and _rel(dq, dqr) <= tol, (name, seed, k, same, eq, _rel(dq, dqr))
            if name in CONSTANT_HESSIAN:
                assert not bool(dq.any()), name   # an exact zero


def _tol(cls, kwargs):
    # NORM at p = 1.5: the third derivative carries a^(p-3) = a^-1.5 of the row residuals a = |r| + 1e-6, which weights
    # the rounding of the smallest residuals (the kernel stores its row weights in fp32, as its H v does) far above the
    # rest, so the gradient is held to 1e-4 there.
    return 1e-4 if cls == "Norm" and kwargs.get("norm_power") == 1.5 else 1e-5


LARGE = [("Quadratic", (4096,), {}), ("Norm", (4096,), {"norm_power": 3.}), ("Rastrigin", (1024,), {})]


@pytest.mark.parametrize("cls,args,kwargs", CASES + LARGE, ids=["%s%s" % (c, a) for c, a, _ in CASES + LARGE])
def test_hess_form_matches_fp64_triple_autograd(cls, args, kwargs):
    for seed in (0, 1):
        problem = getattr(Z, cls)(*args, random_seed=seed, **kwargs) if cls != "IsotropicQuadratic" else \
            Z.IsotropicQuadratic(*args, random_seed=seed)
        _check(problem, cls, seed, tol=_tol(cls, kwargs))


@pytest.mark.parametrize("cls,n,batch", DATA_CASES + [("OutwardSnake", 2048, 64)])
def test_hess_form_data_families(cls, n, batch):
    for seed in (0, 1):
        problem = getattr(Z, cls)(n, random_seed=seed)
        gen = np.random.RandomState(seed)
        ds = Z.random_binary(n, batch, random_seed=seed) if cls == "OutwardSnake" else \
            Z.random_symmetric(n, batch, random_seed=seed)
        data = torch.as_tensor(ds.data[gen.permutation(batch)]).to(DEV)
        _check(problem, cls, seed, data)


def test_hess_form_chunks_pairs_above_the_limit():
    from open_l2o_b200.engine import launch_count
    problem = Z.Norm(300, random_seed=2, norm_power=2.5)
    x = problem.init_tensors(2, DEV)[0].reshape(-1).contiguous()
    k = 2 * _lib.ZOO_MAX_PAIRS + 3
    U, V = _pairs(300, k, 2, False)
    before = launch_count()
    q, dq = problem.kernel(x).hess_form(x, U, V)
    assert launch_count() - before == 3
    qr, dqr = _reference(problem, x, U, V)
    assert abs(float(q) - float(qr)) <= 1e-5 * abs(float(qr)) and _rel(dq, dqr) <= 1e-5


def test_hess_form_deterministic_and_graph_replay():
    for p in (Z.Quadratic(2048, random_seed=0), Z.Norm(300, random_seed=1, norm_power=1.5), Z.Ackley(),
              Z.MinMaxWell(64), Z.DependencyChain(20)):
        x = p.init_tensors(0, DEV)[0].reshape(-1).contiguous()
        U, V = _pairs(x.numel(), 10, 0, False)
        z = p.kernel(x)
        q0, d0 = z.hess_form(x, U, V)
        q1, d1 = z.hess_form(x, U, V)
        assert torch.equal(q0, q1) and torch.equal(d0, d1)
        out = {}
        graph, s = torch.cuda.CUDAGraph(), torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            out["q"], out["d"] = z.hess_form(x, U, V)
        torch.cuda.current_stream().wait_stream(s)
        for _ in range(2):
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(out["q"], q0) and torch.equal(out["d"], d0), type(p)


def test_hutchinson_on_a_bare_family_is_one_launch_and_none_backward():
    from open_l2o_b200.engine import launch_count
    from open_l2o_b200.scale_reg import Regularizer
    problem = Z.Rosenbrock(random_seed=0)
    objective = Z.training_objective(problem)
    x = problem.init_tensors(0, DEV)[0].reshape(-1).clone().requires_grad_(True)
    reg = Regularizer("hessian", 10, seed=0)
    objective([x])
    before = launch_count()
    r = reg(objective, x, lambda t: [t], None)
    assert launch_count() - before == 1
    before = launch_count()
    (d,) = torch.autograd.grad(r, x)
    assert launch_count() - before == 0
    P = reg.probes(objective, 2, "cpu", torch.float64)
    want = O.regularizer("hessian", lambda t: problem.torch_objective([t]), x.detach(), probes=P)
    assert abs(float(r.detach()) - float(want)) <= 1e-5 * abs(float(want))


def test_zoo_hvp_adjoint_through_autograd():
    """The third-order chain through _ZooGrad -> _ZooHvp -> hess_form / hvp, against torch ops in fp64."""
    for problem in (Z.Norm(18, random_seed=0, norm_power=2.5), Z.Beale(), Z.DependencyChain(12)):
        x32 = problem.init_tensors(1, DEV)[0].reshape(-1)
        v = torch.randn(x32.numel(), generator=torch.Generator().manual_seed(4)).to(DEV)
        out = []
        for obj, x, vv in ((problem.objective, x32.clone().requires_grad_(True), v.clone().requires_grad_(True)),
                           (problem.torch_objective, x32.double().cpu().requires_grad_(True),
                            v.double().cpu().requires_grad_(True))):
            (g,) = torch.autograd.grad(obj([x.view(problem.param_shapes[0])]), x, create_graph=True)
            (hv,) = torch.autograd.grad(g, x, grad_outputs=vv, create_graph=True)
            out.append(torch.autograd.grad((hv * hv).sum(), (x, vv)))
        assert _rel(out[0][0], out[1][0]) <= 1e-4 and _rel(out[0][1], out[1][1]) <= 1e-5, type(problem)


# ---- trainers --------------------------------------------------------------------------------------------------------
def _trainer(name, shapes, second, **reg):
    from open_l2o_b200 import baselines_train as bt
    from open_l2o_b200 import hrnn_train as ht
    if name == "HierarchicalRNN":
        return ht.MetaTrainer(shapes, theta=ht._init_theta(3), device=DEV, use_second_derivatives=second,
                              random_seed=3, **reg)
    return bt.TrainableAdamTrainer(shapes, device=DEV, use_second_derivatives=second, random_seed=3,
                                   learning_rate=1e-3, **reg)


def _meta(name, objective, params, second, **reg):
    tr = _trainer(name, [tuple(p.shape) for p in params], second, **reg)
    n = sum(p.numel() for p in params)
    llr = (torch.rand(n, generator=torch.Generator().manual_seed(5)) * 3.0 - 6.0) if name == "HierarchicalRNN" else None
    meta, grad, objs, _ = tr.meta_gradient(objective, params, 5, log_learning_rate=llr, regularize=True)
    return float(meta), grad.double().cpu(), objs, tr


OPTS = ["hessian", "jacob", "hessian-ev", "hessian-esd"]
COMBOS = [(o, flag, second) for o in OPTS for flag in ("reg_optimizer", "reg_optimizee") for second in (False, True)
          if not (flag == "reg_optimizee" and second and o != "jacob")]


@pytest.mark.parametrize("trainer", ["HierarchicalRNN", "TrainableAdam"])
@pytest.mark.parametrize("option,flag,second", COMBOS)
def test_regularized_meta_gradient_kernel_vs_torch_objective(trainer, option, flag, second):
    """The same regularised meta-gradient whether the objective and its derivatives come from the zoo kernels or from
    torch ops (same probes, same start vectors); the objectives agree to fp32 rounding, so the meta-gradients agree
    within a small multiple of it.  reg(x0) against the fp64 oracle."""
    problem = Z.Norm(18, random_seed=4, norm_power=2.5)
    params = problem.init_tensors(7, DEV)
    reg = {flag: True, "reg_option": option, "hessian_itrs": 4, "alpha": 0.5, "beta": 0.1, "regularize_time": "all"}
    mk, gk, ok, tk = _meta(trainer, Z.training_objective(problem), params, second, **reg)
    mt, gt, ot, _ = _meta(trainer, lambda ps: problem.torch_objective(ps), params, second, **reg)
    assert all(math.isfinite(o) for o in ok) and bool(torch.isfinite(gk).all())
    assert abs(mk - mt) <= 1e-4 * max(1.0, abs(mt)), (mk, mt)
    assert _rel(gk, gt) <= 2e-3, _rel(gk, gt)
    plain, _, _, _ = _meta(trainer, Z.training_objective(problem), params, second)
    if flag == "reg_optimizer":
        assert mk != plain     # the term is in the meta objective
    # the regulariser's value at x0 against the oracle
    objective = Z.training_objective(problem)
    x = torch.cat([p.reshape(-1) for p in params]).clone().requires_grad_(True)
    objective([x.view(params[0].shape)])
    gen = torch.Generator().manual_seed(11)
    r = tk.regularizer(objective, x, lambda t: [t.view(params[0].shape)], gen)
    kw = dict(itrs=4)
    if option == "hessian":
        kw["probes"] = tk.regularizer.probes(objective, x.numel(), "cpu", torch.float64)
    elif option == "hessian-esd":
        kw["v0"] = tk.regularizer.probes(objective, x.numel(), "cpu", torch.float64)[0]
    elif option == "hessian-ev":
        kw["v0"] = torch.randn(x.numel(), generator=torch.Generator().manual_seed(11)).double()
    want = O.regularizer(option, lambda t: problem.torch_objective([t.view(params[0].shape)]), x.detach(), **kw)
    r = float(r.detach())
    assert abs(r - float(want)) <= 1e-4 * max(1.0, abs(float(want))), (r, float(want))


@pytest.mark.parametrize("trainer", ["HierarchicalRNN", "TrainableAdam"])
@pytest.mark.parametrize("second", [False, True])
def test_flags_off_is_bitwise_the_plain_trainer(trainer, second):
    problem = Z.Norm(18, random_seed=4, norm_power=2.5)
    params = problem.init_tensors(7, DEV)
    obj = Z.training_objective(problem)
    m0, g0, o0, _ = _meta(trainer, obj, params, second)
    assert math.isfinite(m0)
    m1, g1, o1, _ = _meta(trainer, obj, params, second, reg_option="hessian-esd", hessian_itrs=3, alpha=1.0, beta=1.0,
                          regularize_time="prior", reg_scale=0.1)
    assert m0 == m1 and torch.equal(g0, g1) and o0 == o1


def test_evaluate_uses_the_regularized_gradient():
    problem = Z.Quadratic(20, random_seed=1)
    objective = Z.training_objective(problem)
    params = problem.init_tensors(2, DEV)
    a = _trainer("TrainableAdam", [tuple(params[0].shape)], False).evaluate(objective, params, [5])
    b = _trainer("TrainableAdam", [tuple(params[0].shape)], False, reg_optimizee=True, reg_option="jacob",
                 beta=1.0).evaluate(objective, params, [5])
    assert math.isfinite(b) and a != b


@pytest.mark.parametrize("optimizer", ["HierarchicalRNN", "CoordinatewiseRNN", "TrainableAdam", "GlobalLearningRate",
                                       "LearningRateSchedule"])
def test_scale_metarun_with_the_hessian_regulariser(optimizer, tmp_path):
    from open_l2o_b200 import scale_metarun as smr
    flags = smr.parse(["--optimizer", optimizer, "--cell_cls", "LSTMCell", "--train_dir", str(tmp_path),
                       "--include_optimization_test_problems", "--reg_optimizer", "--reg_option", "hessian",
                       "--num_problems", "1", "--num_meta_iterations", "2", "--fix_unroll", "--fix_unroll_length",
                       "3", "--fix_num_steps", "18", "--fix_num_steps_eval", "3", "--evaluation_epochs", "1",
                       "--meta_learning_rate", "1e-3", "--seed", "2"])
    theta, log = smr.run(flags, out=None)
    assert len(log) == 2 and all(len(m) >= 1 and all(math.isfinite(v) for v in m) for _, m in log), log
    assert bool(torch.isfinite(theta).all())
