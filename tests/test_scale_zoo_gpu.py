"""GPU: the l2o_zoo kernels (value-and-gradient, Hessian-vector product) of L2O-Scale's analytic problem families
against fp64 autograd of their torch restatement, eager vs graph replay, launch counts, HierarchicalRNN meta-gradients
on a zoo problem, and scale_metarun end to end for the five optimizers."""
import math

import numpy as np
import pytest
import torch

from open_l2o_b200 import scale_zoo as Z

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEEDS = (0, 1, 2)


def _rel(a, b):
    a, b = a.double().cpu().reshape(-1), b.double().cpu().reshape(-1)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _reference(problem, x32, v32, data=None):
    """fp64 autograd of the torch restatement at the fp32 point: (f, g, H v)."""
    x = x32.detach().double().cpu().requires_grad_(True)
    d = None if data is None else data.double().cpu()
    f = problem.torch_objective([x.view(problem.param_shapes[0])], d)
    (g,) = torch.autograd.grad(f, x, create_graph=True)
    (hv,) = torch.autograd.grad(g, x, grad_outputs=v32.double().cpu())
    return f.detach(), g.detach(), hv


def _kernel(problem, x32, v32, data=None):
    """The product path: f from the kernel, g by autograd (the kernel's g), H v by double backward (the kernel's)."""
    x = x32.detach().clone().requires_grad_(True)
    f = problem.objective([x.view(problem.param_shapes[0])], data)
    (g,) = torch.autograd.grad(f, x, create_graph=True)
    (hv,) = torch.autograd.grad(g, x, grad_outputs=v32)
    return f.detach(), g.detach(), hv


def _check(problem, seed, data=None, tol=1e-5):
    x = problem.init_tensors(seed, DEV)[0].reshape(-1)
    v = torch.randn(x.numel(), generator=torch.Generator().manual_seed(seed + 100)).to(DEV)
    fk, gk, hk = _kernel(problem, x, v, data)
    fr, gr, hr = _reference(problem, x, v, data)
    torch.cuda.synchronize()
    e = dict(f=abs(float(fk) - float(fr)) / max(abs(float(fr)), 1e-30), g=_rel(gk, gr), hv=_rel(hk, hr))
    assert e["f"] <= tol and e["g"] <= tol and e["hv"] <= tol, (type(problem).__name__, seed, e)


CASES = ([("Quadratic", (n,), {}) for n in (1, 20, 100, 300, 2048)]
         + [("Lasso", (n,), {"lambda_": 0.7}) for n in (20, 300)]
         + [("Norm", (n,), {"norm_power": p}) for n in (18, 300) for p in (1., 1.5, 2., 3.)]
         + [("Rastrigin", (n,), {}) for n in (2, 50, 300)]
         + [("Bowl", (c,), {"angle": a}) for c, a in ((0.1, 0.0), (5.0, np.pi / 4.))]
         + [("IsotropicQuadratic", ([(n,)],), {}) for n in (3, 1000)]
         + [("DependencyChain", (n,), {}) for n in (1, 20, 1000)]
         + [("MinMaxWell", (n,), {}) for n in (2, 64, 1000)]
         + [(c, (), {}) for c in ("Rosenbrock", "Saddle", "LogSumExp", "Ackley", "Beale", "Booth", "StyblinskiTang",
                                  "Matyas", "Branin", "Michalewicz")])


@pytest.mark.parametrize("cls,args,kwargs", CASES, ids=["%s%s" % (c, a) for c, a, _ in CASES])
def test_analytic_family_matches_fp64_autograd(cls, args, kwargs):
    for seed in SEEDS:
        problem = getattr(Z, cls)(*args, random_seed=seed, **kwargs) if cls != "IsotropicQuadratic" else \
            Z.IsotropicQuadratic(*args, random_seed=seed)
        _check(problem, seed)


DATA_CASES = [(c, n, b) for c in ("ProjectionQuadratic", "SumOfQuadratics", "OutwardSnake")
              for n, b in ((12, 10), (64, 128), (300, 300))]


@pytest.mark.parametrize("cls,n,batch", DATA_CASES)
def test_data_family_matches_fp64_autograd(cls, n, batch):
    for seed in SEEDS:
        problem = getattr(Z, cls)(n, random_seed=seed)
        gen = np.random.RandomState(seed)
        ds = Z.random_binary(n, batch, random_seed=seed) if cls == "OutwardSnake" else \
            Z.random_symmetric(n, batch, random_seed=seed)
        data = torch.as_tensor(ds.data[gen.permutation(batch)]).to(DEV)
        _check(problem, seed, data)


def test_wrappers_over_kernel_families():
    for seed in SEEDS:
        for spec in (Z.Spec(Z.Rescale, [Z.Spec(Z.Norm, (18,), {"norm_power": 2.5})], {"scale": 8}),
                     Z.Spec(Z.Rescale, [Z.Spec(Z.Quadratic, (100,), {})], {"scale": 0.1}),
                     Z.Spec(Z.LogObjective, [Z.Spec(Z.Quadratic, (50,), {})], {}),
                     Z.Spec(Z.LogObjective, [Z.Spec(Z.Bowl, (5.0,), {})], {}),
                     Z.Spec(Z.SparseProblem, [Z.Spec(Z.Quadratic, (20,), {})], {})):
            np.random.seed(seed)
            _check(spec.build(), seed)
        np.random.seed(seed)
        st = Z.SumTask([Z.Spec(Z.Quadratic, (11,), {}), Z.Spec(Z.Rosenbrock, (), {}), Z.Spec(Z.Ackley, (), {})])
        ps = st.init_tensors(seed, DEV)
        leaf = [p.detach().clone().requires_grad_(True) for p in ps]
        gk = torch.autograd.grad(st.objective(leaf), leaf)
        ref = [p.detach().double().requires_grad_(True) for p in ps]
        gr = torch.autograd.grad(st.torch_objective(ref), ref)
        assert max(_rel(a, b) for a, b in zip(gk, gr)) <= 1e-5


def test_graph_replay_is_bitwise_eager_and_one_launch():
    from open_l2o_b200.engine import launch_count
    problems = [Z.Quadratic(2048, random_seed=0), Z.Norm(300, random_seed=1, norm_power=1.5), Z.Rosenbrock(),
                Z.MinMaxWell(64), Z.DependencyChain(20)]
    for p in problems:
        x = p.init_tensors(0, DEV)[0].reshape(-1).contiguous()
        v = torch.randn_like(x)
        k = p.kernel(x)
        before = launch_count()
        f0, g0 = k.value_grad(x)
        assert launch_count() - before == 1
        before = launch_count()
        h0 = k.hvp(x, v)
        assert launch_count() - before == 1
        f1, g1 = k.value_grad(x)
        assert torch.equal(f0, f1) and torch.equal(g0, g1)   # run to run
        out = {}
        graph = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
            out["f"], out["g"] = k.value_grad(x)
            out["h"] = k.hvp(x, v)
        torch.cuda.current_stream().wait_stream(s)
        for _ in range(2):
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(out["f"], f0) and torch.equal(out["g"], g0) and torch.equal(out["h"], h0), type(p)


def _hrnn_meta(objective, params, second):
    from open_l2o_b200 import hrnn_train as ht
    shapes = [tuple(p.shape) for p in params]
    tr = ht.MetaTrainer(shapes, theta=ht._init_theta(3), device=DEV, use_second_derivatives=second)
    n = sum(p.numel() for p in params)
    llr = (torch.rand(n, generator=torch.Generator().manual_seed(5)) * 3.0 - 6.0)
    meta, grad, objs, _ = tr.meta_gradient(objective, params, 6, log_learning_rate=llr)
    return float(meta), grad.double().cpu(), objs


def test_hrnn_meta_gradient_kernel_vs_torch_objective():
    """The same meta-gradient, first and second order, whether the optimizee's value, gradient and H v come from the
    kernel or from torch ops.  The objectives agree to fp32 rounding, so the meta-gradients agree within a small
    multiple of it; the second-order term must stand well clear of that difference on at least one problem, so that
    the comparison sees the kernel's H v."""
    seps = []
    for problem in (Z.Quadratic(20, random_seed=4), Z.Rosenbrock(random_seed=0)):
        params = problem.init_tensors(7, DEV)
        got = {}
        for second in (False, True):
            mk, gk, ok = _hrnn_meta(lambda ps: problem.objective(ps), params, second)
            mt, gt, ot = _hrnn_meta(lambda ps: problem.torch_objective(ps), params, second)
            assert all(math.isfinite(o) for o in ok)
            assert abs(mk - mt) <= 1e-4 * max(1.0, abs(mt)), (mk, mt)
            got[second] = (gk, gt, _rel(gk, gt))
            assert got[second][2] <= 1e-3, (type(problem).__name__, second, got[second][2])
        sep = _rel(got[False][1], got[True][1])   # torch: first against second order
        seps.append((sep, got[True][2], type(problem).__name__))
    assert any(sep > 1e-5 and sep >= 10.0 * err for sep, err, _ in seps), seps


@pytest.mark.parametrize("optimizer", ["HierarchicalRNN", "CoordinatewiseRNN", "TrainableAdam", "GlobalLearningRate",
                                       "LearningRateSchedule"])
def test_scale_metarun_runs_each_optimizer(optimizer, tmp_path):
    from open_l2o_b200 import scale_metarun as smr
    flags = smr.parse(["--optimizer", optimizer, "--cell_cls", "LSTMCell", "--train_dir", str(tmp_path),
                       "--include_quadratic_problems", "--include_optimization_test_problems",
                       "--include_softmax_2_class_problems", "--num_problems", "3", "--num_meta_iterations", "1",
                       "--fix_unroll", "--fix_unroll_length", "3", "--fix_num_steps", "6", "--fix_num_steps_eval", "3",
                       "--evaluation_epochs", "1", "--meta_learning_rate", "1e-3", "--seed", "2"])
    theta, log = smr.run(flags, out=None)
    assert len(log) == 3 and all(len(m) >= 1 and all(math.isfinite(v) for v in m) for _, m in log), log
    assert bool(torch.isfinite(theta).all())
    from open_l2o_b200.trainable_baselines import register_optimizers
    theta0 = register_optimizers()[optimizer](device=DEV, **smr.optimizer_kwargs(flags)).theta
    assert theta.shape == theta0.shape and not torch.equal(theta.detach(), theta0)


def test_noisy_problem_gradient_noise_uses_the_generator():
    problem = Z.Quadratic(20, random_seed=0, noise_stdev=0.5)
    x = problem.init_tensors(0, DEV)
    gens = [torch.Generator(device=DEV) for _ in range(2)]
    grads = []
    for g in gens:
        g.manual_seed(9)
        leaf = [t.clone().requires_grad_(True) for t in x]
        grads.append(torch.autograd.grad(Z.training_objective(problem, None, g)(leaf), leaf)[0])
    assert torch.equal(grads[0], grads[1])
    leaf = [t.clone().requires_grad_(True) for t in x]
    plain = torch.autograd.grad(problem.objective(leaf), leaf)[0]
    d = (grads[0] - plain).reshape(-1)
    assert 0.3 < float(d.std()) < 0.7
    sparse = Z.SparseProblem(Z.Spec(Z.Quadratic, (100,), {"random_seed": 0}))
    leaf = [t.clone().requires_grad_(True) for t in sparse.init_tensors(0, DEV)]
    g = torch.autograd.grad(Z.training_objective(sparse, None, gens[0])(leaf), leaf)[0]
    assert 0.8 <= float((g == 0).float().mean()) <= 1.0
