"""GPU: imitation meta-training of the L2O-Scale optimizers (SC/metaopt.py:354-450, 541-548; SC/mt_utils.py;
trainable_optimizer.py:380-389; hierarchical_rnn.py:398-404).  The HierarchicalRNN and CoordinatewiseRNN imitation
meta-gradients against autograd through the fp64 oracles, replay of the recorded gradients against re-evaluation at the
teacher-forced points, and the extended ``train_optimizer`` driver."""
import math
import random

import pytest
import torch

from oracle import crnn_oracle as CR
from oracle import hrnn_oracle as orc   # checker only
from tests.helpers import REL_TOL, hrnn_generic_theta
from tests.test_crnn_gpu import crnn_generic_theta

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SHAPES = [(40, 7), (150,)]
T = 5


def _problem(dtype=torch.float32, device=DEV, seed=0):
    gen = torch.Generator().manual_seed(seed)
    A = torch.randn(60, 40, generator=gen, dtype=torch.float64)
    y = torch.randn(60, 7, generator=gen, dtype=torch.float64)
    C = torch.randn(150, generator=gen, dtype=torch.float64)
    A, y, C = (t.to(device=device, dtype=dtype) for t in (A, y, C))

    def objective(params):
        w, v = params
        return ((A @ w - y) ** 2).mean() + 0.1 * ((v - C) ** 2).mean() + 0.01 * torch.cos(3.0 * v).mean()
    init = [torch.randn(s, generator=gen, dtype=torch.float64) * 0.5 for s in SHAPES]
    return objective, init


def _teacher(k=1):
    from open_l2o_b200.scale_base import teacher_labels
    obj32, init = _problem()
    x0 = torch.cat([p.reshape(-1) for p in init]).float().to(DEV)
    labels, grads = teacher_labels(obj32, x0, SHAPES, [T], "adam", k)
    return obj32, init, labels, grads


def _split(row, dtype):
    out, off = [], 0
    for s in SHAPES:
        n = math.prod(s)
        out.append(row[off:off + n].to(dtype).reshape(s))
        off += n
    return out


def _mse(upds, labs, n):
    return 0.5 * sum(((u.reshape(-1) - l.reshape(-1)) ** 2).sum() for u, l in zip(upds, labs)) / n


def _hrnn_oracle_mt(theta, init, llr, labels, grads, dtype):
    """Autograd through the HierarchicalRNN oracle's unrolled step with x teacher-forced along ``labels`` and the
    weighted mean-square imitation objective, in ``dtype``."""
    th = theta.to(dtype).clone().requires_grad_(True)
    P = orc.unpack_theta(th)
    params = [p.to(dtype) for p in init]
    states, off = [], 0
    for p in params:
        st = orc.initial_state(P, p, torch.Generator().manual_seed(0))
        st["log_learning_rate"] = llr[off:off + p.numel()].to(dtype).reshape(-1, 1)
        off += p.numel()
        states.append(st)
    glob = orc.initial_global_state(P, dtype)
    N, meta = labels.shape[1], 0.0
    for t in range(labels.shape[0]):
        lab, gr = _split(labels[t].cpu(), dtype), _split(grads[t].cpu(), dtype)
        _, states, glob, upds = orc.step(th, params, gr, states, glob)
        meta = meta + _mse(upds, lab, N) / labels.shape[0]
        params = [p - l for p, l in zip(params, lab)]
    (g,) = torch.autograd.grad(meta, th)
    return float(meta.detach()), g.detach().double()


def _crnn_oracle_mt(theta, init, lr0, labels, grads, dtype):
    th = theta.to(dtype).clone().requires_grad_(True)
    P = CR.unpack_theta(th)
    params = [p.to(dtype) for p in init]
    states, off = [], 0
    for p in params:
        st = CR.initial_state(P, p.numel(), torch.Generator(), dtype=dtype)
        st["learning_rate"] = lr0[off:off + p.numel()].to(dtype).reshape(-1, 1)
        off += p.numel()
        states.append(st)
    N, meta = labels.shape[1], 0.0
    for t in range(labels.shape[0]):
        lab, gr = _split(labels[t].cpu(), dtype), _split(grads[t].cpu(), dtype)
        _, states, upds = CR.step(th, params, gr, states)
        meta = meta + _mse(upds, lab, N) / labels.shape[0]
        params = [p - l for p, l in zip(params, lab)]
    (g,) = torch.autograd.grad(meta, th)
    return float(meta.detach()), g.detach().double()


def _check_blocks(spec, g, g64, g32):
    """Each theta block within 1e-5 of its own largest entry, or 3x the fp32 oracle's distance from fp64 where that
    is larger; blocks the reference gradient reaches (and only those) are reached."""
    bad, off = [], 0
    for name, shape in spec:
        n = int(math.prod(shape))
        e, r, f = g[off:off + n], g64[off:off + n], g32[off:off + n]
        off += n
        own = float(r.abs().max())
        assert bool((r != 0).any()) == bool((e != 0).any()), name
        if own == 0.0:
            continue
        err, tol = float((e - r).abs().max()) / own, max(REL_TOL, 3.0 * float((f - r).abs().max()) / own)
        if err > tol:
            bad.append((name, err, tol))
    assert not bad, bad


@pytest.mark.parametrize("theta_kind", ["init", "generic"])
def test_hrnn_imitation_meta_gradient_matches_oracle_autograd(theta_kind):
    from open_l2o_b200 import hrnn_train as ht
    _, init, labels, grads = _teacher()
    theta = orc.init_theta(seed=3) if theta_kind == "init" else hrnn_generic_theta(5)
    n = labels.shape[1]
    llr = (torch.rand(n, generator=torch.Generator().manual_seed(5), dtype=torch.float64) * 3.0 - 6.0).float()
    tr = ht.MetaTrainer(SHAPES, theta=theta, device=DEV)
    meta, g, objs, final = tr.meta_gradient_mt(None, [p.float().to(DEV) for p in init], labels, grads,
                                               log_learning_rate=llr)
    torch.cuda.synchronize()
    assert objs == []
    m64, g64 = _hrnn_oracle_mt(theta, init, llr, labels, grads, torch.float64)
    _, g32 = _hrnn_oracle_mt(theta, init, llr, labels, grads, torch.float32)
    assert abs(float(meta) - m64) <= 1e-5 * abs(m64), (float(meta), m64)
    g = g.detach().cpu().double()
    scale = float(g64.abs().max())
    assert scale > 0 and float((g - g64).abs().max()) <= 1e-5 * scale, float((g - g64).abs().max()) / scale
    _check_blocks(orc.theta_spec(), g, g64, g32)
    x = torch.cat([p.reshape(-1) for p in init]).float().to(DEV)
    for t in range(T):
        x = x - labels[t]
    assert torch.equal(final.x, x)


def test_crnn_imitation_meta_gradient_matches_oracle_autograd():
    from open_l2o_b200 import crnn_train as ct
    _, init, labels, grads = _teacher()
    n = labels.shape[1]
    lr0 = torch.exp(torch.rand(n, generator=torch.Generator().manual_seed(4), dtype=torch.float64) * 3.0 - 6.0).float()
    theta = crnn_generic_theta(7)
    tr = ct.MetaTrainer(SHAPES, theta=theta, device=DEV)
    meta, g, _, _ = tr.meta_gradient_mt(None, [p.float().to(DEV) for p in init], labels, grads, lr0)
    torch.cuda.synchronize()
    m64, g64 = _crnn_oracle_mt(theta, init, lr0, labels, grads, torch.float64)
    _, g32 = _crnn_oracle_mt(theta, init, lr0, labels, grads, torch.float32)
    assert abs(float(meta) - m64) <= 1e-5 * abs(m64), (float(meta), m64)
    _check_blocks(CR.theta_spec(), g.detach().cpu().double(), g64, g32)


@pytest.mark.parametrize("trainer", ["hrnn", "crnn"])
def test_replayed_imitation_unroll_equals_reevaluation(trainer):
    """The recorded gradient rows against evaluating the objective at each teacher-forced point (mt_k = 2: the rows
    are the gradients at the first point of each group); second-order training gives the same meta-gradient, since
    x_t does not depend on theta."""
    from open_l2o_b200 import crnn_train as ct
    from open_l2o_b200 import hrnn_train as ht
    obj32, init, labels, grads = _teacher(k=2)
    make = (lambda **kw: ht.MetaTrainer(SHAPES, theta=hrnn_generic_theta(5), device=DEV, random_seed=1, **kw)) \
        if trainer == "hrnn" else \
        (lambda **kw: ct.MetaTrainer(SHAPES, theta=crnn_generic_theta(7), device=DEV, random_seed=1, **kw))
    p0 = [p.float().to(DEV) for p in init]
    runs = []
    for second, rows in ((False, grads), (False, None), (True, None)):
        tr = make(use_second_derivatives=second)
        meta, g, objs, final = tr.meta_gradient_mt(obj32, p0, labels, rows)
        runs.append((float(meta), g.detach().clone(), final.x.detach().clone(), len(objs)))
    (m0, g0, x0, n0) = runs[0]
    assert n0 == 0 and all(n == T for _, _, _, n in runs[1:])
    for m, g, x, _ in runs[1:]:
        assert abs(m - m0) <= 1e-6 * abs(m0)
        assert float((g - g0).abs().max()) <= 1e-6 * float(g0.abs().max())
        assert torch.equal(x, x0)


def _two_problems():
    obj_a, init_a = _problem()
    tgt = torch.randn(64, generator=torch.Generator().manual_seed(9)).to(DEV)
    return [(obj_a, lambda: [p.float().to(DEV) for p in init_a]),
            (lambda ps: ((ps[0] - tgt) ** 2).mean(), lambda: [torch.zeros(64, device=DEV)])]


@pytest.mark.parametrize("trainer", ["tadam", "hrnn"])
def test_train_optimizer_with_the_recipe_off_is_the_plain_loop(trainer):
    """train_optimizer(if_mt=False, if_cl=False) against the plain sampling loop written out: the same problem draws,
    trainers, partial unrolls and meta-steps.  TrainableAdam's kernels are deterministic, so theta is bitwise the
    same.  The HierarchicalRNN's backward sums d theta with fp64 atomics, whose order varies from run to run, so two
    runs of one loop can differ in theta's last bit: there the log is compared exactly and theta to 1e-6."""
    from open_l2o_b200 import baselines_train as bt
    from open_l2o_b200 import hrnn_train as ht
    problems = _two_problems()

    def make(sh, th):
        if trainer == "tadam":
            return bt.TrainableAdamTrainer(sh, theta=th, device=DEV, learning_rate=1e-3)
        return ht.MetaTrainer(sh, theta=orc.init_theta(seed=3) if th is None else th, device=DEV, learning_rate=1e-4,
                              random_seed=0)
    lens = lambda: iter([2, 3] * 20)
    it = lens()
    theta, log = ht.train_optimizer(make, problems, num_problems=3, num_meta_iterations=2, num_unroll_func=lambda: 2,
                                    num_partial_unroll_itrs_func=lambda: next(it), seed=4, if_mt=False, if_cl=False)
    it, rng, trainers, th, rms, want_log = lens(), random.Random(4), {}, None, None, []
    for _ in range(3):
        k = rng.randrange(len(problems))
        objective, init_fn = problems[k]
        shapes = tuple(tuple(p.shape) for p in init_fn())
        if shapes not in trainers:
            trainers[shapes] = make(shapes, th)
        tr = trainers[shapes]
        if th is not None and tr.theta is not th:
            with torch.no_grad():
                tr.theta.copy_(th)
                tr.rms.copy_(rms)
        for _ in range(2):
            ls = [next(it) for _ in range(2)]
            metas, _, _ = tr._train_unrolls(objective, init_fn(), ls)
            want_log.append((k, metas))
        th, rms = tr.theta, tr.rms
    assert log == want_log and len(set(k for k, _ in log)) == 2
    if trainer == "tadam":
        assert torch.equal(theta.detach(), th.detach())
    else:
        assert float((theta - th).abs().max()) <= 1e-6 * float(th.abs().max())


def test_train_optimizer_imitation_and_curriculum_end_to_end(tmp_path):
    """Imitation runs (mt_ratio 1, mt_k 2), the curriculum's first stage with evaluation, and checkpoints that the
    HierarchicalRNN optimizer loads back."""
    from open_l2o_b200 import hierarchical_rnn as hr
    from open_l2o_b200 import hrnn_train as ht
    problems = _two_problems()[:1]
    opt = hr.HierarchicalRNN(random_seed=0, **hr.metarun_flags())
    before = opt.theta.detach().clone()
    save = str(tmp_path / "model.ckpt")
    params = [torch.empty(s) for s in SHAPES]
    theta, log = ht.train_optimizer(lambda sh, th: opt.meta_trainer(params, learning_rate=1e-4, random_seed=1),
                                    problems, num_problems=1, num_meta_iterations=2, num_unroll_func=lambda: 0,
                                    num_partial_unroll_itrs_func=lambda: 0, seed=0, if_mt=True, mt_ratio=1.0, mt_k=2,
                                    if_cl=True, evaluation_epochs=1, save_path=save)
    assert log == []                                   # imitation runs are not logged
    assert bool(torch.isfinite(theta).all()) and not torch.equal(theta.detach().cpu(), before.cpu())
    ck = torch.load(save + "-0")
    assert list(ck) == [name for name, _ in hr.THETA_SPEC]
    opt.load_variables(ck)
    assert torch.equal(opt.theta.cpu(), torch.cat([v.reshape(-1) for v in ck.values()]))
