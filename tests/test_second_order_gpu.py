"""GPU: second-order meta-gradients (``use_second_derivatives``).  The adjoint of the optimizee gradient g that
l2o_hrnn_coord_bwd / l2o_crnn_bwd write into d_g, against fp64 autograd through the oracles; the existing outputs with
and without d_g; both trainers' second-order meta-gradients against the oracles'; train_optimizer end to end."""
import ctypes
import math

import pytest
import torch

from oracle import crnn_oracle as CR
from oracle import hrnn_oracle as H
from tests.helpers import HRNN_CONVNET, REL_TOL, hrnn_generic_theta, hrnn_ragged_shapes, rel_err
from tests.test_crnn_gpu import crnn_generic_theta
from tests.test_second_order_cpu import crnn_oracle_meta, curved_problem, hrnn_oracle_meta

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HRNN_KEYS = ["parameter", "scl_decay", "inp_decay", "log_learning_rate"] + ["grad_accum%d" % s for s in range(1, 5)] \
    + ["ms%d" % s for s in range(1, 5)]


def _shapes(kind):
    if kind == "small":
        return [(33, 7), (5,), (300,)]
    if kind == "convnet":
        from open_l2o_b200.scale_problems import ConvNet
        return [tuple(s) for s in ConvNet(*HRNN_CONVNET).param_shapes]
    return hrnn_ragged_shapes()   # 301 tensors


def _gradients(shapes, gen, scale=0.3, special=False):
    """Random gradients; with `special`, every 7th tensor all zero and every 7th (offset 1) at 1e-6."""
    out = []
    for j, s in enumerate(shapes):
        g = torch.randn(s, generator=gen, dtype=torch.float64) * scale
        if special and j % 7 == 0:
            g = torch.zeros(s, dtype=torch.float64)
        elif special and j % 7 == 1:
            g = g * (1e-6 / scale)
        out.append(g)
    return out


def _hrnn_planes(states):
    """Oracle per-tensor states -> the engine's [21, N] planes."""
    return torch.cat([torch.cat([st[k].reshape(st[k].shape[0], -1) for k in HRNN_KEYS], 1) for st in states], 0).t()


def _per_tensor(v, shapes):
    return torch.split(v.reshape(-1), [int(math.prod(s)) for s in shapes])


# ---------------------------------------------------------------------------------------------------------------------
# 3. the kernels' d g against the oracle, one step

HRNN_KERNEL_CASES = [("small", "init", False), ("small", "generic", False), ("convnet", "generic", False),
                     ("ragged", "generic", False), ("small", "generic", True)]


@pytest.mark.parametrize("kind,theta_kind,clip", HRNN_KERNEL_CASES)
def test_hrnn_coord_bwd_d_g_matches_oracle(kind, theta_kind, clip):
    """One HierarchicalRNN step from a state two oracle steps in (or, with `clip`, with a third of the log-lrs at -33),
    fed gradients G; every output of the step (x, the 21 planes, the per-tensor and global RNN states) gets a random
    adjoint, so the backward sees generic adjoints of the planes, the raw update and the per-tensor sums.  d L / d G
    through the trainer's step (l2o_hrnn_coord_bwd's d_g plus the host-side per-tensor pieces) against fp64 autograd
    through the oracle, per tensor: 3e-5, or 3x the fp32 oracle's distance where that is larger."""
    from open_l2o_b200 import hrnn_train as ht
    shapes = _shapes(kind)
    gen = torch.Generator().manual_seed(21)
    theta = H.init_theta(3) if theta_kind == "init" else hrnn_generic_theta(5)
    n = sum(int(math.prod(s)) for s in shapes)
    llr = torch.rand(n, generator=gen, dtype=torch.float64) * 3.0 - 6.0
    if clip:
        llr[::3] = -33.0
    # a generic state: two fp64 oracle steps, then rounded to fp32 so that both sides start from the same numbers
    P64 = H.unpack_theta(theta.double())
    params = [torch.randn(s, generator=gen, dtype=torch.float64) * 0.5 for s in shapes]
    states, off = [], 0
    for p in params:
        st = H.initial_state(P64, p, torch.Generator().manual_seed(0), )
        st["log_learning_rate"] = llr[off:off + p.numel()].reshape(-1, 1)
        off += p.numel()
        states.append(st)
    glob = H.initial_global_state(P64, torch.float64)
    for _ in range(2):
        params, states, glob, _ = H.step(theta.double(), params, _gradients(shapes, gen), states, glob)
    params = [p.float().double() for p in params]
    states = [{k: v.detach().float().double() for k, v in st.items()} for st in states]
    glob = glob.detach().float().double()
    G = _gradients(shapes, gen, special=(kind == "ragged"))
    R_x = [torch.randn(s, generator=gen, dtype=torch.float64) for s in shapes]
    R_planes = torch.randn(21, n, generator=gen, dtype=torch.float64)
    R_layer = torch.randn(len(shapes), 20, generator=gen, dtype=torch.float64)
    R_glob = torch.randn(1, 20, generator=gen, dtype=torch.float64)

    def oracle(dtype):
        th = theta.to(dtype)
        Gl = [g.to(dtype).requires_grad_(True) for g in G]
        ps, sts, gl, _ = H.step(th, [p.to(dtype) for p in params], Gl,
                                [{k: v.to(dtype) for k, v in st.items()} for st in states], glob.to(dtype))
        L = sum((r.to(dtype) * p).sum() for r, p in zip(R_x, ps)) + (R_planes.to(dtype) * _hrnn_planes(sts)).sum() \
            + (R_layer.to(dtype) * torch.cat([st["layer"] for st in sts], 0)).sum() + (R_glob.to(dtype) * gl).sum()
        return torch.cat([d.reshape(-1) for d in torch.autograd.grad(L, Gl)])
    want64, want32 = oracle(torch.float64), oracle(torch.float32)

    tr = ht.MetaTrainer(shapes, theta=theta, device=DEV, use_second_derivatives=True)
    Gd = torch.cat([g.reshape(-1) for g in G]).float().to(DEV).requires_grad_(True)
    # a linear objective <G, x>: its gradient is G itself, kept in the graph (x requires grad, second derivatives on)
    lin = lambda ps: sum((gj * p).sum() for gj, p in zip(tr._split(Gd), ps))
    x0 = torch.cat([p.reshape(-1) for p in params]).float().to(DEV).requires_grad_(True)
    zero_flag = torch.stack([torch.stack([(st["ms%d" % s] == 0).all() for s in range(1, 5)]) for st in states])
    st0 = ht.OptimizerState(_hrnn_planes(states).float().contiguous().to(DEV), torch.cat([st["layer"] for st in states], 0)
                            .float().to(DEV), glob.float().to(DEV), zero_flag.to(torch.int32).to(DEV), x0)
    _, _, fin = tr.unroll(lin, st0, 1)
    dev = lambda t: t.float().to(DEV)
    L = (dev(torch.cat([r.reshape(-1) for r in R_x])) * fin.x).sum() + (dev(R_planes) * fin.planes).sum() \
        + (dev(R_layer) * fin.layer).sum() + (dev(R_glob) * fin.global_state).sum()
    (got,) = torch.autograd.grad(L, Gd)
    torch.cuda.synchronize()
    bad = []
    for j, (e, w64, w32) in enumerate(zip(_per_tensor(got.cpu(), shapes), _per_tensor(want64, shapes),
                                          _per_tensor(want32, shapes))):
        err, own = rel_err(e, w64), rel_err(w32, w64)
        if not err <= max(3 * REL_TOL, 3 * own):
            bad.append((j, shapes[j], err, own))
    assert not bad, bad[:10]


CRNN_KERNEL_CASES = [("small", "init"), ("small", "generic"), ("convnet", "generic"), ("ragged", "generic")]


@pytest.mark.parametrize("kind,theta_kind", CRNN_KERNEL_CASES)
def test_crnn_bwd_d_g_matches_oracle(kind, theta_kind):
    """One CoordinatewiseRNN step (crnn_train._Step: l2o_crnn_step, l2o_crnn_bwd) from a state two oracle steps in, with
    random adjoints of the 103 new planes and of the update: d L / d g against fp64 autograd through the oracle, per
    tensor within 1e-5, or 3x the fp32 oracle's distance where that is larger."""
    from open_l2o_b200.crnn_train import _Step
    shapes = _shapes(kind)
    gen = torch.Generator().manual_seed(22)
    theta = CR.init_theta(3) if theta_kind == "init" else crnn_generic_theta(5)
    n = sum(int(math.prod(s)) for s in shapes)
    P64 = CR.unpack_theta(theta.double())
    lr0 = torch.exp(torch.rand(n, generator=gen, dtype=torch.float64) * 3.0 - 6.0)
    params = [torch.randn(s, generator=gen, dtype=torch.float64) * 0.5 for s in shapes]
    states, off = [], 0
    for p in params:
        st = CR.initial_state(P64, p.numel(), gen)
        st["learning_rate"] = lr0[off:off + p.numel()].reshape(-1, 1)
        off += p.numel()
        states.append(st)
    for _ in range(2):
        params, states, _ = CR.step(theta.double(), params, _gradients(shapes, gen), states)
    planes = CR.state_to_planes(states).float()
    G = _gradients(shapes, gen, special=(kind == "ragged"))
    R_planes = torch.randn(103, n, generator=gen, dtype=torch.float64)
    R_upd = torch.randn(n, generator=gen, dtype=torch.float64)

    def oracle(dtype):
        Gl = [g.to(dtype).requires_grad_(True) for g in G]
        sts = CR.planes_to_states(planes.to(dtype), [int(math.prod(s)) for s in shapes])
        _, new, upd = CR.step(theta.to(dtype), [p.to(dtype) for p in params], Gl, sts)
        L = (R_planes.to(dtype) * CR.state_to_planes(new)).sum() \
            + (R_upd.to(dtype) * torch.cat([u.reshape(-1) for u in upd])).sum()
        return torch.cat([d.reshape(-1) for d in torch.autograd.grad(L, Gl)])
    want64, want32 = oracle(torch.float64), oracle(torch.float32)
    Gd = torch.cat([g.reshape(-1) for g in G]).float().to(DEV).requires_grad_(True)
    new, upd = _Step.apply(theta.to(DEV), planes.to(DEV), Gd)
    L = (R_planes.float().to(DEV) * new).sum() + (R_upd.float().to(DEV) * upd).sum()
    (got,) = torch.autograd.grad(L, Gd)
    torch.cuda.synchronize()
    bad = []
    for j, (e, w64, w32) in enumerate(zip(_per_tensor(got.cpu(), shapes), _per_tensor(want64, shapes),
                                          _per_tensor(want32, shapes))):
        err, own = rel_err(e, w64), rel_err(w32, w64)
        if not err <= max(REL_TOL, 3 * own):
            bad.append((j, shapes[j], err, own))
    assert not bad, bad[:10]


# ---------------------------------------------------------------------------------------------------------------------
# 4. a null d_g leaves every existing output as it was

def test_hrnn_coord_bwd_outputs_do_not_depend_on_d_g():
    """The same l2o_hrnn_coord_bwd call with and without d_g (ConvNet shapes, generic weights and inputs): the old-plane
    adjoints bit-identical; d theta, d bias0 and d mean_log_lr up to the order of the fp64 atomics."""
    from open_l2o_b200 import hrnn_train as ht
    shapes = _shapes("convnet")
    gen = torch.Generator().manual_seed(23)
    eng = ht._Engine([int(math.prod(s)) for s in shapes], torch.device(DEV))
    N, nt = eng.N, eng.nt
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=gen) * scale).to(DEV)
    theta = hrnn_generic_theta(5).to(DEV)
    planes = rnd(21, N, scale=0.5)
    planes[10:12] = torch.rand(2, N, generator=gen).to(DEV)        # decays in (0, 1)
    planes[17:21] = planes[17:21].abs() + 1e-3                      # mean squares > 0
    args = (theta, planes, rnd(nt, 32, scale=0.3), planes[12].mean().reshape(1), rnd(N, scale=0.1),
            torch.zeros(nt, 4, dtype=torch.int32, device=DEV), rnd(21, N), rnd(N), rnd(nt, 24))
    a = eng.coord_backward(*args, want_dg=False)
    b = eng.coord_backward(*args, want_dg=True)
    torch.cuda.synchronize()
    assert a[4] is None and b[4] is not None and bool(torch.isfinite(b[4]).all())
    assert torch.equal(a[1], b[1])
    for k in (0, 2, 3):
        assert rel_err(b[k], a[k]) <= 1e-6, k


def _crnn_bwd(theta, planes, g, d_new, d_upd, d_g):
    from open_l2o_b200 import _lib
    from open_l2o_b200.engine import _ptr as _p
    d_old = torch.empty_like(planes)
    d_theta = torch.zeros(theta.numel(), dtype=torch.float64, device=DEV)
    a = _lib.CrnnBwdArgs()
    a.n = int(g.numel())
    a.theta, a.g, a.state_old, a.d_state_new, a.d_update, a.d_state_old = map(_p, (theta, g, planes, d_new, d_upd, d_old))
    a.d_theta, a.d_g = d_theta.data_ptr(), _p(d_g)
    _lib.check(_lib.lib().l2o_crnn_bwd(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "l2o_crnn_bwd")
    return d_old, d_theta


def test_crnn_bwd_outputs_do_not_depend_on_d_g():
    gen = torch.Generator().manual_seed(24)
    n = 354218
    theta = crnn_generic_theta(5).to(DEV)
    planes = (torch.randn(103, n, generator=gen) * 0.5).to(DEV)
    planes[100] = planes[100].abs() + 1e-3
    planes[101] = torch.rand(n, generator=gen).to(DEV)
    planes[102] = planes[102].abs() * 1e-2
    g, d_new, d_upd = ((torch.randn(*s, generator=gen)).to(DEV) for s in ((n,), (103, n), (n,)))
    d_g = torch.empty(n, device=DEV)
    a_old, a_theta = _crnn_bwd(theta, planes, g, d_new, d_upd, None)
    b_old, b_theta = _crnn_bwd(theta, planes, g, d_new, d_upd, d_g)
    torch.cuda.synchronize()
    assert torch.equal(a_old, b_old) and bool(torch.isfinite(d_g).all())
    assert rel_err(b_theta, a_theta) <= 1e-6   # the per-CTA images sum the readout terms with shared-memory atomics


def test_hrnn_coord_bwd_rejects_misaligned_or_overlapping_d_g():
    from open_l2o_b200 import _lib, hrnn_train as ht
    eng = ht._Engine([37, 200], torch.device(DEV))
    N, nt = eng.N, eng.nt
    bufs = dict(theta=torch.zeros(H.theta_count(), device=DEV), state_old=torch.zeros(21, N, device=DEV),
                g=torch.zeros(N, device=DEV), bias0=torch.zeros(nt, 32, device=DEV),
                zero_flag=torch.zeros(nt, 4, dtype=torch.int32, device=DEV), mean_log_lr=torch.zeros(1, device=DEV),
                d_state_new=torch.zeros(21, N, device=DEV), d_upd=torch.zeros(N, device=DEV),
                d_sums=torch.zeros(nt, 24, device=DEV), d_state_old=torch.zeros(21, N, device=DEV),
                d_theta=torch.zeros(H.theta_count(), dtype=torch.float64, device=DEV),
                d_bias0=torch.zeros(nt, 32, dtype=torch.float64, device=DEV),
                d_mean_log_lr=torch.zeros(1, dtype=torch.float64, device=DEV))
    ptrs = {k: v.data_ptr() for k, v in bufs.items()}
    own = torch.zeros(N + 4, device=DEV)
    L = _lib.lib()
    call = lambda d_g: L.l2o_hrnn_coord_bwd(eng._h, ctypes.byref(_lib.HrnnBwdArgs(d_g=d_g, **ptrs)), None)
    assert call(own.data_ptr() + 2) == _lib.L2O_E_INVALID
    for k, t in bufs.items():
        nbytes = t.numel() * t.element_size()
        for d_g in (ptrs[k], ptrs[k] + nbytes - 4):
            assert call(d_g) == _lib.L2O_E_INVALID, k
    assert call(own.data_ptr()) == _lib.L2O_OK
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# 5. the trainers' second-order meta-gradients against the oracles'

def _convnet_problem(dtype, device):
    from open_l2o_b200.scale_problems import ConvNet
    net = ConvNet(*HRNN_CONVNET)
    gen = torch.Generator().manual_seed(31)
    data = torch.rand(2, 32, 32, 3, generator=gen, dtype=torch.float64).to(device=device, dtype=dtype)
    labels = torch.eye(10, dtype=torch.float64)[torch.tensor([3, 7])].to(device=device, dtype=dtype)
    shapes = [tuple(s) for s in net.param_shapes]
    # He-scaled weights and positive biases: the ReLU on the logits (problem_generator.py:696) leaves every class
    # alive, so the objective is not flat (a flat objective has a zero meta-gradient)
    init = [torch.randn(s, generator=gen, dtype=torch.float64) * math.sqrt(2.0 / math.prod(s[:-1])) if len(s) > 1
            else 0.1 + 0.05 * torch.rand(s, generator=gen, dtype=torch.float64) for s in shapes]
    return (lambda ps: net.objective(ps, data, labels)), shapes, init


TRAINER_CASES = [("hrnn", "curved"), ("hrnn", "convnet"), ("crnn", "curved")]


def _trainer_case(which, problem):
    shapes = [(40, 5), (5,), (150,)]
    if problem == "convnet":
        obj64, shapes, init = _convnet_problem(torch.float64, "cpu")
        obj32c, _, _ = _convnet_problem(torch.float32, "cpu")
        obj32, _, _ = _convnet_problem(torch.float32, DEV)
    else:
        obj64, init = curved_problem(shapes, seed=8)
        obj32c, _ = curved_problem(shapes, seed=8, dtype=torch.float32)
        obj32, _ = curved_problem(shapes, seed=8, dtype=torch.float32, device=DEV)
    n = sum(p.numel() for p in init)
    u = torch.rand(n, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    if which == "hrnn":
        theta = hrnn_generic_theta(5)
        # log learning rates, well inside the +-33 clip.  On the ConvNet they must be tiny: every coordinate moves by
        # about lr, and a coherent move of lr over the 32,768 rows of the dense layer shifts the ReLU'd logits by
        # ~10^4 lr, which at e^-10 already kills every class (a flat objective, a zero meta-gradient)
        lr = (u * 1.5 - (12.0 if problem == "convnet" else 1.0)).float()
        oracle = hrnn_oracle_meta
    else:
        theta = crnn_generic_theta(7)
        lr = torch.exp(u + 3.0).float()                   # the CoordinatewiseRNN's first updates are small
        oracle = crnn_oracle_meta
    return theta, shapes, init, lr, oracle, obj64, obj32c, obj32


def _blocks(which):
    spec = H.theta_spec() if which == "hrnn" else CR.theta_spec()
    out, off = [], 0
    for name, shape in spec:
        k = int(math.prod(shape))
        out.append((name, off, off + k))
        off += k
    return out


@pytest.mark.parametrize("which,problem", TRAINER_CASES)
def test_second_order_meta_gradient_matches_oracle(which, problem):
    """T = 3 from a fresh state, then a truncated second unroll of 3 steps from the detached state.  Per theta block:
    within 1e-5 of the block's largest entry, or 3x the fp32 oracle's distance from fp64 where that is larger, or 3x
    the first-order trainer's distance from the first-order fp64 oracle (on the ConvNet the device's convolutions sum in
    another order than the CPU's, and blocks fed by acc - g, which cancels when x barely moves, inherit that; the
    second-order path must add no error of its own).  The first-order gradient must be far outside the tolerance, or
    dropping the term would pass."""
    from open_l2o_b200 import crnn_train as ct, hrnn_train as ht
    theta, shapes, init, lr, oracle, obj64, obj32c, obj32 = _trainer_case(which, problem)
    cls = ht.MetaTrainer if which == "hrnn" else ct.MetaTrainer
    p0 = [p.float().to(DEV) for p in init]
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False   # the ConvNet's convolutions in exact fp32, as the fp32 oracle's
    try:
        runs = []
        for second in (True, False):
            tr = cls(shapes, theta=theta, device=DEV, use_second_derivatives=second)
            m_a, g_a, objs_a, fin = tr.meta_gradient(obj32, p0, 3, lr)
            m_b, g_b, _, _ = tr.meta_gradient(obj32, p0, 3, state=tr.detach_state(fin),
                                              initial_obj=torch.tensor(objs_a[0], device=DEV))
            runs.append((m_a, g_a.detach().double().cpu(), m_b, g_b.detach().double().cpu()))
        torch.cuda.synchronize()
    finally:
        torch.backends.cudnn.allow_tf32 = tf32
    (meta1, g1, meta2, g2), (_, e1, _, e2) = runs
    m1, r1, c64 = oracle(theta, obj64, init, lr, 3, True)
    _, r1_32, c32 = oracle(theta, obj32c, init, lr, 3, True, dtype=torch.float32)
    _, f1, _ = oracle(theta, obj64, init, lr, 3, False)
    m2, r2, _ = oracle(theta, obj64, init, lr, 3, True, carry=c64, initial_obj=c64[3])
    _, r2_32, _ = oracle(theta, obj32c, init, lr, 3, True, dtype=torch.float32, carry=c32, initial_obj=c32[3])
    _, f2, _ = oracle(theta, obj64, init, lr, 3, False, carry=c64, initial_obj=c64[3])
    assert abs(float(meta1) - float(m1)) <= 1e-5 * max(1.0, abs(float(m1)))
    assert abs(float(meta2) - float(m2)) <= 1e-5 * max(1.0, abs(float(m2)))
    for tag, eng, ref, r32, first, eng1 in (("unroll1", g1, r1, r1_32, f1, e1), ("unroll2", g2, r2, r2_32, f2, e2)):
        r32 = r32.double()
        bad, sep = [], []
        for name, lo, hi in _blocks(which):
            own = float(ref[lo:hi].abs().max())
            if own == 0.0:
                continue
            err = float((eng[lo:hi] - ref[lo:hi]).abs().max()) / own
            tol = max(1e-5, 3.0 * float((r32[lo:hi] - ref[lo:hi]).abs().max()) / own,
                      3.0 * float((eng1[lo:hi] - first[lo:hi]).abs().max()) / own)
            if err > tol:
                bad.append((name, err, tol))
            sep.append((float((first[lo:hi] - ref[lo:hi]).abs().max()) / own / tol, name))
        assert not bad, (tag, bad)
        sep.sort(reverse=True)
        # the second-order term is at least 10x the tolerance on a third of the checked blocks or more (with T = 3 some
        # blocks cannot reach it: it needs theta -> x_t -> g_t -> x_t+1 inside the unroll)
        assert sum(s >= 10.0 for s, _ in sep) * 3 >= len(sep), (tag, sep)


# ---------------------------------------------------------------------------------------------------------------------
# 6. end to end

@pytest.mark.parametrize("which", ["hrnn", "crnn"])
def test_train_optimizer_with_second_derivatives(which):
    from open_l2o_b200 import crnn_train as ct, hrnn_train as ht
    mod = ht if which == "hrnn" else ct
    gen = torch.Generator().manual_seed(12)
    tgt = torch.randn(20, 10, generator=gen).to(DEV)
    init = torch.randn(20, 10, generator=gen).to(DEV)
    problems = [(lambda ps: ((ps[0] - tgt) ** 2).mean() + 0.3 * torch.cos(3.0 * ps[0]).mean(), lambda: [init.clone()])]
    theta0 = hrnn_generic_theta(5) if which == "hrnn" else crnn_generic_theta(7)
    # initial learning rates large enough for the optimizee's curvature to show in the meta-gradient
    lr_range = (math.exp(-1.0), math.exp(0.5)) if which == "hrnn" else (math.exp(3.0), math.exp(4.0))
    runs = []
    for second in (False, True):
        trainers = []

        def make(shapes, th):
            tr = mod.MetaTrainer(shapes, theta=theta0, device=DEV, learning_rate=1e-2, random_seed=0,
                                 init_lr_range=lr_range, use_second_derivatives=second)
            trainers.append(tr)
            return tr
        theta, log = mod.train_optimizer(make, problems, num_problems=1, num_meta_iterations=2,
                                         num_unroll_func=lambda: 2, num_partial_unroll_itrs_func=lambda: 5,
                                         select_random_problems=False)
        assert trainers[0].use_second_derivatives is second
        assert len(log) == 2 and all(len(m) == 2 and all(math.isfinite(v) for v in m) for _, m in log)
        assert bool(torch.isfinite(theta).all()) and not torch.equal(theta.detach().cpu(), theta0)
        runs.append(theta.detach().cpu().clone())
    assert not torch.equal(runs[0], runs[1])
    assert mod.MetaTrainer([(3,)], device=DEV).use_second_derivatives is False
