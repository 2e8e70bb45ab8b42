"""Meta-training of the HierarchicalRNN (SURVEY.md 8(f) row 1): BPTT through the unrolled optimizer on the engine
(l2o_hrnn_step_local forward + l2o_hrnn_coord_bwd backward, cross-coordinate pieces as torch autograd) against
torch.autograd through the fp64 CPU oracle's step (SC/optimizer/trainable_optimizer.py:200-470, 586-609)."""
import math

import pytest
import torch

from oracle import hrnn_oracle as orc   # checker only
from tests.helpers import HRNN_CONVNET, HRNN_TILE, hrnn_generic_theta, hrnn_ragged_shapes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _problem(seed=0, dtype=torch.float64, device="cpu"):
    gen = torch.Generator().manual_seed(seed)
    A = torch.randn(40, 30, generator=gen, dtype=torch.float64)
    y = torch.randn(40, 7, generator=gen, dtype=torch.float64)
    C = torch.randn(150, generator=gen, dtype=torch.float64)
    A, y, C = A.to(device=device, dtype=dtype), y.to(device=device, dtype=dtype), C.to(device=device, dtype=dtype)

    def objective(params):
        w, b, v = params
        return ((A @ w + b - y) ** 2).mean() + 0.1 * ((v - C) ** 2).mean() + 0.01 * torch.cos(3.0 * v).mean()
    shapes = [(30, 7), (7,), (150,)]
    init = [torch.randn(s, generator=gen, dtype=torch.float64) * 0.5 for s in shapes]
    return objective, shapes, init


def _oracle_meta_gradient(theta, objective, init, llr, T, carry=None, initial_obj=None, want_carry=False,
                          dtype=torch.float64):
    """Autograd through the oracle's unrolled step in `dtype` (fp64: the reference; fp32: the size of round-off an
    exact fp32 evaluation of the same computation makes).  `objective` must compute in `dtype` too."""
    th = theta.to(dtype).clone().requires_grad_(True)
    P = orc.unpack_theta(th)
    gen = torch.Generator().manual_seed(0)
    if carry is None:
        params = [p.to(dtype) for p in init]
        states, off = [], 0
        for p in params:
            st = orc.initial_state(P, p, gen)
            st["log_learning_rate"] = llr[off:off + p.numel()].to(dtype).reshape(-1, 1)
            off += p.numel()
            states.append(st)
        glob = orc.initial_global_state(P, dtype)
    else:   # truncated BPTT: everything handed over from the previous unroll is a constant
        params = [p.detach() for p in carry[0]]
        states = [{k: v.detach() for k, v in st.items()} for st in carry[1]]
        glob = carry[2].detach()
    objs = []
    for t in range(T):
        ps = [p.detach().requires_grad_(True) for p in params]
        f = objective(ps)
        grads = torch.autograd.grad(f, ps)
        objs.append(objective(params) if t > 0 else f.detach())
        params, states, glob, _ = orc.step(th, params, [g.detach() for g in grads], states, glob)
    allo = torch.stack([o.reshape(()) for o in objs])
    f0 = objs[0].detach() if initial_obj is None else initial_obj
    meta = torch.log(allo / (f0 + 1e-6) + 1e-6).mean()
    g = torch.autograd.grad(meta, th)[0] if meta.requires_grad else torch.zeros_like(th)
    out = (float(meta.detach()), g.detach(), [float(o.detach()) for o in objs],
           torch.cat([p.detach().reshape(-1) for p in params]))
    return out + ((params, states, glob),) if want_carry else out


def _groups():
    out, off = [], 0
    for name, shape in orc.theta_spec():
        n = int(math.prod(shape))
        out.append((name, off, off + n))
        off += n
    return out


def _separable_problem(shapes, seed=1, dtype=torch.float64, device="cpu"):
    """sum over tensors of mean((p - target)^2) + 0.05 mean(cos 2p) (scripts/hrnn_train_check.py): every tensor's
    gradient depends on its own coordinates only, so the oracle's autograd stays cheap at 354 K coordinates."""
    gen = torch.Generator().manual_seed(seed)
    tgt = [torch.randn(s, generator=gen, dtype=torch.float64).to(device=device, dtype=dtype) for s in shapes]

    def objective(params):
        return sum(((p - t) ** 2).mean() + 0.05 * torch.cos(2.0 * p).mean() for p, t in zip(params, tgt))
    init = [torch.randn(s, generator=gen, dtype=torch.float64) * 0.5 for s in shapes]
    return objective, init


def _meta_problem(problem, dtype, device):
    if problem == "toy":
        return _problem(dtype=dtype, device=device)
    if problem == "convnet":
        from open_l2o_b200.scale_problems import ConvNet
        shapes = [tuple(s) for s in ConvNet(*HRNN_CONVNET).param_shapes]
    else:
        shapes = hrnn_ragged_shapes()
    objective, init = _separable_problem(shapes, dtype=dtype, device=device)
    return objective, shapes, init


META_CASES = ([pytest.param("toy", T, "init", False, id=str(T)) for T in (1, 2, 5)]
              + [pytest.param("toy", 5, "generic", False, id="toy-generic-5")]
              + [pytest.param(p, 3, th, clip, id="%s-%s" % (p, "clip" if clip else th))
                 for p in ("convnet", "ragged") for th, clip in (("init", False), ("generic", False), ("generic", True))])


@pytest.mark.parametrize("problem,T,theta_kind,clip", META_CASES)
def test_hrnn_meta_gradient_matches_oracle_autograd(problem, T, theta_kind, clip):
    """The engine's meta-gradient against autograd through the fp64 oracle.  "convnet" (BASELINE #4 shapes, 2,770
    tiles) and "ragged" (> 300 tensors) give coord_bwd_kernel more tiles than CTAs, so its persistent loop walks
    tensors and flushes the per-tensor adjoints on each change; "generic" theta (tests/helpers.hrnn_generic_theta)
    makes every block of theta live and distinct; clip starts a third of the log-lrs at -33 so that the step log-lr is
    clipped, where the gradient passes straight through (HR:674-686)."""
    from open_l2o_b200 import hrnn_train as ht
    obj64, shapes, init = _meta_problem(problem, torch.float64, "cpu")
    obj32, _, _ = _meta_problem(problem, torch.float32, DEV)
    if problem != "toy":   # every backward CTA must walk >= 2 tiles (the grid is min(tiles, 2 x SMs))
        tiles = sum(math.ceil(math.prod(s) / HRNN_TILE) for s in shapes)
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert tiles >= 4 * sms, (tiles, sms)
    theta = orc.init_theta(seed=3) if theta_kind == "init" else hrnn_generic_theta(5)
    n = sum(int(math.prod(s)) for s in shapes)
    llr = (torch.rand(n, generator=torch.Generator().manual_seed(5), dtype=torch.float64) * 3.0 - 6.0).float()
    if clip:
        llr[::3] = -33.0
    meta_ref, g_ref, objs_ref, x_ref = _oracle_meta_gradient(theta, obj64, init, llr, T)
    tr = ht.MetaTrainer(shapes, theta=theta, device=DEV)
    meta, g, objs, final = tr.meta_gradient(obj32, [p.float().to(DEV) for p in init], T, log_learning_rate=llr)
    torch.cuda.synchronize()
    assert abs(float(meta) - meta_ref) <= 1e-5 * max(1.0, abs(meta_ref)), (float(meta), meta_ref)
    for a, b in zip(objs, objs_ref):
        assert abs(a - b) <= 2e-5 * max(1.0, abs(b)), (objs, objs_ref)
    assert float((final.x.detach().cpu().double() - x_ref).abs().max()) <= 2e-5 * float(x_ref.abs().max())
    g = g.detach().cpu().double()
    scale = float(g_ref.abs().max())
    if T == 1:      # a one-step unroll has a constant objective: the meta-gradient vanishes identically
        assert scale == 0.0 and float(g.abs().max()) == 0.0
        return
    assert scale > 0
    worst = []
    for name, lo, hi in _groups():
        e = float((g[lo:hi] - g_ref[lo:hi]).abs().max())
        worst.append((e / scale, name, float(g_ref[lo:hi].abs().max()) / scale))
    worst.sort(reverse=True)
    assert worst[0][0] <= 1e-5, worst[:6]     # measured 1e-7 .. 3e-7 (scripts/hrnn_train_check.py)
    # every block of theta that the reference gradient reaches must be reached here too (and vice versa)
    for name, lo, hi in _groups():
        ref_nz, got_nz = bool((g_ref[lo:hi] != 0).any()), bool((g[lo:hi] != 0).any())
        assert ref_nz == got_nz, (name, ref_nz, got_nz)
    # each block against its own largest entry: 1e-5, or 3x the distance of an exact fp32 evaluation (the fp32 oracle)
    # from fp64 on that block where round-off alone is larger
    obj32c, _, _ = _meta_problem(problem, torch.float32, "cpu")
    g32 = _oracle_meta_gradient(theta, obj32c, init, llr, T, dtype=torch.float32)[1].double()
    bad = []
    for name, lo, hi in _groups():
        own = float(g_ref[lo:hi].abs().max())
        if own == 0.0:
            continue
        e = float((g[lo:hi] - g_ref[lo:hi]).abs().max()) / own
        tol = max(1e-5, 3.0 * float((g32[lo:hi] - g_ref[lo:hi]).abs().max()) / own)
        if e > tol:
            bad.append((name, e, tol, own / scale))
    assert not bad, bad


def test_hrnn_meta_training_rmsprop_step_and_descent():
    """RMSProp with make_finite + clipping (SC/metaopt.py:255-289): the update rule on a known gradient, then a few
    meta-steps on the toy problem move theta along the negative clipped gradient."""
    from open_l2o_b200 import hrnn_train as ht
    obj32, shapes, init = _problem(dtype=torch.float32, device=DEV)
    tr = ht.MetaTrainer(shapes, theta=orc.init_theta(seed=3), device=DEV, learning_rate=1e-3, gradient_clip=0.5,
                        random_seed=7)
    th0 = tr.theta.detach().clone()
    g = torch.zeros_like(th0)
    g[0], g[1], g[2], g[3] = 2.0, float("nan"), -0.25, float("inf")
    used = tr.apply_meta_gradient(g)
    assert used[0] == 0.5 and used[1] == 0.0 and used[2] == -0.25 and used[3] == 0.0
    rms = 0.9 * 1.0 + 0.1 * used ** 2                       # accumulator starts at one (tf.train.RMSPropOptimizer)
    want = th0 - 1e-3 * used / torch.sqrt(rms + 1e-20)
    assert float((tr.theta.detach() - want).abs().max()) <= 1e-7
    p0 = [p.float().to(DEV) for p in init]
    metas = []
    for _ in range(3):
        meta, objs, _ = tr.train_step(obj32, p0, 4)
        assert math.isfinite(meta) and all(math.isfinite(o) for o in objs)
        metas.append(meta)
    assert tr.global_step == 4


def test_hrnn_truncated_bptt_second_unroll_matches_oracle():
    """Partial unrolls (SC/metaopt.py:458-613): the second unroll starts from the DETACHED state the first one left and is
    normalised by the first unroll's initial objective; its meta-gradient against the oracle run the same way."""
    from open_l2o_b200 import hrnn_train as ht
    obj64, shapes, init = _problem(dtype=torch.float64, device="cpu")
    obj32, _, _ = _problem(dtype=torch.float32, device=DEV)
    theta = orc.init_theta(seed=11)
    n = sum(int(math.prod(s)) for s in shapes)
    llr = (torch.rand(n, generator=torch.Generator().manual_seed(6), dtype=torch.float64) * 3.0 - 6.0).float()
    m1, g1, o1, x1, carry = _oracle_meta_gradient(theta, obj64, init, llr, 3, want_carry=True)
    m2, g2, o2, x2 = _oracle_meta_gradient(theta, obj64, init, llr, 4, carry=carry, initial_obj=torch.tensor(o1[0]))
    tr = ht.MetaTrainer(shapes, theta=theta, device=DEV)
    p0 = [p.float().to(DEV) for p in init]
    meta1, ga, objs_a, fin = tr.meta_gradient(obj32, p0, 3, log_learning_rate=llr)
    meta2, gb, objs_b, fin2 = tr.meta_gradient(obj32, p0, 4, state=tr.detach_state(fin),
                                               initial_obj=torch.tensor(objs_a[0], device=DEV))
    torch.cuda.synchronize()
    assert abs(float(meta2) - m2) <= 1e-5 * max(1.0, abs(m2)), (float(meta2), m2)
    for a, b in zip(objs_b, o2):
        assert abs(a - b) <= 2e-5 * max(1.0, abs(b))
    gb = gb.detach().cpu().double()
    scale = float(g2.abs().max())
    assert scale > 0 and float((gb - g2).abs().max()) <= 1e-5 * scale, float((gb - g2).abs().max()) / scale
    # the driver form: two unrolls with a meta-step after each
    tr2 = ht.MetaTrainer(shapes, theta=theta, device=DEV, learning_rate=1e-4)
    metas, values, out = tr2.train_problem(obj32, p0, num_unrolls=2, unroll_len=3, log_learning_rate=llr)
    assert len(metas) == 2 and len(values) == 6 and tr2.global_step == 2
    assert abs(metas[0] - m1) <= 1e-5 * max(1.0, abs(m1))


def test_hierarchical_rnn_meta_trainer_round_trip():
    """HierarchicalRNN.meta_trainer / adopt: train the optimizer's own weights, then step with them."""
    from open_l2o_b200 import hierarchical_rnn as hr
    obj32, shapes, init = _problem(dtype=torch.float32, device=DEV)
    params = [p.float().to(DEV).requires_grad_(True) for p in init]
    opt = hr.HierarchicalRNN(random_seed=0, **hr.metarun_flags())
    tr = opt.meta_trainer(params, learning_rate=1e-4, random_seed=1)
    before = opt.theta.detach().clone()
    tr.train_problem(obj32, [p.detach() for p in params], num_unrolls=2, unroll_len=3)
    opt.adopt(tr)
    assert not torch.equal(opt.theta, before) and torch.equal(opt.theta, tr.theta.detach())
    losses = opt.minimize(lambda *ps: obj32(list(ps)), params, 3)
    assert all(math.isfinite(float(v)) for v in losses)


def test_train_optimizer_loop_on_the_engine():
    """hrnn_train.train_optimizer with real trainers: two problem shapes, unequal partial-unroll lengths, theta and the
    RMSProp accumulator handed on between problems."""
    from open_l2o_b200 import hrnn_train as ht
    obj_a, shapes_a, init_a = _problem(dtype=torch.float32, device=DEV)
    tgt = torch.randn(64, device=DEV)
    problems = [(obj_a, lambda: [p.float().to(DEV) for p in init_a]),
                (lambda ps: ((ps[0] - tgt) ** 2).mean(), lambda: [torch.zeros(64, device=DEV)])]
    lens = iter([2, 3, 2, 3, 2, 3, 2, 3])
    theta0 = orc.init_theta(seed=3)
    theta, log = ht.train_optimizer(lambda sh, th: ht.MetaTrainer(sh, theta=theta0 if th is None else th, device=DEV,
                                                                  learning_rate=1e-4, random_seed=0),
                                    problems, num_problems=2, num_meta_iterations=2, num_unroll_func=lambda: 2,
                                    num_partial_unroll_itrs_func=lambda: next(lens), select_random_problems=False)
    assert [k for k, _ in log] == [0, 0, 1, 1] and all(len(m) == 2 and all(math.isfinite(v) for v in m) for _, m in log)
    assert torch.isfinite(theta).all() and not torch.equal(theta.detach().cpu(), theta0)
