"""GPU: L2O-Scale's baselines.  The step kernels (l2o_tadam_step, l2o_lrsgd_step) and the trainers' meta-gradients
(l2o_tadam_bwd, l2o_lrsgd_bwd) against the oracle (oracle/baselines_oracle.py), graph replay against eager execution,
d_g's independence from the other outputs, and train_optimizer end to end."""
import ctypes
import math

import pytest
import torch

from oracle import baselines_oracle as B
from tests.helpers import HRNN_CONVNET, REL_TOL, hrnn_ragged_shapes, rel_err
from tests.test_baselines_cpu import baseline_oracle_meta, tadam_theta
from tests.test_second_order_cpu import curved_problem

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SPECIAL = [0.0, 1.0, -1.0, 1e-30, -1e-30, 1e30, -1e30, 0.5]   # g values of the extra tensor of every step case
TIGHT = 1e-6   # kernel against the fp32 oracle, TrainableAdam step (same operations, same rounding)


def _shapes(kind):
    if kind == "small":
        return [(33, 7), (5,), (300,)]
    if kind == "convnet":
        from open_l2o_b200.scale_problems import ConvNet
        return [tuple(s) for s in ConvNet(*HRNN_CONVNET).param_shapes]
    if kind == "ragged":
        return hrnn_ragged_shapes()   # 301 tensors
    return [(1,)]


def _check(tag, got, w32, w64, tol32=REL_TOL):
    """NaN where the fp32 oracle has NaN; elsewhere within `tol32` max-norm relative of the fp32 oracle, and of the fp64
    oracle within 1e-5 or 3x the fp32 oracle's own distance from it."""
    got, w32, w64 = (t.detach().double().cpu().reshape(-1) for t in (got, w32, w64))
    nan = torch.isnan(w32)
    assert torch.equal(torch.isnan(got), nan), tag
    ok = ~nan
    if not bool(ok.any()):
        return
    e32, own = rel_err(got[ok], w32[ok]), rel_err(w32[ok], w64[ok])
    assert e32 <= tol32, (tag, e32)
    assert rel_err(got[ok], w64[ok]) <= max(REL_TOL, 3 * own), (tag, rel_err(got[ok], w64[ok]), own)


STEP_CASES = [("small", 0.9), ("convnet", 0.9), ("ragged", 0.9), ("lone", 0.9), ("small", 0.999), ("convnet", 0.999)]


@pytest.mark.parametrize("kind,b1", STEP_CASES)
def test_tadam_steps_match_oracle(kind, b1):
    """Three steps (t = 1..3) through TrainableAdam.apply_gradients and the training form of the kernel, against the
    oracle fed the same gradients: x, update and the m | t | v planes per tensor.  An extra tensor carries
    g in {0, +-1, +-1e-30, +-1e30}: NaN from the first step where g = +-1, as in the oracle.  The kernel rounds every
    operation as the fp32 oracle does, so it must agree with it to 1e-6 (TIGHT), not just 1e-5: terms that move the
    update by less than 1e-5, such as the 1e-10 added to eps (1e-10 / (1e-5 + eps) relative), are then pinned."""
    from open_l2o_b200.trainable_baselines import TrainableAdam, tadam_step_launch
    shapes = _shapes(kind) + [(len(SPECIAL),)]
    if kind == "convnet":
        assert sum(math.prod(s) for s in shapes[:-1]) == 354218
    gen = torch.Generator().manual_seed(5)
    opt = TrainableAdam(learning_rate=1e-3, beta1=b1, beta2=0.99, epsilon=1e-7)
    theta = opt.theta.detach().cpu().clone()
    params = [torch.randn(s, generator=gen) for s in shapes]
    gvars = [p.clone().to(DEV) for p in params]
    grads_all = []
    for _ in range(3):
        gs = [torch.randn(s, generator=gen) * 10.0 ** float(torch.empty(()).uniform_(-3, 1, generator=gen))
              for s in shapes[:-1]]
        grads_all.append(gs + [torch.tensor(SPECIAL)])
    st32 = [B.tadam_initial_state(p.numel(), torch.float32) for p in params]
    p64, st64 = [p.double() for p in params], [B.tadam_initial_state(p.numel()) for p in params]
    for it, grads in enumerate(grads_all):
        gflat = torch.cat([g.reshape(-1) for g in grads]).to(DEV)
        upd = None
        if it > 0:   # (the first apply_gradients creates the slots) the training form: update written, x untouched
            upd = torch.empty_like(gflat)
            tadam_step_launch(opt.theta, gflat, opt.state, torch.empty_like(opt.state), update=upd)
        opt.apply_gradients(zip([g.to(DEV) for g in grads], gvars))
        params, st32, u32 = B.tadam_step(theta, params, grads, st32)
        p64, st64, u64 = B.tadam_step(theta.double(), p64, [g.double() for g in grads], st64)
        if upd is not None:
            for j, (a, b, c) in enumerate(zip(torch.split(upd.cpu(), [math.prod(s) for s in shapes]), u32, u64)):
                _check(("update", it, j), a, b, c, TIGHT)
    torch.cuda.synchronize()
    for j in range(len(shapes)):
        _check(("x", j), gvars[j], params[j], p64[j], TIGHT)
        for k in B.TADAM_KEYS:
            _check((k, j), opt.get_slot(j, k), st32[j][k], st64[j][k], TIGHT)
    assert torch.equal(opt.get_slot(0, "t").cpu(), torch.full((math.prod(shapes[0]), 1), 3.0))
    nan = torch.isnan(gvars[-1].cpu())
    assert nan.tolist() == [False, True, True, False, False, False, False, False]


def test_lrs_steps_past_n_steps_and_glr():
    """A 3-entry schedule for 6 steps (rates[2] from the third step on) and the counter slot; the global rate."""
    from open_l2o_b200.trainable_baselines import GlobalLearningRate, LearningRateSchedule
    gen = torch.Generator().manual_seed(8)
    shapes = [(40, 3), (7,)]
    for which in ("lrs", "glr"):
        opt = LearningRateSchedule(n_steps=3) if which == "lrs" else GlobalLearningRate(initial_rate=0.37)
        if which == "lrs":
            opt.theta.copy_(torch.tensor([0.5, -0.25, 0.125]))
        rates = opt.theta.detach().cpu().clone()
        params = [torch.randn(s, generator=gen) for s in shapes]
        gvars = [p.clone().to(DEV) for p in params]
        itr = 0
        for t in range(6):
            grads = [torch.randn(s, generator=gen) for s in shapes]
            opt.apply_gradients(zip([g.to(DEV) for g in grads], gvars))
            params, itr, _ = B.lrs_step(rates, params, grads, itr if which == "lrs" else 0)
            torch.cuda.synchronize()
            assert all(torch.equal(v.cpu(), p) for v, p in zip(gvars, params)), (which, t)
        if which == "lrs":
            assert int(opt.get_slot(1, "itr")) == 6 and int(opt.state[1]) == 0


@pytest.mark.parametrize("which", ["tadam", "lrs", "glr"])
def test_minimize_graph_replay_matches_eager(which):
    """12 steps of minimize, eager and with graph replay: the same objective values, x and state bit for bit.  The
    schedule (12 distinct rates, more steps than entries would not show a stalled counter) advances under replay."""
    from open_l2o_b200 import engine
    from open_l2o_b200.trainable_baselines import GlobalLearningRate, LearningRateSchedule, TrainableAdam
    gen = torch.Generator().manual_seed(4)
    shapes = [(64, 9), (17,)]
    tgt = [torch.randn(s, generator=gen).to(DEV) for s in shapes]
    init = [torch.randn(s, generator=gen).to(DEV) for s in shapes]
    obj = lambda a, b: ((a - tgt[0]) ** 2).mean() + ((b - tgt[1]) ** 2).mean() + 0.1 * torch.cos(3 * a).mean()
    sched = torch.linspace(2.0, 0.2, 12)
    runs = []
    for graph in (False, True):
        if which == "tadam":
            opt = TrainableAdam(learning_rate=2e-6, beta1=0.8)
        elif which == "lrs":
            opt = LearningRateSchedule(n_steps=12)
            opt.theta.copy_(sched.to(DEV))
        else:
            opt = GlobalLearningRate(initial_rate=1.5)
        vs = [p.clone().requires_grad_(True) for p in init]
        before = engine.launch_count()
        f = opt.minimize(obj, vs, 12, cuda_graph=graph)
        runs.append((f, [v.detach().clone() for v in vs], opt.state.clone(), engine.launch_count() - before))
    (fe, xe, se, le), (fg, xg, sg, lg) = runs
    assert fe == fg and all(torch.equal(a, b) for a, b in zip(xe, xg)) and torch.equal(se, sg)
    assert le == 12 and lg == 13   # graph: 2 eager steps, 1 captured launch, 10 replays
    assert len(set(fg)) == 12
    if which == "lrs":
        assert sg.tolist() == [12, 0]


@pytest.mark.parametrize("which", ["tadam", "lrs"])
def test_reset_state_between_graph_replayed_minimize_calls(which):
    """minimize, reset_state, minimize with the same objective and variables: the second call replays the graph the
    first one captured, so the reset must keep the state buffer.  Against the same sequence run eagerly: objective
    values, x and the state bit for bit; the schedule's counter restarts at 0 and ends at 8."""
    from open_l2o_b200.trainable_baselines import LearningRateSchedule, TrainableAdam
    gen = torch.Generator().manual_seed(6)
    shapes = [(32, 5), (9,)]
    tgt = [torch.randn(s, generator=gen).to(DEV) for s in shapes]
    init = [torch.randn(s, generator=gen).to(DEV) for s in shapes]
    obj = lambda a, b: ((a - tgt[0]) ** 2).mean() + ((b - tgt[1]) ** 2).mean() + 0.1 * torch.cos(3 * a).mean()
    runs = []
    for graph in (False, True):
        if which == "tadam":
            opt = TrainableAdam(learning_rate=2e-6, beta1=0.8)
        else:
            opt = LearningRateSchedule(n_steps=16)
            opt.theta.copy_(torch.linspace(1.5, 0.1, 16).to(DEV))
        vs = [p.clone().requires_grad_(True) for p in init]
        f1 = opt.minimize(obj, vs, 8, cuda_graph=graph)
        state1 = opt.state.clone()
        opt.reset_state()
        assert float(opt.state.abs().max()) == 0
        f2 = opt.minimize(obj, vs, 8, cuda_graph=graph)
        runs.append((f1 + f2, [v.detach().clone() for v in vs], state1, opt.state.clone()))
    (fe, xe, s1e, s2e), (fg, xg, s1g, s2g) = runs
    assert fe == fg and all(torch.equal(a, b) for a, b in zip(xe, xg))
    assert torch.equal(s1e, s1g) and torch.equal(s2e, s2g)
    if which == "lrs":
        assert s2g.tolist() == [8, 0]
    else:
        assert bool((s2g[1] == 8.0).all())   # t restarted at 0


def test_tadam_bwd_with_nonzero_v_matches_oracle():
    """The backward's v != 0 branch (not reachable from the zero state; a hand-set state): d_state_old, d_theta and d_g
    of l2o_tadam_bwd against fp64 autograd through the oracle, for random adjoints of m', v' and the update.  Every
    third coordinate keeps v = 0; g = 0 and g = 1e-25 (g^2 underflows in fp32) take pow's derivatives as 0.  Each output
    within 1e-5 max-norm relative, or 3x the fp32 oracle's distance from fp64 where that is larger; the t plane's
    adjoint is exactly 0 and beta2_logit's gradient is nonzero."""
    from open_l2o_b200 import _lib
    from open_l2o_b200.engine import _ptr as _p
    gen = torch.Generator().manual_seed(31)
    n = 4096
    theta = tadam_theta(lr=1e-3, b1=0.85, b2=0.9, eps=1e-7, dtype=torch.float32)
    m = torch.randn(n, generator=gen) * 0.1
    t = torch.full((n,), 2.0)
    v = torch.rand(n, generator=gen) * 0.09 + 0.01
    v[::3] = 0.0
    g = torch.rand(n, generator=gen) * 1.6 - 0.8
    g[::7] = 0.0
    g[1::11] = 1e-25
    R_m, R_v, R_u = (torch.randn(n, generator=gen) for _ in range(3))

    def oracle(dtype):
        th = theta.to(dtype).requires_grad_(True)
        mm, vv, gg = (a.to(dtype).reshape(-1, 1).requires_grad_(True) for a in (m, v, g))
        _, st, upd = B.tadam_compute_update(th, torch.zeros(n, 1, dtype=dtype), gg,
                                            {"m": mm, "t": t.to(dtype).reshape(-1, 1), "v": vv})
        L = (R_m.to(dtype).reshape(-1, 1) * st["m"]).sum() + (R_v.to(dtype).reshape(-1, 1) * st["v"]).sum() \
            + (R_u.to(dtype).reshape(-1, 1) * upd).sum()
        return [d.reshape(-1) for d in torch.autograd.grad(L, (th, mm, vv, gg))]
    want64, want32 = oracle(torch.float64), oracle(torch.float32)

    dev = lambda a: a.contiguous().to(DEV)
    planes = dev(torch.stack([m, t, v]))
    d_new = dev(torch.stack([R_m, torch.randn(n, generator=gen), R_v]))   # the t adjoint is ignored
    d_old, d_theta, d_g = torch.empty(3, n, device=DEV), torch.zeros(4, dtype=torch.float64, device=DEV), \
        torch.empty(n, device=DEV)
    th_d, g_d, du_d = dev(theta), dev(g), dev(R_u)
    a = _lib.TadamBwdArgs(n=n, theta=_p(th_d), g=_p(g_d), state_old=_p(planes), d_state_new=_p(d_new),
                          d_update=_p(du_d), d_state_old=_p(d_old), d_theta=d_theta.data_ptr(), d_g=_p(d_g))
    _lib.check(_lib.lib().l2o_tadam_bwd(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "l2o_tadam_bwd")
    torch.cuda.synchronize()
    got = [d_theta.cpu(), d_old[0].cpu(), d_old[2].cpu(), d_g.cpu()]
    for name, e, w64, w32 in zip(("theta", "m", "v", "g"), got, want64, want32):
        e = e.double()
        assert bool(torch.isfinite(e).all()), name
        if name == "theta":
            for j in range(4):
                r = float(w64[j])
                err, own = abs(float(e[j]) - r) / abs(r), abs(float(w32[j]) - r) / abs(r)
                assert err <= max(REL_TOL, 3 * own), (name, j, err, own)
        else:
            assert rel_err(e, w64) <= max(REL_TOL, 3 * rel_err(w32, w64)), (name, rel_err(e, w64), rel_err(w32, w64))
    assert float(d_old[1].abs().max()) == 0.0 and float(d_theta[2]) != 0.0


def _problem(which):
    shapes = [(40, 5), (5,), (150,)]
    obj64, init = curved_problem(shapes, seed=8)
    obj32c, _ = curved_problem(shapes, seed=8, dtype=torch.float32)
    obj32, _ = curved_problem(shapes, seed=8, dtype=torch.float32, device=DEV)
    # step sizes of about 1.5: the curvature of the (150,) tensor (about 0.02) shows in the meta-gradient, and the
    # (5,) tensor (about 1) still converges
    if which == "tadam":
        theta = tadam_theta(lr=1.5e-5, b1=0.8, b2=0.99, eps=1e-7, dtype=torch.float32)   # lr / (1e-5 + eps) = 1.5
    elif which == "lrs":
        theta = torch.tensor([1.0, 1.8, 0.6, 1.4])   # n_steps = 4: the second unroll's last two steps reuse rates[3]
    else:
        theta = torch.tensor([1.5])
    return shapes, theta, init, obj64, obj32c, obj32


@pytest.mark.parametrize("which", ["tadam", "lrs", "glr"])
@pytest.mark.parametrize("second", [False, True])
def test_meta_gradient_matches_oracle_autograd(which, second):
    """T = 3 from a fresh state, then a truncated second unroll of 3 steps from the detached state, first and second
    order.  Per theta entry: within 1e-5 relative, or 3x the fp32 oracle's distance from fp64 where that is larger;
    entries the oracle gives exactly 0 (beta2_logit, schedule entries no step used) are exactly 0.  With second
    derivatives the first-order oracle must miss the reference by far more than the tolerance."""
    from open_l2o_b200 import baselines_train as bt
    shapes, theta, init, obj64, obj32c, obj32 = _problem(which)
    cls = {"tadam": bt.TrainableAdamTrainer, "lrs": bt.LearningRateScheduleTrainer,
           "glr": bt.GlobalLearningRateTrainer}[which]
    tr = cls(shapes, theta=theta, device=DEV, use_second_derivatives=second)
    p0 = [p.float().to(DEV) for p in init]
    m1, g1, objs, fin = tr.meta_gradient(obj32, p0, 3)
    m2, g2, _, _ = tr.meta_gradient(obj32, p0, 3, state=tr.detach_state(fin),
                                    initial_obj=torch.tensor(objs[0], device=DEV))
    torch.cuda.synchronize()
    r1m, r1, c64 = baseline_oracle_meta(which, theta, obj64, init, 3, second)
    _, r1_32, c32 = baseline_oracle_meta(which, theta, obj32c, init, 3, second, dtype=torch.float32)
    r2m, r2, _ = baseline_oracle_meta(which, theta, obj64, init, 3, second, carry=c64, initial_obj=c64[3])
    _, r2_32, _ = baseline_oracle_meta(which, theta, obj32c, init, 3, second, dtype=torch.float32, carry=c32,
                                       initial_obj=c32[3])
    assert abs(float(m1) - float(r1m)) <= 1e-5 * max(1.0, abs(float(r1m)))
    assert abs(float(m2) - float(r2m)) <= 1e-5 * max(1.0, abs(float(r2m)))
    for tag, eng, ref, r32 in (("unroll1", g1, r1, r1_32), ("unroll2", g2, r2, r2_32)):
        eng, r32 = eng.detach().double().cpu(), r32.double()
        for j in range(ref.numel()):
            r = float(ref[j])
            if r == 0.0:
                assert float(eng[j]) == 0.0, (tag, j)
                continue
            err, own = abs(float(eng[j]) - r) / abs(r), abs(float(r32[j]) - r) / abs(r)
            assert err <= max(REL_TOL, 3 * own), (tag, j, err, own)
        if second:
            _, first, _ = baseline_oracle_meta(which, theta, obj64, init, 3, False) if tag == "unroll1" else \
                baseline_oracle_meta(which, theta, obj64, init, 3, False, carry=c64, initial_obj=c64[3])
            assert rel_err(first, ref) >= 100 * REL_TOL, (tag, rel_err(first, ref))
    if which == "tadam":
        assert float(g1[2]) == 0.0 and float(g2[2]) == 0.0
    if which == "lrs":
        # unroll 1 scores x_0..x_2 (rates 0, 1; its last step's rates[2] reaches no scored objective); unroll 2 starts
        # from the detached x_3 and scores x_4, x_5, made with rates[3] and the clamped index 4 -> 3
        assert g1[0] != 0 and g1[1] != 0 and float(g1[2:].abs().max()) == 0.0
        assert float(g2[:3].abs().max()) == 0.0 and g2[3] != 0


def test_bwd_outputs_do_not_depend_on_d_g():
    """At the ConvNet size: d_state_old bit-identical with and without d_g, d_theta equal up to the fp64 atomics'
    order; the same for the schedule's backward."""
    from open_l2o_b200 import _lib
    from open_l2o_b200.engine import _ptr as _p
    L = _lib.lib()
    gen = torch.Generator().manual_seed(24)
    n = 354218
    theta = tadam_theta(lr=1e-3, b1=0.9, b2=0.99, dtype=torch.float32).to(DEV)
    planes = torch.stack([torch.randn(n, generator=gen), torch.full((n,), 2.0), torch.zeros(n)]).to(DEV)
    planes[2, ::3] = torch.rand((n + 2) // 3, generator=gen).to(DEV) * 0.1   # some v != 0: the v-chain runs too
    g, d_new, d_upd = (torch.randn(*s, generator=gen).to(DEV) for s in ((n,), (3, n), (n,)))
    g.clamp_(-0.9, 0.9)   # (v != 0 with g^2 > 1 makes v' negative and sqrt(v^ + 1e-10) NaN, as in the reference)

    def tadam(d_g):
        d_old, d_theta = torch.empty_like(planes), torch.zeros(4, dtype=torch.float64, device=DEV)
        a = _lib.TadamBwdArgs(n=n, theta=_p(theta), g=_p(g), state_old=_p(planes), d_state_new=_p(d_new),
                              d_update=_p(d_upd), d_state_old=_p(d_old), d_theta=d_theta.data_ptr(), d_g=_p(d_g))
        _lib.check(L.l2o_tadam_bwd(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "l2o_tadam_bwd")
        return d_old, d_theta
    d_g = torch.empty(n, device=DEV)
    a_old, a_th = tadam(None)
    b_old, b_th = tadam(d_g)
    rates = torch.tensor([0.3, 0.2], device=DEV)
    itr = torch.tensor([5, 0], dtype=torch.int32, device=DEV)

    def lrs(dg):
        d_rates = torch.zeros(2, dtype=torch.float64, device=DEV)
        a = _lib.LrsgdBwdArgs(n=n, rates=_p(rates), n_steps=2, itr=_p(itr, torch.int32), g=_p(g), d_update=_p(d_upd),
                              d_rates=d_rates.data_ptr(), d_g=_p(dg))
        _lib.check(L.l2o_lrsgd_bwd(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "l2o_lrsgd_bwd")
        return d_rates
    d_g2 = torch.empty(n, device=DEV)
    la, lb = lrs(None), lrs(d_g2)
    torch.cuda.synchronize()
    assert torch.equal(a_old, b_old) and bool(torch.isfinite(d_g).all())
    assert rel_err(b_th, a_th) <= 1e-12 and float(a_th[2]) != 0.0
    assert float(la[0]) == 0.0 and rel_err(lb, la) <= 1e-12
    assert torch.equal(d_g2, rates[1] * d_upd)   # index min(5, 1) = 1
    assert rel_err(la[1], (d_upd.double() * g.double()).sum()) <= 1e-6


@pytest.mark.parametrize("which", ["TrainableAdam", "LearningRateSchedule", "GlobalLearningRate"])
def test_train_optimizer_runs_end_to_end(which):
    from open_l2o_b200 import baselines_train as bt
    from open_l2o_b200.trainable_baselines import register_optimizers
    gen = torch.Generator().manual_seed(11)
    tgt = torch.randn(20, 10, generator=gen).to(DEV)
    problems = [(lambda ps: ((ps[0] - tgt) ** 2).mean() + 0.3 * torch.cos(3.0 * ps[0]).mean(),
                 lambda: [torch.randn(20, 10, generator=gen).to(DEV)])]
    kwargs = {"TrainableAdam": dict(learning_rate=1e-5), "LearningRateSchedule": dict(initial_rate=0.0, n_steps=8),
              "GlobalLearningRate": dict(initial_rate=1.0)}[which]
    for second in (False, True):
        opt = register_optimizers()[which](**kwargs)
        theta_before = opt.theta.clone()
        trainers = []

        def make(shapes, th):
            tr = opt.meta_trainer([torch.empty(s) for s in shapes], learning_rate=1e-2, use_second_derivatives=second)
            trainers.append(tr)
            return tr
        theta, log = bt.train_optimizer(make, problems, num_problems=1, num_meta_iterations=2,
                                        num_unroll_func=lambda: 2, num_partial_unroll_itrs_func=lambda: 4,
                                        select_random_problems=False)
        assert len(log) == 2 and all(len(m) == 2 and all(math.isfinite(v) for v in m) for _, m in log), log
        assert trainers[0].global_step == 4 and trainers[0].use_second_derivatives is second
        assert bool(torch.isfinite(theta).all())
        opt.adopt(trainers[0])
        assert not torch.equal(opt.theta, theta_before)
