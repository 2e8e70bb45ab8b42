"""GPU: the CoordinatewiseRNN step (l2o_crnn_step) and meta-gradient (l2o_crnn_bwd) against the oracle
(oracle/crnn_oracle.py), graph replay against eager execution, and one meta-training run."""
import math

import pytest
import torch

from oracle import crnn_oracle as CR
from tests.helpers import HRNN_CONVNET, REL_TOL, hrnn_ragged_shapes, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TILE = 128   # coordinates per tile of l2o_crnn_bwd (l2o_crnn.cu kBwdBlock)


def crnn_generic_theta(seed, dtype=torch.float32):
    """CoordinatewiseRNN weights with no zero or constant block left.  The initial distribution zeroes the lr weights
    and bias (lr' = lr exactly, so a dropped lr term or factor shows nothing), zeroes every LSTM bias (a permuted gate
    row shows nothing) and repeats 2.2 in the decay bias.  Each is redrawn at about init scale: lr weights N(0, 0.3)
    and bias N(0, 0.3), LSTM biases N(0, 0.5), decay bias 2.2 + N(0, 0.5)."""
    base = CR.init_theta(seed, dtype=torch.float64)
    g = torch.Generator().manual_seed(1000 + int(seed))
    out = []
    for name, shape in CR.theta_spec():
        v = CR.unpack_theta(base)[name].reshape(-1).clone()
        noise = lambda s: torch.randn(v.numel(), generator=g, dtype=torch.float64) * s
        if name in ("learning_rate_weights", "learning_rate_bias"):
            v = noise(0.3)
        elif name.endswith("/bias"):
            v = noise(0.5)
        elif name == "decay_bias":
            v = 2.2 + noise(0.5)
        out.append(v)
    return torch.cat(out).to(dtype)


def _shapes(kind):
    if kind == "small":
        return [(33, 7), (5,), (300,)]
    if kind == "convnet":
        from open_l2o_b200.scale_problems import ConvNet
        return [tuple(s) for s in ConvNet(*HRNN_CONVNET).param_shapes]
    if kind == "ragged":
        return [(1,), (TILE - 1,), (TILE,), (TILE + 1,)] + hrnn_ragged_shapes(n_small=40, big=3 * TILE + 5)
    return [(1,)]


CASES = [("small", "init"), ("small", "generic"), ("convnet", "generic"), ("ragged", "generic"), ("lone", "generic"),
         ("small", "saturate")]


@pytest.mark.parametrize("kind,theta_kind", CASES)
def test_crnn_steps_match_oracle(kind, theta_kind):
    """Several engine steps through CoordinatewiseRNN.apply_gradients against the fp32 oracle fed the same gradients:
    x, the applied update and every state plane within 1e-5 max-norm relative.  "saturate" drives lr' to exactly 2 lr
    and decay' to 0 (the sigmoids at +-60)."""
    from open_l2o_b200.coordinatewise_rnn import CoordinatewiseRNN, metarun_args, step_launch
    shapes = _shapes(kind)
    if kind == "convnet":
        assert sum(math.prod(s) for s in shapes) == 354218
    gen = torch.Generator().manual_seed(7)
    opt = CoordinatewiseRNN(random_seed=3, **metarun_args())
    theta = CR.init_theta(3) if theta_kind == "init" else crnn_generic_theta(5)
    if theta_kind == "saturate":
        P = CR.unpack_theta(theta)
        P["learning_rate_weights"].zero_()
        P["learning_rate_bias"].fill_(60.0)
        P["decay_weights"].zero_()
        P["decay_bias"].fill_(-60.0)
    opt.theta.copy_(theta.to(DEV))
    params = [torch.randn(s, generator=gen) for s in shapes]
    gvars = [p.clone().to(DEV) for p in params]
    scales = [10.0 ** float(torch.empty(()).uniform_(-3, 0, generator=gen)) for _ in shapes]
    grads_all = [[torch.randn(s, generator=gen) * c for s, c in zip(shapes, scales)] for _ in range(4)]
    opt.apply_gradients(zip([g.to(DEV) for g in grads_all[0]], gvars))     # creates the slots
    N = opt.N
    lr0 = torch.exp(torch.rand(N, generator=gen, dtype=torch.float64) * (math.log(1e-2) - math.log(1e-6)) + math.log(1e-6))
    opt.reset_state(learning_rate=lr0)
    for v, p in zip(gvars, params):
        v.data.copy_(p.to(DEV))
    P = CR.unpack_theta(theta)
    states = [CR.initial_state(P, p.numel(), gen, dtype=torch.float32) for p in params]
    off = 0
    for st, p in zip(states, params):
        st["learning_rate"] = lr0[off:off + p.numel()].float().reshape(-1, 1)
        off += p.numel()
    assert torch.equal(opt.state.cpu(), CR.state_to_planes(states))
    th64, p64 = theta.double(), [p.double() for p in params]
    s64 = [{k: v.double() for k, v in st.items()} for st in states]
    for grads in grads_all:
        p64, s64, u64 = CR.step(th64, p64, [g.double() for g in grads], s64)
        gflat = torch.cat([g.reshape(-1) for g in grads]).to(DEV)
        upd_eng = torch.empty(N, device=DEV)                 # the training form of the same step: the update itself
        step_launch(opt.theta, gflat, opt.state, torch.empty_like(opt.state), update=upd_eng)
        opt.apply_gradients(zip([g.to(DEV) for g in grads], gvars))
        params, states, upd = CR.step(theta, params, grads, states)
    torch.cuda.synchronize()
    # each quantity within 1e-5 max-norm relative, or 3x the fp32 oracle's own distance from fp64 where that is larger
    # (a plane of one hidden unit can be small everywhere, and then sum order alone moves it by more than 1e-5)
    want, want64, got = CR.state_to_planes(states), CR.state_to_planes(s64), opt.state.cpu()
    flat = lambda ts: torch.cat([t.reshape(-1) for t in ts])
    cmp = {"x": (flat(gvars), flat(params), flat(p64)), "update": (upd_eng, flat(upd), flat(u64))}
    cmp.update({"plane%d" % k: (got[k], want[k], want64[k]) for k in range(want.shape[0])})
    bad = {}
    for k, (e, w32, w64) in cmp.items():
        err, own = rel_err(e, w32), rel_err(w32, w64)
        if not err <= max(REL_TOL, 3 * own):
            bad[k] = (err, own)
    assert not bad, bad
    if theta_kind == "saturate":
        assert torch.equal(got[102], (lr0 * 16).float()) and float(got[101].abs().max()) < 1e-20
    assert torch.equal(opt.get_slot(0, "rnn").cpu(), got[:100, :shapes_numel(shapes[0])].t())
    assert opt.get_slot(len(shapes) - 1, "learning_rate").shape == (shapes_numel(shapes[-1]), 1)


def shapes_numel(s):
    return int(math.prod(s))


def test_crnn_step_launch_update_and_inplace_agree():
    """The training form (separate out planes, update written, x untouched) and the inference form (in place, x -= update)
    compute the same step."""
    from open_l2o_b200.coordinatewise_rnn import CoordinatewiseRNN, metarun_args, step_launch
    gen = torch.Generator().manual_seed(2)
    n = 5000
    opt = CoordinatewiseRNN(random_seed=1, **metarun_args())
    opt.theta.copy_(crnn_generic_theta(1).to(DEV))
    x = torch.randn(n, generator=gen).to(DEV)
    opt.apply_gradients([(torch.randn(n, generator=gen).to(DEV), x)])
    planes = opt.state.clone()
    g = (torch.randn(n, generator=gen) * 0.3).to(DEV)
    new, upd = torch.empty_like(planes), torch.empty(n, device=DEV)
    x0 = x.detach().clone()
    step_launch(opt.theta, g, planes, new, update=upd)
    opt.apply_gradients([(g, x)])
    torch.cuda.synchronize()
    assert torch.equal(new, opt.state) and torch.equal(x0 - upd, x.detach())


def test_crnn_minimize_graph_replay_matches_eager():
    from open_l2o_b200.coordinatewise_rnn import CoordinatewiseRNN, metarun_args
    from open_l2o_b200 import engine
    gen = torch.Generator().manual_seed(4)
    shapes = [(64, 9), (17,)]
    tgt = [torch.randn(s, generator=gen).to(DEV) for s in shapes]
    init = [torch.randn(s, generator=gen).to(DEV) for s in shapes]
    obj = lambda a, b: ((a - tgt[0]) ** 2).mean() + ((b - tgt[1]) ** 2).mean() + 0.1 * torch.cos(3 * a).mean()
    runs = []
    for graph in (False, True):
        opt = CoordinatewiseRNN(random_seed=9, **metarun_args())
        opt.theta.copy_(crnn_generic_theta(2).to(DEV))
        vs = [p.clone().requires_grad_(True) for p in init]
        before = engine.launch_count()
        f = opt.minimize(obj, vs, 12, cuda_graph=graph)
        runs.append((f, [v.detach().clone() for v in vs], opt.state.clone(), engine.launch_count() - before))
    (fe, xe, se, le), (fg, xg, sg, lg) = runs
    assert fe == fg and all(torch.equal(a, b) for a, b in zip(xe, xg)) and torch.equal(se, sg)
    assert le == 12 and lg == 13   # graph: 2 eager steps, 1 captured launch, 10 replays


def _oracle_meta_gradient(theta0, init, tgt, lr0, steps, dtype, carry=None):
    """Autograd through the oracle: meta objective of `steps` steps from `init` (or from a carried, detached state) and
    its gradient w.r.t. theta.  Returns (meta, grad, final params, final states, initial objective)."""
    th = theta0.to(dtype).clone().requires_grad_(True)
    P = CR.unpack_theta(th)
    fobj = lambda ps: sum(((p - t.to(dtype)) ** 2).mean() + 0.05 * torch.cos(2.0 * p).mean() for p, t in zip(ps, tgt))
    if carry is None:
        params = [p.to(dtype) for p in init]
        states, off = [], 0
        for p in params:
            st = CR.initial_state(P, p.numel(), torch.Generator(), dtype=dtype)
            st["learning_rate"] = lr0[off:off + p.numel()].to(dtype).reshape(-1, 1)
            off += p.numel()
            states.append(st)
        f0 = None
    else:
        params, states, f0 = carry
    vals = []
    for t in range(steps):
        leaf = [p.detach().requires_grad_(True) for p in params]
        f = fobj(leaf)
        gr = torch.autograd.grad(f, leaf)
        vals.append(fobj(params) if t > 0 or carry is not None else f.detach())
        params, states, _ = CR.step(th, params, [g.detach() for g in gr], states)
    f0 = vals[0].detach() if f0 is None else f0
    meta = torch.log(torch.stack([v.reshape(()) for v in vals]) / (f0 + 1e-6) + 1e-6).mean()
    (g,) = torch.autograd.grad(meta, th)
    det = ([p.detach() for p in params], [{k: v.detach() for k, v in s.items()} for s in states], f0)
    return meta.detach(), g, det


@pytest.mark.parametrize("theta_kind,shapes", [("init", [(40, 5), (5,), (150,)]), ("generic", [(40, 5), (5,), (150,)]),
                                               ("generic", [(1,), (127,), (129,), (300,)])])
def test_crnn_meta_gradient_matches_oracle_autograd(theta_kind, shapes):
    """T = 3 from a fresh state (the init_vector block included), then a second unroll of 3 steps continuing from the
    detached state of the first (truncated BPTT).  Each theta block within 1e-5 of its own largest entry, or 3x the fp32
    oracle's distance from fp64 where that is larger."""
    from open_l2o_b200 import crnn_train as ct
    gen = torch.Generator().manual_seed(3)
    tgt = [torch.randn(s, generator=gen, dtype=torch.float64) for s in shapes]
    init = [torch.randn(s, generator=gen, dtype=torch.float64) * 0.5 for s in shapes]
    N = sum(p.numel() for p in init)
    lr0 = torch.exp(torch.rand(N, generator=gen, dtype=torch.float64) * 3.0 - 6.0).float()
    theta0 = CR.init_theta(7) if theta_kind == "init" else crnn_generic_theta(7)
    tr = ct.MetaTrainer(shapes, theta=theta0, device=DEV)
    obj32 = lambda ps: sum(((p - t.float().to(DEV)) ** 2).mean() + 0.05 * torch.cos(2.0 * p).mean() for p, t in zip(ps, tgt))
    p0 = [p.float().to(DEV) for p in init]
    meta1, g1, _, fin = tr.meta_gradient(obj32, p0, 3, lr0)
    initial = torch.tensor(float(obj32(p0)), device=DEV)
    meta2, g2, _, _ = tr.meta_gradient(obj32, p0, 3, state=tr.detach_state(fin), initial_obj=initial)
    torch.cuda.synchronize()
    m1_64, r1_64, c64 = _oracle_meta_gradient(theta0, init, tgt, lr0, 3, torch.float64)
    _, r1_32, c32 = _oracle_meta_gradient(theta0, init, tgt, lr0, 3, torch.float32)
    m2_64, r2_64, _ = _oracle_meta_gradient(theta0, init, tgt, lr0, 3, torch.float64, carry=c64)
    _, r2_32, _ = _oracle_meta_gradient(theta0, init, tgt, lr0, 3, torch.float32, carry=c32)
    assert abs(float(meta1) - float(m1_64)) <= 1e-5 and abs(float(meta2) - float(m2_64)) <= 1e-5
    sizes = [math.prod(s) for _, s in CR.theta_spec()]
    names = [n for n, _ in CR.theta_spec()]
    for tag, eng, ref, r32 in (("unroll1", g1, r1_64, r1_32), ("unroll2", g2, r2_64, r2_32)):
        eb, rb, fb = (torch.split(t.detach().double().cpu(), sizes) for t in (eng, ref, r32))
        for name, e, r, f in zip(names, eb, rb, fb):
            den = float(r.abs().max())
            if den == 0.0:
                assert float(e.abs().max()) == 0.0, (tag, name)
                continue
            err, own = float((e - r).abs().max()) / den, float((f - r).abs().max()) / den
            assert err <= max(REL_TOL, 3 * own), (tag, name, err, own)
        if tag == "unroll1":
            assert float(rb[names.index("init_vector")].abs().max()) > 0


def test_crnn_train_optimizer_runs_end_to_end():
    from open_l2o_b200 import crnn_train as ct
    from open_l2o_b200.coordinatewise_rnn import CoordinatewiseRNN, metarun_args
    gen = torch.Generator().manual_seed(11)
    tgt = torch.randn(20, 10, generator=gen).to(DEV)
    problems = [(lambda ps: ((ps[0] - tgt) ** 2).mean(), lambda: [torch.randn(20, 10, generator=gen).to(DEV)])]
    opt = CoordinatewiseRNN(random_seed=5, **metarun_args())
    theta_before = opt.theta.clone()
    trainers = []

    def make(shapes, th):
        tr = opt.meta_trainer([torch.empty(s) for s in shapes], learning_rate=1e-3, random_seed=0)
        trainers.append(tr)
        return tr
    theta, log = ct.train_optimizer(make, problems, num_problems=1, num_meta_iterations=2, num_unroll_func=lambda: 2,
                                    num_partial_unroll_itrs_func=lambda: 5, select_random_problems=False)
    assert len(log) == 2 and all(len(m) == 2 and all(math.isfinite(v) for v in m) for _, m in log)
    assert trainers[0].global_step == 4 and bool(torch.isfinite(theta).all())
    opt.adopt(trainers[0])
    assert not torch.equal(opt.theta, theta_before)
