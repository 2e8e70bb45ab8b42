"""Tensor-core (wgmma) engine parity: 3xTF32 unroll vs the CPU oracle and vs the exact-fp32 FFMA engine."""
import pytest
import torch

from oracle import l2o_oracle as orc
from tests.helpers import REL_TOL, SPECS, arena_to_state, make_handle, rel_err
from tests.test_kernels_gpu import _fused_problem, _run_prerecorded, _theta

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("name", ["dm_identity", "dm_logsign", "rnnprop"])
@pytest.mark.parametrize("n,T", [(777, 20), (256, 1), (5000, 3)])
def test_tc_unroll_fwd_prerecorded(name, n, T):
    from open_l2o_b200.engine import ENGINE_TC
    r = _run_prerecorded(SPECS[name], n=n, T=T, seed=7, engine=ENGINE_TC)
    spec, sf = r["spec"], r["sf"]
    assert rel_err(r["dseq"], torch.stack(r["deltas"])) <= REL_TOL
    assert rel_err(r["xg"], r["x_ref"]) <= REL_TOL
    for t in sorted({0, 1, T // 2, T}):
        got = arena_to_state(r["ckpt"][t * sf * n:(t + 1) * sf * n].cpu(), spec.layers, n)
        for (hg, cg), (hr, cr) in zip(got, r["states"][t]):
            assert rel_err(hg, hr) <= REL_TOL and rel_err(cg, cr) <= REL_TOL, t
    fin = arena_to_state(r["arena"].cpu(), spec.layers, n)
    for (hg, cg), (hr, cr) in zip(fin, r["states"][T]):
        assert rel_err(hg, hr) <= REL_TOL and rel_err(cg, cr) <= REL_TOL


@pytest.mark.parametrize("T", [20, 100])
def test_tc_fused_rastrigin_forward_then_bptt(T):
    """BASELINE config #5 shape at reduced d: tensor-core forward unroll (T=100: error growth over the full unroll)
    feeding the BPTT kernel; both against the fp64 oracle."""
    from open_l2o_b200.engine import ENGINE_TC, OPT_KINDS
    spec = SPECS["dm_identity"]
    n = 2000
    gen = torch.Generator().manual_seed(5)
    theta = _theta(spec, gain=0.05)
    prob, x0 = _fused_problem("rastrigin_sep", n, gen)
    prob64 = orc.FusedProblem("rastrigin_sep", prob.a.double(), prob.b.double(), prob.alpha, prob.fscale)
    g64, res64 = orc.meta_grad(spec, theta.double(), x0.double(), orc.initial_state(spec, n, torch.float64), None, T,
                               grad_of=prob64.f_and_g)
    g32, res32 = orc.meta_grad(spec, theta, x0, orc.initial_state(spec, n), None, T, grad_of=prob.f_and_g)
    h = make_handle(spec)
    h.set_engine(ENGINE_TC)
    sf = h.state_floats
    th = theta.to(DEV)
    arena = h.new_state(n, DEV)
    ckpt = torch.zeros((T + 1) * sf * n, device=DEV)
    x = x0.to(DEV).clone()
    g_rec = torch.empty(T + 1, n, device=DEV)
    fx = torch.zeros(T + 1, dtype=torch.float64, device=DEV)
    h.unroll_fwd(th, n, T, arena, opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=prob.a.to(DEV), opt_b=prob.b.to(DEV),
                 opt_alpha=prob.alpha, opt_fscale=prob.fscale, x=x, ckpt=ckpt, g_rec=g_rec, fx=fx)
    torch.cuda.synchronize()
    slack = max(REL_TOL, 3.0 * rel_err(res32.x_final, res64.x_final))
    assert rel_err(fx, res64.fx) <= slack
    assert rel_err(x, res64.x_final) <= slack
    dtheta = torch.zeros(h.n_theta, dtype=torch.float64, device=DEV)
    h.unroll_bwd(th, n, T, g_rec, ckpt, dtheta, g_rec=g_rec)
    torch.cuda.synchronize()
    gslack = max(REL_TOL, 3.0 * rel_err(g32, g64))
    assert rel_err(dtheta, g64) <= gslack, (rel_err(dtheta, g64), rel_err(g32, g64))


def test_tc_matches_ffma_engine_large():
    """Many tiles per CTA (persistent loop) + ragged tail: tensor-core engine vs exact-fp32 engine."""
    from open_l2o_b200.engine import ENGINE_FFMA, ENGINE_TC, OPT_KINDS
    spec = SPECS["dm_identity"]
    n, T = 76_109, 6
    gen = torch.Generator().manual_seed(8)
    theta = _theta(spec, gain=0.05).to(DEV)
    a, b, x0 = (torch.randn(n, generator=gen).to(DEV) for _ in range(3))
    outs = {}
    for eng in (ENGINE_FFMA, ENGINE_TC):
        h = make_handle(spec)
        h.set_engine(eng)
        arena = h.new_state(n, DEV)
        x = x0.clone()
        fx = torch.zeros(T + 1, dtype=torch.float64, device=DEV)
        g_rec = torch.empty(T + 1, n, device=DEV)
        h.unroll_fwd(theta, n, T, arena, opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=a, opt_b=b, opt_alpha=10.0,
                     opt_fscale=1.0 / n, x=x, g_rec=g_rec, fx=fx)
        torch.cuda.synchronize()
        outs[eng] = (x, arena, fx, g_rec)
    for u, v in zip(outs[ENGINE_TC], outs[ENGINE_FFMA]):
        assert rel_err(u, v) <= REL_TOL


@pytest.mark.parametrize("name", ["dm_identity", "dm_logsign"])
def test_tc_bwd_matches_ffma_bwd(name):
    """Same checkpoints / recorded gradients through both BPTT kernels (multi-tile, ragged tail)."""
    from open_l2o_b200.engine import ENGINE_FFMA, ENGINE_TC
    spec = SPECS[name]
    n, T = 19_021, 5
    gen = torch.Generator().manual_seed(21)
    theta = _theta(spec, gain=0.05).to(DEV)
    from tests.helpers import wild_gradients
    if spec.preprocess_name == "LogAndSign":
        g_rec = torch.stack([wild_gradients(n, gen) for _ in range(T + 1)]).to(DEV)
    else:
        g_rec = (torch.randn(T + 1, n, generator=gen) * 0.5).to(DEV)
    h = make_handle(spec)
    h.set_engine(ENGINE_FFMA)
    sf = h.state_floats
    arena = h.new_state(n, DEV)
    ckpt = torch.zeros((T + 1) * sf * n, device=DEV)
    h.unroll_fwd(theta, n, T, arena, in_seq=g_rec[:T].contiguous(), ckpt=ckpt)
    outs = {}
    for eng in (ENGINE_FFMA, ENGINE_TC):
        h.set_engine(eng)
        d = torch.zeros(h.n_theta, dtype=torch.float64, device=DEV)
        h.unroll_bwd(theta, n, T, g_rec[:T].contiguous(), ckpt, d, g_rec=g_rec)
        torch.cuda.synchronize()
        outs[eng] = d
    assert rel_err(outs[ENGINE_TC], outs[ENGINE_FFMA]) <= REL_TOL


@pytest.mark.parametrize("name", ["dm_identity", "dm_logsign"])
def test_tc_step_operator(name):
    """l2o_step on the tensor-core engine (state in HBM, out-of-place) vs the oracle; chained over 3 steps."""
    from open_l2o_b200.engine import ENGINE_TC
    from tests.helpers import random_state, state_to_arena, wild_gradients
    spec = SPECS[name]
    n = 20000
    gen = torch.Generator().manual_seed(31)
    theta = _theta(spec)
    st = random_state(spec, n, gen)
    x_ref = torch.randn(n, generator=gen)
    h = make_handle(spec)
    h.set_engine(ENGINE_TC)
    th = theta.to(DEV)
    a_in = state_to_arena(st, n).to(DEV)
    x = x_ref.to(DEV).clone()
    for it in range(3):
        g = wild_gradients(n, gen) if spec.preprocess_name == "LogAndSign" else torch.randn(n, generator=gen)
        d_ref, st = orc.net_apply(spec, theta, g.unsqueeze(-1), st)
        x_ref = x_ref + d_ref
        a_out = torch.zeros_like(a_in)
        delta = torch.empty(n, device=DEV)
        h.step(th, g.to(DEV), a_in, a_out, x=x, delta=delta)
        torch.cuda.synchronize()
        assert rel_err(delta, d_ref) <= REL_TOL
        assert rel_err(x, x_ref) <= REL_TOL
        for (hg, cg), (hr, cr) in zip(arena_to_state(a_out.cpu(), spec.layers, n), st):
            assert rel_err(hg, hr) <= REL_TOL and rel_err(cg, cr) <= REL_TOL
        a_in = a_out


@pytest.mark.parametrize("name", ["dm_identity", "dm_logsign"])
def test_tc_imitation_bptt(name):
    """Imitation ("mt") unroll on the tensor-core engine (DM/meta_dm_train.py:463-480): forward over pre-recorded inputs
    records delta_seq; the tensor-core BPTT forms dDelta_t = (delta_t - label_t)/N from it."""
    from open_l2o_b200.engine import ENGINE_TC
    spec = SPECS[name]
    n, T = 18_963, 7
    gen = torch.Generator().manual_seed(13)
    theta = _theta(spec, gain=1.0)
    inputs = torch.randn(T, n, generator=gen)
    labels = torch.randn(T, n, generator=gen) * 0.01
    th64 = theta.double().requires_grad_(True)
    loss64, _, _ = orc.imitation_loss(spec, th64, inputs.double(), labels.double(),
                                      orc.initial_state(spec, n, torch.float64))
    (g64,) = torch.autograd.grad(loss64, th64)
    th32 = theta.clone().requires_grad_(True)
    loss32, _, _ = orc.imitation_loss(spec, th32, inputs, labels, orc.initial_state(spec, n))
    (g32,) = torch.autograd.grad(loss32, th32)
    h = make_handle(spec)
    h.set_engine(ENGINE_TC)   # explicit engine: an unsupported mode would raise instead of falling back
    sf = h.state_floats
    th, seq, lab = theta.to(DEV), inputs.contiguous().to(DEV), labels.to(DEV)
    arena = h.new_state(n, DEV)
    ckpt = torch.zeros((T + 1) * sf * n, device=DEV)
    dseq = torch.zeros(T * n, device=DEV)
    il = torch.zeros(1, dtype=torch.float64, device=DEV)
    h.unroll_fwd(th, n, T, arena, in_seq=seq, ckpt=ckpt, labels=lab, imit_loss=il, n_total=n, delta_seq=dseq)
    assert rel_err(il, loss64) <= REL_TOL
    dtheta = torch.zeros(h.n_theta, dtype=torch.float64, device=DEV)
    h.unroll_bwd(th, n, T, seq, ckpt, dtheta, labels=lab, n_total=n, delta_seq=dseq)
    torch.cuda.synchronize()
    slack = max(REL_TOL, 3.0 * rel_err(g32, g64))
    assert rel_err(dtheta, g64) <= slack, (rel_err(dtheta, g64), rel_err(g32, g64))
    with pytest.raises(Exception):   # imitation mode without the recorded deltas is not a tensor-core mode
        h.unroll_bwd(th, n, T, seq, ckpt, dtheta, labels=lab, n_total=n)


def test_tc_rnnprop_step_fused_adam_features():
    """RNNProp (DM/networks.py:279-300 + DM/meta_rnnprop_train.py:383-388) on the tensor-core engine: l2o_step with the
    fused Adam-feature mode (m, v in/out, p from a DEVICE scalar as the captured graphs use it), fc(2->20)+ELU in the
    epilogue, tanh output; three chained steps against the oracle, incl. the recorded (m~, g~) rows."""
    from open_l2o_b200.engine import ENGINE_TC
    from tests.helpers import random_state, state_to_arena
    spec = SPECS["rnnprop"]
    n = 20000 + 37
    gen = torch.Generator().manual_seed(41)
    theta = _theta(spec)
    st = random_state(spec, n, gen)
    x_ref = torch.randn(n, generator=gen)
    m_ref, v_ref = torch.zeros(n), torch.zeros(n)
    h = make_handle(spec)
    h.set_engine(ENGINE_TC)
    th = theta.to(DEV)
    a_in = state_to_arena(st, n).to(DEV)
    x = x_ref.to(DEV).clone()
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    step_dev = torch.tensor([5], dtype=torch.int32, device=DEV)
    for it in range(3):
        g = torch.randn(n, generator=gen) * (10.0 ** float(torch.randint(-4, 1, (1,), generator=gen)))
        g[::13] = 0.0
        m_ref, v_ref, mt, gt = orc.adam_features(g, m_ref, v_ref, float(5 + it), 0.95, 0.95)
        d_ref, st = orc.net_apply(spec, theta, torch.stack([mt, gt], -1), st)
        x_ref = x_ref + d_ref
        a_out = torch.zeros_like(a_in)
        delta = torch.empty(n, device=DEV)
        feat = torch.empty(2, n, device=DEV)
        h.step(th, g.to(DEV), a_in, a_out, m=m, v=v, beta1=0.95, beta2=0.95, x=x, delta=delta, feat_out=feat,
               step_ptr=step_dev, t_offset=it)
        torch.cuda.synchronize()
        assert rel_err(feat[0], mt) <= REL_TOL and rel_err(feat[1], gt) <= REL_TOL
        assert rel_err(m, m_ref) <= REL_TOL and rel_err(v, v_ref) <= REL_TOL
        assert rel_err(delta, d_ref) <= REL_TOL
        assert rel_err(x, x_ref) <= REL_TOL
        for (hg, cg), (hr, cr) in zip(arena_to_state(a_out.cpu(), spec.layers, n), st):
            assert rel_err(hg, hr) <= REL_TOL and rel_err(cg, cr) <= REL_TOL
        a_in = a_out


def test_tc_rnnprop_fused_unroll_matches_ffma():
    """RNNProp fused unroll (in-kernel separable optimizee, Adam moments carried in registers, checkpoints and
    (m~, g~) rows recorded) on the tensor-core engine vs the exact-fp32 engine, multi-tile with a ragged tail."""
    from open_l2o_b200.engine import ENGINE_FFMA, ENGINE_TC, OPT_KINDS
    spec = SPECS["rnnprop"]
    n, T = 37_979, 6
    gen = torch.Generator().manual_seed(9)
    theta = _theta(spec).to(DEV)
    a, b, x0 = (torch.randn(n, generator=gen).to(DEV) for _ in range(3))
    outs = {}
    for eng in (ENGINE_FFMA, ENGINE_TC):
        h = make_handle(spec)
        h.set_engine(eng)
        arena = h.new_state(n, DEV)
        x = x0.clone()
        m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        fx = torch.zeros(T + 1, dtype=torch.float64, device=DEV)
        g_rec = torch.empty(T + 1, n, device=DEV)
        feat = torch.empty(T, 2, n, device=DEV)
        ckpt = torch.zeros((T + 1) * h.state_floats * n, device=DEV)
        h.unroll_fwd(theta, n, T, arena, opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=a, opt_b=b, opt_alpha=10.0,
                     opt_fscale=1.0 / n, x=x, ckpt=ckpt, m=m, v=v, beta1=0.95, beta2=0.95, step0=3, g_rec=g_rec,
                     feat_rec=feat, fx=fx)
        torch.cuda.synchronize()
        outs[eng] = (x, arena, fx, g_rec, feat, m, v, ckpt)
    for u, w in zip(outs[ENGINE_TC], outs[ENGINE_FFMA]):
        assert rel_err(u, w) <= REL_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("n,T", [(19021, 5), (38188, 20), (100, 3)])
def test_tc_rnnprop_bptt_two_pass_matches_ffma(n, T):
    """RNNProp (fc(20) + ELU, tanh output) BPTT on the tensor-core engine — layer-2 pass, hand-over buffer, layer-1 pass
    with the fc layer's own gradient — against the exact-fp32 engine on the same checkpoints, features and deltas
    (DM/networks.py:279-300, DM/meta.py:319-376).  Several tiles per CTA and a ragged tail."""
    from open_l2o_b200.engine import ENGINE_FFMA, ENGINE_TC, OPT_KINDS
    spec = SPECS["rnnprop"]
    gen = torch.Generator().manual_seed(31)
    theta = _theta(spec, gain=0.3).to(DEV)
    a, b, x0 = (torch.randn(n, generator=gen).to(DEV) for _ in range(3))
    h = make_handle(spec)
    h.set_engine(ENGINE_FFMA)
    arena = h.new_state(n, DEV)
    x = x0.clone()
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    g_rec = torch.empty(T + 1, n, device=DEV)
    feat = torch.empty(T, 2, n, device=DEV)
    dseq = torch.empty(T, n, device=DEV)
    ckpt = torch.zeros((T + 1) * h.state_floats * n, device=DEV)
    h.unroll_fwd(theta, n, T, arena, opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=a, opt_b=b, opt_alpha=10.0,
                 opt_fscale=1.0 / n, x=x, ckpt=ckpt, m=m, v=v, beta1=0.95, beta2=0.95, step0=1, g_rec=g_rec,
                 feat_rec=feat, delta_seq=dseq)
    outs = {}
    for eng in (ENGINE_FFMA, ENGINE_TC):
        h.set_engine(eng)
        d = torch.zeros(h.n_theta, dtype=torch.float64, device=DEV)
        kw = {}
        if eng == ENGINE_TC:
            kw = dict(delta_seq=dseq, scratch=torch.empty(T, n, 20, device=DEV))
        h.unroll_bwd(theta, n, T, feat, ckpt, d, g_rec=g_rec, **kw)
        torch.cuda.synchronize()
        outs[eng] = d
    ref = outs[ENGINE_FFMA]
    assert float(ref.abs().max()) > 0
    # every block of theta on its own scale (the fc layer's gradient is orders of magnitude below the LSTM's)
    off = 0
    for name, cnt in (("fc_w", 40), ("fc_b", 20), ("w1", 40 * 80), ("b1", 80), ("w2", 40 * 80), ("b2", 80), ("wo", 20), ("bo", 1)):
        u, w = outs[ENGINE_TC][off:off + cnt], ref[off:off + cnt]
        assert rel_err(u, w) <= 2e-5, (name, rel_err(u, w))
        off += cnt
    assert off == h.n_theta
    with pytest.raises(Exception):   # without the hand-over buffer the tensor-core engine refuses an fc net
        h.unroll_bwd(theta, n, T, feat, ckpt, torch.zeros_like(ref), g_rec=g_rec, delta_seq=dseq)


@pytest.mark.gpu
def test_tc_bptt_tanh_output_net_uses_recorded_deltas():
    """A tanh-output DM net (DM/networks.py:227-232) on the tensor-core BPTT: tanh' of the output layer comes
    from the deltas the forward pass recorded; against the exact-fp32 engine (which recomputes y) on the same checkpoints.
    Without the recorded deltas the tensor-core engine refuses such a net."""
    import dataclasses
    from open_l2o_b200.engine import ENGINE_FFMA, ENGINE_TC
    spec = dataclasses.replace(SPECS["dm_logsign"], tanh_output=True, scale=0.5)
    n, T = 19_005, 6
    gen = torch.Generator().manual_seed(17)
    theta = _theta(spec, gain=0.6).to(DEV)
    from tests.helpers import wild_gradients
    g_rec = torch.stack([wild_gradients(n, gen) for _ in range(T + 1)]).to(DEV)
    h = make_handle(spec)
    h.set_engine(ENGINE_FFMA)
    arena = h.new_state(n, DEV)
    ckpt = torch.zeros((T + 1) * h.state_floats * n, device=DEV)
    dseq = torch.empty(T, n, device=DEV)
    h.unroll_fwd(theta, n, T, arena, in_seq=g_rec[:T].contiguous(), ckpt=ckpt, delta_seq=dseq)
    assert float(dseq.abs().max()) > 0.05 * spec.scale     # the output layer is really in its nonlinear range
    outs = {}
    for eng in (ENGINE_FFMA, ENGINE_TC):
        h.set_engine(eng)
        d = torch.zeros(h.n_theta, dtype=torch.float64, device=DEV)
        h.unroll_bwd(theta, n, T, g_rec[:T].contiguous(), ckpt, d, g_rec=g_rec, delta_seq=dseq)
        torch.cuda.synchronize()
        outs[eng] = d
    assert rel_err(outs[ENGINE_TC], outs[ENGINE_FFMA]) <= REL_TOL
    with pytest.raises(Exception):
        h.unroll_bwd(theta, n, T, g_rec[:T].contiguous(), ckpt, torch.zeros_like(outs[ENGINE_TC]), g_rec=g_rec)
