"""Segmented BPTT: l2o_unroll_bwd_carry chains against one l2o_unroll_bwd, recomputed checkpoints against the
forward's, and MetaOptimizer with forced segment lengths against the unsegmented program.

The per-coordinate arithmetic of a chain of segments is the whole sweep's: the carried adjoint state and lambda pass
through HBM exactly, and lambda keeps the summation order of one sweep.  So the carries a chain hands on are bitwise
those of one sweep.  dtheta is not bitwise: both engines sum dW over a CTA's steps in fp32 before the fp64 atomics
(the exact-fp32 engine in shared memory over the whole launch, the tensor-core engine per 64-coordinate tile), and a
segment boundary ends such a sum early.  dtheta is therefore compared at DTHETA_TOL; a single segment with a zero carry
groups every sum as l2o_unroll_bwd does and is compared at fp64-atomic reordering level."""
import numpy as np
import pytest
import torch

from oracle import l2o_oracle as orc
from tests.helpers import REL_TOL, SPECS, assert_theta_close, make_handle, rel_err

pytestmark = pytest.mark.gpu

DTHETA_TOL = 2e-5
ATOMIC_TOL = 1e-12

KERNEL_SPECS = {
    "identity": SPECS["dm_identity"],
    "logsign": SPECS["dm_logsign"],
    "rnnprop": SPECS["rnnprop"],
    "tanh": orc.NetSpec(layers=(20, 20), scale=0.1, tanh_output=True),
}


def _forward(spec, n, T, seed):
    """A fused Rastrigin unroll recording everything a BPTT reads: checkpoints, g_rec, the deltas, RNNProp's features."""
    from open_l2o_b200.engine import OPT_KINDS
    h = make_handle(spec)
    g = torch.Generator().manual_seed(seed)
    theta = orc.init_theta(spec, seed=seed, out_gain=0.05).cuda()
    a, b, x = (torch.randn(n, generator=g).cuda() for _ in range(3))
    state = h.new_state(n, "cuda")
    ckpt = torch.zeros((T + 1) * h.state_size(n), device="cuda")
    g_rec = torch.zeros(T + 1, n, device="cuda")
    delta = torch.zeros(T, n, device="cuda")
    kw, in_seq = {}, g_rec
    if h.n_in == 2:
        in_seq = torch.zeros(T, 2, n, device="cuda")
        kw = dict(m=torch.zeros(n, device="cuda"), v=torch.zeros(n, device="cuda"), step0=1, feat_rec=in_seq)
    h.unroll_fwd(theta, n, T, state, opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=a, opt_b=b, opt_alpha=10.0,
                 opt_fscale=1.0 / n, x=x, ckpt=ckpt, g_rec=g_rec, delta_seq=delta, **kw)
    return h, theta, ckpt, g_rec, delta, in_seq


def _chain(h, theta, n, bounds, ckpt, g_rec, delta, in_seq, scratch):
    """l2o_unroll_bwd_carry over the segments [bounds[k], bounds[k+1]), last first, from a zero carry."""
    slot = h.state_size(n)
    dth = torch.zeros(h.n_theta, dtype=torch.float64, device="cuda")
    d_state = torch.zeros(slot, device="cuda")
    lam = torch.zeros(n, device="cuda")
    for t0, t1 in reversed(list(zip(bounds[:-1], bounds[1:]))):
        h.unroll_bwd_carry(theta, n, t1 - t0, in_seq[t0:], ckpt[t0 * slot:], dth, d_state, lam, g_rec=g_rec[t0:],
                           delta_seq=delta[t0:], scratch=scratch)
    return dth, d_state, lam


@pytest.mark.parametrize("engine", ["ffma", "tc"])
@pytest.mark.parametrize("net", list(KERNEL_SPECS))
def test_carry_chain_matches_one_sweep(engine, net):
    from open_l2o_b200.engine import ENGINE_FFMA, ENGINE_TC
    spec = KERNEL_SPECS[net]
    n, T = 3001, 9   # a ragged last tile on both engines
    h, theta, ckpt, g_rec, delta, in_seq = _forward(spec, n, T, seed=3)
    h.set_engine(ENGINE_FFMA if engine == "ffma" else ENGINE_TC)
    scratch = torch.zeros(T, n, 20, device="cuda") if h.n_in == 2 else None
    ref = torch.zeros(h.n_theta, dtype=torch.float64, device="cuda")
    h.unroll_bwd(theta, n, T, in_seq, ckpt, ref, g_rec=g_rec, delta_seq=delta, scratch=scratch)
    one, d_state1, lam1 = _chain(h, theta, n, [0, T], ckpt, g_rec, delta, in_seq, scratch)
    torch.cuda.synchronize()
    assert rel_err(one, ref) <= ATOMIC_TOL
    # the carry out of a whole sweep: lambda = sum_{tau > 0} g_tau, and an adjoint state that is not trivially zero
    assert rel_err(lam1, g_rec[1:].double().sum(0)) <= 1e-5
    assert float(d_state1.abs().max()) > 0
    for bounds in ([0, 1, T], [0, T - 1, T], [0, 2, 6, T], list(range(T + 1))):
        dth, d_state, lam = _chain(h, theta, n, bounds, ckpt, g_rec, delta, in_seq, scratch)
        torch.cuda.synchronize()
        assert torch.equal(d_state, d_state1) and torch.equal(lam, lam1), bounds
        assert rel_err(dth, ref) <= DTHETA_TOL, (bounds, rel_err(dth, ref))


# ---------------------------------------------------------------------------------------------------------------
# MetaOptimizer
# ---------------------------------------------------------------------------------------------------------------
DM = {"net": "CoordinateWiseDeepLSTM", "net_options": {"layers": (20, 20), "scale": 0.1}}
DM_LOGSIGN = {"net": "CoordinateWiseDeepLSTM", "net_options": {"layers": (20, 20), "preprocess_name": "LogAndSign",
                                                              "preprocess_options": {"k": 5}, "scale": 0.01}}
RNNPROP = {"net": "RNNprop", "net_options": {"layers": (20, 20), "preprocess_name": "fc", "preprocess_options": {"dim": 20},
                                             "scale": 0.01, "tanh_output": True}}


def _workload(name):
    """(optimizer class name, net config, problem, net_assignments, regime)."""
    from open_l2o_b200 import problems
    return {
        "rastrigin_fused": ("MetaOptimizer", {"cw": DM}, problems.rastrigin_separable(num_dims=3000), None, "fused"),
        "quadratic_diag_fused": ("MetaOptimizer", {"cw": DM}, problems.quadratic_diag(num_dims=2000), None, "fused"),
        "quadratic_external": ("MetaOptimizer", {"cw": DM}, problems.quadratic(batch_size=16, num_dims=10), None,
                               "external"),
        "mlp_external": ("MetaOptimizer", {"cw": DM_LOGSIGN}, problems.mlp(layers=(12,), in_dim=20, n_classes=5,
                                                                           batch_size=16), None, "external"),
        "lasso_producer": ("MetaOptimizer", {"cw": DM}, problems.lasso(batch_size=16, num_dims=10), None, "external"),
        "rnnprop_fused": ("RNNpropMetaOptimizer", {"rp": RNNPROP}, problems.rastrigin_separable(num_dims=3000), None,
                          "fused"),
        "rnnprop_external": ("RNNpropMetaOptimizer", {"rp": RNNPROP},
                             problems.mlp(layers=(12,), in_dim=20, n_classes=5, batch_size=16), None, "external"),
        "two_nets": ("MetaOptimizer", {"a": DM, "b": DM_LOGSIGN}, problems.simple_multi_optimizer(num_dims=3),
                     [("a", ["x_0", "x_2"]), ("b", ["x_1"])], "external"),
        "random_scaling": ("MetaOptimizer", {"cw": DM}, problems.quadratic(batch_size=16, num_dims=10), None, "scaled"),
    }[name]


def _program(name, T, segment):
    from open_l2o_b200 import meta
    cls, cfg, problem, assign, regime = _workload(name)
    kw = dict(cfg) if segment is None else dict(cfg, _bptt_segment=segment)
    opt = getattr(meta, cls)(**kw)
    ms = opt.meta_minimize(problem, T, learning_rate=0.003, net_assignments=assign)
    prog = opt.program
    assert (prog.fused is not None) == (regime == "fused"), name
    meta.Session().run(ms.reset)
    return opt, ms, prog


def _feed(name, opt, prog, it, T):
    feed = {opt.step_placeholder: it * T + 1}
    if _workload(name)[4] == "scaled":
        g = torch.Generator().manual_seed(10 + it)
        for p, v in zip(prog.scale_placeholders, prog.variables):
            feed[p] = np.exp(torch.rand(v["shape"], generator=g).numpy() * 2 - 1)
    return feed


@pytest.mark.parametrize("S", [1, 3, 7, 10])
@pytest.mark.parametrize("name", ["rastrigin_fused", "quadratic_diag_fused", "quadratic_external", "mlp_external",
                                  "lasso_producer", "rnnprop_fused", "rnnprop_external", "two_nets", "random_scaling"])
def test_meta_optimizer_segments_match_full(name, S):
    """Three training unrolls (the third replays the captured graph in the external regime).  Before each unroll the
    segmented program takes the full program's theta and Adam slots, so every unroll starts from the same point: fx,
    x and the committed state are bitwise equal (fx up to its fp64 atomics), dtheta and theta within DTHETA_TOL.  On the
    first unroll every recomputed checkpoint slot is bitwise the full program's."""
    from open_l2o_b200 import meta
    T = 10
    opt_a, ms_a, full = _program(name, T, None)
    opt_b, ms_b, seg = _program(name, T, S)
    assert not full.segmented and seg.segmented == (S < T)
    sess = meta.Session()
    for it in range(3):
        theta_before = {k: net.theta.clone() for k, net in full.nets.items()}
        for k in full.nets:
            seg.nets[k].theta.copy_(full.nets[k].theta)
            for s in ("m", "v"):
                seg.adam[k][s].copy_(full.adam[k][s])
        out_a = sess.run([ms_a.fx, ms_a.x, ms_a.update, ms_a.step], feed_dict=_feed(name, opt_a, full, it, T))
        out_b = sess.run([ms_b.fx, ms_b.x, ms_b.update, ms_b.step], feed_dict=_feed(name, opt_b, seg, it, T))
        torch.cuda.synchronize()
        assert rel_err(seg.last_fx, full.last_fx) <= ATOMIC_TOL, it
        for xa, xb in zip(out_a[1], out_b[1]):
            assert np.array_equal(xa, xb), it
        assert torch.equal(seg.X, full.X), it
        for ra, rb in zip(full.runs, seg.runs):
            assert torch.equal(ra.state, rb.state), it
            if ra.net.handle.n_in == 2:
                assert torch.equal(ra.m, rb.m) and torch.equal(ra.v, rb.v), it
        for k in full.nets:
            d = full.dtheta[k]
            assert rel_err(seg.dtheta[k], d) <= DTHETA_TOL, (it, k)
            # Adam's first moves are ~ lr sign(g): entries whose gradient is at round-off level may step differently
            big = d.abs() > 1e-4 * float(d.abs().max())
            assert rel_err(seg.nets[k].theta[big], full.nets[k].theta[big]) <= DTHETA_TOL, (it, k)
        if it == 0 and seg.segmented:
            # recompute every segment again from the boundary store, at the theta the unroll ran with
            theta_after = {k: net.theta.clone() for k, net in seg.nets.items()}
            for k in seg.nets:
                seg.nets[k].theta.copy_(theta_before[k])
            for ra, rb in zip(full.runs, seg.runs):
                for j, (t0, t1) in enumerate(zip(seg.plan.bounds[:-1], seg.plan.bounds[1:])):
                    seg._recompute(rb, j)
                    torch.cuda.synchronize()
                    assert torch.equal(rb.ckpt[:(t1 - t0 + 1) * rb.slot],
                                       ra.ckpt[t0 * ra.slot:(t1 + 1) * ra.slot]), (j, t0, t1)
            for k in seg.nets:
                seg.nets[k].theta.copy_(theta_after[k])


def test_segmented_training_matches_oracle():
    """Fused Rastrigin with segments of 3 steps over T = 10 against the oracle's autograd trainer, three unrolls."""
    from open_l2o_b200 import meta, problems
    n, T = 3000, 10
    optimizer = meta.MetaOptimizer(cw=DM, _bptt_segment=3)
    step, update, reset, fx, x = optimizer.meta_minimize(problems.rastrigin_separable(num_dims=n), T,
                                                         learning_rate=0.001)
    prog = optimizer.program
    assert prog.segmented and prog.plan.bounds == [0, 3, 6, 9, 10]
    sess = meta.Session()
    sess.run(reset)
    spec = orc.NetSpec(layers=(20, 20), scale=0.1)
    prob = orc.FusedProblem("rastrigin_sep", prog.const_vals["b"].cpu(), prog.const_vals["c"].cpu(), alpha=10.0,
                            fscale=1.0 / n)
    tr = orc.MetaTrainerOracle(spec, next(iter(prog.nets.values())).theta.cpu().clone(), None, lr=0.001,
                               grad_of=prob.f_and_g)
    tr.reset(prog.X.cpu().clone())
    for it in range(3):
        cost, xs, _, _ = sess.run([fx, x, update, step])
        res = tr.run_unroll(T)
        assert abs(cost - float(res.fx[-1])) <= 1e-5 * abs(float(res.fx[-1]))
        assert rel_err(xs[0], res.x_final) <= REL_TOL
        assert_theta_close(next(iter(prog.nets.values())).theta, tr, it)
