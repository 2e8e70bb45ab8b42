"""GPU tests of the confocal_microscopy_3d producer (l2o_confocal_grad, DM/problems.py:701-956) and of meta-training
the two registry problems it came with (DM/util.py:215-230) against the oracle."""
import types

import numpy as np
import pytest
import torch

from oracle import l2o_oracle as orc
from tests import confocal_oracle as co
from tests.helpers import REL_TOL, assert_theta_close, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("B,P,roi", [(32, 5, (28, 28, 28)), (3, 1, (5, 7, 9)), (1, 8, (32, 32, 32))])
@pytest.mark.parametrize("scaled", [False, True])
def test_confocal_grad_matches_fp64_autograd(B, P, roi, scaled):
    """f and df/dx in one launch vs autograd of the oracle's dense loss in fp64.  theta spans [-0.2, 1.2]: the quantile
    map extrapolates linearly outside [0, 1].  With ``scale`` the kernel sees x = theta / scale, as run_epoch feeds the
    random-scaling trick (DM/util.py:40-54)."""
    from open_l2o_b200 import engine
    gen = torch.Generator().manual_seed(11 + P)
    rows = 6 * P + 1
    theta = torch.rand(rows, B, generator=gen) * 1.4 - 0.2
    sim = torch.rand(rows, B, generator=gen)
    sc = torch.exp(torch.rand(rows, B, generator=gen) * 6 - 3) if scaled else None
    x = theta / sc if scaled else theta
    xd = x.double().requires_grad_(True)
    f_ref = co.confocal_f(xd * sc.double() if scaled else xd, sim.double(), B, P, roi)
    (g_ref,) = torch.autograd.grad(f_ref, xd)
    g = torch.empty(rows * B, device=DEV)
    f = torch.zeros((), dtype=torch.float64, device=DEV)
    engine.confocal_grad(x.reshape(-1).to(DEV), sim.to(DEV), g, B, P, roi, f=f,
                         scale=sc.reshape(-1).to(DEV) if scaled else None)
    torch.cuda.synchronize()
    f_ref = float(f_ref.detach())
    assert abs(float(f) - f_ref) <= REL_TOL * abs(f_ref), (float(f), f_ref)
    assert rel_err(g, g_ref) <= REL_TOL, rel_err(g, g_ref)


def _flat(xs):
    return np.concatenate([np.asarray(a).reshape(-1) for a in xs])


def _train_confocal(monkeypatch, disable_fused, graphs=True, T=20):
    """get_config("confocal_microscopy_3d") meta-trained for three unrolls, then reset and two more.  Returns the
    initial theta, x and simulated constants, and per unroll (fx, x, theta, library launches)."""
    from open_l2o_b200 import engine, meta, util
    monkeypatch.setenv("L2O_DISABLE_FUSED", "1" if disable_fused else "0")
    monkeypatch.setenv("L2O_CUDA_GRAPH", "1" if graphs else "0")
    problem, net_config, net_assignments = util.get_config("confocal_microscopy_3d")
    optimizer = meta.MetaOptimizer(**net_config)
    ms = optimizer.meta_minimize(problem, T, learning_rate=0.001, net_assignments=net_assignments)
    prog = optimizer.program
    theta0 = next(iter(prog.nets.values())).theta.cpu().clone()
    sess = meta.Session()
    sess.run(ms.reset)
    x0 = prog.X.cpu().clone()
    sim0 = torch.stack([prog.const_vals[c["name"]].reshape(-1).cpu() for c in prog.constants])
    out = []
    for it in range(5):
        if it == 3:
            sess.run(ms.reset)
        n0 = engine.launch_count()
        cost, xs, _, _ = sess.run([ms.fx, ms.x, ms.update, ms.step])
        torch.cuda.synchronize()
        out.append((cost, _flat(xs), next(iter(prog.nets.values())).theta.cpu().clone(), engine.launch_count() - n0))
    return prog, (theta0, x0, sim0), out


def test_confocal_bound_producer_matches_autograd_and_oracle(monkeypatch):
    T = 20
    prog, init, fused = _train_confocal(monkeypatch, False, T=T)
    assert prog.producer is not None and prog.producer.kind == "confocal_psf"
    # the simulated constants are rows of the one buffer the kernel reads
    assert all(prog.const_vals[n].data_ptr() == prog.producer.sim[k].data_ptr()
               for k, n in enumerate(prog.producer.constants))
    prog_ag, init_ag, autograd = _train_confocal(monkeypatch, True, T=T)
    assert prog_ag.producer is None and not prog_ag._graph_failed and True in prog_ag._graphs
    assert all(torch.equal(a, b) for a, b in zip(init, init_ag))
    theta0, x0, sim0 = init
    # an eager unroll (the first two) runs the same library kernels on both paths plus one producer launch per gradient
    for it in range(2):
        assert fused[it][3] - autograd[it][3] == T + 1, (fused[it][3], autograd[it][3])
    for it in range(5):
        (c, x, th, _), (ca, xa, tha, _) = fused[it], autograd[it]
        assert abs(c - ca) <= REL_TOL * abs(ca), (it, c, ca)
        assert rel_err(x, xa) <= REL_TOL, (it, rel_err(x, xa))

    B, P, roi = 32, 5, (28, 28, 28)
    spec = orc.NetSpec(layers=(20, 20))
    with torch.device(DEV):   # the oracle's torch ops, run on the device for speed
        sim = sim0.to(DEV)
        tr = orc.MetaTrainerOracle(spec, theta0.to(DEV), lambda x: co.confocal_f(x, sim, B, P, roi), lr=0.001)
        tr.reset(x0.to(DEV))
        for it in range(3):
            res = tr.run_unroll(T)
            ref_fx, ref_x = float(res.fx[-1]), res.x_final.detach().cpu()
            for c, x, th, _ in (fused[it], autograd[it]):
                assert abs(c - ref_fx) <= REL_TOL * abs(ref_fx), (it, c, ref_fx)
                assert rel_err(x, ref_x) <= REL_TOL, (it, rel_err(x, ref_x))
            tr_cpu = types.SimpleNamespace(theta=tr.theta.cpu(), last_grad=tr.last_grad.cpu())
            assert_theta_close(fused[it][2], tr_cpu, it)
            assert_theta_close(autograd[it][2], tr_cpu, it)


def test_confocal_graph_replay_after_reset_equals_eager(monkeypatch):
    """Unroll 3 is captured into a CUDA graph and unrolls 4-5 replay it after a reset refilled x and the simulated
    constants in place; an all-eager run gives the same numbers.  They differ only through the fp64 atomics of fx and
    of the BPTT's dtheta, whose order is not fixed."""
    prog, _, graph = _train_confocal(monkeypatch, False, graphs=True)
    assert not prog._graph_failed and True in prog._graphs
    _, _, eager = _train_confocal(monkeypatch, False, graphs=False)
    for it in range(5):
        (c, x, th, _), (ce, xe, the, _) = graph[it], eager[it]
        assert abs(c - ce) <= 1e-9 * abs(ce), (it, c, ce)
        assert rel_err(x, xe) <= 1e-6 and rel_err(th, the) <= 1e-6, (it, rel_err(x, xe), rel_err(th, the))


def test_square_cos_training_matches_oracle():
    """get_config("square_cos"): 128 x 2 coordinates on the graph-captured autograd path, three T = 20 unrolls."""
    from open_l2o_b200 import meta, util
    T = 20
    problem, net_config, net_assignments = util.get_config("square_cos")
    optimizer = meta.MetaOptimizer(**net_config)
    ms = optimizer.meta_minimize(problem, T, learning_rate=0.001, net_assignments=net_assignments)
    prog = optimizer.program
    assert prog.fused is None and prog.producer is None
    sess = meta.Session()
    sess.run(ms.reset)
    w, y, wcos = (prog.const_vals[k].cpu() for k in ("w", "y", "wcos"))
    tr = orc.MetaTrainerOracle(orc.NetSpec(layers=(20, 20)), next(iter(prog.nets.values())).theta.cpu().clone(),
                               lambda x: co.square_cos_f(x, w, y, wcos), lr=0.001)
    tr.reset(prog.X.cpu().clone().reshape(128, 2))
    for it in range(3):
        cost, xs, _, _ = sess.run([ms.fx, ms.x, ms.update, ms.step])
        res = tr.run_unroll(T)
        assert abs(cost - float(res.fx[-1])) <= REL_TOL * abs(float(res.fx[-1])), (it, cost, float(res.fx[-1]))
        assert rel_err(xs[0], res.x_final) <= REL_TOL
        assert_theta_close(next(iter(prog.nets.values())).theta, tr, it)
