"""Training-trajectory parity at the BASELINE configs' OWN shapes (VERDICT r1 "untested configs"): Lasso m=250 n=500
unroll 100 (config #2), the target-line net (LogAndSign k=5, scale 0.01, MLP optimizee, external-gradient regime with
CUDA-graph replay), RNNProp on the 784-100-10 MLP (config #3).  Every run goes through the public
``MetaOptimizer.meta_minimize`` + ``Session.run([fx, x, update, step])`` surface and is compared with the CPU oracle
(``MetaTrainerOracle`` = DM/meta.py:319-414 + DM/util.py:31-75) on identical tensors."""
import numpy as np
import pytest
import torch

from oracle import l2o_oracle as orc
from tests.helpers import REL_TOL, assert_theta_close, rel_err

pytestmark = pytest.mark.gpu


def _net(prog):
    return next(iter(prog.nets.values()))


def _lasso_data(B, seed=2, m=250, n=500):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(B, m, n, generator=g) / (m ** 0.5)      # DM/problems.py:137-175 caller's synthetic data
    b = torch.randn(B, m, 1, generator=g)
    return A, b


def test_lasso_m250_n500_T100_training_trajectory():
    """BASELINE config #2's optimizee shape (m=250, n=500, unroll 100) on a batch the oracle's autograd BPTT finishes
    in seconds: 3 x (unroll + BPTT + TF-Adam + carry-over) against the oracle."""
    from open_l2o_b200 import meta, problems
    B, T = 8, 100
    A, b = _lasso_data(B)
    optimizer = meta.MetaOptimizer(cw={"net": "CoordinateWiseDeepLSTM", "net_options": {"layers": (20, 20), "scale": 0.1}})
    ms = optimizer.meta_minimize(problems.lasso_fixed(A, b), T, learning_rate=0.001)
    prog = optimizer.program
    sess = meta.Session()
    sess.run(ms.reset)
    spec = orc.NetSpec(layers=(20, 20), scale=0.1)
    tr = orc.MetaTrainerOracle(spec, _net(prog).theta.cpu().clone(), lambda x: orc.lasso_f(x, A, b), lr=0.001)
    tr.reset(prog.X.cpu().clone().reshape(B, 500))
    for it in range(3):
        cost, xs, _, _ = sess.run([ms.fx, ms.x, ms.update, ms.step])
        res = tr.run_unroll(T)
        assert abs(cost - float(res.fx[-1])) <= REL_TOL * abs(float(res.fx[-1])), it
        assert rel_err(xs[0], res.x_final) <= REL_TOL, it
        assert_theta_close(_net(prog).theta, tr, it)


def test_lasso_full_size_B128_unrolls():
    """BASELINE config #2 at its FULL size (B=128 -> 64,000 coordinates, T=100), two training unrolls.  The oracle's
    autograd graph does not fit at this size, so: x_T and every f(x_t) against the oracle's no-grad unroll driven by
    the engine's own theta; d-theta of the tensor-core BPTT against the exact-fp32 engine on the same checkpoints
    (that engine is checked against the oracle's autograd at B=8 above and in test_kernels_gpu); theta against
    TF-Adam applied by the oracle to that d-theta."""
    from open_l2o_b200 import meta, problems
    from open_l2o_b200.engine import ENGINE_AUTO, ENGINE_FFMA
    B, T = 128, 100
    A, b = _lasso_data(B)
    optimizer = meta.MetaOptimizer(cw={"net": "CoordinateWiseDeepLSTM", "net_options": {"layers": (20, 20), "scale": 0.1}})
    ms = optimizer.meta_minimize(problems.lasso_fixed(A, b), T, learning_rate=0.001)
    prog = optimizer.program
    sess = meta.Session()
    sess.run(ms.reset)
    spec = orc.NetSpec(layers=(20, 20), scale=0.1)
    net = _net(prog)
    x = prog.X.cpu().clone().reshape(B, 500)
    state = orc.initial_state(spec, B * 500)
    m, v = torch.zeros(net.theta.numel()), torch.zeros(net.theta.numel())
    r = prog.runs[0]
    for it in range(2):
        theta_k = net.theta.cpu().clone()
        cost, xs, _, _ = sess.run([ms.fx, ms.x, ms.update, ms.step])
        with torch.no_grad():
            res = orc.unroll(spec, theta_k, x, state, lambda z: orc.lasso_f(z, A, b), T)
        assert abs(cost - float(res.fx[-1])) <= REL_TOL * abs(float(res.fx[-1])), it
        assert abs(float(prog.last_fx.sum()) - float(res.loss)) <= REL_TOL * abs(float(res.loss)), it
        assert rel_err(xs[0], res.x_final) <= REL_TOL, it
        assert rel_err(prog.last_fx, res.fx) <= REL_TOL, it
        # same checkpoints / recorded gradients through the exact-fp32 BPTT, (a) in one launch and (b) in 1,000-
        # coordinate chunks summed in fp64 (no long fp32 accumulation anywhere) = the reference.  This gradient is a
        # sum of 6.4 M terms with heavy cancellation (|dtheta| up to 2e5): the bar is 1e-5, or 3x the distance the
        # exact-fp32 engine itself has from the reference when that is larger.
        d_auto = prog.dtheta[r.key].clone()
        hnd = r.net.handle
        hnd.set_engine(ENGINE_FFMA)
        d_ffma = torch.zeros_like(d_auto)
        hnd.unroll_bwd(theta_k.cuda(), r.n, T, r.g_rec, r.ckpt, d_ffma, g_rec=r.g_rec)
        d_ref = torch.zeros_like(d_auto)
        ck4 = r.ckpt.view(T + 1, 4, r.n, 20)
        for lo in range(0, r.n, 1000):
            hi = min(r.n, lo + 1000)
            hnd.unroll_bwd(theta_k.cuda(), hi - lo, T, r.g_rec[:, lo:hi].contiguous(),
                           ck4[:, :, lo:hi, :].contiguous().view(-1), d_ref, g_rec=r.g_rec[:, lo:hi].contiguous())
        hnd.set_engine(ENGINE_AUTO)
        torch.cuda.synchronize()
        e_tc, e_ff = rel_err(d_auto, d_ref), rel_err(d_ffma, d_ref)
        assert e_tc <= max(REL_TOL, 3.0 * e_ff), (it, e_tc, e_ff)
        theta_ref, m, v = orc.tf_adam_step(theta_k, d_auto.float().cpu(), m, v, it + 1, lr=0.001)
        big = d_ref.abs().cpu() > 1e-4 * float(d_ref.abs().max())
        assert rel_err(net.theta.cpu()[big], theta_ref[big]) <= REL_TOL, it
        x, state = res.x_final, res.state_final


def _mlp_f(prog, hidden_act=torch.sigmoid):
    data, labels = prog.const_vals["data"], prog.const_vals["labels"]
    shapes = [v["shape"] for v in prog.variables]

    def f(xflat):
        d, l = data.cpu().to(xflat.dtype), labels.cpu().long()
        off, ts = 0, []
        for s in shapes:
            k = int(np.prod(s))
            ts.append(xflat[off:off + k].view(s))
            off += k
        h = d
        for li in range(0, len(ts) - 2, 2):
            h = hidden_act(h @ ts[li] + ts[li + 1])
        return torch.nn.functional.cross_entropy(h @ ts[-2] + ts[-1], l)
    return f


def test_target_line_net_training_trajectory_with_graph_replay_and_reset():
    """The north-star target line's configuration (DM/util.py:99-109: LogAndSign k=5, scale 0.01, LSTM-20x2) on the
    reference's own MNIST-MLP shape 784-20-10 (DM/problems.py:254-288; 15,910 coordinates), unroll 20, external-gradient
    regime.  Five training unrolls: calls 1-2 run eagerly, call 3 is captured into a CUDA graph, calls 4-5 REPLAY it -
    so the replay is what is compared.  Then ``reset`` (new x, new data/labels written in place) and two more unrolls
    replayed from the same graph must follow the oracle on the NEW problem instance (ADVICE r1: stale constants)."""
    from open_l2o_b200 import meta, problems, util
    T = 20
    optimizer = meta.MetaOptimizer(cw=util.get_default_net_config(None))
    ms = optimizer.meta_minimize(problems.mlp(layers=(20,)), T, learning_rate=0.001)
    prog = optimizer.program
    assert prog.N == 784 * 20 + 20 + 20 * 10 + 10 and prog.fused is None
    sess = meta.Session()
    spec = orc.NetSpec(layers=(20, 20), preprocess_name="LogAndSign", preprocess_options={"k": 5}, scale=0.01)
    tr = orc.MetaTrainerOracle(spec, _net(prog).theta.cpu().clone(), None, lr=0.001)
    for epoch, n_unrolls in enumerate([5, 2]):
        sess.run(ms.reset)
        tr.f = _mlp_f(prog)                       # closes over the CURRENT constants
        tr.reset(prog.X.cpu().clone())
        for it in range(n_unrolls):
            cost, xs, _, _ = sess.run([ms.fx, ms.x, ms.update, ms.step])
            res = tr.run_unroll(T)
            tag = (epoch, it)
            assert abs(cost - float(res.fx[-1])) <= REL_TOL * abs(float(res.fx[-1])), tag
            assert rel_err(np.concatenate([a.reshape(-1) for a in xs]), res.x_final) <= REL_TOL, tag
            assert_theta_close(_net(prog).theta, tr, tag)
    assert True in prog._graphs, "the training unroll was never captured into a CUDA graph"


def test_rnnprop_mlp_784_100_10_training_trajectory():
    """BASELINE config #3 at its own size: RNNProp (fc(2->20)+ELU, tanh output, scale 0.01, beta 0.95) on the
    784-100-10 sigmoid MLP (79,510 coordinates), unroll 20: two training unrolls with the ``step`` placeholder fed as
    DM/util.py:59-60 does, then one evaluation unroll (no meta-step)."""
    from open_l2o_b200 import meta_rnnprop_train, problems, util
    T = 20
    _, net_config, _ = util.get_config("mlp", net_name="RNNprop")
    optimizer = meta_rnnprop_train.MetaOptimizer(0, 0.95, 0.95, **net_config)
    ms, scale, var_x, constants, subsets, seq_step, *_mt = optimizer.meta_minimize(
        problems.mlp(layers=(100,)), T, learning_rate=0.001)
    prog = optimizer.program
    assert prog.N == 79510
    sess = meta_rnnprop_train.Session()
    sess.run(ms.reset)
    spec = orc.NetSpec(layers=(20, 20), preprocess_name="fc", preprocess_options={"dim": 20}, scale=0.01,
                       tanh_output=True, rnnprop=True)
    # RNNProp divides every gradient by its own running magnitude, so for the many coordinates of this MLP whose
    # gradient sits at 1e-7..1e-9 the last-bit differences between cuBLAS and the CPU's matmul are amplified to
    # percent-level differences of g~ (measured: x differs by 6e-5 with EITHER engine when each side differentiates
    # the optimizee itself).  "Identical inputs" (SURVEY.md 8(c)) therefore means identical gradient tensors: the oracle
    # replays the gradients the engine recorded, f(x) itself stays the oracle's own.
    f_cpu = _mlp_f(prog)
    rec = {"t": 0}

    def grad_of(xflat):
        g = prog.runs[0].g_rec[min(rec["t"], T)].detach().cpu().clone()
        rec["t"] += 1
        return f_cpu(xflat), g

    tr = orc.MetaTrainerOracle(spec, _net(prog).theta.cpu().clone(), None, lr=0.001, grad_of=grad_of)
    tr.reset(prog.X.cpu().clone())
    for it in range(3):
        train = it < 2
        fetch = [ms.fx, ms.x, ms.update] + ([ms.step] if train else [])
        out = sess.run(fetch, feed_dict={seq_step: it * T + 1})
        rec["t"] = 0
        res = tr.run_unroll(T, train=train)
        assert abs(out[0] - float(res.fx[-1])) <= REL_TOL * abs(float(res.fx[-1])), it
        assert rel_err(np.concatenate([a.reshape(-1) for a in out[1]]), res.x_final.detach()) <= REL_TOL, it
        if train:
            assert_theta_close(_net(prog).theta, tr, it)


def test_rnnprop_imitation_task_matches_oracle():
    """DM/meta_rnnprop_train.py:441-555: RNNProp imitation unrolls - raw gradients in, the task's own Adam moments,
    p = float(step + t), loss = sum_t 0.5 ||label - delta||^2 / N, own Adam slots, (state, m, v) carried by update_mt."""
    from open_l2o_b200 import meta_rnnprop_train, problems, util
    T, lr = 6, 0.001
    _, net_config, _ = util.get_config("mlp", net_name="RNNprop")
    optimizer = meta_rnnprop_train.MetaOptimizer(1, 0.95, 0.95, **net_config)
    (ms, scale, var_x, constants, subsets, seq_step, loss_mt, steps_mt, update_mt, reset_mt, mt_labels,
     mt_inputs) = optimizer.meta_minimize(problems.mlp(layers=(12,), in_dim=20, n_classes=5, batch_size=16), T,
                                          learning_rate=lr)
    prog = optimizer.program
    n = prog.N
    sess = meta_rnnprop_train.Session()
    sess.run(ms.reset)
    sess.run(reset_mt[0])
    spec = orc.NetSpec(layers=(20, 20), preprocess_name="fc", preprocess_options={"dim": 20}, scale=0.01,
                       tanh_output=True, rnnprop=True)
    theta = _net(prog).theta.cpu().clone()
    am, av = torch.zeros_like(theta), torch.zeros_like(theta)
    state = orc.initial_state(spec, n)
    m, v = torch.zeros(n), torch.zeros(n)
    gen = torch.Generator().manual_seed(4)
    for it in range(2):
        inputs = torch.randn(T, n, generator=gen) * 0.3
        labels = torch.randn(T, n, generator=gen) * 0.01
        feats = []
        for t in range(T):
            m, v, mt, gt = orc.adam_features(inputs[t], m, v, float(it * T + 1 + t), 0.95, 0.95)
            feats.append(torch.stack([mt, gt], -1))
        th = theta.clone().requires_grad_(True)
        loss_ref, state_next, _ = orc.imitation_loss(spec, th, torch.stack(feats), labels, state)
        (g,) = torch.autograd.grad(loss_ref, th)
        theta, am, av = orc.tf_adam_step(theta, g, am, av, it + 1, lr=lr)
        state = tuple((h.detach(), c.detach()) for h, c in state_next)
        cost = sess.run([loss_mt[0], update_mt[0], steps_mt[0]],
                        feed_dict={mt_inputs[0][0]: inputs.numpy(), mt_labels[0][0]: labels.numpy(),
                                   seq_step: it * T + 1})[0]
        assert abs(cost - float(loss_ref)) <= REL_TOL * abs(float(loss_ref)), it
        big = g.abs() > 1e-5 * float(g.abs().max())
        assert rel_err(_net(prog).theta.cpu()[big], theta[big]) <= REL_TOL, it


def test_reset_after_graph_capture_matches_eager(monkeypatch):
    """ADVICE r1 (high): ``reset`` must not leave captured graphs reading stale constants.  Same seed, same calls, with
    and without CUDA graphs: 3 unrolls, reset, 2 unrolls - bit-for-bit the same costs and parameters."""
    from open_l2o_b200 import meta, problems

    def run():
        optimizer = meta.MetaOptimizer(cw={"net": "CoordinateWiseDeepLSTM", "net_options": {"layers": (20, 20)}})
        ms = optimizer.meta_minimize(problems.quadratic(batch_size=128, num_dims=10), 20, learning_rate=0.001)
        sess, out = meta.Session(), []
        for n_unrolls in (4, 3):
            sess.run(ms.reset)
            for _ in range(n_unrolls):
                cost, xs, _, _ = sess.run([ms.fx, ms.x, ms.update, ms.step])
                out.append((cost, xs[0].copy()))
        return out, optimizer.program

    monkeypatch.setenv("L2O_CUDA_GRAPH", "1")
    graphed, prog = run()
    assert True in prog._graphs
    monkeypatch.setenv("L2O_CUDA_GRAPH", "0")
    eager, prog2 = run()
    assert not prog2._graphs
    for (c1, x1), (c2, x2) in zip(graphed, eager):
        assert abs(c1 - c2) <= 1e-6 * abs(c2)
        assert rel_err(x1, x2) <= 1e-6
