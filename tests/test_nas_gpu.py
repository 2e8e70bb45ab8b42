"""GPU tests of the NAS-cell producer l2o_nas_grad (DM/problems.py:540-634) and of meta-training get_config("nas")
through it, on the seeded synthetic CIFAR-10 of test_cifar_gpu."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import l2o_oracle as orc
from tests.helpers import REL_TOL, SPECS, assert_theta_close, rel_err
from tests.test_cifar_gpu import N_TEST, ROOT, _pixels, _split, data_dir  # noqa: F401  (data_dir is a fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_COORDS = 7578
SIZES = [432, 16, 2304, 16, 2304, 16, 2304, 16, 160, 10]
BIASES = (1, 3, 5, 7)   # the conv biases: their true gradient is zero (batch norm removes the channel mean)
LAYERS = ("z0", "za", "z1", "zb")   # node0, node0_onto_node2, node1, node1_onto_node3


def _views(x):
    from open_l2o_b200.problems import NAS_VARIABLES
    out, off = [], 0
    for (_, shape), n in zip(NAS_VARIABLES, SIZES):
        out.append(x[off:off + n].view(shape))
        off += n
    return out


def nas_f(x, images, labels, idx):
    """The torch build's loss on the rows ``idx`` in x's dtype; ``x`` is the flat arena."""
    from open_l2o_b200.problems import nas_forward
    pix = _pixels(images, idx).permute(0, 2, 3, 1)
    return nas_forward(_views(x), pix.to(x.dtype), labels.index_select(0, idx.long()))


def kernel_decisions(ws, B):
    """The ReLU decisions of the last l2o_nas_grad call, from the fp32 values it took them from
    (l2o_nas_workspace_layout): the four conv layers' [B, 16, 32, 32] masks and the logits' ReLU."""
    from open_l2o_b200 import engine
    off = engine.nas_workspace_layout(B)

    def f32(name, n):
        return ws[off[name]:off[name] + 4 * n].view(torch.float32)
    bn = f32("bn", 128).view(4, 2, 16)
    masks = [((f32(name, B * 16384).view(B, 32, 32, 16) - bn[k, 0]) * bn[k, 1] > 0).permute(0, 3, 1, 2)
             for k, name in enumerate(LAYERS)]
    return masks, f32("dl", B * 16).view(B, 16)[:, :10] != 0


def max_flips(B):
    """Decisions fp64 may take differently from the fp32 kernel: 4 * 16,384 ReLUs per image, each within fp32 rounding
    (~1e-6 of the O(1) normalised value after a 144-term fp32 sum) of its kink with probability ~1e-6.  A flip moves
    one position's gradient only, ~1 / (B * 1024) of a channel's, and the reference takes the kernel's decisions."""
    return max(8, int(1e-5 * B * 4 * 16384))


def fp64_grad(x, images, labels, idx, dec, scale=None):
    """f, df/dx and the flip count of the torch build's NAS cell in fp64 on the rows ``idx``, with the ReLU decisions
    ``dec`` (kernel_decisions) in place of its own."""
    F = torch.nn.functional
    xd = x.detach().double().requires_grad_(True)
    masks, live = dec
    flips = 0
    with torch.enable_grad():
        w0, b0, wa, ba, w1, b1, wb, bb, wf, bf = _views(xd * scale.double() if scale is not None else xd)

        def conv(h, w, b, mask):
            nonlocal flips
            y = F.batch_norm(F.conv2d(h, w.permute(3, 2, 0, 1), padding=1) + b.reshape(1, -1, 1, 1), None, None,
                             training=True, eps=1e-3)
            flips += int(((y.detach() > 0) != mask).sum())
            return y * mask
        node0 = conv(_pixels(images, idx).double(), w0, b0, masks[0])
        n0o2 = conv(node0, wa, ba, masks[1])
        node1 = conv(node0, w1, b1, masks[2])
        n1o3 = conv(node1, wb, bb, masks[3])
        node3 = F.avg_pool2d(node1, 3, 1, padding=1, count_include_pad=False) + n0o2 + n1o3 + node0
        logits = node3.mean(dim=(2, 3)) @ wf + bf
        flips += int(((logits.detach() > 0) != live).sum())
        f = F.cross_entropy(logits * live, labels.index_select(0, idx.long()).long())
        (g,) = torch.autograd.grad(f, xd)
    return float(f.detach()), g, flips


def assert_grad_close(g, g_ref, what=""):
    """Per variable: max-abs error <= 1e-5 of that variable's max |g|; the conv biases, whose true gradient is zero,
    against the max over all variables."""
    gmax = float(g_ref.abs().max())
    err_all = (g.double() - g_ref.to(g.device)).abs()
    off = 0
    for k, n in enumerate(SIZES):
        err = float(err_all[off:off + n].max())
        ref = gmax if k in BIASES else float(g_ref[off:off + n].abs().max())
        assert err <= REL_TOL * ref, (what, k, err, ref)
        off += n


def _init(gen, scaled=False):
    """An arena with every variable at N(0, 0.05^2) and the fc weights at N(0, 1) (the mean over 1024 positions
    makes the features small); with ``scaled``, x = theta / scale."""
    x = torch.randn(N_COORDS, generator=gen) * 0.05
    x[sum(SIZES[:8]):sum(SIZES[:9])] *= 20
    sc = torch.exp(torch.rand(N_COORDS, generator=gen) * 2 - 1) if scaled else None
    return (x / sc if scaled else x), sc


def _call(data_dir, x, B, seed=5, counter=None, scale=None, mode="train"):
    from open_l2o_b200 import engine
    images, labels = _split(data_dir, mode)
    g = torch.empty_like(x)
    f = torch.zeros((), dtype=torch.float64, device=DEV)
    idx = torch.empty(B, dtype=torch.int32, device=DEV)
    if counter is None:
        counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    ws = torch.empty(engine.nas_workspace_bytes(B), dtype=torch.uint8, device=DEV)
    engine.nas_grad(images, labels, x, g, B, seed, counter, ws, f=f, scale=scale, idx_out=idx)
    return f, g, idx, counter, ws


@pytest.mark.parametrize("B", [1, 2, 7, 128, 129, 1024, 200])
@pytest.mark.parametrize("mode", ["train", "test"])
@pytest.mark.parametrize("scaled", [False, True])
def test_nas_grad_matches_fp64_autograd(data_dir, B, mode, scaled):  # noqa: F811
    """f and df/dx on the recorded indices against fp64 autograd of the torch build, taking the kernel's ReLU
    decisions.  B = 200 and 1024 have CTAs walk several images through all seven stages."""
    gen = torch.Generator().manual_seed(B * 10 + scaled)
    x, sc = _init(gen, scaled)
    x = x.to(DEV)
    sc = sc.to(DEV) if scaled else None
    f, g, idx, counter, ws = _call(data_dir, x, B, scale=sc, mode=mode)
    torch.cuda.synchronize()
    images, labels = _split(data_dir, mode)
    assert int(counter) == 1 and int(idx.min()) >= 0 and int(idx.max()) < images.shape[0]
    f_ref, g_ref, flips = fp64_grad(x, images, labels, idx, kernel_decisions(ws, B), sc)
    assert flips <= max_flips(B), flips
    assert abs(float(f) - f_ref) <= REL_TOL * abs(f_ref), (float(f), f_ref)
    assert_grad_close(g, g_ref, (B, mode, scaled))


def test_nas_indices_match_the_mnist_producer(data_dir):  # noqa: F811
    """The same seed, counter and N draw the same indices as l2o_mnist_grad; each call advances the counter by one."""
    from open_l2o_b200 import engine
    images, _ = _split(data_dir)
    N = images.shape[0]
    mimg = torch.randint(0, 256, (N, 784), dtype=torch.uint8, device=DEV)
    mlab = torch.randint(0, 10, (N,), dtype=torch.uint8, device=DEV)
    x = _init(torch.Generator().manual_seed(0))[0].to(DEV)
    xm = torch.randn((784 + 1) * 20 + 21 * 10, device=DEV) * 0.01
    for seed, start, B in ((5, 41, 128), (7, 2 ** 33 + 3, 3)):
        c = torch.full((1,), start, dtype=torch.int64, device=DEV)
        _, _, a, _, _ = _call(data_dir, x, B, seed=seed, counter=c)
        assert int(c) == start + 1
        cm = torch.full((1,), start, dtype=torch.int64, device=DEV)
        im = torch.empty(B, dtype=torch.int32, device=DEV)
        engine.mnist_grad(mimg, mlab, xm, torch.empty_like(xm), (20,), B, "sigmoid", seed, cm, idx_out=im)
        assert torch.equal(a, im) and int(cm) == start + 1


def test_nas_grad_is_deterministic(data_dir):  # noqa: F811
    x, sc = _init(torch.Generator().manual_seed(3), True)
    x, sc = x.to(DEV), sc.to(DEV)
    f1, g1, i1, _, _ = _call(data_dir, x, 200, scale=sc, counter=torch.full((1,), 9, dtype=torch.int64, device=DEV))
    f2, g2, i2, _, _ = _call(data_dir, x, 200, scale=sc, counter=torch.full((1,), 9, dtype=torch.int64, device=DEV))
    assert torch.equal(i1, i2) and float(f1) == float(f2) and torch.equal(g1, g2)


class _Replay:
    """The optimizee the oracle runs: the cell on the batches the engine recorded, with the gradients it recorded."""

    def __init__(self, data_dir, g_rec):  # noqa: F811
        self.images, self.labels = _split(data_dir)
        self.g_rec = g_rec
        self.idx, self.t = None, 0

    def start(self, idx):
        self.idx, self.t = idx, 0

    def __call__(self, x):
        idx = self.idx[self.t]
        g = self.g_rec[self.t].double()
        self.t += 1
        return nas_f(x, self.images, self.labels, idx), g.detach()


@pytest.mark.parametrize("rnnprop", [False, True])
def test_nas_bound_producer_meta_training_matches_oracle(data_dir, rnnprop, monkeypatch):  # noqa: F811
    """get_config("nas"), T = 20, two unrolls: per-step fx, x and dtheta against the oracle replaying the engine's
    recorded batches and gradients, and every gradient of the first unroll against fp64 autograd."""
    from open_l2o_b200 import engine, meta, meta_rnnprop_train, util
    T = 20
    calls, real = [], engine.nas_grad

    def spy(images, labels, x, g, batch, seed, counter, ws, **kw):
        real(images, labels, x, g, batch, seed, counter, ws, **kw)
        if not torch.cuda.is_current_stream_capturing():
            calls.append((x.clone(), kw["idx_out"].clone(), g.clone(), kernel_decisions(ws, batch)))
    monkeypatch.setattr(engine, "nas_grad", spy)
    problem, net_config, _ = util.get_config("nas", net_name="RNNprop" if rnnprop else None, data_dir=data_dir)
    if rnnprop:
        optimizer = meta_rnnprop_train.MetaOptimizer(0, 0.95, 0.95, **net_config)
        ms = optimizer.meta_minimize(problem, T, learning_rate=0.001)[0]
        sess = meta_rnnprop_train.Session()
    else:
        optimizer = meta.MetaOptimizer(**net_config)
        ms = optimizer.meta_minimize(problem, T, learning_rate=0.001)
        sess = meta.Session()
    prog = optimizer.program
    assert prog.producer is not None and prog.producer.kind == "nas"
    sess.run(ms.reset)
    net = next(iter(prog.nets.values()))
    spec = SPECS["rnnprop" if rnnprop else "dm_logsign"]
    rep = _Replay(data_dir, prog.runs[0].g_rec)
    with torch.device(DEV):
        tr = orc.MetaTrainerOracle(spec, net.theta.detach().double().clone(), None, lr=0.001, grad_of=rep)
        tr.reset(prog.X.detach().double().clone())
    for it in range(2):
        cost, xs, _, _ = sess.run([ms.fx, ms.x, ms.update, ms.step])
        torch.cuda.synchronize()
        assert int(prog.producer.counter) == (it + 1) * (T + 1)
        rep.start(prog.producer.idx.clone())
        with torch.device(DEV):
            res = tr.run_unroll(T)
        fx = prog.last_fx.cpu()
        assert rel_err(fx, res.fx.detach()) <= REL_TOL, (it, rel_err(fx, res.fx.detach()))
        fx_ref = float(res.fx[-1].detach())
        assert abs(cost - fx_ref) <= REL_TOL * abs(fx_ref), (it, cost, fx_ref)
        assert rel_err(np.concatenate([a.reshape(-1) for a in xs]), res.x_final.detach()) <= REL_TOL, it
        dth = next(iter(prog.dtheta.values()))
        assert rel_err(dth, tr.last_grad) <= 10 * REL_TOL, (it, rel_err(dth, tr.last_grad))
        if it == 0:
            images, labels = _split(data_dir)
            assert len(calls) == T + 1
            for t, (xc, ic, gc, dec) in enumerate(calls):
                assert torch.equal(ic, prog.producer.idx[t]) and torch.equal(gc, prog.runs[0].g_rec[t]), t
                _, g_ref, flips = fp64_grad(xc, images, labels, ic, dec)
                assert flips <= max_flips(len(ic)), (t, flips)
                assert_grad_close(gc, g_ref, ("step", t))
        assert_theta_close(net.theta.detach().cpu(), types.SimpleNamespace(
            theta=tr.theta.detach().cpu().float(), last_grad=tr.last_grad.detach().cpu()), it)


def test_nas_graph_replay_advances_the_producer_counter(data_dir):  # noqa: F811
    from open_l2o_b200 import meta, util
    T = 10
    problem, net_config, _ = util.get_config("nas", data_dir=data_dir)
    optimizer = meta.MetaOptimizer(**net_config)
    ms = optimizer.meta_minimize(problem, T, learning_rate=0.001)
    prog = optimizer.program
    sess = meta.Session()
    sess.run(ms.reset)
    seen = []
    for it in range(4):
        sess.run([ms.fx, ms.update, ms.step])
        torch.cuda.synchronize()
        assert int(prog.producer.counter) == (it + 1) * (T + 1), it
        idx = prog.producer.idx.clone().cpu()
        assert not any(torch.equal(idx, s) for s in seen), it
        seen.append(idx)
    assert not prog._graph_failed and True in prog._graphs


def test_nas_eval_epoch_producer_draws_per_evaluation(data_dir):  # noqa: F811
    from open_l2o_b200 import meta, util
    T = 10
    problem, net_config, _ = util.get_config("nas", mode="test", data_dir=data_dir)
    optimizer = meta.MetaOptimizer(**net_config)
    loss, update, reset, cost_op, _ = optimizer.meta_loss(problem, T)
    sess = meta.Session()
    sess.run(reset)
    _, costs = util.run_eval_epoch(sess, cost_op, [update], 3)
    assert len(costs) == 3 and all(np.isfinite(costs))
    prog = optimizer.program
    assert prog.producer.kind == "nas" and int(prog.producer.counter) == 3 * (T + 1)
    assert int(prog.producer.idx.max()) < N_TEST


def test_nas_without_batch_norm_meta_trains_on_the_autograd_path(data_dir):  # noqa: F811
    from open_l2o_b200 import meta, problems, util
    problem = problems.nas(batch_norm=False, data_dir=data_dir)
    optimizer = meta.MetaOptimizer(**{"cw": util.get_default_net_config(None)})
    ms = optimizer.meta_minimize(problem, 5, learning_rate=0.001)
    prog = optimizer.program
    assert prog.producer is None and prog.fused is None
    sess = meta.Session()
    sess.run(ms.reset)
    costs = [sess.run([ms.fx, ms.update, ms.step])[0] for _ in range(2)]
    assert all(np.isfinite(costs))


def test_train_dm_runs_nas_on_a_local_cifar10(data_dir):  # noqa: F811
    env = dict(os.environ, PYTHONPATH=ROOT)
    cmd = [sys.executable, "-m", "open_l2o_b200.train_dm", "--problem", "nas", "--if_cl", "--num_epochs", "2",
           "--evaluation_period", "1", "--evaluation_epochs", "1", "--min_num_eval", "1"]
    r = subprocess.run(cmd, cwd=os.path.dirname(data_dir), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
