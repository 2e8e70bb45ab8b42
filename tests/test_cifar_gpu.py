"""GPU tests of the CIFAR-10 ConvNet producer l2o_cifar_conv_grad (DM/problems.py:369-458) and of meta-training
get_config("cifar_conv") through it, on a seeded synthetic CIFAR-10 written into a temporary directory."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import l2o_oracle as orc
from tests.cifar_fixture import write_cifar10
from tests.helpers import REL_TOL, SPECS, assert_theta_close, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_COORDS = 13610
SIZES = [432, 16, 12800, 32, 320, 10]
BIASES = (1, 3)   # the conv biases: their true gradient is zero (batch norm removes the channel mean)
N_TRAIN, N_TEST = 3000, 700


@pytest.fixture(scope="module")
def data_dir(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("cifar_conv") / "cifar10")
    write_cifar10(path, n_train=N_TRAIN, n_test=N_TEST, seed=9)
    return path


def _split(data_dir, mode="train"):
    from open_l2o_b200.cifar_data import device_split
    return device_split(data_dir, mode, DEV)


def _views(x):
    from open_l2o_b200.problems import CIFAR10_VARIABLES
    out, off = [], 0
    for (_, shape), n in zip(CIFAR10_VARIABLES, SIZES):
        out.append(x[off:off + n].view(shape))
        off += n
    return out


def _pixels(images, idx):
    """NCHW fp32 pixels of the rows ``idx``: fp32(p) / fp32(255), as the reader defines them."""
    from open_l2o_b200.cifar_data import device_values
    return device_values(images.device)[images.index_select(0, idx.long()).long()].view(-1, 3, 32, 32)


def conv_f(x, images, labels, idx):
    """The torch build's loss on the rows ``idx`` in x's dtype; ``x`` is the flat arena."""
    from open_l2o_b200.problems import cifar10_forward
    pix = _pixels(images, idx).permute(0, 2, 3, 1)
    return cifar10_forward(_views(x), pix.to(x.dtype), labels.index_select(0, idx.long()))


def _windows(y):
    """NHWC [B, H, W, C] -> the 2x2 / 2 pooling windows [B, H/2, W/2, C, 4] in row-major window order."""
    Bn, H, W, C = y.shape
    return y.reshape(Bn, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(Bn, H // 2, W // 2, C, 4)


def _decide(y):
    """ReLU + max-pool decisions on normalised NHWC values: the first maximum of ReLU(y) in each window, and whether
    y > 0 there (the ReLU passes the gradient)."""
    a = _windows(y).clamp_min(0)
    arg = torch.zeros(a.shape[:-1], dtype=torch.long, device=y.device)
    best = a[..., 0]
    for t in range(1, 4):
        better = a[..., t] > best
        arg, best = torch.where(better, t, arg), torch.where(better, a[..., t], best)
    return arg, _windows(y).gather(-1, arg[..., None])[..., 0] > 0


def kernel_decisions(ws, B):
    """The ReLU and max-pool decisions the last l2o_cifar_conv_grad call took, from the fp32 values it took them from
    (l2o_cifar_conv_workspace_layout): conv1's and conv2's windows, and the logits' ReLU."""
    from open_l2o_b200 import engine
    off = engine.cifar_conv_workspace_layout(B)

    def f32(name, n):
        return ws[off[name]:off[name] + 4 * n].view(torch.float32)
    bn = f32("bn", 96)
    y1 = (f32("z1", B * 3600).view(B, 15, 15, 16) - bn[:16]) * bn[16:32]   # fp32, (z - mu) * rstd as the kernel
    y2 = (f32("z2", B * 128).view(B, 2, 2, 32) - bn[32:64]) * bn[64:96]
    return _decide(y1[:, :14, :14]), _decide(y2), f32("dl", B * 16).view(B, 16)[:, :10] != 0


# As for mnist_conv (§3.17): a pre-activation within fp32 rounding of a ReLU or max-pool kink (B * 826 such decisions
# here) may be decided differently by the fp32 kernel and an fp64 forward, and one flip moves a channel's gradient by
# about 1 / sqrt(B H W).  The fp64 reference therefore takes the kernel's decisions, and the count of decisions it would
# take otherwise is bounded here: with N(0, 0.05^2) weights the normalised values are O(1), an fp32 rounding is ~1e-7 of
# them, so at B = 1024 fewer than one flip is expected per call.
MAX_FLIPS = 8


def fp64_grad(x, images, labels, idx, dec, scale=None, dtype=torch.float64):
    """f, df/dx and the flip count of the torch build's ConvNet in fp64 (or ``dtype``; fp32 with TF32 off) on the rows
    ``idx``, with the ReLU and max-pool decisions ``dec`` (kernel_decisions) in place of its own."""
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        return _ref_grad(x, images, labels, idx, dec, scale, dtype)


def _ref_grad(x, images, labels, idx, dec, scale, dtype):
    F = torch.nn.functional
    xd = x.detach().to(dtype).requires_grad_(True)
    flips = 0
    with torch.enable_grad():
        w1, b1, w2, b2, wf, bf = _views(xd * scale.to(dtype) if scale is not None else xd)
        h = _pixels(images, idx).to(dtype)
        for (w, b), (arg, live), crop in (((w1, b1), dec[0], 14), ((w2, b2), dec[1], 2)):
            y = F.batch_norm(F.conv2d(h, w.permute(3, 2, 0, 1), stride=2) + b.reshape(1, -1, 1, 1), None, None,
                             training=True, eps=1e-3)
            y = y.permute(0, 2, 3, 1)[:, :crop, :crop, :]
            own_arg, own_live = _decide(y.detach())
            flips += int(((own_arg != arg) & (own_live | live)).sum() + (own_live != live).sum())
            p = _windows(y).gather(-1, arg[..., None])[..., 0] * live   # [B, H/2, W/2, C]
            h = p.permute(0, 3, 1, 2)
        logits = p.reshape(p.shape[0], -1) @ wf + bf
        flips += int(((logits.detach() > 0) != dec[2]).sum())
        f = F.cross_entropy(logits * dec[2], labels.index_select(0, idx.long()).long())
        (g,) = torch.autograd.grad(f, xd)
    return float(f.detach()), g, flips


def assert_grad_close(g, g_ref, what="", g32=None):
    """Per variable: max-abs error <= 1e-5 of that variable's max |g|; the conv biases, whose true gradient is zero,
    against the max over all variables.  With ``g32``, an fp32 torch reference taking the same decisions (given at
    B = 1 only), the bar is the larger of that and three times g32's own error: at B = 1 each BN2 channel is normalised
    over 4 positions only, and its backward amplifies fp32 rounding past 1e-5 in any fp32 evaluation."""
    gmax = float(g_ref.abs().max())
    err_all = (g.double() - g_ref.to(g.device)).abs()
    err32 = (g32.double() - g_ref).abs() if g32 is not None else torch.zeros_like(g_ref)
    off = 0
    for k, n in enumerate(SIZES):
        err = float(err_all[off:off + n].max())
        ref = gmax if k in BIASES else float(g_ref[off:off + n].abs().max())
        bar = max(REL_TOL * ref, 3 * float(err32[off:off + n].max()))
        assert err <= bar, (what, k, err, ref, bar)
        off += n


def _init(gen, scaled=False):
    """An arena with every variable (the biases too) at N(0, 0.05^2); with ``scaled``, x = theta / scale."""
    x = torch.randn(N_COORDS, generator=gen) * 0.05
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
    ws = torch.empty(engine.cifar_conv_workspace_bytes(B), dtype=torch.uint8, device=DEV)
    engine.cifar_conv_grad(images, labels, x, g, B, seed, counter, ws, f=f, scale=scale, idx_out=idx)
    return f, g, idx, counter, ws


@pytest.mark.parametrize("B", [1, 2, 7, 128, 129, 1024, 200])
@pytest.mark.parametrize("mode", ["train", "test"])
@pytest.mark.parametrize("scaled", [False, True])
def test_cifar_conv_grad_matches_fp64_autograd(data_dir, B, mode, scaled):
    """f and df/dx on the recorded indices against fp64 autograd of the torch build, taking the kernel's ReLU and
    max-pool decisions.  B = 200 and 1024 have CTAs walk several images through all five stages."""
    gen = torch.Generator().manual_seed(B * 10 + scaled)
    x, sc = _init(gen, scaled)
    x = x.to(DEV)
    sc = sc.to(DEV) if scaled else None
    f, g, idx, counter, ws = _call(data_dir, x, B, scale=sc, mode=mode)
    torch.cuda.synchronize()
    images, labels = _split(data_dir, mode)
    assert int(counter) == 1 and int(idx.min()) >= 0 and int(idx.max()) < images.shape[0]
    dec = kernel_decisions(ws, B)
    f_ref, g_ref, flips = fp64_grad(x, images, labels, idx, dec, sc)
    assert flips <= MAX_FLIPS, flips
    assert abs(float(f) - f_ref) <= REL_TOL * abs(f_ref), (float(f), f_ref)
    # only at B = 1 is BN2 normalised over 4 positions per channel; every larger batch keeps the plain 1e-5 bar
    g32 = fp64_grad(x, images, labels, idx, dec, sc, dtype=torch.float32)[1] if B == 1 else None
    assert_grad_close(g, g_ref, (B, mode, scaled), g32)


def test_cifar_conv_indices_match_the_mnist_producer(data_dir):
    """The same seed, counter and N draw the same indices as l2o_mnist_grad; each call advances the counter by one."""
    from open_l2o_b200 import engine
    images, _ = _split(data_dir)
    N = images.shape[0]
    mimg = torch.randint(0, 256, (N, 784), dtype=torch.uint8, device=DEV)
    mlab = torch.randint(0, 10, (N,), dtype=torch.uint8, device=DEV)
    x = _init(torch.Generator().manual_seed(0))[0].to(DEV)
    xm = torch.randn((784 + 1) * 20 + 21 * 10, device=DEV) * 0.01
    for seed, start, B in ((5, 41, 128), (6, 0, 1000), (7, 2 ** 33 + 3, 3)):
        c = torch.full((1,), start, dtype=torch.int64, device=DEV)
        _, _, a, _, _ = _call(data_dir, x, B, seed=seed, counter=c)
        assert int(c) == start + 1
        _, _, b, _, _ = _call(data_dir, x, B, seed=seed, counter=c)
        assert int(c) == start + 2 and not torch.equal(a, b)
        cm = torch.full((1,), start, dtype=torch.int64, device=DEV)
        im = torch.empty(B, dtype=torch.int32, device=DEV)
        engine.mnist_grad(mimg, mlab, xm, torch.empty_like(xm), (20,), B, "sigmoid", seed, cm, idx_out=im)
        assert torch.equal(a, im) and int(cm) == start + 1


def test_cifar_conv_grad_is_deterministic(data_dir):
    x, sc = _init(torch.Generator().manual_seed(3), True)
    x, sc = x.to(DEV), sc.to(DEV)
    f1, g1, i1, _, _ = _call(data_dir, x, 200, scale=sc, counter=torch.full((1,), 9, dtype=torch.int64, device=DEV))
    f2, g2, i2, _, _ = _call(data_dir, x, 200, scale=sc, counter=torch.full((1,), 9, dtype=torch.int64, device=DEV))
    assert torch.equal(i1, i2) and float(f1) == float(f2) and torch.equal(g1, g2)


class _Replay:
    """The optimizee the oracle runs: the ConvNet on the batches the engine recorded, one per evaluation in order, with
    the gradients the engine recorded (``g_rec``)."""

    def __init__(self, data_dir, g_rec):
        self.images, self.labels = _split(data_dir)
        self.g_rec = g_rec
        self.idx, self.t = None, 0

    def start(self, idx):
        self.idx, self.t = idx, 0

    def __call__(self, x):
        idx = self.idx[self.t]
        g = self.g_rec[self.t].double()
        self.t += 1
        return conv_f(x, self.images, self.labels, idx), g.detach()


@pytest.mark.parametrize("rnnprop", [False, True])
def test_cifar_conv_bound_producer_meta_training_matches_oracle(data_dir, rnnprop, monkeypatch):
    """get_config("cifar_conv"), T = 20, two unrolls: per-step fx, x and dtheta against the oracle replaying the
    engine's [T+1][B] recorded batches and gradients; the counter advances by T + 1 per unroll; and every gradient the
    first unroll recorded against fp64 autograd at the x and batch it was computed at."""
    from open_l2o_b200 import engine, meta, meta_rnnprop_train, util
    T = 20
    calls, real = [], engine.cifar_conv_grad

    def spy(images, labels, x, g, batch, seed, counter, ws, **kw):   # x, indices, g and decisions of every eager
        real(images, labels, x, g, batch, seed, counter, ws, **kw)      # (not graph-captured) evaluation
        if not torch.cuda.is_current_stream_capturing():
            calls.append((x.clone(), kw["idx_out"].clone(), g.clone(), kernel_decisions(ws, batch)))
    monkeypatch.setattr(engine, "cifar_conv_grad", spy)
    problem, net_config, _ = util.get_config("cifar_conv", net_name="RNNprop" if rnnprop else None, data_dir=data_dir)
    if rnnprop:
        optimizer = meta_rnnprop_train.MetaOptimizer(0, 0.95, 0.95, **net_config)
        ms = optimizer.meta_minimize(problem, T, learning_rate=0.001)[0]
        sess = meta_rnnprop_train.Session()
    else:
        optimizer = meta.MetaOptimizer(**net_config)
        ms = optimizer.meta_minimize(problem, T, learning_rate=0.001)
        sess = meta.Session()
    prog = optimizer.program
    assert prog.producer is not None and prog.producer.kind == "cifar_conv"
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
        if it == 0:   # every recorded gradient row of the eager first unroll against fp64 at its x and batch
            images, labels = _split(data_dir)
            assert len(calls) == T + 1
            for t, (xc, ic, gc, dec) in enumerate(calls):
                assert torch.equal(ic, prog.producer.idx[t]) and torch.equal(gc, prog.runs[0].g_rec[t]), t
                _, g_ref, flips = fp64_grad(xc, images, labels, ic, dec)
                assert flips <= MAX_FLIPS, (t, flips)
                assert_grad_close(gc, g_ref, ("step", t))
        assert_theta_close(net.theta.detach().cpu(), types.SimpleNamespace(
            theta=tr.theta.detach().cpu().float(), last_grad=tr.last_grad.detach().cpu()), it)


def test_cifar_conv_graph_replay_advances_the_producer_counter(data_dir):
    """Unrolls 3 and 4 replay one captured graph and still draw new batches; the counter advances by T + 1 per
    unroll."""
    from open_l2o_b200 import meta, util
    T = 10
    problem, net_config, _ = util.get_config("cifar_conv", data_dir=data_dir)
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
        assert len({tuple(r.tolist()) for r in idx}) == T + 1
        assert not any(torch.equal(idx, s) for s in seen), it
        seen.append(idx)
    assert not prog._graph_failed and True in prog._graphs


def test_cifar_conv_eval_epoch_producer_draws_per_evaluation(data_dir):
    """util.run_eval_epoch over a meta_loss of get_config("cifar_conv", mode="test"): T + 1 draws per unroll."""
    from open_l2o_b200 import meta, util
    T = 10
    problem, net_config, _ = util.get_config("cifar_conv", mode="test", data_dir=data_dir)
    optimizer = meta.MetaOptimizer(**net_config)
    loss, update, reset, cost_op, _ = optimizer.meta_loss(problem, T)
    sess = meta.Session()
    sess.run(reset)
    _, costs = util.run_eval_epoch(sess, cost_op, [update], 3)
    assert len(costs) == 3 and all(np.isfinite(costs))
    prog = optimizer.program
    assert prog.producer.kind == "cifar_conv" and int(prog.producer.counter) == 3 * (T + 1)
    assert int(prog.producer.idx.max()) < N_TEST


def test_cifar_without_batch_norm_meta_trains_on_the_autograd_path(data_dir):
    from open_l2o_b200 import meta, problems, util
    problem = problems.cifar10(batch_norm=False, data_dir=data_dir)
    optimizer = meta.MetaOptimizer(**{"cw": util.get_default_net_config(None)})
    ms = optimizer.meta_minimize(problem, 5, learning_rate=0.001)
    prog = optimizer.program
    assert prog.producer is None and prog.fused is None
    sess = meta.Session()
    sess.run(ms.reset)
    costs = [sess.run([ms.fx, ms.update, ms.step])[0] for _ in range(2)]
    assert all(np.isfinite(costs))


def test_train_dm_runs_cifar_conv_on_a_local_cifar10(data_dir):
    """From a directory holding cifar10/, the default data directory of cifar_conv."""
    env = dict(os.environ, PYTHONPATH=ROOT)
    cmd = [sys.executable, "-m", "open_l2o_b200.train_dm", "--problem", "cifar_conv", "--if_cl", "--num_epochs", "2",
           "--evaluation_period", "1", "--evaluation_epochs", "1", "--min_num_eval", "1"]
    r = subprocess.run(cmd, cwd=os.path.dirname(data_dir), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
