"""GPU tests of the MNIST MLP producer l2o_mnist_grad (DM/problems.py:254-288) and of meta-training the registry's
MNIST problems through it, on a seeded synthetic MNIST written into a temporary directory."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import l2o_oracle as orc
from tests.helpers import REL_TOL, SPECS, assert_theta_close, rel_err
from tests.mnist_fixture import write_mnist

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def data_dir(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("mnist") / "MNIST-data")
    write_mnist(path, n_train=6000, n_test=1000, seed=7)
    return path


def _split(data_dir, mode="train"):
    from open_l2o_b200.mnist_data import device_split
    return device_split(data_dir, mode, DEV)


def _arena_size(layers):
    n, k = 0, 784
    for w in tuple(layers) + (10,):
        n, k = n + (k + 1) * w, w
    return n


def mlp_f(x, images, labels, idx, layers, activation):
    """The reference's loss (sigmoid/ReLU MLP, mean sparse softmax cross entropy) on the rows ``idx``, in x's dtype;
    ``x`` is the flat arena w0, b0, w1, b1, ..."""
    h = (images.index_select(0, idx.long()).float() * float(np.float32(1.0 / 255.0))).to(x.dtype)
    off, k = 0, 784
    widths = tuple(layers) + (10,)
    for i, w in enumerate(widths):
        W = x[off:off + k * w].view(k, w)
        b = x[off + k * w:off + k * w + w]
        off += k * w + w
        h = h @ W + b
        if i < len(widths) - 1:
            h = torch.sigmoid(h) if activation == "sigmoid" else torch.relu(h)
        k = w
    return torch.nn.functional.cross_entropy(h, labels.index_select(0, idx.long()).long())


def _call(data_dir, x, layers, act, B, seed=5, counter=None, scale=None):
    from open_l2o_b200 import engine
    images, labels = _split(data_dir)
    g = torch.empty_like(x)
    f = torch.zeros((), dtype=torch.float64, device=DEV)
    idx = torch.empty(B, dtype=torch.int32, device=DEV)
    if counter is None:
        counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    engine.mnist_grad(images, labels, x, g, layers, B, act, seed, counter, f=f, scale=scale, idx_out=idx)
    return f, g, idx, counter


CASES = [((20,), "sigmoid", 128), ((20,), "relu", 128), ((20, 20), "sigmoid", 128), ((20, 20), "relu", 100),
         ((64, 64, 64, 64), "sigmoid", 128), ((64, 64, 64, 64), "relu", 1000), ((7,), "sigmoid", 3)]


@pytest.mark.parametrize("layers,act,B", CASES)
@pytest.mark.parametrize("scaled", [False, True])
def test_mnist_grad_matches_fp64_autograd(data_dir, layers, act, B, scaled):
    """f and df/dx on the recorded indices against fp64 autograd.  B = 100, 1000 and 3 leave the last CTAs of the
    cluster ragged or empty.  With ``scale`` the kernel sees x = theta / scale, as run_epoch feeds the random-scaling
    trick (DM/util.py:40-54)."""
    gen = torch.Generator().manual_seed(len(layers) * 100 + B)
    n = _arena_size(layers)
    theta = torch.randn(n, generator=gen) * 0.1
    sc = torch.exp(torch.rand(n, generator=gen) * 2 - 1) if scaled else None
    x = (theta / sc if scaled else theta).to(DEV)
    f, g, idx, _ = _call(data_dir, x, layers, act, B, scale=sc.to(DEV) if scaled else None)
    torch.cuda.synchronize()
    images, labels = _split(data_dir)
    assert int(idx.min()) >= 0 and int(idx.max()) < images.shape[0]
    xd = x.double().requires_grad_(True)
    f_ref = mlp_f(xd * sc.to(DEV).double() if scaled else xd, images, labels, idx, layers, act)
    (g_ref,) = torch.autograd.grad(f_ref, xd)
    f_ref = float(f_ref.detach())
    assert abs(float(f) - f_ref) <= REL_TOL * abs(f_ref), (float(f), f_ref)
    assert rel_err(g, g_ref) <= REL_TOL, rel_err(g, g_ref)


def test_mnist_indices_stream(data_dir):
    """In range; the same seed and counter draw the same indices and the counter advances by one per call; a different
    seed draws others; 100 calls fill 10 equal bins of [0, N) within 5 sigma of uniform."""
    n = _arena_size((20,))
    x = torch.randn(n, device=DEV) * 0.01
    N = _split(data_dir)[0].shape[0]
    _, _, a, c = _call(data_dir, x, (20,), "sigmoid", 128, counter=torch.full((1,), 41, dtype=torch.int64, device=DEV))
    assert int(c) == 42
    _, _, b, c = _call(data_dir, x, (20,), "sigmoid", 128, counter=torch.full((1,), 41, dtype=torch.int64, device=DEV))
    assert torch.equal(a, b) and int(c) == 42
    _, _, d, _ = _call(data_dir, x, (20,), "sigmoid", 128, counter=c)
    assert int(c) == 43 and not torch.equal(a, d)
    _, _, e, _ = _call(data_dir, x, (20,), "sigmoid", 128, seed=6, counter=torch.full((1,), 41, dtype=torch.int64,
                                                                                      device=DEV))
    assert not torch.equal(a, e)
    counter = torch.zeros(1, dtype=torch.int64, device=DEV)
    draws = []
    for _ in range(100):
        draws.append(_call(data_dir, x, (20,), "sigmoid", 128, counter=counter)[2].clone())
    assert int(counter) == 100
    draws = torch.cat(draws).cpu().numpy()
    assert draws.min() >= 0 and draws.max() < N
    hist = np.bincount(draws * 10 // N, minlength=10)
    m = draws.size / 10
    sigma = np.sqrt(draws.size * 0.1 * 0.9)
    assert np.all(np.abs(hist - m) <= 5 * sigma), hist


def test_mnist_grad_is_deterministic(data_dir):
    layers = (64, 64)
    x = torch.randn(_arena_size(layers), device=DEV) * 0.1
    f1, g1, i1, _ = _call(data_dir, x, layers, "relu", 1000, counter=torch.full((1,), 9, dtype=torch.int64, device=DEV))
    f2, g2, i2, _ = _call(data_dir, x, layers, "relu", 1000, counter=torch.full((1,), 9, dtype=torch.int64, device=DEV))
    assert torch.equal(i1, i2) and float(f1) == float(f2) and torch.equal(g1, g2)


def test_mnist_grad_rejects_shapes_outside_its_limits(data_dir):
    from open_l2o_b200 import _lib
    images, labels = _split(data_dir)
    x = torch.zeros(_arena_size((65,)), device=DEV)
    g, counter = torch.empty_like(x), torch.zeros(1, dtype=torch.int64, device=DEV)
    for hidden, B in (((65,), 128), ((20,), 1025), ((20,) * 5, 128)):
        a = _lib.MnistArgs()
        a.batch, a.num_examples, a.n_layers, a.activation = B, images.shape[0], len(hidden) + 1, 0
        for k, w in enumerate(hidden[:4]):
            a.hidden[k] = w
        a.counter, a.images, a.labels = counter.data_ptr(), images.data_ptr(), labels.data_ptr()
        a.x, a.g = x.data_ptr(), g.data_ptr()
        assert _lib.lib().l2o_mnist_grad(ctypes.byref(a), None) == _lib.L2O_E_INVALID, (hidden, B)
    assert int(counter) == 0


def test_out_of_limit_mlp_meta_trains_on_the_autograd_path(data_dir):
    from open_l2o_b200 import meta, problems, util
    problem = problems.mnist((65,), data_dir=data_dir)
    optimizer = meta.MetaOptimizer(**{"cw": util.get_default_net_config(None)})
    ms = optimizer.meta_minimize(problem, 5, learning_rate=0.001)
    prog = optimizer.program
    assert prog.producer is None and prog.fused is None
    sess = meta.Session()
    sess.run(ms.reset)
    costs = [sess.run([ms.fx, ms.update, ms.step])[0] for _ in range(2)]
    assert all(np.isfinite(costs))


class _Replay:
    """The optimizee the oracle runs: the MLP on the batches the engine recorded, one per evaluation in order; the
    gradient is fp64 autograd of it, or (``g_rec``) the gradient the engine recorded."""

    def __init__(self, data_dir, layers, act, g_rec=None):
        self.images, self.labels = _split(data_dir)
        self.layers, self.act, self.g_rec = layers, act, g_rec
        self.idx, self.t = None, 0

    def start(self, idx):
        self.idx, self.t = idx, 0

    def __call__(self, x):
        idx = self.idx[self.t]
        f = lambda v: mlp_f(v, self.images, self.labels, idx, self.layers, self.act)   # noqa: E731
        if self.g_rec is not None:
            g = self.g_rec[self.t].double()
        else:
            xg = x.detach().requires_grad_(True)
            with torch.enable_grad():
                (g,) = torch.autograd.grad(f(xg), xg)
        self.t += 1
        return f(x), g.detach()


def _parity(data_dir, rnnprop):
    from open_l2o_b200 import meta, meta_rnnprop_train, util
    T = 20
    problem, net_config, _ = util.get_config("mnist", net_name="RNNprop" if rnnprop else None, data_dir=data_dir)
    if rnnprop:
        optimizer = meta_rnnprop_train.MetaOptimizer(0, 0.95, 0.95, **net_config)
        ms = optimizer.meta_minimize(problem, T, learning_rate=0.001)[0]
        sess = meta_rnnprop_train.Session()
    else:
        optimizer = meta.MetaOptimizer(**net_config)
        ms = optimizer.meta_minimize(problem, T, learning_rate=0.001)
        sess = meta.Session()
    prog = optimizer.program
    assert prog.producer is not None and prog.producer.kind == "mnist_mlp"
    sess.run(ms.reset)
    net = next(iter(prog.nets.values()))
    spec = SPECS["rnnprop" if rnnprop else "dm_logsign"]
    # RNNProp divides each gradient by its running magnitude, so it replays the engine's gradients (see
    # test_parity_configs_gpu); the DM net sees the oracle's own fp64 gradient
    rep = _Replay(data_dir, (20,), "sigmoid", g_rec=prog.runs[0].g_rec if rnnprop else None)
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
        assert_theta_close(net.theta.detach().cpu(), tr_cpu(tr), it)


def tr_cpu(tr):
    import types
    return types.SimpleNamespace(theta=tr.theta.detach().cpu().float(), last_grad=tr.last_grad.detach().cpu())


@pytest.mark.parametrize("rnnprop", [False, True])
def test_mnist_bound_producer_meta_training_matches_oracle(data_dir, rnnprop):
    """get_config("mnist"), T = 20, two unrolls: per-step fx, x and dtheta against the oracle replaying the engine's
    [T+1][B] recorded batches; the counter advances by T + 1 per unroll."""
    _parity(data_dir, rnnprop)


def _graph_run(data_dir, segment, unrolls=4, T=10):
    from open_l2o_b200 import meta, util
    problem, net_config, _ = util.get_config("mnist", data_dir=data_dir)
    kw = {"_bptt_segment": segment} if segment else {}
    optimizer = meta.MetaOptimizer(**net_config, **kw)
    ms = optimizer.meta_minimize(problem, T, learning_rate=0.001)
    prog = optimizer.program
    sess = meta.Session()
    sess.run(ms.reset)
    out = []
    for it in range(unrolls):
        sess.run([ms.fx, ms.update, ms.step])
        torch.cuda.synchronize()
        out.append((int(prog.producer.counter), prog.producer.idx.clone().cpu(),
                    next(iter(prog.dtheta.values())).clone().cpu()))
    return prog, out


def test_mnist_graph_replay_advances_the_producer_counter(data_dir):
    """Unrolls 3 and 4 replay one captured graph and still draw new batches; the counter advances by T + 1 per unroll
    with and without BPTT segments, whose recomputation draws nothing; dtheta agrees up to summation order."""
    T = 10
    prog, full = _graph_run(data_dir, None, T=T)
    assert not prog._graph_failed and True in prog._graphs and not prog.segmented
    prog_s, seg = _graph_run(data_dir, 3, T=T)
    assert prog_s.segmented and not prog_s._graph_failed and True in prog_s._graphs
    for it, ((c, idx, d), (cs, idx_s, ds)) in enumerate(zip(full, seg)):
        assert c == cs == (it + 1) * (T + 1), (it, c, cs)
        assert torch.equal(idx, idx_s), it
        if it > 0:
            assert not torch.equal(idx, full[it - 1][1]), it
        assert len({tuple(r.tolist()) for r in idx}) == T + 1
    for it in range(2):
        assert rel_err(seg[it][2], full[it][2]) <= REL_TOL, (it, rel_err(seg[it][2], full[it][2]))


def test_mnist_eval_epoch_producer_draws_per_evaluation(data_dir):
    """util.run_eval_epoch over a meta_loss of get_config("mnist", path=...): test split, T + 1 draws per unroll."""
    from open_l2o_b200 import meta, util
    T = 10
    problem, net_config, _ = util.get_config("mnist", path=None, mode="test", data_dir=data_dir)
    optimizer = meta.MetaOptimizer(**net_config)
    loss, update, reset, cost_op, _ = optimizer.meta_loss(problem, T)
    sess = meta.Session()
    sess.run(reset)
    _, costs = util.run_eval_epoch(sess, cost_op, [update], 3)
    assert len(costs) == 3 and all(np.isfinite(costs))
    prog = optimizer.program
    assert int(prog.producer.counter) == 3 * (T + 1)
    assert int(prog.producer.idx.max()) < 1000   # the 1,000 test images of the fixture


def test_train_dm_runs_on_a_local_mnist(data_dir, tmp_path):
    env = dict(os.environ, PYTHONPATH=ROOT)
    cwd = os.path.dirname(data_dir)   # holds MNIST-data/, the default data_dir
    cmd = [sys.executable, "-m", "open_l2o_b200.train_dm", "--problem", "mnist", "--if_cl", "--num_epochs", "2",
           "--evaluation_period", "1", "--evaluation_epochs", "1", "--min_num_eval", "1"]
    r = subprocess.run(cmd, cwd=cwd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode != 0 and "FileNotFoundError" in r.stderr and "MNIST-data" in r.stderr, r.stderr[-2000:]
