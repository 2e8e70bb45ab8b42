"""The LISTA-family kernels against the fp64 oracle: every layer's x_k, every parameter gradient, the loss kernel, a
short layer-wise training run, CUDA-graph replay and the launch count of a training step."""
import os

import numpy as np
import pytest
import torch

from open_l2o_b200 import lista, lista_train as lt
from open_l2o_b200.engine import adam_step, launch_count
from oracle import lista_oracle as lo
from tests import lista_cases as lc

pytestmark = pytest.mark.gpu

SHAPES = [(256, 512, 128), (256, 512, 1024), (250, 500, 128), (25, 50, 128), (5, 10, 128), (250, 500, 9)]
MODELS = ("lista", "lista_cp", "lista_cpss", "alista")
_shares = lambda m: (False,) if m == "alista" else (False, True)
# (250, 500, 9) leaves a partial cluster of rows.  M > N only without ALISTA, whose analytic W needs A A^T invertible.
# New cases go last, so the ids of the earlier ones do not move.
CASES = [(m, s, sh) for m in MODELS for s in SHAPES[:5] for sh in _shares(m)] + \
        [(m, s, sh) for m in MODELS for s in SHAPES[5:] for sh in _shares(m)] + \
        [(m, (512, 256, 129), sh) for m in MODELS[:3] for sh in _shares(m)]
K = 16
# Entries whose |z| lands within fp32 rounding of the row's rank threshold can be selected by one side and not the
# other (z carries ~1e-7 relative error from the fp32 GEMMs, the oracle's is ~1e-16).  The oracle is then run with the
# kernel's masks, so such a flip does not propagate; the count of flips per [B, N] mask is bounded here.
MAX_FLIPS = 4
# The same holds for |z| against theta_k: soft shrinkage is continuous there, but its derivative is not, so the oracle's
# backward also takes the kernel's classification |z| > theta_k (from the recorded z_k).


def _oracle_leaves(m, dtype=torch.float64):
    return {n: v.detach().cpu().to(dtype).clone().requires_grad_(True) for n, v in m.variables.items()}


def _oracle_forward(m, P, data, k1, sels=None, lives=None, zs_out=None):
    nm, T = m.name, m.T
    y = data[:, :m.M].cpu().to(next(iter(P.values())).dtype)
    A = m.A.cpu().to(y.dtype)
    if m.W_const is not None:
        W = m.W_const.cpu().to(y.dtype)[None]
    elif m.share_W:
        W = P[nm + "_W"][None]
    else:
        first = 2 if m.form == lista.LISTA else 1
        W = torch.stack([P[nm + "_W%d" % i] for i in range(first, T + 1)])
    theta = torch.cat([P[nm + "_theta%d" % i] for i in range(1, T + 1)])
    step = torch.cat([P[nm + "_step_size%d" % i] for i in range(1, T + 1)]) if nm + "_step_size1" in P else None
    B1 = P.get(nm + "_B")
    ranks = None if m.ss_rank is None else m.ss_rank.cpu().tolist()
    return lo.forward(m.form, A, B1, W, theta, step, y, k1, m.one_W, ranks, sels, lives, zs_out)


def _rel(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("name,shape,share_W", CASES)
def test_forward_and_gradients_match_fp64(name, shape, share_W):
    M, N, B = shape
    m = lc.generic_model(name, M, N, share_W)
    for k in range(K):
        m.create_cell(k)
    data = torch.as_tensor(lista.make_data(M, N, B, seed=7)["train"]).cuda()
    loss = m.loss_and_grad(data, lista.TASK_SC)
    torch.cuda.synchronize()
    bufs = m._bufs_for(B, True)
    sels = None if bufs["sel"] is None else [bufs["sel"][k].cpu().bool() for k in range(K)]
    theta = m._block(m.name + "_theta1", K)
    lives = [((bufs["zs"][k].abs() > theta[k]) & (bufs["zs"][k] != 0)).cpu() for k in range(K)]
    P = _oracle_leaves(m)
    xs_ref, _ = _oracle_forward(m, P, data, K, sels, lives)
    for k in range(K):
        assert _rel(bufs["xs"][k], xs_ref[k]) <= 1e-5, (k, _rel(bufs["xs"][k], xs_ref[k]))
    # the oracle's own classification differs from the kernel's only at rounding ties
    with torch.no_grad():
        Pd = {n: v.detach() for n, v in P.items()}
        _, own_sel = _oracle_forward(m, Pd, data, K)
        zs_ref = []
        _oracle_forward(m, Pd, data, K, sels, lives, zs_ref)
    for k in range(K):
        own_live = (zs_ref[k].abs() > Pd[m.name + "_theta%d" % (k + 1)]) & (zs_ref[k] != 0)
        assert int((own_live != lives[k]).sum()) <= MAX_FLIPS, k
        if sels is not None:
            assert int((own_sel[k] != sels[k]).sum()) <= MAX_FLIPS, k
    xt = data[:, M:].cpu().double()
    ref_loss = lo.sc_loss(xs_ref[-1], xt)
    assert abs(float(loss.sum()) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss))
    ref_loss.backward()
    grads = {n: (l.grad if l.grad is not None else torch.zeros_like(l)) for n, l in P.items()}
    for vname, ref in grads.items():
        got = m._grad_span(vname, 1).view(ref.shape)
        if ref.abs().max() == 0:
            assert got.abs().max() == 0, vname
            continue
        err = float((got.cpu() - ref).abs().max() / ref.abs().max())   # each variable against its own magnitude
        assert err <= 1e-5, (vname, err)


@pytest.mark.parametrize("shape", [(250, 500), (25, 50), (5, 10)])
def test_lasso_loss_kernel_matches_fp64(shape):
    M, N = shape
    m = lc.generic_model("lista", M, N, False)
    for k in range(4):
        m.create_cell(k)
    data = torch.as_tensor(lista.make_data(M, N, 128, seed=3)["train"]).cuda()
    lam = 0.005
    loss = m.loss_and_grad(data, lista.TASK_LASSO, lam, k1=4)
    torch.cuda.synchronize()
    x = m._bufs_for(128, True)["xs"][3].cpu().double().requires_grad_(True)
    ref = lo.lasso_loss(x, m.A.cpu().double(), data[:, :M].cpu().double(), lam)
    ref.backward()
    assert abs(float(loss.sum()) - float(ref)) <= 1e-5 * abs(float(ref))
    assert _rel(m._bufs_for(128, True)["d_xk"], x.grad) <= 1e-5


class _OracleTrainer(lt.KernelTrainer):
    """The same schedule and batches, with the fp64 oracle's forward, autograd and Keras Adam.  `mirror`, a second
    kernel model, supplies the discrete decisions at the oracle's own (fp32-rounded) weights: support masks and
    |z| > theta.  Both jump at rounding ties (a flipped selection moves x by theta), and one flip in one step sends two
    otherwise equal training runs apart."""

    def __init__(self, model, *a, mirror=None, **kw):
        super().__init__(model, *a, **kw)
        self.mirror = mirror
        self.P = _oracle_leaves(model)
        self.mo = {n: torch.zeros_like(v) for n, v in self.P.items()}
        self.vo = {n: torch.zeros_like(v) for n, v in self.P.items()}

    def create_cell(self, k):
        self.model.num_cells += 1

    def begin_stage(self, lr, gscale):
        self.lr, self.t, self.gs = lr, 0, np.asarray(gscale, np.float64)
        for d in (self.mo, self.vo):
            for v in d.values():
                v.zero_()

    def step(self, batch):
        k1 = self.model.num_cells
        for v in self.P.values():
            v.grad = None
        xs, _ = _oracle_forward(self.model, self.P, batch, k1, *self._kernel_masks(batch, k1))
        rows = 0.5 * ((xs[-1] - batch[:, self.model.M:].cpu().double()) ** 2).sum(dim=1)
        rows.sum().backward()
        self.t += 1
        with torch.no_grad():
            for n, v in self.P.items():
                g = v.grad if v.grad is not None else torch.zeros_like(v)
                lo.keras_adam_step(v, g * self.gs[self.model.births[n]], self.mo[n], self.vo[n], self.t, self.lr)
        return rows.detach()

    def _kernel_masks(self, data, k1):
        km = self.mirror
        km.load_state_dict({n: v.detach().float() for n, v in self.P.items()})
        km.forward(data, k1, record=True)
        b = km._bufs_for(data.shape[0], True)
        th = km._block(km.name + "_theta1", km.T)
        sels = None if b["sel"] is None else [b["sel"][k].cpu().bool() for k in range(k1)]
        return sels, [((b["zs"][k].abs() > th[k]) & (b["zs"][k] != 0)).cpu() for k in range(k1)]

    def validate(self):
        k1 = self.model.num_cells
        xs, _ = _oracle_forward(self.model, {n: v.detach() for n, v in self.P.items()}, self.val, k1,
                                *self._kernel_masks(self.val, k1))
        return float(lo.nmse_db(xs[-1], self.val[:, self.model.M:].cpu().double()))


class _Recorded:
    """Records the epochs each stage of train_layerwise ran and every validation metric."""

    def begin_stage(self, lr, gscale):
        self.stage_epochs = getattr(self, "stage_epochs", []) + [0]
        super().begin_stage(lr, gscale)

    def train_epoch(self):
        self.stage_epochs[-1] += 1
        super().train_epoch()

    def validate(self):
        v = super().validate()
        self.vals = getattr(self, "vals", []) + [float(v)]
        return v


# LISTA-CPSS with per-layer W is not compared as a trajectory: on this overfitting run its fp32 and fp64 runs part
# after ~40 epochs although every step agrees (test_layerwise_training_steps_match_the_oracle).  The worst gradients
# are dtheta_k that cancel to 1e-4 of their terms, where fp32 inputs leave 1e-3 relative error; Adam divides them by
# their own running magnitude, so their sign errors become full-size steps and the runs go apart.
@pytest.mark.parametrize("name,share_W", [("lista", False), ("lista", True), ("lista_cp", False), ("lista_cp", True),
                                          ("lista_cpss", True), ("alista", False)])
def test_layerwise_training_follows_the_oracle(name, share_W, monkeypatch):
    """Three layers on a training set small enough to overfit, so the validation metric stalls and early stopping
    ends stages before the epoch cap.  The oracle-driven trainer takes the kernels' discrete decisions (support masks
    and |z| > theta at its own weights, see _OracleTrainer) and runs the stages the kernels' early stopping chose: a
    strict '<' between two validation metrics that differ by less than fp32 noise can go either way, and after that
    the two runs would train different schedules.  On that schedule every epoch's training loss and validation metric
    must agree.  fit_stage's stopping rule itself is tested on the CPU."""
    M, N, T, epochs, lr = 32, 64, 3, 15, 1e-2
    d = lista.make_data(M, N, (64, 128, 8), seed=5)
    W = lista.alista_weight(d["A"]) if name == "alista" else None
    train, val = torch.as_tensor(d["train"]).cuda(), torch.as_tensor(d["val"]).cuda()
    runs = []
    for base in (lt.KernelTrainer, _OracleTrainer):
        m = lt.build_model(name, d["A"], T, 0.4, share_W, 5.0, 20.0, W)
        kw = {} if base is lt.KernelTrainer else {"mirror": lt.build_model(name, d["A"], T, 0.4, share_W, 5.0, 20.0, W)}
        tr = type("Run", (_Recorded, base), {})(m, train, val, lista.TASK_SC, 0.0, 16, 128, 4, seed=3, **kw)
        lt.train_layerwise(tr, T, base_lr=lr, epochs=epochs)
        runs.append(tr)
        if base is lt.KernelTrainer:   # the oracle replays the kernels' stage lengths
            lengths = iter(tr.stage_epochs)

            def replay(train_epoch, validate, epochs, patience=lt.PATIENCE):
                hist = []
                for _ in range(next(lengths)):
                    train_epoch()
                    hist.append(float(validate()))
                return hist
            monkeypatch.setattr(lt, "fit_stage", replay)
    k, o = runs
    assert k.stage_epochs == o.stage_epochs and len(k.stage_epochs) == 3 * T
    assert min(k.stage_epochs) < epochs, k.stage_epochs      # early stopping fired
    np.testing.assert_allclose(k.losses, o.losses, rtol=2e-4)
    np.testing.assert_allclose(k.vals, o.vals, rtol=0, atol=2e-3)   # NMSE in dB
    assert k.losses[-1] < k.losses[0]


def test_layerwise_training_steps_match_the_oracle():
    """LISTA-CPSS (per-layer W) through the same layer-wise run as the trajectory test: at every step, x_k and every
    scaled gradient of the kernels against the fp64 oracle at the kernels' own weights (and masks).  Gradients are
    checked per variable at 2e-3: a dtheta_k can cancel to 1e-4 of the sum of its terms, and fp32 terms carry 1e-7."""
    M, N, T = 32, 64, 3
    d = lista.make_data(M, N, (64, 128, 8), seed=5)
    train, val = torch.as_tensor(d["train"]).cuda(), torch.as_tensor(d["val"]).cuda()
    m = lt.build_model("lista_cpss", d["A"], T, 0.4, False, 5.0, 20.0)
    tr = lt.KernelTrainer(m, train, val, lista.TASK_SC, 0.0, 16, 128, 4, seed=3)
    kernel_step, worst = tr.step, {"x": 0.0, "grad": 0.0, "steps": 0}

    def checked_step(batch):
        k1 = m.num_cells
        P = _oracle_leaves(m)
        m.loss_and_grad(batch, lista.TASK_SC, 0.0, tr.gscale)
        torch.cuda.synchronize()
        b = m._bufs_for(batch.shape[0], True)
        th = m._block(m.name + "_theta1", T)
        sels = [b["sel"][k].cpu().bool() for k in range(k1)]
        lives = [((b["zs"][k].abs() > th[k]) & (b["zs"][k] != 0)).cpu() for k in range(k1)]
        xs, _ = _oracle_forward(m, P, batch, k1, sels, lives)
        lo.sc_loss(xs[-1], batch[:, M:].cpu().double()).backward()
        gs = tr.gscale.cpu().double()
        worst["x"] = max(worst["x"], max(_rel(b["xs"][k], xs[k]) for k in range(k1)))
        for n, v in P.items():
            ref = (v.grad if v.grad is not None else torch.zeros_like(v)) * gs[m.births[n]]
            got = m._grad_span(n, 1).view(ref.shape).cpu()
            if ref.abs().max() == 0:
                assert got.abs().max() == 0, n
            else:
                worst["grad"] = max(worst["grad"], _rel(got, ref))
        worst["steps"] += 1
        return kernel_step(batch)      # the real step: the kernels' forward, backward and Adam

    tr.step = checked_step
    lt.train_layerwise(tr, T, base_lr=1e-2, epochs=15)
    assert worst["steps"] > 100 and worst["x"] <= 1e-5 and worst["grad"] <= 2e-3, worst


def test_lasso_test_mode_final_output_over_several_batches(tmp_path):
    """--test with --task lasso saves x_K of every row of a file longer than one test batch."""
    M, N, T = 25, 50, 4
    d = lista.make_data(M, N, (8, 8, 300), seed=4, out_dir=str(tmp_path))
    m = lc.generic_model("lista", M, N, False, seed=4, T=T)       # the A of make_data(..., seed=4)
    ck = tmp_path / "models" / "exp" / "replicate_1"
    for k in range(T):
        os.makedirs(ck / ("layer_%d" % (k + 1)))
        np.savez(ck / ("layer_%d" % (k + 1)) / "model.npz", **m.state_dict())
        m.create_cell(k)
    res = lt.run("lista", task="lasso", num_layers=T, test=True, test_files=["test_data.npy"], test_batch_size=128,
                 base_dir=str(tmp_path), data_dir=str(tmp_path), exp_name="exp")
    saved = np.load(ck / "test_data_final_output.npy")
    ref = m.forward(torch.as_tensor(d["test"]).cuda(), T)[-1].cpu().numpy()     # all 300 rows in one forward
    assert saved.shape == (300, N)
    np.testing.assert_array_equal(saved, ref)
    assert len(res["test_data.npy"]) == T


def test_graph_replay_equals_eager_and_launches_do_not_grow_with_layers():
    M, N, B = 256, 512, 128
    data = torch.as_tensor(lista.make_data(M, N, B, seed=2)["train"]).cuda()
    counts = {}
    for T in (4, 16):
        m = lc.generic_model("lista_cpss", M, N, True, T=T)
        for k in range(T):
            m.create_cell(k)
        tr = lt.KernelTrainer(m, data, data, lista.TASK_SC, 0.0, B, B, 1)
        tr.begin_stage(1e-3, lt.gradient_scales(T - 1, 1, T))
        tr.step(data)      # allocate the buffers outside the count and the capture
        torch.cuda.synchronize()
        c0 = launch_count()
        tr.step(data)
        torch.cuda.synchronize()
        counts[T] = launch_count() - c0
    assert counts[4] == counts[16] == 5     # forward, loss, backward (2), Adam

    m = lc.generic_model("lista_cpss", M, N, True)
    for k in range(K):
        m.create_cell(k)
    tr = lt.KernelTrainer(m, data, data, lista.TASK_SC, 0.0, B, B, 1)
    tr.begin_stage(1e-3, lt.gradient_scales(K - 1, 1, K))
    start = m.params.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        tr.step(data)            # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        m.loss_and_grad(data, lista.TASK_SC, 0.0, tr.gscale)
        adam_step(m.params, m.grads, tr.m, tr.v, 1, lr=1e-3, eps=lt.KERAS_EPS)
    for run in ("eager", "graph"):
        m.params.copy_(start)
        tr.m.zero_()
        tr.v.zero_()
        if run == "eager":
            m.loss_and_grad(data, lista.TASK_SC, 0.0, tr.gscale)
            adam_step(m.params, m.grads, tr.m, tr.v, 1, lr=1e-3, eps=lt.KERAS_EPS)
            torch.cuda.synchronize()
            eager = (m.params.clone(), m.grads.clone())
        else:
            g.replay()
            torch.cuda.synchronize()
    assert torch.equal(m.grads, eager[1]) and torch.equal(m.params, eager[0])
    assert not torch.equal(m.params, start)
