"""CPU tests of the LISTA family: the oracle against plain ISTA, the support-selection rank, Keras Adam, the analytic
ALISTA weight, the layer-wise schedule on a stub step, the models' variables, and ABI argument checks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from open_l2o_b200 import _lib, lista, lista_train as lt
from oracle import lista_oracle as lo
from tests import lista_cases as lc


def _ista(A, y, lam, K):
    """K steps of ISTA from x = 0 with step 1/L and threshold lam/L, L = 1.001 ||A||_2^2."""
    L = 1.001 * np.linalg.norm(A, 2) ** 2
    x = np.zeros((y.shape[0], A.shape[1]))
    out = []
    for _ in range(K):
        z = x + (y - x @ A.T) @ A / L
        x = np.sign(z) * np.maximum(np.abs(z) - lam / L, 0.0)
        out.append(x)
    return out


@pytest.mark.parametrize("share_W", [False, True])
def test_lista_at_initial_weights_is_ista(share_W):
    d = lista.make_data(20, 40, 16, seed=1)
    A = d["A"].astype(np.float64)
    y = d["train"][:, :20].astype(np.float64)
    lam, K = 0.1, 6
    L = 1.001 * np.linalg.norm(A, 2) ** 2
    B1 = A.T / L
    W = np.eye(40) - B1 @ A
    Ws = torch.tensor(np.stack([W] * (1 if share_W else K - 1)))
    step = torch.ones(K, dtype=torch.float64) if share_W else None
    xs, _ = lo.forward(lo.LISTA, torch.tensor(A), torch.tensor(B1), Ws, torch.full((K,), lam / L, dtype=torch.float64),
                       step, torch.tensor(y), K, share_W)
    for x, ref in zip(xs, _ista(A, y, lam, K)):
        np.testing.assert_allclose(x.numpy(), ref, rtol=0, atol=1e-12)


def test_coupled_cell_with_A_over_L_is_ista():
    d = lista.make_data(15, 30, 8, seed=2)
    A, y, K, lam = d["A"].astype(np.float64), d["train"][:, :15].astype(np.float64), 5, 0.05
    L = 1.001 * np.linalg.norm(A, 2) ** 2
    xs, _ = lo.forward(lo.COUPLED, torch.tensor(A), None, torch.tensor(A / L)[None], torch.full((K,), lam / L,
                       dtype=torch.float64), None, torch.tensor(y), K, share_W=True)
    for x, ref in zip(xs, _ista(A, y, lam, K)):
        np.testing.assert_allclose(x.numpy(), ref, rtol=0, atol=1e-12)


def test_percentile_rank_hand_cases():
    # (n - 1) q / 100 rounded half to even
    assert lo.ss_rank(11, 25.0) == 2      # 2.5 -> 2
    assert lo.ss_rank(11, 35.0) == 4      # 3.5 -> 4
    assert lo.ss_rank(11, 0.0) == 0
    assert lo.ss_rank(11, 100.0) == 10
    assert lo.ss_rank(512, 1.2) == 6      # 6.132
    assert lo.ss_rank(512, 13.0) == 66    # 66.43
    np.testing.assert_array_equal(lista.ss_ranks(16, 512, 1.2, 13.0),
                                  [lo.ss_rank(512, min((k + 1) * 1.2, 13.0)) for k in range(16)])
    # strict > at the row threshold and at theta
    z = torch.tensor([[5.0, -4.0, 3.0, 3.0, 1.0, 0.5]])
    sel = lo.ss_select(z, torch.tensor(0.2), 2)          # threshold |z| = 3 at rank 2
    assert sel.tolist() == [[True, True, False, False, False, False]]
    sel = lo.ss_select(z, torch.tensor(4.0), 3)          # threshold 3, but |z| must also exceed theta = 4
    assert sel.tolist() == [[True, False, False, False, False, False]]
    x, _ = lo.shrink_ss(z, torch.tensor(0.2), 2)
    np.testing.assert_allclose(x.numpy(), [[5.0, -4.0, 2.8, 2.8, 0.8, 0.3]], rtol=1e-6)


def _random_cell(form, M, N, K, share_W, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    S = 1 if share_W else (K if form == lo.COUPLED else K - 1)
    A = r(M, N) / np.sqrt(M)
    W = (A / 2 if form == lo.COUPLED else torch.eye(N, dtype=torch.float64) / 2) + 0.05 * r(S, M if form == lo.COUPLED
                                                                                           else N, N)
    return dict(A=A, B1=A.T / 2 if form == lo.LISTA else None, W=W, theta=0.1 + 0.05 * r(K).abs(),
                step=1 + 0.2 * r(K), y=r(5, M))


@pytest.mark.parametrize("form", [lo.LISTA, lo.COUPLED])
@pytest.mark.parametrize("share_W", [False, True])
def test_oracle_layer_ranges_and_per_layer_shrinkage(form, share_W):
    M, N, K = 6, 9, 5
    c = _random_cell(form, M, N, K, share_W, seed=form + 2 * share_W)
    args = lambda: (form, c["A"], c["B1"], c["W"], c["theta"], c["step"], c["y"])
    ranks = [2, -1, N - 1, N + 5, 0]
    full, used = lo.forward(*args(), K, share_W, ranks)
    assert used[1] is None and all(u is not None for i, u in enumerate(used) if i != 1)
    for j in range(1, K):      # a pass [j, K) from x_j reproduces layers j .. K-1, bit for bit
        part, pused = lo.forward(*args(), K, share_W, ranks, k0=j, x0=full[j - 1])
        assert len(part) == K - j
        for k in range(j, K):
            assert torch.equal(part[k - j], full[k]), (j, k)
            assert (pused[k - j] is None) == (used[k] is None)
    # x0 = None is x_0 = 0; k0 = 0 with an explicit zero x0 is the same pass
    z0, _ = lo.forward(*args(), K, share_W, ranks, x0=torch.zeros(5, N, dtype=torch.float64))
    assert all(torch.equal(a, b) for a, b in zip(z0, full))
    # a negative rank is soft shrinkage in that layer only
    zs = []
    xs, _ = lo.forward(*args(), 2, share_W, [-1, -1], zs_out=zs)
    soft, _ = lo.forward(*args(), 2, share_W)
    for k in range(2):
        assert torch.equal(xs[k], soft[k]) and torch.equal(xs[k], lo.shrink_free(zs[k], c["theta"][k]))
    # ranks >= N read as N - 1
    _, a = lo.forward(*args(), K, share_W, [N - 1] * K)
    _, b = lo.forward(*args(), K, share_W, [N + 5] * K)
    assert all(torch.equal(u, v) for u, v in zip(a, b)) and any(bool(u.any()) for u in a)


def test_abi_exact_inputs_keep_every_sum_exact():
    """The premise of test_lista_abi_gpu's bit-exact tests, on every parametrization: the abs-sum bound of every sum
    the kernels form stays below 2^24, so integer inputs give exact fp32 results; and the inputs reach the edges
    they are there for: |z| == theta, z == 0 and -0.0, ties at the support-selection threshold just above theta (where
    '>' against '>=' decides), and N - 1 against N - 2 changing a mask where the rank clamps."""
    cases = [(lc.exact_case(*c), 0, lc.K) for c in lc.EXACT_CASES]
    cases += [(lc.exact_case(f, (12, 16, 13), "clamp", "perlayer", seed=3), k0, k1) for f in (lo.LISTA, lo.COUPLED)
              for k0, k1 in lc.RANGES]
    cases.append((lc.exact_case(lo.LISTA, (24, 16, 13), "mixed", "perlayer", seed=5), 0, lc.K))
    cases.append((lc.exact_case(lo.COUPLED, (24, 16, 13), "mixed", "perlayer", seed=5), 0, lc.K))
    seen = dict(theta_ties=0, zeros=0, negative_zeros=0, rank_ties=0, clamp=0)
    for P, k0, k1 in cases:
        assert lc.exact_bound(P, k0, k1) < 2 ** 24
        ref = lc.oracle(P, k0, k1, d_xk=None)
        for l in range(k1 - k0):
            z, th = ref["zs"][l], float(P["theta"][k0 + l])
            seen["theta_ties"] += int((z.abs() == th).sum())
            seen["zeros"] += int((z == 0).sum())
            seen["negative_zeros"] += int(((z == 0) & torch.signbit(z)).sum())
            if P["ranks"] is None or int(P["ranks"][k0 + l]) < 0:
                continue
            N = P["N"]
            srt = z.abs().sort(dim=1, descending=True).values
            thr = srt[:, min(int(P["ranks"][k0 + l]), N - 1)][:, None]
            seen["rank_ties"] += int(((z.abs() == thr) & (z.abs() > th)).sum())
            if N > 1 and int(P["ranks"][k0 + l]) >= N - 1:
                seen["clamp"] += int(((z.abs() == srt[:, N - 2:N - 1]) & (z.abs() > srt[:, N - 1:]) &
                                      (z.abs() > th)).sum())
    assert all(v >= 10 for v in seen.values()), seen


def test_keras_adam_one_step_closed_form():
    g = torch.tensor([0.5, -2.0, 0.0], dtype=torch.float64)
    p = torch.tensor([1.0, 1.0, 1.0], dtype=torch.float64)
    m, v = torch.zeros(3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64)
    lr = 0.01
    lo.keras_adam_step(p, g, m, v, 1, lr)
    # m = 0.1 g, v = 0.001 g^2, lr_t = lr sqrt(0.001) / 0.1  =>  step = lr g / (|g| + 1e-7 / sqrt(0.001))
    ref = 1.0 - lr * g.numpy() / (np.abs(g.numpy()) + 1e-7 / np.sqrt(0.001))
    np.testing.assert_allclose(p.numpy(), ref, rtol=1e-12)


def test_alista_weight_constraint_and_optimality():
    A = lista.make_data(25, 50, 1, seed=3)["A"]
    W = lista.alista_weight(A).astype(np.float64)
    A64 = A.astype(np.float64)
    np.testing.assert_allclose(np.diag(W.T @ A64), 1.0, atol=1e-5)
    # KKT of min ||A^T w_i||^2 s.t. a_i^T w_i = 1: A A^T w_i is parallel to a_i
    G = A64 @ A64.T @ W
    mu = np.sum(G * A64, axis=0) / np.sum(A64 * A64, axis=0)
    np.testing.assert_allclose(G, A64 * mu, atol=1e-4 * np.abs(G).max())


def test_make_data_layout(tmp_path):
    d = lista.make_data(8, 16, (10, 4, 3), p=0.25, seed=0, out_dir=str(tmp_path))
    assert d["train"].shape == (10, 24) and d["val"].shape == (4, 24) and d["test"].shape == (3, 24)
    np.testing.assert_allclose(np.linalg.norm(d["A"], axis=0), 1.0, rtol=1e-5)
    y, x = d["train"][:, :8], d["train"][:, 8:]
    np.testing.assert_allclose(y, x @ d["A"].T, atol=1e-5)
    for f in ("A.npy", "train_data.npy", "val_data.npy", "test_data.npy"):
        assert os.path.exists(tmp_path / f)


def test_gradient_scales():
    np.testing.assert_array_equal(lt.gradient_scales(2, 0, 5), [0, 0, 1, 0, 0])
    np.testing.assert_allclose(lt.gradient_scales(2, 1, 5), [0.09, 0.3, 1, 0, 0], rtol=1e-6)
    np.testing.assert_allclose(lt.gradient_scales(2, 2, 5), [0.09, 0.3, 1, 0, 0], rtol=1e-6)
    np.testing.assert_array_equal(lt.gradient_scales(0, 0, 3), [1, 0, 0])


def test_fit_stage_stops_after_five_epochs_without_strict_improvement():
    vals = iter([3.0, 2.0, 2.0, 2.5, 1.9, 1.9, 1.9, 1.9, 1.9, 1.9, 0.1])
    n = []
    hist = lt.fit_stage(lambda: n.append(1), lambda: next(vals), epochs=100)
    assert hist == [3.0, 2.0, 2.0, 2.5, 1.9, 1.9, 1.9, 1.9, 1.9, 1.9] and len(n) == 10
    assert len(lt.fit_stage(lambda: None, lambda: 1.0, epochs=3)) == 3


class _Stub:
    """A trainer whose variables are one scalar per layer; records what each stage would train."""

    def __init__(self, K, plateau=2):
        self.K, self.plateau = K, plateau
        self.cells, self.stages, self.loaded, self.saved = [], [], [], []
        self.w = np.zeros(K)
        self.epoch = 0

    def create_cell(self, k):
        self.cells.append(k)

    def begin_stage(self, lr, gscale):
        self.stages.append((len(self.cells) - 1, lr, np.asarray(gscale).copy()))
        self.epoch = 0

    def train_epoch(self):
        self.w += self.stages[-1][2]     # a variable moves only where its multiplier is nonzero
        self.epoch += 1

    def validate(self):
        return max(self.plateau - self.epoch, 0)

    def save(self, path):
        np.savez(path, w=self.w)
        self.saved.append(path)

    def load(self, path):
        self.loaded.append(path)
        self.w = np.load(path)["w"]


def test_train_layerwise_schedule_and_resume(tmp_path):
    K = 3
    s = _Stub(K)
    lt.train_layerwise(s, K, base_lr=1e-3, epochs=50, model_dir=str(tmp_path))
    assert s.cells == [0, 1, 2] and len(s.stages) == 3 * K
    for i, (layer, lr, g) in enumerate(s.stages):
        assert layer == i // 3
        assert lr == pytest.approx(1e-3 * lt.STAGE_LR[i % 3])
        np.testing.assert_allclose(g, lt.gradient_scales(layer, i % 3, K))
    # each stage ran 2 improving epochs and then 5 without improvement: 7 epochs.  Layer 0's variable: three stages
    # at age 0, frozen in stage 1 of each later layer, then 0.3 and 0.09 in their stages 2 and 3
    np.testing.assert_allclose(s.w, [7 * (3 + 0.6 + 0.18), 7 * (3 + 0.6), 7 * 3])
    assert [os.path.basename(os.path.dirname(p)) for p in s.saved] == ["layer_1", "layer_2", "layer_3"]
    # resume: remove the last layer's checkpoint; layers 1-2 are skipped and layer 2 is restored
    os.remove(tmp_path / "layer_3" / "model.npz")
    r = _Stub(K)
    lt.train_layerwise(r, K, base_lr=1e-3, epochs=50, model_dir=str(tmp_path))
    assert r.cells == [0, 1, 2] and [st[0] for st in r.stages] == [2, 2, 2]
    assert [os.path.basename(os.path.dirname(p)) for p in r.loaded] == ["layer_2"]


def test_models_variables_on_cpu():
    A = lista.make_data(6, 12, 1, seed=0)["A"]
    m = lista.Lista(A, 4, 0.4, device="cpu")
    assert list(m.variables) == ["Lista_B", "Lista_W2", "Lista_W3", "Lista_W4", "Lista_theta1", "Lista_theta2",
                                 "Lista_theta3", "Lista_theta4"]
    assert m.layer_variables(0) == ["Lista_B", "Lista_theta1"] and m.layer_variables(2) == ["Lista_W3", "Lista_theta3"]
    L = 1.001 * np.linalg.norm(A.astype(np.float64), 2) ** 2
    np.testing.assert_allclose(m.variables["Lista_theta1"].numpy(), 0.4 / L, rtol=1e-6)
    np.testing.assert_allclose(m.variables["Lista_B"].numpy(), A.T / L, rtol=1e-5)
    ms = lista.Lista(A, 4, 0.4, share_W=True, device="cpu")
    assert ms.births["Lista_W"] == 1 and "Lista_step_size3" in ms.variables
    cp = lista.ListaCpss(A, 4, 0.4, 1.2, 13.0, share_W=False, device="cpu")
    np.testing.assert_array_equal(cp.variables["ListaCpss_W3"].numpy(), A)   # W_k = A, not A / L
    al = lista.Alista(A, lista.alista_weight(A), 4, 0.4, 1.2, 13.0, device="cpu")
    assert list(al.variables) == ["Alista_theta%d" % i for i in range(1, 5)] + \
        ["Alista_step_size%d" % i for i in range(1, 5)]
    with pytest.raises(NotImplementedError):
        lista.ListaCp(A, 4, 0.4, D=np.eye(12), device="cpu")
    with pytest.raises(NotImplementedError):
        lt.run(task="cs")
    with pytest.raises(ValueError):
        m.create_cell(1)


def _args(**kw):
    a = _lib.IstaArgs()
    fake = 1 << 20      # aligned non-null addresses: the checks run before any launch and never dereference
    a.form, a.batch, a.m, a.n, a.num_layers, a.k0, a.k1, a.share_W = lista.COUPLED, 4, 8, 16, 4, 0, 4, 0
    a.A = a.W = a.theta = a.y = a.xs = a.zs = a.rs = fake
    a.ldy = 24
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.skipif(not os.path.exists(_lib.LIB_PATH), reason="library not built")
def test_ista_abi_rejects_bad_arguments_without_gpu():
    L = _lib.lib()
    nb = C.c_size_t()
    assert L.l2o_ista_workspace_bytes(C.byref(_args()), C.byref(nb)) == _lib.L2O_OK
    assert nb.value == 4 * (4 * 4 * 16 + 4 * 8 * 2)
    bad = [dict(form=2), dict(batch=0), dict(k0=2, k1=2), dict(k1=5), dict(k0=-1), dict(A=None), dict(W=None),
           dict(theta=None), dict(y=None), dict(ldy=7), dict(share_W=2), dict(y=(1 << 20) + 2),
           dict(form=lista.LISTA, B1=None)]
    for kw in bad:
        assert L.l2o_ista_workspace_bytes(C.byref(_args(**kw)), C.byref(nb)) == _lib.L2O_E_INVALID, kw
        assert L.l2o_ista_fwd(C.byref(_args(**kw)), None) == _lib.L2O_E_INVALID, kw
    assert L.l2o_ista_fwd(C.byref(_args(xs=None)), None) == _lib.L2O_E_INVALID
    assert L.l2o_ista_fwd(C.byref(_args(n=4096, ldy=4096)), None) == _lib.L2O_E_UNSUPPORTED
    # the shared-memory plan binds before M, N <= 2048: coupled 4 (8 (2M + 3N) + 2048) bytes <= 200 KB
    assert L.l2o_ista_workspace_bytes(C.byref(_args(m=1024, n=1365, ldy=1024)), C.byref(nb)) == _lib.L2O_OK
    assert L.l2o_ista_workspace_bytes(C.byref(_args(m=1024, n=1366, ldy=1024)), C.byref(nb)) == \
        _lib.L2O_E_UNSUPPORTED
    lista_args = dict(form=lista.LISTA, B1=1 << 20)   # LISTA: 4 (8 (M + 4N) + 2048) bytes
    assert L.l2o_ista_workspace_bytes(C.byref(_args(m=1024, n=1280, ldy=1024, **lista_args)), C.byref(nb)) == \
        _lib.L2O_OK
    assert L.l2o_ista_workspace_bytes(C.byref(_args(m=1024, n=1281, ldy=1024, **lista_args)), C.byref(nb)) == \
        _lib.L2O_E_UNSUPPORTED
    # the largest plans of each form (run on the GPU by test_lista_abi_gpu) and their +1 neighbours in M and in N
    largest = [({}, (1024, 1365)), ({}, (2048, 682)), ({}, (3, 2046)),
               (lista_args, (1024, 1280)), (lista_args, (2048, 1024)), (lista_args, (4, 1535))]
    for kw, (m, n) in largest:
        assert L.l2o_ista_workspace_bytes(C.byref(_args(m=m, n=n, ldy=m, **kw)), C.byref(nb)) == _lib.L2O_OK, (m, n)
        for mm, nn in ((m + 1, n), (m, n + 1)):
            assert L.l2o_ista_workspace_bytes(C.byref(_args(m=mm, n=nn, ldy=mm, **kw)), C.byref(nb)) == \
                _lib.L2O_E_UNSUPPORTED, (mm, nn)
    g = _lib.IstaGrads()
    assert L.l2o_ista_bwd(C.byref(_args()), C.byref(g), None) == _lib.L2O_E_INVALID          # no d_xk / dtheta
    g.d_xk = g.dtheta = g.scratch = 1 << 20
    assert L.l2o_ista_bwd(C.byref(_args(rs=None)), C.byref(g), None) == _lib.L2O_E_INVALID   # coupled needs r_k
    g.dtheta = (1 << 20) + 4
    assert L.l2o_ista_bwd(C.byref(_args()), C.byref(g), None) == _lib.L2O_E_INVALID          # misaligned double
    la = _lib.IstaLossArgs()
    assert L.l2o_ista_loss_grad(C.byref(la), None) == _lib.L2O_E_INVALID
    la.task, la.batch, la.m, la.n, la.x, la.d_x, la.x_true, la.ldx = 0, 2, 3, 4, 1 << 20, 1 << 20, None, 4
    assert L.l2o_ista_loss_grad(C.byref(la), None) == _lib.L2O_E_INVALID
