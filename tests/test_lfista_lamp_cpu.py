"""LFISTA and LAMP without a GPU: the fp64 oracle at initial weights against plain FISTA and AMP loops, the models'
variables against the reference's, model selection, and the C ABI's argument checks for the two forms."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from open_l2o_b200 import _lib, lista, lista_train as lt
from tests import lfista_lamp_cases as fc


def _problem(M=20, N=40, B=6, seed=0):
    d = lista.make_data(M, N, B, seed=seed)
    return d["A"], torch.as_tensor(d["train"][:, :M], dtype=torch.float64)


def _soft(z, t):
    return np.sign(z) * np.maximum(np.abs(z) - t, 0.0)


def test_lfista_oracle_at_initial_weights_is_fista():
    A, y = _problem()
    T, lam = 12, 0.4
    m = lista.Lfista(A, T, lam, device="cpu")
    P = {n: v.double() for n, v in m.variables.items()}
    xs = fc.model_forward(m, P, y, T)
    L = 1.001 * np.linalg.norm(A.astype(np.float64), 2) ** 2
    t, mom = fc.fista_momenta_ref(T)
    A64, Y = A.astype(np.float64), y.numpy()
    x = xp = np.zeros((Y.shape[0], A.shape[1]))
    for k in range(T):
        u = x + mom[k] * (x - xp) if k >= 1 else x
        xp, x = x, _soft(u - (u @ A64.T - Y) @ A64 / L, lam / L)
        # the arena holds fp32 weights: W (1 + m_k) rounded once, so compare at fp32 rounding of the weights
        np.testing.assert_allclose(xs[k].numpy(), x, rtol=0, atol=2e-6 * max(1.0, np.abs(x).max()))
    assert m.variables["Lfista_Wg3"].numpy() == pytest.approx(
        (np.eye(A.shape[1], dtype=np.float32) - m.variables["Lfista_We1"].numpy() @ A) * np.float32(1 + mom[2]),
        abs=1e-6)


def test_lamp_oracle_at_initial_weights_is_amp():
    A, y = _problem()
    T, lam = 10, 0.4
    m = lista.Lamp(A, T, lam, device="cpu")
    P = {n: v.double() for n, v in m.variables.items()}
    xs = fc.model_forward(m, P, y, T)
    M = A.shape[0]
    L = 1.001 * np.linalg.norm(A.astype(np.float64), 2) ** 2
    A64, Y = A.astype(np.float64), y.numpy()
    x, v = np.zeros((Y.shape[0], A.shape[1])), np.zeros_like(Y)
    for k in range(T):
        b = (x != 0).sum(axis=1, keepdims=True) / M if k else 0.0
        v = Y - x @ A64.T + b * v
        theta = lam * np.linalg.norm(v, axis=1, keepdims=True) / np.sqrt(M)
        x = _soft(x + v @ A64 / L, theta)
        np.testing.assert_allclose(xs[k].numpy(), x, rtol=0, atol=1e-6 * max(1.0, np.abs(x).max()))


def test_lamp_oracle_zero_row_has_no_theta_gradient():
    A, y = _problem(B=3)
    y[1] = 0.0
    m = lista.Lamp(A, 3, 0.4, device="cpu")
    P = fc.model_leaves(m)
    xs = fc.model_forward(m, P, y, 3)
    (xs[-1] ** 2).sum().backward()
    for n, p in P.items():
        assert torch.isfinite(p.grad).all(), n


def test_lfista_variables_match_reference():
    A, _ = _problem(M=6, N=9)
    M, N, T, lam = 6, 9, 5, 0.4
    m = lista.Lfista(A, T, lam, share_W=True, device="cpu")    # share_W is accepted and ignored
    L = 1.001 * np.linalg.norm(A.astype(np.float64), 2) ** 2
    B = A.T / np.float32(L)
    W = np.eye(N, dtype=np.float32) - B @ A
    _, mom = fc.fista_momenta_ref(T)
    want = {"Lfista_We1": ((N, M), 0, B)}
    for i in range(1, T):
        want["Lfista_Wg%d" % (i + 1)] = ((N, N), i, W * (1 + mom[i]))
        want["Lfista_Wm%d" % (i + 1)] = ((N, N), i, -mom[i] * W)
    for i in range(T):
        want["Lfista_theta%d" % (i + 1)] = ((1,), i, np.float32(lam / L))
    assert set(m.variables) == set(want)
    for n, (shape, birth, init) in want.items():
        assert tuple(m.variables[n].shape) == shape, n
        assert m.births[n] == birth, n
        np.testing.assert_allclose(m.variables[n].numpy(), np.broadcast_to(init, shape), rtol=1e-6, atol=1e-7)
    assert m.layer_variables(1) == ["Lfista_Wg2", "Lfista_Wm2", "Lfista_theta2"]
    assert m.share_W is False and m.one_W is False
    # Lfista_Wm2 is created with layer 1 and no layer reads it: the oracle gives it no gradient
    P = fc.model_leaves(m)
    y = torch.rand(3, M, dtype=torch.float64)
    (fc.model_forward(m, P, y, T)[-1] ** 2).sum().backward()
    assert not P["Lfista_Wm2"].grad.any()
    assert P["Lfista_Wm3"].grad.abs().max() > 0


@pytest.mark.parametrize("share_W", [False, True])
def test_lamp_variables_match_reference(share_W):
    A, _ = _problem(M=6, N=9)
    T, lam = 4, 0.4
    m = lista.Lamp(A, T, lam, share_W=share_W, device="cpu")
    assert m.name == "Lamp"
    L = 1.001 * np.linalg.norm(A.astype(np.float64), 2) ** 2
    want = {}
    if share_W:
        want["Lamp_W"] = ((6, 9), 0, A / np.float32(L))
        for i in range(T):
            want["Lamp_step_size%d" % (i + 1)] = ((1,), i, 1.0)
    else:
        for i in range(T):
            want["Lamp_W%d" % (i + 1)] = ((6, 9), i, A / np.float32(L))
    for i in range(T):
        want["Lamp_lam%d" % (i + 1)] = ((1,), i, lam)   # model_lam itself, not lam / L
    assert set(m.variables) == set(want)
    for n, (shape, birth, init) in want.items():
        assert tuple(m.variables[n].shape) == shape, n
        assert m.births[n] == birth, n
        np.testing.assert_allclose(m.variables[n].numpy(), np.broadcast_to(init, shape).astype(np.float32),
                                   rtol=1e-6)
    with pytest.raises(NotImplementedError):
        lista.Lamp(A, T, lam, D=np.eye(6), device="cpu")
    with pytest.raises(NotImplementedError):
        lista.Lfista(A, T, lam, D=np.eye(6), device="cpu")


def test_build_model_and_cli_accept_lfista_and_lamp(monkeypatch):
    A, _ = _problem(M=6, N=9)
    assert isinstance(lt.build_model("lfista", A, 3, 0.4, False, 1.2, 13.0, device="cpu"), lista.Lfista)
    lp = lt.build_model("lamp", A, 3, 0.4, True, 1.2, 13.0, device="cpu")
    assert isinstance(lp, lista.Lamp) and lp.share_W and lp.name == "Lamp"
    for name in ("step_lista", "tista", "glista"):
        with pytest.raises(NotImplementedError) as e:
            lt.build_model(name, A, 3, 0.4, False, 1.2, 13.0, device="cpu")
        assert "LFISTA" not in str(e.value) and "LAMP" not in str(e.value)
    seen = []
    monkeypatch.setattr(lt, "run", lambda **kw: seen.append(kw["model_name"]))
    lt.main(["--model_name", "lfista"])
    lt.main(["--model_name", "lamp"])
    assert seen == ["lfista", "lamp"]
    with pytest.raises(SystemExit):
        lt.main(["--model_name", "tista"])


def _args(form, **kw):
    a = _lib.IstaArgs()
    fake = 1 << 20      # aligned non-null addresses: the checks run before any launch and never dereference
    a.form, a.batch, a.m, a.n, a.num_layers, a.k0, a.k1, a.share_W = form, 4, 8, 16, 4, 0, 4, 0
    a.theta = a.y = a.xs = a.zs = a.rs = a.W = fake
    if form == lista.LFISTA:
        a.B1 = a.W2 = fake
    else:
        a.A = a.rowrec = fake
    a.ldy = 24
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.skipif(not os.path.exists(_lib.LIB_PATH), reason="library not built")
def test_two_state_abi_rejects_bad_arguments_without_gpu():
    L = _lib.lib()
    nb = C.c_size_t()
    fake = 1 << 20
    for form in (lista.LFISTA, lista.LAMP):
        assert L.l2o_ista_workspace_bytes(C.byref(_args(form)), C.byref(nb)) == _lib.L2O_OK
        assert nb.value == 4 * (4 * 4 * 16 + 4 * 8 * 2)   # the four forms' workspace
    bad = [(lista.LFISTA, dict(B1=None)), (lista.LFISTA, dict(W=None)), (lista.LFISTA, dict(W2=None)),
           (lista.LFISTA, dict(share_W=1)), (lista.LFISTA, dict(step=fake)), (lista.LFISTA, dict(ss_rank=fake)),
           (lista.LFISTA, dict(W2=fake + 2)), (lista.LFISTA, dict(s2_in=fake + 1)),
           (lista.LAMP, dict(A=None)), (lista.LAMP, dict(W=None)), (lista.LAMP, dict(ss_rank=fake)),
           (lista.LAMP, dict(rowrec=fake + 2)), (lista.LAMP, dict(theta=None)), (4, {}), (-1, {})]
    for form, kw in bad:
        assert L.l2o_ista_workspace_bytes(C.byref(_args(form, **kw)), C.byref(nb)) == _lib.L2O_E_INVALID, (form, kw)
        assert L.l2o_ista_fwd(C.byref(_args(form, **kw)), None) == _lib.L2O_E_INVALID, (form, kw)
    # layers that read no Wg / Wm need none
    assert L.l2o_ista_workspace_bytes(C.byref(_args(lista.LFISTA, k1=2, W2=None)), C.byref(nb)) == _lib.L2O_OK
    assert L.l2o_ista_workspace_bytes(C.byref(_args(lista.LFISTA, k1=1, W=None, W2=None)), C.byref(nb)) == \
        _lib.L2O_OK
    assert L.l2o_ista_workspace_bytes(C.byref(_args(lista.LAMP, share_W=1, step=fake)), C.byref(nb)) == _lib.L2O_OK
    # LFISTA 4 (8 (M + 5N) + 2048) bytes, LAMP 4 (8 (2M + 3N) + 2048) bytes <= 200 KB, and M, N <= 2048
    largest = [(lista.LFISTA, (1144, 1000)), (lista.LFISTA, (2044, 820)), (lista.LFISTA, (2048, 819)),
               (lista.LFISTA, (4, 1228)), (lista.LAMP, (1024, 1365)), (lista.LAMP, (2048, 682)),
               (lista.LAMP, (3, 2046))]
    for form, (m, n) in largest:
        assert L.l2o_ista_workspace_bytes(C.byref(_args(form, m=m, n=n, ldy=m)), C.byref(nb)) == _lib.L2O_OK, (m, n)
        for mm, nn in ((m + 1, n), (m, n + 1)):
            assert L.l2o_ista_workspace_bytes(C.byref(_args(form, m=mm, n=nn, ldy=mm)), C.byref(nb)) == \
                _lib.L2O_E_UNSUPPORTED, (form, mm, nn)
    g = _lib.IstaGrads()
    g.d_xk = g.dtheta = g.scratch = g.dB1 = fake
    for form, kw in [(lista.LAMP, dict(rowrec=None)), (lista.LAMP, dict(rs=None)), (lista.LAMP, dict(zs=None)),
                     (lista.LFISTA, dict(zs=None))]:
        assert L.l2o_ista_bwd(C.byref(_args(form, **kw)), C.byref(g), None) == _lib.L2O_E_INVALID, (form, kw)
    g.dB1 = None
    assert L.l2o_ista_bwd(C.byref(_args(lista.LFISTA)), C.byref(g), None) == _lib.L2O_E_INVALID     # no dWe
    g.dB1, g.dW2 = fake, fake + 4
    assert L.l2o_ista_bwd(C.byref(_args(lista.LFISTA)), C.byref(g), None) == _lib.L2O_E_INVALID     # misaligned
    g.dW2, g.d_s2_in = None, fake + 2
    assert L.l2o_ista_bwd(C.byref(_args(lista.LAMP)), C.byref(g), None) == _lib.L2O_E_INVALID       # misaligned
