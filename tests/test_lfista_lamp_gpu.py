"""The LFISTA and LAMP kernels against the fp64 oracle: every layer's x_k and every variable's gradient, exact integer
inputs, layer ranges carried through the second state, a deterministic backward, training steps, CUDA-graph replay
and the launch count of a training step."""
import ctypes as C

import numpy as np
import pytest
import torch

from open_l2o_b200 import _lib, lista, lista_train as lt
from open_l2o_b200.engine import _ptr, _stream, adam_step, launch_count
from oracle import lista_oracle as lo
from tests import lfista_lamp_cases as fc

pytestmark = pytest.mark.gpu

K = 16
SHAPES = [(256, 512, 128), (256, 512, 1024), (250, 500, 9), (25, 50, 128), (5, 10, 128), (512, 256, 129)]
CASES = [("lfista", s, False) for s in SHAPES] + [("lamp", s, sh) for s in SHAPES for sh in (False, True)]
# Entries within fp32 rounding of the threshold can be classified differently by the kernel and the oracle; the
# oracle runs with the kernel's classification, and the flips per [B, N] mask are bounded.
MAX_FLIPS = 4


def _rel(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _built(name, M, N, share_W, T=K, seed=0):
    m = fc.generic_model(name, M, N, share_W, seed=seed, T=T)
    for k in range(T):
        m.create_cell(k)
    return m


def _kernel_lives(m, bufs, k1, V=None):
    """The kernel's classification of every layer, from its records and the variables V it ran with (default the
    model's): LFISTA |z| > theta_k, z != 0; LAMP r != 0 and |r| >= max(sqrt(rvar) lam_k, 0) with the recorded
    sqrt(rvar)."""
    V = m.variables if V is None else V
    lives = []
    for k in range(k1):
        z = bufs["zs"][k]
        if m.form == lista.LFISTA:
            th = V[m.name + "_theta%d" % (k + 1)]
            lives.append(((z.abs() > th) & (z != 0)).cpu())
        else:
            th = torch.clamp_min(bufs["rowrec"][k][:, :1] * V[m.name + "_lam%d" % (k + 1)], 0.0)
            lives.append(((z.abs() >= th) & (z != 0)).cpu())
    return lives


@pytest.mark.parametrize("name,shape,share_W", CASES)
def test_forward_and_gradients_match_fp64(name, shape, share_W):
    M, N, B = shape
    m = _built(name, M, N, share_W)
    data = torch.as_tensor(lista.make_data(M, N, B, seed=7)["train"]).cuda()
    loss = m.loss_and_grad(data, lista.TASK_SC)
    torch.cuda.synchronize()
    bufs = m._bufs_for(B, True)
    lives = _kernel_lives(m, bufs, K)
    P = fc.model_leaves(m)
    y = data[:, :M].cpu().double()
    rec = []
    xs_ref = fc.model_forward(m, P, y, K, lives=lives, rec=rec)
    for k in range(K):
        assert _rel(bufs["xs"][k], xs_ref[k]) <= 1e-5, (k, _rel(bufs["xs"][k], xs_ref[k]))
    if m.form == lista.LAMP:
        for k in range(K):
            r, sq, b, v = rec[k]
            assert _rel(bufs["rs"][k], v) <= 1e-5, k
            assert _rel(bufs["rowrec"][k][:, 0], sq[:, 0]) <= 1e-5, k
            assert torch.equal(bufs["rowrec"][k][:, 1].cpu(), b[:, 0].detach().float()), k   # fp32 count / M
    # the oracle's own classification differs from the kernel's only at rounding ties
    with torch.no_grad():
        Pd = {n: v.detach() for n, v in P.items()}
        zs_ref, rec_ref = [], []
        fc.model_forward(m, Pd, y, K, lives=lives, zs_out=zs_ref, rec=rec_ref)
    for k in range(K):
        if m.form == lista.LFISTA:
            own = (zs_ref[k].abs() > Pd[m.name + "_theta%d" % (k + 1)]) & (zs_ref[k] != 0)
        else:
            r, sq, _, _ = rec_ref[k]
            own = (r.abs() >= torch.clamp_min(sq * Pd[m.name + "_lam%d" % (k + 1)], 0)) & (r != 0)
        assert int((own != lives[k]).sum()) <= MAX_FLIPS, k
    ref_loss = lo.sc_loss(xs_ref[-1], data[:, M:].cpu().double())
    assert abs(float(loss.sum()) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss))
    for x in xs_ref:
        x.retain_grad()
    ref_loss.backward()
    scales = _scalar_term_sums(m, P, xs_ref, lives, rec)
    for vname, leaf in P.items():
        ref = leaf.grad if leaf.grad is not None else torch.zeros_like(leaf)
        got = m._grad_span(vname, 1).view(ref.shape).cpu()
        if ref.abs().max() == 0:
            assert got.abs().max() == 0, vname
            continue
        # each matrix against its own magnitude; each scalar against the sum of its terms' magnitudes, since a
        # signed sum over a few rows can cancel far below its terms
        err = float((got - ref).abs().max() / max(float(ref.abs().max()), scales.get(vname, 0.0)))
        assert err <= 1e-5, (vname, err)
    if m.form == lista.LFISTA:
        assert not m._grad_span("Lfista_Wm2", 1).any()


def _scalar_term_sums(m, P, xs_ref, lives, rec):
    """Sum of |term| of every per-layer scalar gradient: LFISTA dtheta_k = -sum sign(z) live dx_{k+1}; LAMP
    dlam_k = sum_b g_b sqrt(rvar_b) with g_b = -sum_n sign(r) live dx_{k+1}, and ds_k = <v_k, dr_k W_k^T>."""
    out = {}
    for k in range(len(xs_ref)):
        d = xs_ref[k].grad.abs() * lives[k].double()
        if m.form == lista.LFISTA:
            out[m.name + "_theta%d" % (k + 1)] = float(d.sum())
        else:
            sq = rec[k][1]
            out[m.name + "_lam%d" % (k + 1)] = float((d.sum(dim=1, keepdim=True) * sq.detach()).sum())
            if m.share_W:
                W = P[m.name + "_W"].detach().abs()
                out[m.name + "_step_size%d" % (k + 1)] = float((rec[k][3].detach().abs() * (d @ W.T)).sum())
    return out


def _integer_lfista(M, N, B, T, seed):
    """LFISTA on inputs whose every fp32 sum is an exact integer: sparse {-1, 0, 1} weights, integer y, x_true and
    theta."""
    g = torch.Generator().manual_seed(seed)
    A = lista.make_data(M, N, 1, seed=seed)["A"]
    m = lista.Lfista(A, T, 0.4)
    for vname, v in m.variables.items():
        if "_theta" in vname:
            v.fill_(float(torch.randint(0, 3, (1,), generator=g)))
        else:
            w = torch.randint(-1, 2, v.shape, generator=g) * (torch.rand(v.shape, generator=g) < 0.15)
            v.copy_(w.float())
    for k in range(T):
        m.create_cell(k)
    data = torch.randint(-3, 4, (B, M + N), generator=g).float().cuda()
    return m, data


@pytest.mark.parametrize("shape", [(12, 20, 9), (7, 33, 16), (30, 8, 17)])
def test_lfista_exact_integers_match_bit_for_bit(shape):
    M, N, B = shape
    T = 4
    m, data = _integer_lfista(M, N, B, T, seed=sum(shape))
    m.loss_and_grad(data, lista.TASK_SC)
    torch.cuda.synchronize()
    bufs = m._bufs_for(B, True)
    P = fc.model_leaves(m)
    xs_ref = fc.model_forward(m, P, data[:, :M].cpu().double(), T)   # the oracle's own classification
    assert float(max(x.abs().max() for x in xs_ref)) < 2 ** 20
    for k in range(T):
        assert torch.equal(bufs["xs"][k].cpu().double(), xs_ref[k].detach()), k
    lo.sc_loss(xs_ref[-1], data[:, M:].cpu().double()).backward()
    for vname, leaf in P.items():
        ref = leaf.grad if leaf.grad is not None else torch.zeros_like(leaf)
        assert torch.equal(m._grad_span(vname, 1).view(ref.shape).cpu(), ref), vname


def _pass(m, y, k0, k1, x_in=None, s2_in=None, d_xk=None, d_s2=None):
    """One forward [k0, k1) through the C ABI with fresh records, and with d_xk its backward into fresh gradient
    arenas.  Returns the records, d_x_in, d_s2_in and the gradient arena."""
    B = y.shape[0]
    L = k1 - k0
    z = lambda *s: torch.empty(*s, dtype=torch.float32, device="cuda")
    bufs = {"xs": z(L, B, m.N), "zs": z(L, B, m.N), "sel": None,
            "rs": z(L, B, m.M) if m.form == lista.LAMP else None,
            "rowrec": z(L, B, 2) if m.form == lista.LAMP else None}
    a = m._args(y, y.stride(0), B, k1, bufs, True)
    a.k0 = k0
    a.x_in, a.s2_in = _ptr(x_in), _ptr(s2_in)
    lib = _lib.lib()
    _lib.check(lib.l2o_ista_fwd(C.byref(a), _stream()), "l2o_ista_fwd")
    if d_xk is None:
        return bufs
    m.grads.fill_(float("nan"))
    S = m.M if m.form == lista.LAMP else m.N
    out = {"d_x_in": z(B, m.N), "d_s2_in": z(B, S)}
    nbytes = C.c_size_t()
    _lib.check(lib.l2o_ista_workspace_bytes(C.byref(a), C.byref(nbytes)), "workspace")
    scratch = torch.empty((nbytes.value + 3) // 4, dtype=torch.float32, device="cuda")
    W, dW, B1, dB1, step, dstep = m._weights()
    g = _lib.IstaGrads()
    g.d_xk, g.d_x_in, g.d_s2, g.d_s2_in = _ptr(d_xk), _ptr(out["d_x_in"]), _ptr(d_s2), _ptr(out["d_s2_in"])
    g.dW, g.dB1, g.dW2 = _ptr(dW, torch.float64, "dW"), _ptr(dB1, torch.float64, "dB1"), \
        _ptr(m._second()[1], torch.float64, "dW2")
    g.dtheta, g.dstep = _ptr(m._theta_grad(), torch.float64, "dtheta"), _ptr(dstep, torch.float64, "dstep")
    g.scratch = _ptr(scratch)
    _lib.check(lib.l2o_ista_bwd(C.byref(a), C.byref(g), _stream()), "l2o_ista_bwd")
    torch.cuda.synchronize()
    bufs.update(out)
    bufs["grads"] = m.grads.clone()
    return bufs


@pytest.mark.parametrize("name,share_W", [("lfista", False), ("lamp", False), ("lamp", True)])
@pytest.mark.parametrize("j", [1, 2, 5])
def test_split_pass_reproduces_full_pass(name, share_W, j):
    M, N, B, T = 40, 72, 19, 8
    m = _built(name, M, N, share_W, T=T, seed=3)
    y = torch.as_tensor(lista.make_data(M, N, B, seed=5)["train"][:, :M]).cuda().contiguous()
    d_xk = torch.randn(B, N, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    full = _pass(m, y, 0, T, d_xk=d_xk)
    s2_in = full["xs"][j - 2] if (name == "lfista" and j >= 2) else (full["rs"][j - 1] if name == "lamp" else None)
    top = _pass(m, y, j, T, x_in=full["xs"][j - 1], s2_in=s2_in, d_xk=d_xk)
    bot = _pass(m, y, 0, j, d_xk=top["d_x_in"], d_s2=top["d_s2_in"])
    for rec in ("xs", "zs", "rs", "rowrec"):
        if full[rec] is not None:
            assert torch.equal(torch.cat([bot[rec], top[rec]]), full[rec]), rec
    # per-layer variables: each comes from one of the two passes, bit for bit; a variable every layer shares
    # (We, a shared W) is the sum of the two passes' parts
    for vname in m.variables:
        got_top, got_bot = (p[vname] for p in (_grad_views(m, top["grads"]), _grad_views(m, bot["grads"])))
        want = _grad_views(m, full["grads"])[vname]
        birth = m.births[vname]
        if vname.endswith(("_We1", "_W")):
            assert torch.allclose(got_top + got_bot, want, rtol=1e-12, atol=1e-300), vname
        else:   # a variable of layer k, Wm_k included (it reads x_{k-1}), belongs to the pass that runs layer k
            assert torch.equal(got_top if birth >= j else got_bot, want), vname
            assert not (got_bot if birth >= j else got_top).any(), vname
    assert torch.equal(bot["d_x_in"], full["d_x_in"])
    assert torch.equal(bot["d_s2_in"], full["d_s2_in"])


def _grad_views(m, arena):
    out = {}
    for vname, v in m.variables.items():
        off = (v.data_ptr() - m.params.data_ptr()) // 4
        out[vname] = arena[off:off + v.numel()].view(v.shape)
    return out


@pytest.mark.parametrize("name,share_W", [("lfista", False), ("lamp", False), ("lamp", True)])
def test_backward_is_deterministic_at_a_partial_batch(name, share_W):
    M, N, B = 250, 500, 13
    m = _built(name, M, N, share_W)
    data = torch.as_tensor(lista.make_data(M, N, B, seed=9)["train"]).cuda()
    m.loss_and_grad(data, lista.TASK_SC)
    first = m.grads.clone()
    m.grads.fill_(float("nan"))
    m.loss_and_grad(data, lista.TASK_SC)
    torch.cuda.synchronize()
    assert torch.equal(first, m.grads)


@pytest.mark.parametrize("name,share_W", [("lfista", False), ("lamp", False), ("lamp", True)])
def test_training_steps_follow_the_oracle(name, share_W):
    """Layer-wise steps on the kernels: each step's gradient (with the stage's 0.3^age multipliers) against the
    oracle's at the same weights, and the Adam update against Keras Adam applied to that gradient."""
    M, N, B, T = 25, 50, 64, 4
    d = lista.make_data(M, N, 4 * B, seed=11)
    m = lt.build_model(name, d["A"], T, 0.4, share_W, 1.2, 13.0)
    train = torch.as_tensor(d["train"]).cuda()
    tr = lt.KernelTrainer(m, train, train, lista.TASK_SC, 0.0, B, B, 2)
    for k in range(T):
        tr.create_cell(k)
        for stage in range(3):
            gs = lt.gradient_scales(k, stage, T)
            tr.begin_stage(1e-3, gs)
            for i in range(2):
                batch = train[i * B:(i + 1) * B]
                P = fc.model_leaves(m)
                V = {n: v.detach().clone() for n, v in m.variables.items()}
                p0 = m.params.double().cpu()
                mv = (tr.m.double().cpu(), tr.v.double().cpu())
                tr.step(batch)
                torch.cuda.synchronize()
                lives = _kernel_lives(m, m._bufs_for(B, True), k + 1, V)
                xs = fc.model_forward(m, P, batch[:, :M].cpu().double(), k + 1, lives=lives)
                lo.sc_loss(xs[-1], batch[:, M:].cpu().double()).backward()
                for vname, leaf in P.items():
                    g = torch.zeros_like(leaf) if leaf.grad is None else leaf.grad
                    g = g * float(gs[m.births[vname]])
                    got = _grad_views(m, m.grads.cpu())[vname]
                    if g.abs().max() == 0:
                        assert not got.any(), vname
                    else:
                        assert float((got - g).abs().max() / g.abs().max()) <= 1e-5, (k, stage, vname)
                p, mm, vv = p0.clone(), mv[0].clone(), mv[1].clone()
                lo.keras_adam_step(p, m.grads.cpu(), mm, vv, tr.t, tr.lr, eps=lt.KERAS_EPS)
                assert float((m.params.double().cpu() - p).abs().max()) <= 1e-6, (k, stage)
    ev = lt.evaluate(m, train, lista.TASK_SC, 0.0, B)
    assert len(ev) == T and all(np.isfinite(ev))


@pytest.mark.parametrize("name,share_W", [("lfista", False), ("lamp", True)])
def test_graph_replay_equals_eager_and_launches_do_not_grow_with_layers(name, share_W):
    M, N, B = 256, 512, 128
    data = torch.as_tensor(lista.make_data(M, N, B, seed=2)["train"]).cuda()
    counts = {}
    for T in (4, 16):
        m = _built(name, M, N, share_W, T=T)
        tr = lt.KernelTrainer(m, data, data, lista.TASK_SC, 0.0, B, B, 1)
        tr.begin_stage(1e-3, lt.gradient_scales(T - 1, 1, T))
        tr.step(data)      # allocate the buffers outside the count and the capture
        torch.cuda.synchronize()
        c0 = launch_count()
        tr.step(data)
        torch.cuda.synchronize()
        counts[T] = launch_count() - c0
    assert counts[4] == counts[16] == 5     # forward, loss, backward (2), Adam

    m = _built(name, M, N, share_W)
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


def test_lamp_keras_output_layout():
    M, N, B, T = 25, 50, 16, 3
    m = _built("lamp", M, N, False, T=T)
    data = torch.as_tensor(lista.make_data(M, N, B, seed=4)["train"]).cuda()
    out = m(data)
    assert out.shape == (B, M + T * (M + N))
    y = data[:, :M]
    assert torch.equal(out[:, :M], y) and torch.equal(out[:, M:2 * M], y)      # v_0 = y
    xs = m.forward(data, T).clone()
    for k in range(T):
        assert torch.equal(out[:, 2 * M + k * (M + N):2 * M + k * (M + N) + N], xs[k])
