"""Tensor-core engine with the gate scales folded into its weight image.

The forward images B1 / B2 hold every gate column of the extended weight matrix [W; b] multiplied by -s_g (s_g = log2e
for i, f, o and 2 log2e for j), with snt.LSTM's forget bias +1 added to the f bias row first, so the MMA delivers the
exponents the epilogues feed to ex2.  The dX images T1 / T2 stay unscaled.  These tests read the image back through
l2o_tc_weight_image with a generic theta (no zero biases, no repeated constants), and run one forward and one BPTT with
that theta against the fp64 oracle at full and ragged tile counts: state, checkpoints, x and f(x) of the forward, and
dtheta and the carries (the adjoint of the initial state, lambda) of the backward."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import l2o_oracle as orc
from tests.helpers import REL_TOL, SPECS, arena_to_state, make_handle, random_state, rel_err, state_to_arena

pytestmark = pytest.mark.gpu

NETS = ["dm_identity", "dm_logsign", "rnnprop"]
H = 20
LOG2E = np.float32(1.4426950408889634)
GATE_SCALE = [-LOG2E, np.float32(-2.0) * LOG2E, -LOG2E, -LOG2E]   # i | j | f | o


def generic_theta(spec, seed):
    """init_theta plus N(0, 0.1) on every LSTM and input-projection entry: nonzero, distinct biases, so a gate scale
    or the forget bias on the wrong column shows.  The output layer keeps its small init."""
    th = orc.init_theta(spec, seed=seed, out_gain=0.05)
    g = torch.Generator().manual_seed(100 + seed)
    k = th.numel() - (H + 1)
    th[:k] += 0.1 * torch.randn(k, generator=g)
    return th


# ---- the image layout (cwlstm_tc.cuh), restated --------------------------------------------------------------------
def gate_ref_col(n):
    return (2 * ((n >> 3) & 1) + (n & 1)) * H + 5 * ((n & 7) >> 1) + (n >> 4)


def vec_unit(c, base):
    return 5 * ((c - base) & 3) + ((c - base) >> 2)


def unit_col(u, base):
    return base + 4 * (u % 5) + u // 5


def img_index(k, n, ncols):
    return ((k >> 2) * (ncols // 8) + (n >> 3)) * 32 + (n & 7) * 4 + (k & 3)


def dx_gate_col(k):
    return (k & ~7) + 2 * (k & 3) + ((k >> 2) & 1)


def dx_unit(c):
    return -1 if 2 * ((c % 24) >> 3) + (c & 1) >= 5 else 5 * ((c & 7) >> 1) + 2 * ((c % 24) >> 3) + (c & 1)


class Geo:
    def __init__(self, spec):
        fc = spec.preprocess_name == "fc"
        self.F = 20 if fc else (2 if spec.preprocess_name == "LogAndSign" else 1)
        self.fc = fc
        self.h1, self.h2, self.one = (24, 44, 20) if fc else (4, 24, self.F)
        self.l1 = (0, 6) if fc else (0, 3)   # k-blocks
        self.l2 = (2, 8) if fc else (0, 6)
        self.n1, self.n2 = (48 if fc else 24), 48

    def ext(self, P, l2, c, col):
        """extended weight of layer l2 at operand-row column c and reference gate column col (0: a zero row)"""
        w, b = (P["lstm_2/w_gates"], P["lstm_2/b_gates"]) if l2 else (P["lstm_1/w_gates"], P["lstm_1/b_gates"])
        if c == self.one:
            return b[col]
        in_h1, in_h2 = self.h1 <= c < self.h1 + H, self.h2 <= c < self.h2 + H
        if not l2:
            if in_h1:
                return w[self.F + vec_unit(c, self.h1), col]
            if self.fc and c < H:
                return w[vec_unit(c, 0), col]
            if not self.fc and c < self.F:
                return w[c, col]
            return np.float32(0)
        if in_h1:
            return w[vec_unit(c, self.h1), col]
        if in_h2:
            return w[H + vec_unit(c, self.h2), col]
        return np.float32(0)


def _image(h, theta, with_transposed):
    from open_l2o_b200 import _lib
    L = _lib.lib()
    floats = L.l2o_tc_weight_image(h._h, None, None, with_transposed, None)
    assert floats > 0
    img = torch.full((floats,), float("nan"), device="cuda")
    th = theta.cuda()
    assert L.l2o_tc_weight_image(h._h, ctypes.c_void_p(th.data_ptr()), ctypes.c_void_p(img.data_ptr()),
                                 with_transposed, None) == floats
    torch.cuda.synchronize()
    return img.cpu().numpy()


def _check_split(hi, lo, want):
    """hi is tf32, and hi + lo is the fp32 value before the split up to lo's own tf32 rounding"""
    assert (hi.view(np.uint32) & 0x1FFF == 0).all()
    assert np.all(np.abs((hi.astype(np.float64) + lo) - want) <= 2.0 ** -20 * np.abs(want))


@pytest.mark.parametrize("name", NETS)
def test_weight_image_columns_are_scaled(name):
    spec = SPECS[name]
    h = make_handle(spec)
    theta = generic_theta(spec, seed=11)
    P = {m + "/" + k: v.numpy().astype(np.float32) for m, d in orc.unpack_theta(spec, theta).items() for k, v in d.items()}
    G = Geo(spec)
    img = _image(h, theta, 1)
    assert img.size == (G.l1[1] - G.l1[0] + G.l2[1] - G.l2[0]) * 8 * 80 * 2 + 80 * (G.n1 + G.n2) * 2
    assert np.isfinite(img).all()
    # B1h | B1l | B2h | B2l: -s_g (w + [c == 1, g == f])
    off = 0
    for l2, (lo_kb, hi_kb) in ((False, G.l1), (True, G.l2)):
        K = 8 * (hi_kb - lo_kb)
        want = np.zeros(K * 80)
        idx = np.zeros(K * 80, dtype=np.int64)
        for k in range(K):
            c = 8 * lo_kb + k
            for n in range(80):
                col = gate_ref_col(n)
                gate = col // H
                w = np.float32(G.ext(P, l2, c, col))
                if c == G.one and gate == 2:
                    w = np.float32(w + np.float32(1.0))
                want[k * 80 + n] = np.float32(GATE_SCALE[gate] * w)
                idx[k * 80 + n] = img_index(k, n, 80)
        _check_split(img[off + idx], img[off + K * 80 + idx], want)
        off += 2 * K * 80
    # T1h | T1l | T2h | T2l: the unscaled weights, K = 80 gates in dx_gate_col order
    for l2, nc in ((False, G.n1), (True, G.n2)):
        want = np.zeros(80 * nc)
        idx = np.zeros(80 * nc, dtype=np.int64)
        for k in range(80):
            for n in range(nc):
                u = dx_unit(n)
                if u >= 0:
                    c = unit_col(u, G.h1 if n // 24 == 0 else (G.h2 if l2 else 0))
                    want[k * nc + n] = G.ext(P, l2, c, gate_ref_col(dx_gate_col(k)))
                idx[k * nc + n] = img_index(k, n, nc)
        _check_split(img[off + idx], img[off + 80 * nc + idx], want)
        off += 2 * 80 * nc
    assert off == img.size
    # the forward's image is the BPTT's first part
    fwd = _image(h, theta, 0)
    assert np.array_equal(fwd, img[:fwd.size])


def _oracle(spec, theta, x0, state0, prob, T, dtype):
    """fp64 / fp32 oracle: fx, x_T, per-step states, dtheta and the adjoint of the initial state"""
    th = theta.to(dtype).clone().requires_grad_(True)
    st = tuple((hh.to(dtype).clone().requires_grad_(True), cc.to(dtype).clone().requires_grad_(True)) for hh, cc in state0)
    p = orc.FusedProblem("rastrigin_sep", prob.a.to(dtype), prob.b.to(dtype), prob.alpha, prob.fscale)
    mv0 = None
    if spec.rnnprop:
        n = x0.numel()
        mv0 = (torch.zeros(n, dtype=dtype, device=x0.device), torch.zeros(n, dtype=dtype, device=x0.device))
    states, s, x, mv = [st], st, x0.to(dtype), mv0
    for _ in range(T):   # the per-step states, as the checkpoints hold them
        r = orc.unroll(spec, th, x, s, None, 1, mv0=mv, step0=len(states), grad_of=p.f_and_g)
        s, x, mv = r.state_final, r.x_final, r.mv_final
        states.append(s)
    res = orc.unroll(spec, th, x0.to(dtype), st, None, T, mv0=mv0, grad_of=p.f_and_g)
    leaves = [th] + [v for pair in st for v in pair]
    grads = torch.autograd.grad(res.loss, leaves)
    return dict(fx=res.fx.detach(), x=res.x_final.detach(), states=[tuple((a.detach(), b.detach()) for a, b in q)
                                                                   for q in states],
                dtheta=grads[0], d_state=torch.cat([g.reshape(-1) for g in grads[1:]]))


@pytest.mark.parametrize("name", NETS)
@pytest.mark.parametrize("n", [64 * 3, 1000, 64 * 140 + 37])
def test_forward_and_bptt_with_generic_theta_match_fp64(name, n):
    from open_l2o_b200.engine import ENGINE_TC, OPT_KINDS
    spec, T = SPECS[name], 6
    dev = "cuda"
    gen = torch.Generator().manual_seed(n)
    theta = generic_theta(spec, seed=3)
    a, b, x0 = (torch.randn(n, generator=gen) for _ in range(3))
    state0 = random_state(spec, n, gen, amp=0.5, dtype=torch.float64)
    prob = orc.FusedProblem("rastrigin_sep", a.to(dev), b.to(dev), alpha=10.0, fscale=1.0 / n)
    r64 = _oracle(spec, theta.to(dev), x0.to(dev), [(p.to(dev), q.to(dev)) for p, q in state0], prob, T, torch.float64)
    r32 = _oracle(spec, theta.to(dev), x0.to(dev), [(p.to(dev), q.to(dev)) for p, q in state0], prob, T, torch.float32)

    h = make_handle(spec)
    h.set_engine(ENGINE_TC)
    th = theta.to(dev)
    arena = state_to_arena([(p.float(), q.float()) for p, q in state0], n).to(dev)
    ckpt = torch.zeros((T + 1) * h.state_size(n), device=dev)
    g_rec = torch.zeros(T + 1, n, device=dev)
    # RNNProp's tanh output needs the recorded deltas in its BPTT; the DM nets run without them, so their forward takes
    # the full-tile instantiation when n is a multiple of 64
    delta = torch.zeros(T, n, device=dev) if spec.tanh_output else None
    fx = torch.zeros(T + 1, dtype=torch.float64, device=dev)
    x = x0.to(dev).clone()
    kw, in_seq = {}, g_rec
    if h.n_in == 2:
        in_seq = torch.zeros(T, 2, n, device=dev)
        kw = dict(m=torch.zeros(n, device=dev), v=torch.zeros(n, device=dev), step0=1, feat_rec=in_seq)
    h.unroll_fwd(th, n, T, arena, opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=prob.a, opt_b=prob.b, opt_alpha=10.0,
                 opt_fscale=1.0 / n, x=x, ckpt=ckpt, g_rec=g_rec, delta_seq=delta, fx=fx, **kw)
    torch.cuda.synchronize()

    def slack(key):
        return max(REL_TOL, 3.0 * rel_err(r32[key], r64[key]))
    assert rel_err(fx, r64["fx"]) <= slack("fx")
    assert rel_err(x, r64["x"]) <= slack("x")
    sf = h.state_floats

    def check_state(got, t):
        for g2, r2, f2 in zip(arena_to_state(got.cpu(), spec.layers, n), r64["states"][t], r32["states"][t]):
            for u, v, w in zip(g2, r2, f2):
                assert rel_err(u, v) <= max(REL_TOL, 3.0 * rel_err(w, v)), (t, rel_err(u, v), rel_err(w, v))
    for t in range(T + 1):   # checkpoint slot t holds the state before step t
        check_state(ckpt[t * sf * n:(t + 1) * sf * n], t)
    check_state(arena, T)

    dth = torch.zeros(h.n_theta, dtype=torch.float64, device=dev)
    d_state = torch.zeros(h.state_size(n), device=dev)
    lam = torch.zeros(n, device=dev)
    scratch = torch.zeros(T, n, 20, device=dev) if h.n_in == 2 else None
    h.unroll_bwd_carry(th, n, T, in_seq, ckpt, dth, d_state, lam, g_rec=g_rec, delta_seq=delta, scratch=scratch)
    torch.cuda.synchronize()
    assert rel_err(dth, r64["dtheta"]) <= slack("dtheta"), (rel_err(dth, r64["dtheta"]), slack("dtheta"))
    assert rel_err(d_state, r64["d_state"]) <= slack("d_state"), (rel_err(d_state, r64["d_state"]), slack("d_state"))
    assert rel_err(lam, g_rec[1:].double().sum(0)) <= REL_TOL
