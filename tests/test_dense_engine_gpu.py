"""The dense engine (l2o_dense_step / l2o_dense_unroll_bwd, the KernelDeepLSTM path) against an fp64 reference.

DenseNetHandle is driven directly, over a grid of shapes that reaches what the network-level tests cannot: several
128-row CTAs with a ragged last one, the largest features and hidden width (a dtheta image of 121 KB of shared
memory), tanh outputs, a Linear-only net, n_in != n_out both ways (a stride that uses K where O belongs shows only
there), and a 100-step unroll.  Every theta block, biases included, is random, and the initial state is random, so
every term of the backward carries gradient from t = 0 on.  The BPTT's dtheta is compared block by block (gate rows of
the inputs, recurrent gate rows, gate biases, output Linear) with fp64 autograd, each on its own scale.  The last test meta-trains two filter banks through one KernelDeepLSTM with
MetaOptimizer, eagerly and from a captured CUDA graph."""
import types

import numpy as np
import pytest
import torch

from oracle import l2o_oracle as orc
from tests.helpers import REL_TOL, arena_to_state, assert_theta_close, rel_err, state_to_arena, wild_gradients

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOGSIGN_K = 5.0

# id: (layers, K, O, LogAndSign, tanh output, scale, R, T)
CASES = {
    "ragged_33cta": ((20, 20), 9, 9, False, False, 0.1, 4133, 20),
    "max_f_h": ((32, 32), 64, 64, True, False, 0.1, 300, 7),
    "tanh_one_row_tail": ((32,), 25, 25, True, True, 0.5, 129, 5),
    "mixed_1_32": ((1, 32), 6, 6, False, False, 0.1, 128, 5),
    "mixed_32_1": ((32, 1), 6, 6, False, False, 0.1, 128, 5),
    "linear_only": ((), 16, 16, True, True, 1.0, 1, 3),
    "k128_o3": ((20,), 128, 3, False, False, 0.1, 257, 4),
    "k5_o40": ((20,), 5, 40, False, False, 0.1, 200, 4),
    "long_unroll": ((20, 20), 9, 9, False, False, 0.1, 1000, 100),
}
IMITATION = ["ragged_33cta", "max_f_h", "tanh_one_row_tail", "k128_o3", "k5_o40", "linear_only", "long_unroll"]


# ---------------------------------------------------------------------------------------------------------- reference
def dense_shapes(layers, K, O, logsign):
    """(module, variable, shape) of theta in the engine's order: lstm_l/w_gates [kin + H, 4H], lstm_l/b_gates [4H],
    linear/w [top, O], linear/b [O]."""
    out, kin = [], 2 * K if logsign else K
    for i, h in enumerate(layers, start=1):
        out += [(f"lstm_{i}", "w_gates", (kin + h, 4 * h)), (f"lstm_{i}", "b_gates", (4 * h,))]
        kin = h
    return out + [("linear", "w", (kin, O)), ("linear", "b", (O,))]


def theta_blocks(layers, K, O, logsign):
    """(name, offset, count) per theta block; a gate matrix splits into its input rows and its recurrent rows."""
    off, out = 0, []
    for mod, var, shape in dense_shapes(layers, K, O, logsign):
        cnt = int(np.prod(shape))
        if var == "w_gates":
            k_in = shape[0] - shape[1] // 4
            out += [(f"{mod}/w_gates[inputs]", off, k_in * shape[1]), (f"{mod}/w_gates[h]", off + k_in * shape[1],
                                                                        cnt - k_in * shape[1])]
        else:
            out.append((f"{mod}/{var}", off, cnt))
        off += cnt
    return out


def ref_apply(layers, K, O, logsign, tanh, scale, theta, inp, state):
    """One step of the row-wise net in the dtype of theta.  inp: [K, R] (element (k, r) at k * R + r, the engine's
    layout); state: tuple over layers of (h, c) [R, H].  Preprocessing interleaves (log, sign) per input like
    orc.kernel_net_apply; snt.LSTM with forget bias +1 and gates i|j|f|o (orc.lstm_cell); Linear [top, O]; scale with
    optional tanh.  Returns (delta [O, R], next state)."""
    w, off = {}, 0
    for mod, var, shp in dense_shapes(layers, K, O, logsign):
        n = int(np.prod(shp))
        w.setdefault(mod, {})[var] = theta[off:off + n].reshape(shp)
        off += n
    rows = inp.t()
    u = orc.log_and_sign(rows.unsqueeze(-1), LOGSIGN_K).reshape(rows.shape[0], -1) if logsign else rows
    out, nxt = u, []
    for li in range(1, len(layers) + 1):
        h, c = state[li - 1]
        hn, cn = orc.lstm_cell(out, h, c, w[f"lstm_{li}"]["w_gates"], w[f"lstm_{li}"]["b_gates"])
        nxt.append((hn, cn))
        out = hn
    y = out @ w["linear"]["w"] + w["linear"]["b"]
    y = torch.tanh(y) * scale if tanh else y * scale
    return y.t(), tuple(nxt)


def random_theta(layers, K, O, logsign, gen, gain=1.0, out_gain=1.0):
    """Every block random at gain / sqrt(fan_in), biases included (a zero bias hides a bias read from the wrong place)."""
    parts, fan = [], None
    for mod, var, shp in dense_shapes(layers, K, O, logsign):
        if var in ("w_gates", "w"):
            fan = shp[0]
        g = out_gain if mod == "linear" else gain
        parts.append(torch.randn(int(np.prod(shp)), generator=gen, dtype=torch.float64) * (g / np.sqrt(fan)))
    return torch.cat(parts).float()


def random_state(layers, R, gen, amp=0.5):
    return tuple(((torch.rand(R, h, generator=gen, dtype=torch.float64) * 2 - 1).mul(amp).float(),
                  (torch.rand(R, h, generator=gen, dtype=torch.float64) * 2 - 1).mul(amp).float()) for h in layers)


def inputs(K, R, logsign, gen, amp=0.5):
    if logsign:
        return wild_gradients(K * R, gen).view(K, R)
    return (torch.randn(K, R, generator=gen, dtype=torch.float64) * amp).float()


class Case:
    """One grid case: handle, theta, initial state and the input sequence [T, K, R]."""

    def __init__(self, name, seed=0):
        from open_l2o_b200.engine import DenseNetHandle
        self.name = name
        (self.layers, self.K, self.O, self.logsign, self.tanh, self.scale, self.R, self.T) = CASES[name]
        gen = torch.Generator().manual_seed(1234 + seed)
        self.h = DenseNetHandle(self.layers, self.K, self.O, preprocess_name="LogAndSign" if self.logsign else "identity",
                                preprocess_options={"k": LOGSIGN_K} if self.logsign else None, scale=self.scale,
                                tanh_output=self.tanh)
        # the tanh cases drive the output Linear hard enough that tanh is far from linear there
        self.theta = random_theta(self.layers, self.K, self.O, self.logsign, gen, gain=1.5,
                                  out_gain=3.0 if self.tanh else 1.0)
        assert self.theta.numel() == self.h.n_theta
        self.s0 = random_state(self.layers, self.R, gen)
        self.in_seq = torch.stack([inputs(self.K, self.R, self.logsign, gen) for _ in range(self.T)])
        self.gen = gen

    def ref(self, dtype, theta=None, in_seq=None, s0=None):
        """fp64 / fp32 reference forward: the deltas [T, O, R] and the states after each step."""
        theta = self.theta.to(dtype) if theta is None else theta
        in_seq = self.in_seq if in_seq is None else in_seq
        s = tuple((h.to(dtype), c.to(dtype)) for h, c in (self.s0 if s0 is None else s0))
        ds, ss = [], []
        for t in range(in_seq.shape[0]):
            d, s = ref_apply(self.layers, self.K, self.O, self.logsign, self.tanh, self.scale, theta,
                             in_seq[t].to(dtype), s)
            ds.append(d)
            ss.append(s)
        return torch.stack(ds), ss

    def forward(self, theta=None, in_seq=None, s0=None):
        """T engine steps recording checkpoints like meta.py: slot t -> slot t + 1 of one arena."""
        theta = (self.theta if theta is None else theta).to(DEV)
        in_seq = (self.in_seq if in_seq is None else in_seq).to(DEV).contiguous()
        T, _, R = in_seq.shape
        slot = self.h.state_floats * R
        ckpt = torch.zeros(max((T + 1) * slot, 1), device=DEV)
        if slot:
            ckpt[:slot].copy_(state_to_arena(self.s0 if s0 is None else s0, R).to(DEV))
        deltas = torch.empty(T, self.O, R, device=DEV)
        for t in range(T):
            self.h.step(theta, in_seq[t], ckpt[t * slot:(t + 1) * slot] if slot else None,
                        ckpt[(t + 1) * slot:(t + 2) * slot] if slot else None, delta=deltas[t])
        return deltas, (ckpt if slot else None), in_seq

    def arena_states(self, ckpt, R):
        """tuple over steps t = 1..T of tuple over layers of (h, c) from the checkpoint arena."""
        slot, out = self.h.state_floats * R, []
        for t in range(1, self.T + 1):
            a, off, st = ckpt[t * slot:(t + 1) * slot], 0, []
            for H in self.layers:
                st.append((a[off:off + R * H].view(R, H), a[off + R * H:off + 2 * R * H].view(R, H)))
                off += 2 * R * H
            out.append(tuple(st))
        return out


def slack(ref32, ref64):
    """max(1e-5, 3 x the fp32 reference's distance from fp64), on the max-norm relative scale of rel_err."""
    return max(REL_TOL, 3.0 * rel_err(ref32, ref64))


# ---------------------------------------------------------------------------------------------------------- the oracle
@pytest.mark.parametrize("logsign,tanh", [(False, False), (True, True)])
def test_reference_matches_kernel_net_oracle(logsign, tanh):
    """With n_in = n_out = K the local reference is orc.kernel_net_apply on a [kw, kh, cin, cout] filter bank."""
    gen = torch.Generator().manual_seed(5)
    kernel_shape, cin, cout, layers = [3, 2], 4, 5, (7, 3)
    K, R = 6, 20
    theta = random_theta(layers, K, K, logsign, gen, gain=1.5, out_gain=3.0).double()
    g = (wild_gradients(K * R, gen) if logsign else torch.randn(K * R, generator=gen)).double()
    s0 = tuple((h.double(), c.double()) for h, c in random_state(layers, R, gen))
    d_ref, s_ref = orc.kernel_net_apply(kernel_shape, layers, theta, g.view(*kernel_shape, cin, cout), s0,
                                        preprocess_k=LOGSIGN_K if logsign else None, scale=0.3, tanh_output=tanh)
    d, s = ref_apply(layers, K, K, logsign, tanh, 0.3, theta, g.view(K, R), s0)
    assert rel_err(d.reshape(-1), d_ref.reshape(-1)) <= 1e-14
    for (h, c), (hr, cr) in zip(s, s_ref):
        assert rel_err(h, hr) <= 1e-14 and rel_err(c, cr) <= 1e-14


# ---------------------------------------------------------------------------------------------------------- step
@pytest.mark.parametrize("name", list(CASES))
def test_dense_step_chain_matches_fp64(name):
    cs = Case(name)
    d64, s64 = cs.ref(torch.float64)
    d32, s32 = cs.ref(torch.float32)
    if cs.tanh:   # the output layer really is nonlinear here
        assert float((d64 / cs.scale).abs().max()) > 0.5
    x0 = torch.randn(cs.O, cs.R, generator=cs.gen)
    deltas, ckpt, _ = cs.forward()
    # x += delta over the same chain, in a second pass with x given
    x = x0.to(DEV).clone()
    slot = cs.h.state_floats * cs.R
    buf = [torch.empty(max(slot, 1), device=DEV), torch.empty(max(slot, 1), device=DEV)]
    if slot:
        buf[0].copy_(state_to_arena(cs.s0, cs.R).to(DEV))
    for t in range(cs.T):
        cs.h.step(cs.theta.to(DEV), cs.in_seq[t].to(DEV).contiguous(), buf[t % 2] if slot else None,
                  buf[(t + 1) % 2] if slot else None, x=x.view(-1))
    torch.cuda.synchronize()
    worst = 0.0
    for t in range(cs.T):
        e = rel_err(deltas[t], d64[t])
        assert e <= slack(d32[t], d64[t]), (name, t, "delta", e)
        worst = max(worst, e / slack(d32[t], d64[t]))
    if cs.layers:
        states = cs.arena_states(ckpt, cs.R)
        for t in range(cs.T):
            for li, ((h, c), (h64, c64), (h32, c32)) in enumerate(zip(states[t], s64[t], s32[t])):
                assert rel_err(h, h64) <= slack(h32, h64), (name, t, li, "h", rel_err(h, h64))
                assert rel_err(c, c64) <= slack(c32, c64), (name, t, li, "c", rel_err(c, c64))
                worst = max(worst, rel_err(h, h64) / slack(h32, h64), rel_err(c, c64) / slack(c32, c64))
    x64 = x0.double() + d64.sum(0)
    x32 = x0 + d32.sum(0)
    assert rel_err(x, x64) <= slack(x32, x64), (name, "x", rel_err(x, x64))
    print(f"{name}: worst step error / tolerance {worst:.3f}")


@pytest.mark.parametrize("name", ["ragged_33cta", "max_f_h", "tanh_one_row_tail", "mixed_32_1", "k128_o3"])
def test_dense_step_row_slice_and_aliasing_bitwise(name):
    """A contiguous slice of rows run as its own call gives the same bits as in the full call (any stride slip between
    in / state / delta / x shows with zero tolerance); in place equals out of place; x += delta is one fp32 add; the
    x-only and the delta-only call agree."""
    cs = Case(name)
    R, th, g = cs.R, cs.theta.to(DEV), cs.in_seq[0].to(DEV).contiguous()
    s_in = state_to_arena(cs.s0, R).to(DEV) if cs.layers else None
    s_out = torch.empty_like(s_in) if cs.layers else None
    delta = torch.empty(cs.O, R, device=DEV)
    x0 = torch.randn(cs.O, R, generator=cs.gen).to(DEV)
    cs.h.step(th, g, s_in, s_out, delta=delta)
    x = x0.clone()
    cs.h.step(th, g, s_in, torch.empty_like(s_in) if cs.layers else None, x=x)
    assert torch.equal(x, x0 + delta)
    x = x0.clone()
    d2 = torch.empty_like(delta)
    cs.h.step(th, g, s_in, torch.empty_like(s_in) if cs.layers else None, x=x, delta=d2)
    assert torch.equal(d2, delta) and torch.equal(x, x0 + delta)
    if cs.layers:   # in place
        s_ip = s_in.clone()
        d_ip = torch.empty_like(delta)
        cs.h.step(th, g, s_ip, s_ip, delta=d_ip)
        assert torch.equal(s_ip, s_out) and torch.equal(d_ip, delta)
    # a slice of rows that starts and ends inside a CTA of the full call
    a = min(37, R - 1)
    b = min(R, a + 200)
    n = b - a
    g_sl = g[:, a:b].contiguous()
    st_sl = tuple((h[a:b], c[a:b]) for h, c in cs.s0)
    s_in_sl = state_to_arena(st_sl, n).to(DEV) if cs.layers else None
    s_out_sl = torch.empty_like(s_in_sl) if cs.layers else None
    d_sl = torch.empty(cs.O, n, device=DEV)
    cs.h.step(th, g_sl, s_in_sl, s_out_sl, delta=d_sl)
    torch.cuda.synchronize()
    assert torch.equal(d_sl, delta[:, a:b])
    if cs.layers:
        full = arena_to_state(s_out, cs.layers, R)
        part = arena_to_state(s_out_sl, cs.layers, n)
        for (h, c), (hs, css) in zip(full, part):
            assert torch.equal(hs, h[a:b]) and torch.equal(css, c[a:b])


# ---------------------------------------------------------------------------------------------------------- BPTT
def _ref_dtheta(cs, objective):
    """d objective / d theta by autograd through the reference unroll, in fp64 and in fp32."""
    out = {}
    for dt in (torch.float64, torch.float32):
        th = cs.theta.to(dt).requires_grad_(True)
        d, _ = cs.ref(dt, theta=th)
        (g,) = torch.autograd.grad(objective(d, dt), th)
        out[dt] = g.detach()
    return out[torch.float64], out[torch.float32]


def _assert_blocks(cs, got, g64, g32, tag):
    got = got.detach().cpu()
    worst = 0.0
    for blk, off, cnt in theta_blocks(cs.layers, cs.K, cs.O, cs.logsign):
        e, tol = rel_err(got[off:off + cnt], g64[off:off + cnt]), slack(g32[off:off + cnt], g64[off:off + cnt])
        assert float(g64[off:off + cnt].abs().max()) > 0.0, (cs.name, tag, blk)   # every block carries gradient
        assert e <= tol, (cs.name, tag, blk, e, tol)
        worst = max(worst, e / tol)
    print(f"{cs.name} {tag}: worst block error / tolerance {worst:.3f}")
    return worst


def _g_rec_case(cs):
    """g_rec [T + 1, O, R]; the input sequence is g_rec[:T] when K = O (as meta.py records it), its own draw if not."""
    g_rec = torch.randn(cs.T + 1, cs.O, cs.R, generator=cs.gen) * 0.5
    if cs.K == cs.O and not cs.logsign:
        cs.in_seq = g_rec[:cs.T].clone()
    elif cs.K == cs.O:   # LogAndSign: keep the wild inputs and use them as the recorded gradients too
        g_rec[:cs.T] = cs.in_seq
    return g_rec


@pytest.mark.parametrize("name", list(CASES))
def test_dense_bptt_g_rec_every_block_matches_fp64(name):
    """g_rec mode: dtheta of sum_t <delta_t, lambda_t> with lambda_t = sum_{tau > t} g_rec[tau]."""
    cs = Case(name)
    g_rec = _g_rec_case(cs)
    lam = torch.flip(torch.cumsum(torch.flip(g_rec[1:], [0]), 0), [0])   # lam[t] = sum_{tau = t+1..T} g_rec[tau]
    g64, g32 = _ref_dtheta(cs, lambda d, dt: (d * lam.to(dt)).sum())
    _, ckpt, in_seq = cs.forward()
    dtheta = torch.zeros(cs.h.n_theta, dtype=torch.float64, device=DEV)
    cs.h.unroll_bwd(cs.theta.to(DEV), cs.K * cs.R, cs.T, in_seq, ckpt, dtheta, g_rec=g_rec.to(DEV).contiguous())
    torch.cuda.synchronize()
    _assert_blocks(cs, dtheta, g64, g32, "g_rec")


@pytest.mark.parametrize("name", IMITATION)
def test_dense_bptt_imitation_every_block_matches_fp64(name):
    """Imitation mode: dtheta of sum_t 0.5 ||label_t - delta_t||^2 / n_total, n_total larger than this call's elements
    (one subset of a multi-subset task).

    This dtheta is J^T r summed over rows and steps, with the residual r_t = (delta_t - label_t) / n_total, and the
    engine forms r from its own fp32 deltas.  The sum cancels strongly, so it is far more sensitive to r than to the
    backward: on an H100 at T = 100 (long_unroll) the engine's deltas are 3.8e-7 from fp64 (fp32 autograd: 5.2e-7),
    yet J^T r computed in fp64 at the engine's residual is already 2.0e-5 from the fp64 gradient in lstm_2/b_gates,
    while fp32 autograd's own residual happens to move that block by only 6.4e-6.  So the backward is checked against
    fp64 autograd at the engine's residual (engine within 2e-6 of it on every block), and the gradient of the loss
    itself against plain fp64 autograd with that measured residual effect added to the slack."""
    cs = Case(name)
    d64, _ = cs.ref(torch.float64)
    labels = (d64 + torch.randn(d64.shape, generator=cs.gen, dtype=torch.float64) * d64.std()).float()
    n_total = 3 * cs.K * cs.R
    g64, g32 = _ref_dtheta(cs, lambda d, dt: 0.5 * ((labels.to(dt) - d) ** 2).sum() / n_total)
    deltas, ckpt, in_seq = cs.forward()
    dtheta = torch.zeros(cs.h.n_theta, dtype=torch.float64, device=DEV)
    cs.h.unroll_bwd(cs.theta.to(DEV), cs.K * cs.R, cs.T, in_seq, ckpt, dtheta, labels=labels.to(DEV).contiguous(),
                    n_total=n_total)
    torch.cuda.synchronize()
    r_eng = (deltas.cpu().double() - labels.double()) / n_total
    b64, b32 = _ref_dtheta(cs, lambda d, dt: (d * r_eng.to(dt)).sum())
    _assert_blocks(cs, dtheta, b64, b32, "imitation at the engine's residual")
    got = dtheta.cpu()
    for blk, off, cnt in theta_blocks(cs.layers, cs.K, cs.O, cs.logsign):
        s = slice(off, off + cnt)
        tol = slack(g32[s], g64[s]) + rel_err(b64[s], g64[s])
        assert rel_err(got[s], g64[s]) <= tol, (name, "imitation", blk, rel_err(got[s], g64[s]), tol)


# ---------------------------------------------------------------------------------------------------------- contract
@pytest.mark.parametrize("name", ["ragged_33cta", "tanh_one_row_tail"])
def test_dense_bptt_accumulates_into_dtheta(name):
    """dtheta is accumulated (+=): a pre-filled vector plus two calls on two row sets that share theta equals the
    pre-fill plus the fp64 gradient over all rows."""
    cs = Case(name)
    g_rec = torch.randn(cs.T + 1, cs.O, cs.R, generator=cs.gen) * 0.5
    lam = torch.flip(torch.cumsum(torch.flip(g_rec[1:], [0]), 0), [0])
    g64, g32 = _ref_dtheta(cs, lambda d, dt: (d * lam.to(dt)).sum())
    pre = torch.randn(cs.h.n_theta, generator=cs.gen, dtype=torch.float64) * float(g64.abs().max())
    dtheta = pre.to(DEV)
    cut = cs.R // 2 + 3
    for a, b in ((0, cut), (cut, cs.R)):
        s0 = tuple((h[a:b], c[a:b]) for h, c in cs.s0)
        _, ckpt, in_seq = cs.forward(in_seq=cs.in_seq[:, :, a:b], s0=s0)
        cs.h.unroll_bwd(cs.theta.to(DEV), cs.K * (b - a), cs.T, in_seq, ckpt, dtheta,
                        g_rec=g_rec[:, :, a:b].to(DEV).contiguous())
    torch.cuda.synchronize()
    _assert_blocks(cs, dtheta.cpu() - pre, g64, g32, "two calls")


def test_dense_empty_calls_launch_nothing_and_tc_is_refused():
    """T = 0 and rows = 0 BPTT calls return without a launch and leave dtheta untouched (an empty step is covered at the
    C-ABI level in tests/test_dense_args_cpu.py: an empty tensor has no address to pass as its input)."""
    from open_l2o_b200.engine import ENGINE_TC, L2OError, launch_count
    cs = Case("max_f_h")
    th = cs.theta.to(DEV)
    _, ckpt, in_seq = cs.forward()
    g_rec = torch.zeros(cs.T + 1, cs.O, cs.R, device=DEV)
    pre = torch.randn(cs.h.n_theta, generator=cs.gen, dtype=torch.float64).to(DEV)
    dtheta = pre.clone()
    torch.cuda.synchronize()
    n0 = launch_count()
    cs.h.unroll_bwd(th, cs.K * cs.R, 0, in_seq, ckpt, dtheta, g_rec=g_rec)
    cs.h.unroll_bwd(th, 0, cs.T, in_seq, ckpt, dtheta, g_rec=g_rec)
    torch.cuda.synchronize()
    assert launch_count() == n0
    assert torch.equal(dtheta, pre)
    with pytest.raises(L2OError):
        cs.h.set_engine(ENGINE_TC)


# ---------------------------------------------------------------------------------------------------------- meta-training
def test_two_filter_banks_one_kernel_net_training_matches_oracle(monkeypatch):
    """Two conv filter banks with the same [3, 3] kernel ([3,3,4,40]: 160 rows, [3,3,40,8]: 320 rows) trained by one
    KernelDeepLSTM (32, 32) with LogAndSign, so two per-variable BPTT runs add into one dtheta whose 15,145 floats
    (59 KB) need the shared-memory opt-in above 48 KB; the biases go to a coordinate-wise net.  Three unrolls
    (eager, eager, then CUDA-graph capture and replay) of forward + BPTT + TF-Adam against the oracle's autograd."""
    from open_l2o_b200 import meta
    from open_l2o_b200.variables import get_variable, random_normal_initializer
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)   # the optimizee's convolutions in fp32, as the oracle's
    kw = kh = 3
    c0, c1, c2, T = 4, 40, 8, 5
    gen = torch.Generator().manual_seed(17)
    data = torch.randn(4, c0, 6, 6, generator=gen)
    target = torch.randn(4, c2, 6, 6, generator=gen)
    data_d, target_d = data.to(DEV), target.to(DEV)

    def conv_loss(w1, b1, w2, b2, dat, tgt):   # HWIO filters, as the reference stores them
        hid = torch.tanh(torch.nn.functional.conv2d(dat, w1.permute(3, 2, 0, 1), b1, padding=1))
        out = torch.nn.functional.conv2d(hid, w2.permute(3, 2, 0, 1), b2, padding=1)
        return ((out - tgt) ** 2).mean()

    def problem():
        w1 = get_variable("c1/w", shape=[kw, kh, c0, c1], initializer=random_normal_initializer(stddev=0.2))
        b1 = get_variable("c1/b", shape=[c1], initializer=random_normal_initializer(stddev=0.2))
        w2 = get_variable("c2/w", shape=[kw, kh, c1, c2], initializer=random_normal_initializer(stddev=0.1))
        b2 = get_variable("c2/b", shape=[c2], initializer=random_normal_initializer(stddev=0.2))
        return conv_loss(w1, b1, w2, b2, data_d, target_d)

    conv_opts = {"kernel_shape": [kw, kh], "layers": (32, 32), "scale": 0.1, "preprocess_name": "LogAndSign",
                 "preprocess_options": {"k": LOGSIGN_K}}
    net_config = {"conv": {"net": "KernelDeepLSTM", "net_options": conv_opts},
                  "cw": {"net": "CoordinateWiseDeepLSTM", "net_options": {"layers": (20, 20), "scale": 0.1}}}
    optimizer = meta.MetaOptimizer(**net_config)
    ms = optimizer.meta_minimize(problem, T, learning_rate=0.001,
                                 net_assignments=[("conv", ["c1/w", "c2/w"]), ("cw", ["c1/b", "c2/b"])])
    prog = optimizer.program
    assert prog.nets["conv"].theta.numel() == 15_145
    assert sum(r.key == "conv" for r in prog.runs) == 2
    sess = meta.Session()
    sess.run(ms.reset)
    th = {k: prog.nets[k].theta.cpu().clone() for k in ("conv", "cw")}
    adam = {k: (torch.zeros_like(v), torch.zeros_like(v)) for k, v in th.items()}
    names = [v["name"] for v in prog.variables]
    shapes = {v["name"]: v["shape"] for v in prog.variables}
    views = {}
    for j, nm in enumerate(names):
        n = int(np.prod(shapes[nm]))
        views[nm] = slice(prog.var_off[j], prog.var_off[j] + n)

    def f_of(xf):
        return conv_loss(*(xf[views[nm]].view(shapes[nm]) for nm in ("c1/w", "c1/b", "c2/w", "c2/b")), data, target)

    spec_cw = orc.NetSpec(layers=(20, 20), scale=0.1)
    x = prog.X.cpu().clone()
    s_conv = {nm: tuple((torch.zeros(shapes[nm][2] * shapes[nm][3], 32), torch.zeros(shapes[nm][2] * shapes[nm][3], 32))
                        for _ in range(2)) for nm in ("c1/w", "c2/w")}
    bias_idx = torch.cat([torch.arange(prog.N)[views[nm]] for nm in ("c1/b", "c2/b")])
    s_cw = orc.initial_state(spec_cw, c1 + c2)
    for it in range(3):
        cost, xs, _, _ = sess.run([ms.fx, ms.x, ms.update, ms.step])
        p = {k: v.clone().requires_grad_(True) for k, v in th.items()}
        xc, sc, sw_, total = x, dict(s_conv), s_cw, 0.0
        for t in range(T):
            xg = xc.detach().requires_grad_(True)
            (g,) = torch.autograd.grad(f_of(xg), xg)
            g = g.detach()
            total = total + f_of(xc)
            upd = torch.zeros(prog.N, dtype=xc.dtype)
            for nm in ("c1/w", "c2/w"):
                d, sc[nm] = orc.kernel_net_apply([kw, kh], (32, 32), p["conv"], g[views[nm]].view(shapes[nm]), sc[nm],
                                                 preprocess_k=LOGSIGN_K, scale=0.1)
                upd = upd.index_add(0, torch.arange(prog.N)[views[nm]], d.reshape(-1))
            db, sw_ = orc.net_apply(spec_cw, p["cw"], g[bias_idx].unsqueeze(-1), sw_)
            xc = xc + upd.index_add(0, bias_idx, db)
        fx_T = f_of(xc)
        total = total + fx_T
        grads = torch.autograd.grad(total, [p["conv"], p["cw"]])
        assert abs(cost - float(fx_T.detach())) <= REL_TOL * abs(float(fx_T.detach())), it
        got_x = torch.cat([torch.as_tensor(np.asarray(a)).reshape(-1) for a in xs])
        want_x = torch.cat([xc.detach()[views[nm]] for nm in names])
        assert rel_err(got_x, want_x) <= REL_TOL, it
        for k, g in zip(("conv", "cw"), grads):
            th[k], m_, v_ = orc.tf_adam_step(th[k], g, adam[k][0], adam[k][1], it + 1, lr=0.001)
            adam[k] = (m_, v_)
            assert_theta_close(prog.nets[k].theta, types.SimpleNamespace(theta=th[k], last_grad=g), tag=(it, k))
        x = xc.detach()
        s_conv = {nm: tuple((h.detach(), c.detach()) for h, c in s) for nm, s in sc.items()}
        s_cw = tuple((h.detach(), c.detach()) for h, c in sw_)
    # the third unroll ran from a captured graph, BPTT launches (59 KB of dynamic shared memory) included
    assert not prog._graph_failed and True in prog._graphs
