"""CPU: the chunked fp64 references that tests/test_scale_bwd_tiles_gpu.py compares the L2O-Scale backward kernels
with (l2o_crnn_bwd, l2o_tadam_bwd, l2o_lrsgd_bwd), against whole-problem autograd through the oracles.

The CoordinatewiseRNN and the baselines are coordinate-wise, so the vector-Jacobian product of one step splits over
coordinate chunks: the per-coordinate adjoints (old planes, g) of a chunk are those of the whole problem, and d theta is
the sum of the chunks' d theta.  That is what lets the GPU tests build an fp64 reference at millions of coordinates in
bounded memory.  The one term that is not coordinate-wise, the CoordinatewiseRNN's per-tensor "decay := 0 if
ALL(ms == 0)" (SC/optimizer/utils.py:129-130), is inactive in every state with ms > 0, and the chunked reference
refuses states where it could fire."""
import math
from functools import partial

import pytest
import torch

from oracle import baselines_oracle as B
from oracle import crnn_oracle as CR
from tests.test_baselines_cpu import tadam_theta
from tests.test_crnn_gpu import crnn_generic_theta

CHUNK = 1 << 16   # coordinates per chunk of the references


def _leaf(t, dtype):
    return t.detach().to(dtype).requires_grad_(True)


def crnn_vjp(theta, planes, g, d_new, d_upd, dtype):
    """One CoordinatewiseRNN step through the oracle in `dtype`, on the inputs' device, over one tensor of n
    coordinates: (d theta, d planes_old [103, n], d g) of L = <d_new, planes'> + <d_upd, update>."""
    n = g.numel()
    assert bool((planes[100] > 0).all()), "ms == 0 somewhere: the per-tensor decay predicate is not coordinate-wise"
    th, pl, gg = _leaf(theta, dtype), _leaf(planes, dtype), _leaf(g.reshape(-1), dtype)
    _, new, upd = CR.step(th, [torch.zeros_like(gg)], [gg], CR.planes_to_states(pl, [n]))
    L = (d_new.to(dtype) * CR.state_to_planes(new)).sum() + (d_upd.to(dtype) * upd[0]).sum()
    return torch.autograd.grad(L, (th, pl, gg))


def tadam_vjp(theta, planes, g, d_new, d_upd, dtype):
    """One TrainableAdam step through the oracle: (d theta [4], d planes_old [3, n], d g) of
    L = <d_new, planes'> + <d_upd, update>.  The step count t is a constant (its plane's adjoint is 0)."""
    n = g.numel()
    th, pl, gg = _leaf(theta, dtype), _leaf(planes, dtype), _leaf(g.reshape(-1, 1), dtype)
    st = B.planes_to_states(pl, [n])[0]
    st["t"] = st["t"].detach()
    _, new, upd = B.tadam_compute_update(th, torch.zeros_like(gg), gg, st)
    L = (d_new.to(dtype) * B.state_to_planes([new])).sum() + (d_upd.to(dtype).reshape(-1, 1) * upd).sum()
    d_th, d_pl, d_g = torch.autograd.grad(L, (th, pl, gg))
    return d_th, d_pl, d_g.reshape(-1)


def lrs_vjp(rates, planes, g, d_new, d_upd, dtype, itr=0):
    """One LearningRateSchedule step (GlobalLearningRate: a one-entry table) through the oracle: (d rates, None, d g) of
    L = <d_upd, update>.  The schedule keeps no planes."""
    th, gg = _leaf(rates, dtype), _leaf(g.reshape(-1), dtype)
    _, _, upd = B.lrs_compute_update(th, torch.zeros_like(gg), gg, itr)
    d_rates, d_g = torch.autograd.grad((d_upd.to(dtype) * upd).sum(), (th, gg))
    return d_rates, None, d_g


def chunked_vjp(vjp, theta, planes, g, d_new, d_upd, dtype, chunk=CHUNK, each=None):
    """`vjp` over coordinate chunks [lo, hi) of at most `chunk` coordinates.  d theta is summed over the chunks in fp64
    and returned.  The per-coordinate adjoints of each chunk go to each(lo, hi, d_planes, d_g); without `each` they are
    concatenated and returned too: (d theta, d planes_old, d g).  planes / d_new may be None (no planes)."""
    n = g.numel()
    cut = lambda t, lo, hi: None if t is None else t[..., lo:hi]
    d_theta, parts = None, []
    for lo in range(0, n, chunk):
        hi = min(n, lo + chunk)
        dt, dp, dg = vjp(theta, cut(planes, lo, hi), g[lo:hi], cut(d_new, lo, hi), d_upd[lo:hi], dtype)
        d_theta = dt.double() if d_theta is None else d_theta + dt.double()
        if each is not None:
            each(lo, hi, dp, dg)
        else:
            parts.append((dp, dg))
    if each is not None:
        return d_theta
    dps = None if planes is None else torch.cat([p for p, _ in parts], 1)
    return d_theta, dps, torch.cat([q for _, q in parts])


# ---------------------------------------------------------------------------------------------------------------------
# generic states

def crnn_generic_planes(theta, n, seed, device="cpu", chunk=CHUNK):
    """CoordinatewiseRNN planes [103, n] (fp32) of a generic state: per-coordinate learning rates exp(U(-6, -3)), then
    two fp64 oracle steps with gradients N(0, 0.3^2), rounded to fp32.  Drawn in chunks from one generator on
    `device`, so the state at 4 M coordinates costs one chunk of fp64 memory."""
    gen = torch.Generator(device=device).manual_seed(seed)
    th = theta.double().to(device)
    init = CR.unpack_theta(th)["init_vector"].reshape(-1, 1)
    out = torch.empty(103, n, device=device)
    for lo in range(0, n, chunk):
        m = min(n, lo + chunk) - lo
        lr = torch.exp(torch.rand(m, generator=gen, dtype=torch.float64, device=device) * 3.0 - 6.0)
        ones = torch.ones(1, m, dtype=torch.float64, device=device)
        pl = torch.cat([init.expand(100, m), ones, ones, lr.reshape(1, m)], 0)
        for _ in range(2):
            gr = torch.randn(m, generator=gen, dtype=torch.float64, device=device) * 0.3
            _, new, _ = CR.step(th, [torch.zeros(m, dtype=torch.float64, device=device)], [gr],
                                CR.planes_to_states(pl, [m]))
            pl = CR.state_to_planes(new)
        out[:, lo:lo + m] = pl.float()
    return out


def tadam_generic_planes(n, seed, device="cpu"):
    """TrainableAdam planes m | t | v (fp32) of a hand-set state with v != 0 (the v-chain of the backward runs): t = 2,
    m ~ N(0, 0.1^2), v ~ U(0.01, 0.1) with every third coordinate at v = 0; and gradients g ~ U(-0.8, 0.8) (|g| < 1
    keeps 1 - pow(g^2, b2) > 0) with every 7th at 0 and every 11th (offset 1) at 1e-25, whose square underflows."""
    gen = torch.Generator(device=device).manual_seed(seed)
    m = torch.randn(n, generator=gen, device=device) * 0.1
    v = torch.rand(n, generator=gen, device=device) * 0.09 + 0.01
    v[::3] = 0.0
    g = torch.rand(n, generator=gen, device=device) * 1.6 - 0.8
    g[::7] = 0.0
    g[1::11] = 1e-25
    return torch.stack([m, torch.full((n,), 2.0, device=device), v]), g


TADAM_THETA = dict(lr=1e-3, b1=0.85, b2=0.9, eps=1e-7)   # (tests/test_baselines_gpu.py: the v != 0 backward test)


# ---------------------------------------------------------------------------------------------------------------------
# the chunked references against whole-problem autograd

SHAPES = [(33, 7), (5,), (300,), (129,)]   # 665 coordinates: chunks of 100 cross every tensor boundary


def _close(a, b, tol=1e-12):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).abs().max()) <= tol * max(float(b.abs().max()), 1e-300)


def test_crnn_chunked_reference_matches_whole_problem_autograd():
    """Autograd through CR.step over the four tensors at once (per-tensor states, the form the other tests use) against
    the chunked single-tensor reference with chunks of 100 coordinates: d theta, every plane's adjoint and d g."""
    theta = crnn_generic_theta(5)
    sizes = [math.prod(s) for s in SHAPES]
    n = sum(sizes)
    planes = crnn_generic_planes(theta, n, seed=1)
    gen = torch.Generator().manual_seed(2)
    g = torch.randn(n, generator=gen) * 0.3
    d_new, d_upd = torch.randn(103, n, generator=gen), torch.randn(n, generator=gen)
    th, pl, gg = _leaf(theta, torch.float64), _leaf(planes, torch.float64), _leaf(g, torch.float64)
    G = list(torch.split(gg, sizes))
    _, new, upd = CR.step(th, [torch.zeros_like(x) for x in G], G, CR.planes_to_states(pl, sizes))
    L = (d_new.double() * CR.state_to_planes(new)).sum() + (d_upd.double() * torch.cat(upd)).sum()
    w_th, w_pl, w_g = torch.autograd.grad(L, (th, pl, gg))
    c_th, c_pl, c_g = chunked_vjp(crnn_vjp, theta, planes, g, d_new, d_upd, torch.float64, chunk=100)
    off = 0
    for name, shape in CR.theta_spec():
        k = math.prod(shape)
        assert _close(c_th[off:off + k], w_th[off:off + k]), name
        if name != "init_vector":   # (the planes are given: the init vector reaches no output)
            assert float(w_th[off:off + k].abs().max()) > 0, name
        off += k
    for p in range(103):
        assert _close(c_pl[p], w_pl[p]) and float(w_pl[p].abs().max()) > 0, p
    assert _close(c_g, w_g)


def test_tadam_chunked_reference_matches_whole_problem_autograd():
    """The same for TrainableAdam from a state with v != 0: d theta (each of the 4 entries), the m and v adjoints, d g,
    and the t plane's adjoint exactly 0."""
    n = sum(math.prod(s) for s in SHAPES)
    theta = tadam_theta(dtype=torch.float32, **TADAM_THETA)
    planes, g = tadam_generic_planes(n, seed=3)
    gen = torch.Generator().manual_seed(4)
    d_new, d_upd = torch.randn(3, n, generator=gen), torch.randn(n, generator=gen)
    sizes = [math.prod(s) for s in SHAPES]
    th, pl, gg = _leaf(theta, torch.float64), _leaf(planes, torch.float64), _leaf(g, torch.float64)
    sts = B.planes_to_states(pl, sizes)
    for st in sts:
        st["t"] = st["t"].detach()
    G = list(torch.split(gg, sizes))
    _, new, upd = B.tadam_step(th, [torch.zeros_like(x) for x in G], G, sts)
    L = (d_new.double() * B.state_to_planes(new)).sum() + (d_upd.double() * torch.cat(upd)).sum()
    w_th, w_pl, w_g = torch.autograd.grad(L, (th, pl, gg))
    c_th, c_pl, c_g = chunked_vjp(tadam_vjp, theta, planes, g, d_new, d_upd, torch.float64, chunk=100)
    for j in range(4):
        assert float(w_th[j]) != 0.0 and _close(c_th[j:j + 1], w_th[j:j + 1]), j
    for p in (0, 2):
        assert _close(c_pl[p], w_pl[p]), p
    assert float(c_pl[1].abs().max()) == 0.0 and float(w_pl[1].abs().max()) == 0.0
    assert _close(c_g, w_g) and bool(torch.isfinite(c_g).all())


@pytest.mark.parametrize("n_steps,itr", [(3, 5), (1, 0)])
def test_lrs_chunked_reference_is_the_closed_form(n_steps, itr):
    """LearningRateSchedule with a clamped index (itr 5, 3 entries: rates[2]) and GlobalLearningRate: d rates is
    sum(d_upd g) at the used entry and 0 elsewhere, d g = rate d_upd."""
    gen = torch.Generator().manual_seed(5)
    n = 665
    rates = torch.rand(n_steps, generator=gen) + 0.1
    g, d_upd = torch.randn(n, generator=gen), torch.randn(n, generator=gen)
    d_r, _, d_g = chunked_vjp(partial(lrs_vjp, itr=itr), rates, None, g, None, d_upd, torch.float64, chunk=100)
    idx = min(itr, n_steps - 1)
    want = torch.zeros(n_steps, dtype=torch.float64)
    want[idx] = (d_upd.double() * g.double()).sum()
    assert _close(d_r, want) and torch.equal(d_g, rates[idx].double() * d_upd.double())
