"""The L2O-DM meta-gradient at benchmark scale, from the fp64 oracle run over coordinate chunks.

Both fused problems (rastrigin_sep, quadratic_diag) are separable and every L2O-DM net (identity, LogAndSign, RNNProp,
whose Adam features are per coordinate) acts coordinate-wise, so the meta-loss sum_t f(x_t) is a sum over coordinates.
Each chunk of coordinates is therefore its own unroll:
  - dtheta is the sum of the chunks' oracle meta-gradients, and fx_t the sum of their fx_t;
  - x_T, the final LSTM state, RNNProp's m and v and the gradient rows g_0..g_T are the chunks' concatenated.
Every chunk keeps the whole problem's fscale (1/n), not 1/chunk.  The sums over chunks are formed in fp64 whatever the
oracle's dtype, so the fp32 run measures the round-off of the unroll and its autograd, not of the chunk sum.

One chunk of CHUNK coordinates at T = 100 keeps its autograd graph under BUDGET_BYTES: tests/test_dm_scale_gpu.py
asserts it with torch.cuda.max_memory_allocated, and measured 4.0 GiB (identity, LogAndSign) to 4.5 GiB (RNNProp) in
fp64 on an H100 80GB HBM3."""
from dataclasses import dataclass
from typing import Optional

import torch

from oracle import l2o_oracle as orc

CHUNK = 16384
BUDGET_BYTES = 8 << 30


@dataclass
class ChunkedResult:
    dtheta: torch.Tensor      # [n_theta] fp64
    fx: torch.Tensor          # [T + 1] fp64
    x: torch.Tensor           # [n] x_T
    state: tuple              # over layers of (h, c) [n, H]
    mv: Optional[tuple]       # RNNProp's (m, v) [n] after the unroll
    g_rec: torch.Tensor       # [T + 1, n] the gradient rows g_0..g_T


def chunked_meta_grad(spec, theta, prob, x0, T, dtype, *, state0=None, mv0=None, step0=1, beta1=0.95, beta2=0.95,
                      chunk=CHUNK, device=None):
    """orc.meta_grad of the fused problem `prob` (an orc.FusedProblem over all n coordinates) run chunk by chunk in
    `dtype` on `device` (default: x0's).  state0 defaults to the zero state, mv0 (RNNProp) to zeros."""
    device = x0.device if device is None else torch.device(device)
    n = x0.numel()
    if state0 is None:
        state0 = orc.initial_state(spec, n, dtype)
    if spec.rnnprop and mv0 is None:
        mv0 = (torch.zeros(n, dtype=dtype), torch.zeros(n, dtype=dtype))
    cast = lambda t: t.to(device=device, dtype=dtype)
    th = cast(theta)
    dtheta = torch.zeros(th.numel(), dtype=torch.float64, device=device)
    fx = torch.zeros(T + 1, dtype=torch.float64, device=device)
    x = torch.empty(n, dtype=dtype, device=device)
    state = tuple((torch.empty(n, h, dtype=dtype, device=device), torch.empty(n, h, dtype=dtype, device=device))
                  for h in spec.layers)
    mv = (torch.empty(n, dtype=dtype, device=device), torch.empty(n, dtype=dtype, device=device)) if spec.rnnprop \
        else None
    g_rec = torch.empty(T + 1, n, dtype=dtype, device=device)
    for lo in range(0, n, chunk):
        hi = min(n, lo + chunk)
        part = orc.FusedProblem(prob.kind, cast(prob.a[lo:hi]), cast(prob.b[lo:hi]), prob.alpha, prob.fscale)
        st = tuple((cast(h[lo:hi]), cast(c[lo:hi])) for h, c in state0)
        kw = dict(mv0=(cast(mv0[0][lo:hi]), cast(mv0[1][lo:hi])), step0=step0, beta1=beta1, beta2=beta2) \
            if spec.rnnprop else {}
        g, res = orc.meta_grad(spec, th, cast(x0[lo:hi]), st, None, T, grad_of=part.f_and_g, **kw)
        dtheta += g.double()
        fx += res.fx.detach().double()
        x[lo:hi] = res.x_final.detach()
        for (h, c), (hr, cr) in zip(state, res.state_final):
            h[lo:hi] = hr.detach()
            c[lo:hi] = cr.detach()
        if spec.rnnprop:
            mv[0][lo:hi] = res.mv_final[0].detach()
            mv[1][lo:hi] = res.mv_final[1].detach()
        g_rec[:T, lo:hi] = torch.stack(res.grads).detach()
        g_rec[T, lo:hi] = part.f_and_g(res.x_final.detach())[1]
        del g, res
    return ChunkedResult(dtheta, fx, x, state, mv, g_rec)
