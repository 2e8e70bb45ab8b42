"""CPU reference of the l2o_minimax_* contract (include/l2o_b200.h): iterations [t0, t1) of a Twin-L2O unroll from
any (u, v, state), and the meta-gradient l2o_minimax_bwd computes for them.

MO.do_fit restates the reference's whole loop, so its segments start at iteration 1 and end at multiples of
2 unroll_unit.  This runs any range, with the ABI's semantics:
- iteration t odd: net 0 updates u from [df/du, df/dv]; even: net 1 updates v from [df/dv, df/du], both at the
  current (u, v), detached;
- the active net's h and c are multiplied by `rescale` before its cells;
- t < warm_end: x += sign(delta) lr[t-1] (no gradient), else x += delta out_mul;
- l_t = f after a min step, -f after a max step; l_t reaches the nets only through its own update delta_t (the other
  variable, and x before the update, are detached), and through delta_t's h/c chain back to t0, whose entering
  states are constants.
The rows run as one batch (row p dim + i is coordinate i of problem p), so the cells see the same [R][.] operands as
MO.do_fit's.
"""
from __future__ import annotations

import copy

import torch

from oracle import minimax_oracle as MO


def _loss_grads(loss, d, u, v):
    """df/du, df/dv [B][dim] of every problem at (u, v) [B][dim]."""
    if loss == 4:
        return torch.bmm(d, v.unsqueeze(2)).squeeze(2), torch.bmm(d.transpose(1, 2), u.unsqueeze(2)).squeeze(2)
    a, b = d[:, 0:1], d[:, 1:2]
    return MO.grad_u(loss, (a, b), u, v), MO.grad_v(loss, (a, b), u, v)


def _loss_value(loss, d, u, v):
    """f [B] of every problem."""
    if loss == 4:
        return (u * torch.bmm(d, v.unsqueeze(2)).squeeze(2)).sum(1)
    return MO.loss_value(loss, (d[:, 0], d[:, 1]), u[:, 0], v[:, 0])


def segment(nets, loss, data, u, v, state, t0, t1, warm_end, lr, rescale, out_mul=1.0, coef=None, weight=None,
            dtype=torch.float64):
    """Run iterations [t0, t1) in `dtype`.

    nets: the two MO.Net (copied, then cast to dtype); data [B][2] (a, b) or [B][dim][dim] A; u, v [R]; state
    [2][4][R][H] (h1, c1, h2, c2 of net 0, then of net 1); lr[t-1] the sign-step size of iteration t (read for
    t < warm_end only); coef [t1-t0] the weight of each l_t and weight [B] each problem's (None: all 1).

    Returns a dict of per-iteration records, index t - t0:
      u, v [n][R] after the iteration; state [n][2][4][R][H] after it; ckpt [n][R][4H+2] the active net's inputs and
      h1, c1, h2, c2 before it; dl [n][R] d l_t / d x_t of the updated x; l [n][B]; delta [n][R] the net's output;
    and, when coef is given, grads: per net the gradient of sum_t coef[t-t0] weight[p] l_t(p) w.r.t. its parameters in
    parameter order (zeros where no path reaches them)."""
    nets = [copy.deepcopy(n).to(dtype) for n in nets]
    d = torch.as_tensor(data).to(dtype)
    B = d.shape[0]
    R = u.numel()
    dim = R // B
    if loss == 4:
        d = d.reshape(B, dim, dim)
    u = u.detach().to(dtype).reshape(B, dim).clone()
    v = v.detach().to(dtype).reshape(B, dim).clone()
    st = state.detach().to(dtype).clone()
    hs = {n: [st[n, 0], st[n, 2]] for n in (0, 1)}
    cs = {n: [st[n, 1], st[n, 3]] for n in (0, 1)}
    w = None if weight is None else torch.as_tensor(weight).to(dtype).reshape(B)
    rec = {k: [] for k in ("u", "v", "state", "ckpt", "dl", "l", "delta")}
    total = None
    for t in range(t0, t1):
        n = 0 if t % 2 == 1 else 1
        ud, vd = u.detach(), v.detach()
        gu, gv = _loss_grads(loss, d, ud, vd)
        x0, x1 = (gu, gv) if n == 0 else (gv, gu)
        x0, x1 = x0.reshape(R, 1), x1.reshape(R, 1)
        rec["ckpt"].append(torch.cat([x0, x1, hs[n][0], cs[n][0], hs[n][1], cs[n][1]], 1).detach())
        out, new_h, new_c = nets[n](x0, x1, [rescale * h for h in hs[n]], [rescale * c for c in cs[n]])
        delta = out.reshape(B, dim)
        x = ud if n == 0 else vd
        new = x + torch.sign(delta.detach()) * lr[t - 1] if t < warm_end else x + delta * out_mul
        hs[n], cs[n] = list(new_h), list(new_c)
        cu, cv = (new, vd) if n == 0 else (ud, new)
        f = _loss_value(loss, d, cu, cv)
        lt = f if n == 0 else -f
        gu1, gv1 = _loss_grads(loss, d, cu.detach(), cv.detach())
        rec["dl"].append((gu1 if n == 0 else -gv1).reshape(R))
        if coef is not None:
            term = float(coef[t - t0]) * (lt if w is None else w * lt)
            total = term.sum() if total is None else total + term.sum()
        u, v = cu, cv
        rec["u"].append(u.detach().reshape(R))
        rec["v"].append(v.detach().reshape(R))
        rec["l"].append(lt.detach())
        rec["delta"].append(delta.detach().reshape(R))
        rec["state"].append(torch.stack([torch.stack([hs[m][0], cs[m][0], hs[m][1], cs[m][1]]) for m in (0, 1)])
                            .detach())
    out = {k: torch.stack(val) for k, val in rec.items()}
    if coef is not None:
        params = [list(nets[0].parameters()), list(nets[1].parameters())]
        flat = params[0] + params[1]
        if total is not None and total.requires_grad:
            gs = torch.autograd.grad(total, flat, allow_unused=True)
        else:
            gs = [None] * len(flat)
        gs = [torch.zeros_like(p) if g is None else g for p, g in zip(flat, gs)]
        out["grads"] = [list(gs[:len(params[0])]), list(gs[len(params[0]):])]
    return out
