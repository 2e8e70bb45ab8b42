"""fp64 CPU restatement of L2O-Minimax's Twin-L2O training and evaluation loop (MM = Model_Free_L2O/L2O-Minimax/
Twin-L2O.py: do_fit :91, fit_optimizer :470, ToyLoss :612, Optimizer :676).

The nets are torch.nn.LSTMCell / nn.Linear themselves, so the gate order (i, f, g, o) and the two biases are the
reference's by construction, and the meta-gradient is autograd through the per-problem loop with the reference's
detach pattern:
- the optimizer inputs are gradients at detached (u, v);
- the active net's h and c are multiplied by `rescale` before its cells;
- x += sign(delta) sche_lr[t-1] while t < 0.2 optim_it (no gradient through sign), then x += delta out_mul;
- reward_t = (l_t + l_{t-1}) / B, l_{t-1} keeping its graph; the updated variable is detached after each reward;
- every 2 unroll_unit iterations the rewards so far are back-propagated and both Adams step, before that iteration's
  own reward; then the variables and states are detached and l_{t-1} is zeroed.
The one deviation, shared with the kernels: each of the R = B dim coordinates carries its own LSTM state (the
reference allocates [B, H] states and slices them to B rows, which only runs at dim = 1).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn as nn


class Net(nn.Module):
    def __init__(self, hidden: int):
        super().__init__()
        self.hidden_sz = hidden
        self.recurs = nn.LSTMCell(2, hidden)
        self.recurs2 = nn.LSTMCell(hidden, hidden)
        self.output = nn.Linear(hidden, 1)

    def forward(self, inp, second, hidden, cell):
        h0, c0 = self.recurs(torch.cat((inp, second), 1), (hidden[0], cell[0]))
        h1, c1 = self.recurs2(h0, (hidden[1], cell[1]))
        return self.output(h1), (h0, h1), (c0, c1)


def sche_lr(optim_it: int) -> list:
    return list(np.arange(1e-4, 1e-1, (1e-1 - 1e-4) / int(0.2 * optim_it)))


def is_warm(iteration: int, optim_it: int) -> bool:
    return iteration < 0.2 * optim_it


def loss_value(kind, d, u, v):
    if kind == 1:
        return d[0] * u * u - d[1] * v * v
    if kind == 2:
        return d[0] * u * u - d[1] * v * v + 2 * v * u
    if kind == 3:
        return (-1) * d[1] * v * torch.sin(math.pi * u * d[0])
    return torch.dot(u, torch.matmul(d, v))


def grad_u(kind, d, u, v):
    if kind == 1:
        return 2 * u * d[0]
    if kind == 2:
        return 2 * u * d[0] + 2 * v
    if kind == 3:
        return (-1) * d[1] * v * torch.cos(d[0] * math.pi * u) * d[0] * math.pi
    return torch.matmul(d, v)


def grad_v(kind, d, u, v):
    if kind == 1:
        return (-2) * d[1] * v
    if kind == 2:
        return (-2) * d[1] * v + 2 * u
    if kind == 3:
        return (-1) * d[1] * torch.sin(d[0] * math.pi * u)
    return torch.matmul(d.t(), u)


def do_fit(nets, kind, data, u0, v0, state0, unroll_unit, optim_it, rescale, out_mul=1.0, train=True,
           meta_opts=None, select=None, dtype=torch.float64):
    """One do_fit.  nets = (net_min, net_max); data[p] is (a, b) or A; u0, v0 [B][dim]; state0[n] = (h [2][R][H],
    c [2][R][H]).  meta_opts: the two torch.optim.Adam (or None: record gradients only).  select(t, traj_u) -> the
    problems whose rewards enter the loss (curriculum), or None for all.  dtype: the precision of the variables, states
    and problem data (the nets must already be in it); float32 gives the rounding error an fp32 implementation of the
    same loop is entitled to.
    Returns per-iteration records (u, v, the [h1, c1, h2, c2] of both nets after the iteration, l_t) and per-segment gradients
    (a list over boundaries of [grads of net_min params, grads of net_max params], None where no path reached them)."""
    B, dim = len(u0), u0[0].numel()
    lr = sche_lr(optim_it)
    data = [d.to(dtype) for d in data]
    u = [x.clone().to(dtype).requires_grad_(True) for x in u0]
    v = [x.clone().to(dtype).requires_grad_(True) for x in v0]
    hs = {n: [h.clone().to(dtype) for h in state0[n][0]] for n in (0, 1)}
    cs = {n: [c.clone().to(dtype) for c in state0[n][1]] for n in (0, 1)}
    reward = {0: [None] * B, 1: [None] * B}
    loss_prev = [0.0] * B
    recs, seg_grads = [], []
    traj_u = np.zeros((B, optim_it, dim))
    for it in range(1, optim_it + 1):
        n = 0 if it % 2 == 1 else 1
        ud, vd = [x.detach() for x in u], [x.detach() for x in v]
        gu = [grad_u(kind, data[p], ud[p], vd[p]) for p in range(B)]
        gv = [grad_v(kind, data[p], ud[p], vd[p]) for p in range(B)]
        first, second = (gu, gv) if n == 0 else (gv, gu)
        inp = torch.cat(first).view(B * dim, 1)
        sec = torch.cat(second).view(B * dim, 1)
        h_in = [rescale * h for h in hs[n]]
        c_in = [rescale * c for c in cs[n]]
        upd, new_h, new_c = nets[n](inp, sec, h_in, c_in)
        upd = upd.split(dim, dim=0)
        xs = u if n == 0 else v
        new_x = []
        for p in range(B):
            if is_warm(it, optim_it):
                new_x.append(xs[p] + torch.sign(upd[p].view(dim)) * lr[it - 1])
            else:
                new_x.append(xs[p] + upd[p].view(dim) * out_mul)
        if n == 0:
            u = new_x
        else:
            v = new_x
        hs[n], cs[n] = list(new_h), list(new_c)
        if it % (2 * unroll_unit) == 0:
            if train:
                chosen = range(B) if select is None else select(it, traj_u)
                total = None
                for p in chosen:
                    for side in (0, 1):
                        if reward[side][p] is not None:
                            total = reward[side][p] if total is None else total + reward[side][p]
                params = [list(nets[0].parameters()), list(nets[1].parameters())]
                if meta_opts is not None:
                    for o in meta_opts:
                        o.zero_grad()
                grads = [[None] * len(params[0]), [None] * len(params[1])]
                if total is not None and total.requires_grad:
                    flat = params[0] + params[1]
                    gs = torch.autograd.grad(total, flat, allow_unused=True)
                    grads = [list(gs[:len(params[0])]), list(gs[len(params[0]):])]
                    if meta_opts is not None:
                        for pp, g in zip(flat, gs):
                            pp.grad = None if g is None else g.clone()
                        for o in meta_opts:
                            o.step()
                seg_grads.append(grads)
            reward = {0: [None] * B, 1: [None] * B}
            u = [x.detach().requires_grad_(True) for x in u]
            v = [x.detach().requires_grad_(True) for x in v]
            for m in (0, 1):
                hs[m] = [h.detach() for h in hs[m]]
                cs[m] = [c.detach() for c in cs[m]]
            loss_prev = [0.0] * B
        for p in range(B):
            traj_u[p, it - 1] = u[p].detach().numpy()
        ls = []
        for p in range(B):
            f = loss_value(kind, data[p], u[p], v[p])
            lt = f if n == 0 else -f
            r = (lt + loss_prev[p]) / B
            reward[n][p] = r if reward[n][p] is None else reward[n][p] + r
            loss_prev[p] = lt.clone()
            ls.append(float(lt.detach()))
        recs.append(dict(u=torch.stack([x.detach() for x in u]), v=torch.stack([x.detach() for x in v]),
                         state=[torch.stack([hs[m][0], cs[m][0], hs[m][1], cs[m][1]]).detach()
                                for m in (0, 1)], l=ls))
        # the variable just updated is detached; the other one is already a leaf, and requires grad
        if n == 0:
            u, v = [x.detach() for x in u], [x.detach().requires_grad_(True) for x in v]
        else:
            u, v = [x.detach().requires_grad_(True) for x in u], [x.detach() for x in v]
    return recs, seg_grads


def loss3_distance(s: float, a: float) -> float:
    """MM :353-373: the distance of s = sum |u| to the nearest k / a, k = 0, 1, ..., searched until it grows past s."""
    best, k = 100000, 0
    while True:
        dist = abs(s - k / a)
        if dist < best:
            best = dist
        elif dist > s:
            break
        k += 1
    return best


def eval_score(kind, data, recs, burn):
    """fit_optimizer's score (MM :586-597): mean over problems of sum_{t >= burn} dist_u^2 + dist_v^2."""
    B = len(data)
    tot = 0.0
    for p in range(B):
        s = 0.0
        for rec in recs[burn:]:
            su = float(rec["u"][p].abs().sum())
            sv = float(rec["v"][p].abs().sum())
            du = loss3_distance(su, float(data[p][0])) if kind == 3 else su
            s += du * du + sv * sv
        tot += s
    return tot / B
