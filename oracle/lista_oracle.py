"""Torch-CPU restatement of model-based L2O's LISTA family (MB/ = Model_Base_L2O/ of the reference), in any dtype.

Checker only: the product path never imports this.  Cell forms (row-major, y [B,M], x [B,N], A [M,N], x_0 = 0):
  LISTA   (MB/models/lista.py:32-45)                 z_k = y B1^T + s_k x_k W_k^T   (layer 0: no W term)
  coupled (MB/models/lista_cp.py, lista_cpss.py, alista.py)  z_k = x_k + s_k (y - x_k A^T) W_k
shrinkage (MB/models/utils.py): shrink_free and shrink_ss; losses and metrics (MB/utils.py); Keras Adam.
Backward passes come from autograd.  W is a tensor of slots: LISTA [S,N,N] (slot k-1 for layer k), coupled [S,M,N]
(slot k), one slot when W is shared; step is None (every s_k = 1) or [K].
"""
from __future__ import annotations

import numpy as np
import torch

LISTA, COUPLED = 0, 1


def ss_rank(n: int, q: float) -> int:
    """tfp.stats.percentile(|z|, 100 - q, interpolation='nearest') as an index into |z| sorted descending: round half
    to even of (n - 1) q / 100, in float64."""
    return int(min(max(np.round((n - 1) * np.float64(q) / 100.0), 0), n - 1))


def shrink_free(z, theta, live=None):
    """sign(z) relu(|z| - theta).  `live` replaces the classification |z| > theta (a constant mask), so a backward can
    follow another computation's rounding at the kink."""
    if live is None:
        return torch.sign(z) * torch.relu(z.abs() - theta)
    return live.to(z.dtype) * (z - torch.sign(z) * theta)


def ss_select(z, theta, rank: int):
    """Support-selection mask: |z| > theta and |z| > the row's |z| at descending rank `rank` (strict)."""
    a = z.abs()
    thres = torch.sort(a, dim=1, descending=True).values[:, rank:rank + 1]
    return (a > theta) & (a > thres)


def shrink_ss(z, theta, rank: int, sel=None, live=None):
    """shrink_ss; `sel` replaces the computed mask (the mask is a stop_gradient constant either way), `live` as in
    shrink_free."""
    if sel is None:
        sel = ss_select(z.detach(), theta.detach(), rank)
    idx = sel.to(z.dtype)
    return idx * z + shrink_free((1.0 - idx) * z, theta, None if live is None else live & ~sel), sel


def w_slot(form, W, k, share_W):
    if share_W:
        return W[0]
    return W[k] if form == COUPLED else W[k - 1]


def forward(form, A, B1, W, theta, step, y, k1, share_W=False, ranks=None, sels=None, lives=None, zs_out=None, k0=0,
            x0=None):
    """x_{k0+1} .. x_k1 of layers k0 .. k1-1 from x_{k0} = x0 (zeros when None), and the support masks used (None per
    layer without support selection).  theta, step, ranks and the W slots are indexed by absolute layer; ranks[k] < 0
    means soft shrinkage in layer k and ranks[k] >= N reads as N - 1.  sels / lives: masks to use in place of the
    computed support selection / |z| > theta classification, one per layer of the pass.  zs_out: a list that
    receives every z_k."""
    B, N = y.shape[0], A.shape[1]
    x = torch.zeros(B, N, dtype=y.dtype, device=y.device) if x0 is None else x0
    by = y @ B1.T if form == LISTA else None
    xs, used = [], []
    for k in range(k0, k1):
        s = 1.0 if step is None else step[k]
        if form == LISTA:
            z = by if k == 0 else by + s * (x @ w_slot(form, W, k, share_W).T)
        else:
            z = x + s * ((y - x @ A.T) @ w_slot(form, W, k, share_W))
        if zs_out is not None:
            zs_out.append(z)
        live = None if lives is None else lives[k - k0]
        rank = -1 if ranks is None else min(int(ranks[k]), N - 1)
        if rank < 0:
            x, m = shrink_free(z, theta[k], live), None
        else:
            x, m = shrink_ss(z, theta[k], rank, None if sels is None else sels[k - k0], live)
        xs.append(x)
        used.append(m)
    return xs, used


def abs_sum_bound(form, A, B1, W, step, y, k1, share_W=False, k0=0, x0=None, d_xk=None):
    """The largest sum of absolute terms over every GEMM, product and reduction that a pass [k0, k1) forms: forward
    r_k, y B1^T, the W products and z_k; with d_xk, the backward's dx_k, ds_k and dtheta_k partials and the per-layer
    dW / dB1 sums over the batch.  It bounds every partial sum in any order, since shrinkage never grows |z| and dz_k
    is dx_{k+1} or 0.  Below 2^24, integer inputs keep all of them exact in fp32."""
    ab = lambda t: None if t is None else t.abs()
    A, B1, W, y = ab(A), ab(B1), ab(W), ab(y)
    N = A.shape[1] if A is not None else B1.shape[0]
    s = lambda k: 1.0 if step is None else abs(float(step[k]))
    X = [torch.zeros(y.shape[0], N, dtype=y.dtype) if x0 is None else x0.abs()]
    R, terms = [], []
    by = y @ B1.T if form == LISTA else None
    for k in range(k0, k1):
        Wk = w_slot(form, W, k, share_W)
        if form == LISTA:
            u = (X[-1] @ Wk.T) if k > 0 else torch.zeros_like(by)
            z = by + s(k) * u
            terms += [by, u]
        else:
            r = y + X[-1] @ A.T
            u = r @ Wk
            z = X[-1] + s(k) * u
            R.append(r)
            terms += [r, u]
        terms.append(z)
        X.append(z)
    if d_xk is not None:
        D = d_xk.abs()
        for k in range(k1 - 1, k0 - 1, -1):
            l, Wk = k - k0, w_slot(form, W, k, share_W)
            terms.append(D.sum().reshape(1))                                   # dtheta_k
            if form == COUPLED:
                u = D @ Wk.T
                v = s(k) * u @ A
                terms += [u, v, (R[l] * u).sum().reshape(1), s(k) * R[l].T @ D]   # ds_k, dW_k
                D = D + v
            else:
                terms.append(D.T @ y)                                          # this layer's dB1 term
                if k == 0:
                    D = torch.zeros_like(D)
                    continue
                u = D @ Wk
                terms += [u, (X[l] * u).sum().reshape(1), s(k) * D.T @ X[l]]      # ds_k, dW_k
                D = s(k) * u
            terms.append(D)
    return max(float(t.max()) for t in terms)


def sc_loss(x, x_true):
    """utils.MSE: tf.nn.l2_loss(x - x_true) over the whole batch (MB/utils.py:13-20)."""
    return 0.5 * ((x - x_true) ** 2).sum()


def lasso_loss(x, A, y, lam):
    """utils.LassoLoss: 0.5 l2_loss(x A^T - y) + lam ||x||_1 (MB/utils.py:33-38)."""
    return 0.5 * (0.5 * ((x @ A.T - y) ** 2).sum()) + lam * x.abs().sum()


def nmse_db(x, x_true):
    """utils.NMSE / EvalNMSE: mean over rows of 10 log10((mse + 1e-10) / (mean x_true^2 + 1e-10))."""
    mse = ((x_true - x) ** 2).mean(dim=1) + 1e-10
    den = (x_true ** 2).mean(dim=1) + 1e-10
    return (10.0 * torch.log10(mse / den)).mean()


def lasso_objective(x, A, y, lam):
    """utils.LassoObjective: mean over rows of 0.5 ||x A^T - y||^2 + lam ||x||_1 (MB/utils.py:52-64)."""
    return (0.5 * ((x @ A.T - y) ** 2).sum(dim=1) + lam * x.abs().sum(dim=1)).mean()


def keras_adam_step(p, g, m, v, t: int, lr: float, b1=0.9, b2=0.999, eps=1e-7):
    """Keras Adam (ResourceApplyAdam, the TF-1 formula): in place on p, m, v; t is the 1-based step."""
    lr_t = lr * np.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)
    m.mul_(b1).add_((1.0 - b1) * g)
    v.mul_(b2).add_((1.0 - b2) * g * g)
    p.sub_(lr_t * m / (v.sqrt() + eps))
