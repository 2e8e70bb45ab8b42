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


def forward(form, A, B1, W, theta, step, y, k1, share_W=False, ranks=None, sels=None, lives=None, zs_out=None):
    """x_1 .. x_k1 and the support masks used (None per layer without support selection).  sels / lives: per-layer
    masks to use in place of the computed support selection / |z| > theta classification.  zs_out: a list that
    receives every z_k."""
    B, N = y.shape[0], A.shape[1]
    x = torch.zeros(B, N, dtype=y.dtype, device=y.device)
    by = y @ B1.T if form == LISTA else None
    xs, used = [], []
    for k in range(k1):
        s = 1.0 if step is None else step[k]
        if form == LISTA:
            z = by if k == 0 else by + s * (x @ w_slot(form, W, k, share_W).T)
        else:
            z = x + s * ((y - x @ A.T) @ w_slot(form, W, k, share_W))
        if zs_out is not None:
            zs_out.append(z)
        live = None if lives is None else lives[k]
        if ranks is None:
            x, m = shrink_free(z, theta[k], live), None
        else:
            x, m = shrink_ss(z, theta[k], int(ranks[k]), None if sels is None else sels[k], live)
        xs.append(x)
        used.append(m)
    return xs, used


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
