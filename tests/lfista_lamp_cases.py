"""fp64 restatements of the LFISTA and LAMP cells (MB/models/lfista.py, MB/models/lamp.py with shrink_lamp of
MB/models/utils.py), and what the LFISTA / LAMP tests share.  Backward passes come from autograd.

Row-major: y [B, M], x [B, N], A [M, N].  Every layer's classification can be replaced by a given mask (`lives`), so
the oracle follows the kernel's decisions where |z| lands within rounding of the threshold."""
import math

import numpy as np
import torch

from open_l2o_b200 import lista


def lfista_forward(We, Wg, Wm, theta, y, k1, k0=0, x0=None, xm0=None, lives=None, zs_out=None):
    """x_{k0+1} .. x_k1 of z_k = y We^T + [k>=1] x_k Wg_k^T + [k>=2] x_{k-1} Wm_k^T, x_{k+1} = shrink_free(z_k).
    Wg, Wm: slot k-1 for layer k.  x0 = x_{k0}, xm0 = x_{k0-1} (zeros when None)."""
    B, N = y.shape[0], We.shape[0]
    zero = torch.zeros(B, N, dtype=y.dtype, device=y.device)
    x = zero if x0 is None else x0
    xm = zero if xm0 is None else xm0
    by = y @ We.T
    xs = []
    for k in range(k0, k1):
        z = by
        if k >= 1:
            z = z + x @ Wg[k - 1].T
        if k >= 2:
            z = z + xm @ Wm[k - 1].T
        if zs_out is not None:
            zs_out.append(z)
        if lives is None:
            xn = torch.sign(z) * torch.relu(z.abs() - theta[k])
        else:
            xn = lives[k - k0].to(z.dtype) * (z - torch.sign(z) * theta[k])
        xm, x = x, xn
        xs.append(x)
    return xs


def lamp_forward(A, W, lam, step, y, k1, share_W=False, k0=0, x0=None, v0=None, lives=None, rec=None):
    """x_{k0+1} .. x_k1 and v_{k0} .. v_{k1-1} of v_k = y - x_k A^T + b_k v_{k-1} (b_k = ||x_k||_0 / M, a constant;
    b_0 = 0), r_k = x_k + s_k v_k W_k, x_{k+1} = sign(r) max(|r| - theta, 0) with theta = max(sqrt(||v_k||^2 / M)
    lam_k, 0).  W: slots [S, M, N], slot k (one when shared); step None (all 1) or [K].  The gradient of theta follows
    tf.maximum (to sqrt(rvar) lam_k where it is >= 0), and is 0 for a row with rvar = 0.  `lives` replaces
    [r != 0, |r| >= theta].  rec: a list that receives (r_k, sqrt(rvar_k), b_k, v_k) per layer."""
    B, M = y.shape
    N = A.shape[1]
    x = torch.zeros(B, N, dtype=y.dtype, device=y.device) if x0 is None else x0
    v = torch.zeros(B, M, dtype=y.dtype, device=y.device) if v0 is None else v0
    xs, vs = [], []
    for k in range(k0, k1):
        b = torch.zeros(B, 1, dtype=y.dtype, device=y.device)
        if k > 0:
            b = (x.detach() != 0).sum(dim=1, keepdim=True).to(y.dtype) / M
        v = y - x @ A.T + b * v
        rvar = (v ** 2).sum(dim=1, keepdim=True) / M
        pos = rvar > 0
        sq = torch.where(pos, torch.sqrt(torch.where(pos, rvar, torch.ones_like(rvar))), torch.zeros_like(rvar))
        raw = sq * lam[k]
        th = torch.where(raw >= 0, raw, torch.zeros_like(raw))
        s = 1.0 if step is None else step[k]
        r = x + s * (v @ (W[0] if share_W else W[k]))
        live = ((r != 0) & (r.abs() >= th)) if lives is None else lives[k - k0]
        x = live.to(r.dtype) * (r - torch.sign(r) * th)
        if rec is not None:
            rec.append((r, sq, b, v))
        xs.append(x)
        vs.append(v)
    return xs, vs


def model_leaves(m, dtype=torch.float64):
    return {n: v.detach().cpu().to(dtype).clone().requires_grad_(True) for n, v in m.variables.items()}


def lfista_params(m, P):
    nm, T = m.name, m.T
    Wg = torch.stack([P[nm + "_Wg%d" % i] for i in range(2, T + 1)])
    Wm = torch.stack([P[nm + "_Wm%d" % i] for i in range(2, T + 1)])
    theta = torch.cat([P[nm + "_theta%d" % i] for i in range(1, T + 1)])
    return P[nm + "_We1"], Wg, Wm, theta


def lamp_params(m, P):
    nm, T = m.name, m.T
    W = P[nm + "_W"][None] if m.share_W else torch.stack([P[nm + "_W%d" % i] for i in range(1, T + 1)])
    lam = torch.cat([P[nm + "_lam%d" % i] for i in range(1, T + 1)])
    step = torch.cat([P[nm + "_step_size%d" % i] for i in range(1, T + 1)]) if m.share_W else None
    return W, lam, step


def model_forward(m, P, y, k1, lives=None, zs_out=None, rec=None):
    """The model's x_1 .. x_k1 from the oracle, with the variables P (name -> tensor)."""
    if m.form == lista.LFISTA:
        We, Wg, Wm, theta = lfista_params(m, P)
        return lfista_forward(We, Wg, Wm, theta, y, k1, lives=lives, zs_out=zs_out)
    W, lam, step = lamp_params(m, P)
    xs, _ = lamp_forward(m.A.to(y.device, y.dtype), W, lam, step, y, k1, m.share_W, lives=lives, rec=rec)
    return xs


def generic_model(name, M, N, share_W, seed=0, T=16, device="cuda"):
    """A model at generic (perturbed) weights that keep the recurrence bounded."""
    from open_l2o_b200 import lista_train as lt
    d = lista.make_data(M, N, 1, seed=seed)
    m = lt.build_model(name, d["A"], T, 0.4, share_W, 1.2, 13.0, None, device)
    g = torch.Generator(device="cpu").manual_seed(seed + 1)
    for vname, v in m.variables.items():
        noise = torch.rand(v.shape, generator=g) - 0.5
        if "_theta" in vname or "_lam" in vname:
            v.copy_((v.cpu() * (1 + noise)).to(v.device))
        elif "_step_size" in vname:
            v.copy_((1 + 0.4 * noise).to(v.device))
        elif name == "lamp" or vname.endswith("_We1"):
            v.copy_((v.cpu() * (1 + 0.2 * noise)).to(v.device))
        else:
            v.copy_((v.cpu() + 0.02 * noise / np.sqrt(N)).to(v.device))
    return m


def fista_momenta_ref(T):
    """The reference's t_k and m_k, restated: t = [1, 1], t_{i+2} = (1 + sqrt(1 + 4 t_{i+1}^2)) / 2."""
    t = [1.0, 1.0]
    for _ in range(T):
        t.append((1 + math.sqrt(1 + 4 * t[-1] ** 2)) / 2)
    return t, [(t[i + 1] - 1) / t[i + 2] for i in range(T)]
