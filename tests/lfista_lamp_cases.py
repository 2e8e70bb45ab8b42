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


# ------------------------------------------------------------------------------------------------ C-ABI problems
# The C-ABI tests call l2o_ista_fwd / l2o_ista_bwd on problem dictionaries laid out as the ABI takes them:
#   LFISTA  We [N, M] (the B1 slot), W = Wg_1 .. Wg_{K-1} [K-1, N, N], W2 = Wm_1 .. Wm_{K-1} [K-1, N, N] (Wm_1 is
#           never read), theta [K]; the second state is x_{k-1} [B, N]
#   LAMP    A [M, N], W [K or 1, M, N], theta = lam [K], step [K] with a shared W (else None); the second state is
#           v_{k-1} [B, M]
# plus y, x_in, s2_in, d_xk, d_s2 (the gradient of the pass's last second state: x_{k1-1} or v_{k1-1}) and gscale.
K2 = 6   # layers of the C-ABI tests' problems


def n_slots2(form, share_W):
    if form == lista.LFISTA:
        return K2 - 1
    return 1 if share_W else K2


def slot_birth2(form, g, share_W):
    """The layer that creates W (or Wm) slot g: its gradient multiplier's index."""
    if form == lista.LFISTA:
        return g + 1
    return 0 if share_W else g


def _s2_width(P):
    return P["N"] if P["form"] == lista.LFISTA else P["M"]


def exact_problem2(form, M, N, B, seed, share_W=False, gscale=(1.0, 0.5, 2.0, 0.25, 4.0, 1.0)):
    """Inputs whose every fp32 product and partial sum is exact (exact_bound2 checks it): sparse {-1, 0, 1} weights
    with a nonzero in every row and column, small integer y, x_in, s2_in, d_xk and d_s2 (zeros stored as -0.0), a
    power-of-two gscale.  LFISTA: integer theta_k, among them 0 and a negative value (shrinkage then grows |z|).
    LAMP: M a power of two, so b_k = ||x_k||_0 / M is dyadic, and every lam_k <= 0, so the threshold
    max(sqrt(rvar) lam_k, 0) is exactly 0; only sqrt(rvar) and dlam_k at the lam_k = 0 layers are then inexact (dlam_k
    at lam_k < 0 is exactly 0).  Steps in {1, -1, 2} with a shared W."""
    g = torch.Generator().manual_seed(seed)

    def sparse(*shape):
        rows, cols = shape[-2], shape[-1]
        pick = torch.zeros(shape, dtype=torch.bool)
        pick[..., torch.arange(rows), torch.randint(0, cols, (rows,), generator=g)] = True
        pick[..., torch.randint(0, rows, (cols,), generator=g), torch.arange(cols)] = True
        sign = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
        return torch.where(pick, sign, torch.tensor(-0.0))

    def ints(lo_, hi, *shape):
        v = torch.randint(lo_, hi + 1, shape, generator=g).float()
        return torch.where(v == 0, torch.tensor(-0.0), v)

    P = dict(form=form, M=M, N=N, B=B, share_W=share_W)
    S = n_slots2(form, share_W)
    if form == lista.LFISTA:
        assert not share_W
        P.update(A=None, We=sparse(N, M), W=sparse(S, N, N), W2=sparse(S, N, N), step=None,
                 theta=torch.tensor([1.0, 0.0, 2.0, -1.0, 0.0, 1.0]))
    else:
        assert M & (M - 1) == 0, "b_k = ||x_k||_0 / M is dyadic only for M a power of two"
        P.update(A=sparse(M, N), We=None, W=sparse(S, M, N), W2=None,
                 theta=torch.tensor([0.0, -1.0, 0.0, -0.5, 0.0, -2.0]),
                 step=torch.tensor([1.0, -1.0, 2.0, 1.0, 2.0, -1.0]) if share_W else None)
    S2 = _s2_width(P)
    P["y"] = ints(-3, 3, B, M)
    P["x_in"] = ints(-2, 2, B, N)
    P["s2_in"] = ints(-2, 2, B, S2)
    P["d_xk"] = ints(-1, 1, B, N)
    P["d_s2"] = ints(-1, 1, B, S2)
    P["gscale"] = torch.tensor(gscale, dtype=torch.float32)
    return P


def generic_problem2(form, M, N, B, share_W, seed=0):
    """generic_model's weights at K = 6, make_data rows, a gscale with a zero, no x_in / s2_in / d_s2 (a model's
    pass), and the sparse-coding loss gradient as d_xk: random d_xk would let dtheta_k, dlam_k and ds_k cancel far
    below fp32 reach."""
    name = "lfista" if form == lista.LFISTA else "lamp"
    m = generic_model(name, M, N, share_W, seed=seed, T=K2, device="cpu")
    V = {n: v.detach().clone() for n, v in m.variables.items()}
    P = dict(form=form, M=M, N=N, B=B, share_W=share_W)
    if form == lista.LFISTA:
        We, Wg, Wm, theta = lfista_params(m, V)
        P.update(A=None, We=We, W=Wg, W2=Wm, theta=theta, step=None)
    else:
        W, lam, step = lamp_params(m, V)
        P.update(A=m.A.detach().cpu().float(), We=None, W=W, W2=None, theta=lam, step=step)
    d = lista.make_data(M, N, B, p=min(1.0, max(0.1, 3.0 / N)), seed=seed + 7)["train"]
    P.update(y=torch.as_tensor(d[:, :M]).clone(), x_in=None, s2_in=None, d_s2=None, d_xk=None,
             gscale=torch.tensor([1.0, 0.3, 0.0, 0.09, 0.5, 2.0]))
    if form == lista.LAMP:
        # At M << N, r_0 = s_0 y W_0 sits far below sqrt(rvar_0) lam_0, and every x_k and gradient would be 0: scale
        # the lam_k down until layer 0 passes the largest entries of the rows
        y = P["y"].double()
        r0 = (y @ P["W"][0].double()).abs().amax(dim=1) * (1.0 if P["step"] is None else abs(float(P["step"][0])))
        reach = float((r0 / (y ** 2).mean(dim=1).sqrt().clamp_min(1e-30)).max())
        P["theta"] = P["theta"] * min(1.0, 0.5 * reach / float(P["theta"].max()))
    x_K = oracle2(P, d_xk=None)["xs"][-1]
    P["d_xk"] = (x_K - torch.as_tensor(d[:, M:]).double()).float()
    return P


def sub_rows2(P, rows):
    """The same problem on a gather of its rows."""
    Q = dict(P)
    Q["B"] = len(rows)
    for key in ("y", "x_in", "s2_in", "d_xk", "d_s2"):
        if P[key] is not None:
            Q[key] = P[key][rows].clone()
    return Q


def _arg(P, v, key):
    return P[key] if isinstance(v, str) else v


def _run2(P, k0, k1, x_in, s2_in, d_xk, d_s2, lives):
    """The fp64 pass [k0, k1) with autograd leaves, and its backward from sum(d_xk x_k1) + sum(d_s2 s2_k1)."""
    form, B, N = P["form"], P["B"], P["N"]
    leaf = lambda t: None if t is None else t.double().clone().requires_grad_(True)
    x_in, s2_in = _arg(P, x_in, "x_in"), _arg(P, s2_in, "s2_in")
    d_xk, d_s2 = _arg(P, d_xk, "d_xk"), _arg(P, d_s2, "d_s2")
    R = dict(theta=leaf(P["theta"]), W=leaf(P["W"]), y=P["y"].double(),
             x0=leaf(x_in if x_in is not None else torch.zeros(B, N)),
             s0=leaf(s2_in if s2_in is not None else torch.zeros(B, _s2_width(P))))
    if form == lista.LFISTA:
        R.update(We=leaf(P["We"]), W2=leaf(P["W2"]), zs=[], rec=None)
        R["xs"] = lfista_forward(R["We"], R["W"], R["W2"], R["theta"], R["y"], k1, k0=k0, x0=R["x0"], xm0=R["s0"],
                                 lives=lives, zs_out=R["zs"])
        s2_out = R["xs"][-2] if len(R["xs"]) >= 2 else R["x0"]
    else:
        R.update(step=leaf(P["step"]), A=P["A"].double(), rec=[])
        R["xs"], vs = lamp_forward(R["A"], R["W"], R["theta"], R["step"], R["y"], k1, P["share_W"], k0=k0,
                                   x0=R["x0"], v0=R["s0"], lives=lives, rec=R["rec"])
        R["zs"] = [r for r, _, _, _ in R["rec"]]
        s2_out = vs[-1]
    if d_xk is not None:
        for t in R["xs"] + [v for _, _, _, v in R["rec"] or []]:
            t.retain_grad()
        loss = (d_xk.double() * R["xs"][-1]).sum()
        if d_s2 is not None:
            loss = loss + (d_s2.double() * s2_out).sum()
        loss.backward()
    return R


def _grad(t):
    return None if t is None else (torch.zeros_like(t) if t.grad is None else t.grad.detach())


def _lives2(P, R, k0):
    """Each layer's classification as the oracle made it: LFISTA |z| > theta_k, z != 0; LAMP r != 0 and
    |r| >= max(sqrt(rvar) lam_k, 0)."""
    out = []
    for l, z in enumerate(R["zs"]):
        z, k = z.detach(), k0 + l
        if P["form"] == lista.LFISTA:
            out.append((z.abs() > R["theta"][k].detach()) & (z != 0))
        else:
            th = torch.clamp_min(R["rec"][l][1].detach() * R["theta"][k].detach(), 0.0)
            out.append((z != 0) & (z.abs() >= th))
    return out


def oracle2(P, k0=0, k1=K2, x_in="P", s2_in="P", d_xk="P", d_s2="P", lives=None):
    """fp64 pass [k0, k1) from x_in (x_{k0}) and s2_in (LFISTA x_{k0-1}, LAMP v_{k0-1}), with the records the kernel
    writes (xs, zs: LFISTA z_k / LAMP r_k, LAMP rs = v_k and rowrec = (sqrt(rvar_k), b_k)) and, with d_xk, the
    gradients of sum(d_xk x_k1) + sum(d_s2 s2_k1) laid out as the C ABI returns them, times gscale[birth layer]:
    d_x_in, d_s2_in, dW, dW2 (LFISTA), dB1 (LFISTA's We), dtheta (LAMP: dlam), dstep.  scale_dtheta and scale_dstep
    are the sums of the magnitudes of each per-layer scalar's terms, which can cancel far below them."""
    lives_given = lives
    R = _run2(P, k0, k1, x_in, s2_in, _arg(P, d_xk, "d_xk"), _arg(P, d_s2, "d_s2"), lives)
    form, share_W = P["form"], P["share_W"]
    st = lambda ts: torch.stack([t.detach() for t in ts])
    out = {"xs": st(R["xs"]), "zs": st(R["zs"]), "rs": None, "rowrec": None}
    if form == lista.LAMP:
        out["rs"] = st([v for _, _, _, v in R["rec"]])
        out["rowrec"] = st([torch.cat([sq, b], dim=1) for _, sq, b, _ in R["rec"]])
    if _arg(P, d_xk, "d_xk") is None:
        return out
    gs = torch.ones(K2, dtype=torch.float64) if P["gscale"] is None else P["gscale"].double()

    def slots(t):
        t = _grad(t)
        if t is None:
            return None
        t = t.clone()
        for s in range(t.shape[0]):
            t[s] *= gs[slot_birth2(form, s, share_W)]
        return t

    out.update(d_x_in=_grad(R["x0"]), d_s2_in=_grad(R["s0"]), dW=slots(R["W"]), dtheta=_grad(R["theta"]) * gs,
               dW2=slots(R.get("W2")), dB1=None, dstep=None)
    if form == lista.LFISTA:
        out["dB1"] = _grad(R["We"]) * gs[0]
    elif R["step"] is not None:
        out["dstep"] = _grad(R["step"]) * gs
    lives = _lives2(P, R, k0) if lives_given is None else lives_given
    sth, sds = torch.zeros(K2, dtype=torch.float64), torch.zeros(K2, dtype=torch.float64)
    for l, k in enumerate(range(k0, k1)):
        d = _grad(R["xs"][l]).abs() * lives[l].double()      # |dL/dr_k| (|dL/dz_k|)
        if form == lista.LFISTA:
            sth[k] = d.sum()                                   # dtheta_k = -sum sign(z) dz
        else:
            _, sq, _, v = R["rec"][l]
            sth[k] = (d.sum(dim=1, keepdim=True) * sq.detach()).sum()     # dlam_k = sum_b g_b sqrt(rvar_b)
            if R["step"] is not None:                                      # ds_k = <v_k, dr_k W_k^T>
                Wk = R["W"][0 if share_W else k].detach().abs()
                sds[k] = (v.detach().abs() * (d @ Wk.T)).sum()
    out.update(scale_dtheta=sth * gs.abs(), scale_dstep=sds * gs.abs())
    return out


def _gran(t):
    """The largest power of two, at most 1, that divides every entry of t (t holds dyadic rationals, exact in
    fp64)."""
    t = t.detach().double().reshape(-1)
    t = t[t != 0]
    e = 0
    while t.numel() and not bool((torch.frac(t * 2.0 ** e) == 0).all()):
        e += 1
        assert e <= 60, "not a dyadic rational"
    return 2.0 ** -e


def exact_bound2(P, k0=0, k1=K2):
    """The largest ratio, over every sum a pass [k0, k1) and its backward form in fp32, of the sum of its terms'
    magnitudes to the granularity (the largest power of two dividing every term): LFISTA's z_k and its dx_k / Wm
    carry, LAMP's v_k, r_k, dv_k (with the b_{k+1} dv_{k+1} carry) and dx_k, the dtheta_k / ds_k partials and each
    layer's dW / dWm / dWe / d_s2_in terms.  Below 2^24 every partial sum, in any order, is an exact fp32 value."""
    R = _run2(P, k0, k1, "P", "P", "P", "P", None)
    lives = _lives2(P, R, k0)
    g, ab = _gran, lambda t: t.detach().abs()
    ratios = []

    def term(bound, gran):
        ratios.append(float(bound.max()) / gran if bound.numel() else 0.0)

    y, x0, s0 = R["y"], R["x0"].detach(), R["s0"].detach()
    ins = [x0] + [x.detach() for x in R["xs"]]             # x_k of pass layer l is ins[l]
    dxs = [_grad(x) for x in R["xs"]]
    if P["form"] == lista.LFISTA:
        We, Wg, Wm = (R[k].detach() for k in ("We", "W", "W2"))
        gw = min(g(We), g(Wg), g(Wm))
        xm = [s0] + ins[:-1]                                  # x_{k-1} of pass layer l
        term(ab(y) @ ab(We).T, g(y) * gw)
        for l, k in enumerate(range(k0, k1)):
            b = ab(y) @ ab(We).T
            if k >= 1:
                b = b + ab(ins[l]) @ ab(Wg[k - 1]).T
            if k >= 2:
                b = b + ab(xm[l]) @ ab(Wm[k - 1]).T
            term(b, min(g(y), g(ins[l]), g(xm[l])) * gw)
        carry = _arg(P, "P", "d_s2").double()
        for l in range(k1 - k0 - 1, -1, -1):
            k, dz = k0 + l, dxs[l] * lives[l]
            term(ab(dz).sum().reshape(1), g(dz))                                # dtheta_k
            term(ab(dz).T @ ab(y), g(dz) * g(y))                                # this layer's dWe part
            dx = ab(carry)
            if k >= 1:
                dx = dx + ab(dz) @ ab(Wg[k - 1])
                term(ab(dz).T @ ab(ins[l]), g(dz) * g(ins[l]))                  # dWg_k
            term(dx, min(g(dz) * gw, g(carry)))
            carry = dz @ Wm[k - 1] if k >= 2 else torch.zeros_like(dz)
            if k >= 2:
                term(ab(dz) @ ab(Wm[k - 1]), g(dz) * gw)
                term(ab(dz).T @ ab(xm[l]), g(dz) * g(xm[l]))                    # dWm_k
        return max(ratios)
    A, W = R["A"], R["W"].detach()
    gw = min(g(A), g(W))
    step = lambda k: 1.0 if R["step"] is None else float(R["step"][k].detach())
    vs = [s0] + [v.detach() for _, _, _, v in R["rec"]]    # v_{k-1} of pass layer l is vs[l]
    bs = [b.detach() for _, _, b, _ in R["rec"]]
    for l, k in enumerate(range(k0, k1)):
        Wk = W[0 if P["share_W"] else k]
        term(ab(bs[l] * vs[l]), g(bs[l]) * g(vs[l]))
        term(ab(y) + ab(ins[l]) @ ab(A).T + ab(bs[l] * vs[l]),
             min(g(y), g(ins[l]) * gw, g(bs[l]) * g(vs[l])))                    # v_k
        term(ab(ins[l]) + abs(step(k)) * (ab(vs[l + 1]) @ ab(Wk)),
             min(g(ins[l]), g(torch.tensor([step(k)])) * g(vs[l + 1]) * gw))      # r_k
    for l in range(k1 - k0 - 1, -1, -1):
        k, Wk = k0 + l, W[0 if P["share_W"] else k]
        gs_ = g(torch.tensor([step(k)]))
        dr, v, dv = dxs[l] * lives[l], vs[l + 1], _grad(R["rec"][l][3])
        u = dr @ Wk.T
        carry = dv - step(k) * u                                                # d_s2 or b_{k+1} dv_{k+1}
        term(ab(dr) @ ab(Wk).T, g(dr) * gw)
        term((ab(v) * ab(u)).sum().reshape(1), g(v) * g(u))                     # ds_k
        term(abs(step(k)) * ab(u) + ab(carry), min(gs_ * g(u), g(carry)))       # dv_k
        term(ab(dr) + ab(dv) @ ab(A), min(g(dr), g(dv) * gw))                   # dx_k
        term(abs(step(k)) * ab(v).T @ ab(dr), gs_ * g(v) * g(dr))               # dW_k
        term(ab(bs[l] * dv), g(bs[l]) * g(dv))                                  # the carry to layer k - 1
    return max(ratios)


# ------------------------------------------------------------------------------------------------ C-ABI cases
# (form, (M, N, B), share_W, seed) of the exact problems: M or N below 8 (CTAs with empty column slices), partial
# clusters of rows; LAMP's M = 4 keeps b_k's dyadic granularity within fp32 reach over K = 6 layers
EXACT2_CASES = [(lista.LFISTA, (12, 5, 9), False, 0), (lista.LFISTA, (6, 20, 13), False, 1),
                (lista.LAMP, (4, 12, 9), False, 0), (lista.LAMP, (4, 12, 9), True, 0),
                (lista.LAMP, (4, 3, 13), False, 2), (lista.LAMP, (4, 3, 13), True, 2)]
RANGES2 = [(k0, k1) for k0 in range(K2) for k1 in range(k0 + 1, K2 + 1)]
SPLITS2 = [(1, 3), (2, 4), (2, 5)]     # [0, a), [a, b), [b, K)


def exact_case2(case):
    form, (M, N, B), share_W, seed = case
    return exact_problem2(form, M, N, B, seed, share_W=share_W)


def s2_after(P, rec, x_in):
    """The second state a pass leaves for the next one: LFISTA x_{k1-1} (the pass's x_in after one layer), LAMP
    v_{k1-1}.  rec: the pass's records ([L, B, *])."""
    if P["form"] == lista.LAMP:
        return rec["rs"][-1]
    return rec["xs"][-2] if rec["xs"].shape[0] >= 2 else x_in
