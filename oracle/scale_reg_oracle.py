"""fp64 CPU restatement of L2O-Scale's four regularisers and of the meta objective's regulariser term, from their
definitions on an explicit Hessian (the product path, ``open_l2o_b200.scale_reg``, never forms H)."""
import torch


def gradient_and_hessian(f, x):
    """g and H of ``f(flat x) -> scalar`` at x, fp64."""
    x = x.detach().double().cpu()
    g = torch.autograd.functional.jacobian(f, x)
    H = torch.autograd.functional.hessian(f, x)
    return g, H


def _unit(v):
    return v / (torch.sqrt(v @ v) + 1e-6)


def jacob(g):
    return (g * g).mean()


def hutchinson(H, probes):
    return torch.stack([p @ H @ p for p in probes.double()]).mean()


def power_iteration(H, v0, itrs):
    v, lam = _unit(v0.double()), None
    for _ in range(itrs):
        v = _unit(v)
        w = H @ v
        lam = w @ v
        v = _unit(w)
    return lam


def lanczos(H, v0, itrs):
    """(alphas, betas) of ``itrs`` Lanczos steps with full re-orthogonalisation from the unit vector v0."""
    v = v0.double()
    vs, al, be = [v], [], []
    w = H @ v
    al.append(w @ v)
    w = w - al[-1] * v
    for _ in range(1, itrs):
        be.append(torch.sqrt(w @ w))
        v = w
        for u in vs:
            v = v - (v @ u) * u
        v = _unit(v)
        vs.append(v)
        w = H @ v
        al.append(w @ v)
        w = w - al[-1] * v - be[-1] * vs[-2]
    return torch.stack(al), torch.stack(be) if be else torch.zeros(0, dtype=torch.float64)


def tridiagonal(al, be):
    return torch.diag(al) + torch.diag(be, 1) + torch.diag(be, -1)


def regularizer(option, f, x, probes=None, v0=None, itrs=10):
    """reg(x) of ``option`` for ``f(flat x)``: probes [k, n] (hessian), the unit start (hessian-esd) or the raw
    N(0, I) start v0 (hessian-ev)."""
    g, H = gradient_and_hessian(f, x)
    if option == "jacob":
        return jacob(g)
    if option == "hessian":
        return hutchinson(H, probes)
    if option == "hessian-ev":
        return power_iteration(H, v0, itrs)
    if option == "hessian-esd":
        return lanczos(H, v0, itrs)[0].sum()
    raise ValueError(option)


def switch(regularize_time, i, num_unrolls, reg_scale):
    """SC/metaopt.py:458-475, restated."""
    if regularize_time == "posterior":
        return i > int(num_unrolls * reg_scale + 1)
    if regularize_time == "prior":
        return i < int(num_unrolls * reg_scale + 1)
    if regularize_time == "none":
        return False
    return True


def loop_term(option, f, xs, alpha, on, **kw):
    """alpha sum_t reg(x_t) over the unroll's points xs when the switch is on, else 0."""
    if not on:
        return torch.zeros((), dtype=torch.float64)
    return alpha * sum(regularizer(option, f, x, **kw) for x in xs)
