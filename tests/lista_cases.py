"""Problems, the fp64 reference and the parametrizations shared by the LISTA-family tests: models at generic
(perturbed) weights, the ABI tests' problem dictionaries (integer inputs whose every fp32 sum is exact, and generic
weights), and the oracle of one pass [k0, k1) with its records and gradients laid out as the C ABI returns them."""
import numpy as np
import torch

from open_l2o_b200 import lista, lista_train as lt
from oracle import lista_oracle as lo

K = 4   # layers of the ABI tests' problems


def generic_model(name, M, N, share_W, seed=0, T=16):
    """A model at generic (perturbed) weights that keep the 16-layer recurrence bounded."""
    d = lista.make_data(M, N, 1, seed=seed)
    A = d["A"]
    W = lista.alista_weight(A) if name == "alista" else None
    m = lt.build_model(name, A, T, 0.4, share_W, 1.2, 13.0, W)
    g = torch.Generator(device="cpu").manual_seed(seed + 1)
    L = float(m.scale)
    for vname, v in m.variables.items():
        noise = torch.rand(v.shape, generator=g) - 0.5
        if "_theta" in vname:
            v.copy_((v.cpu() * (1 + noise)).to(v.device))
        elif "_step_size" in vname:
            v.copy_((1 + 0.4 * noise).to(v.device))
        elif vname.endswith("_B"):
            v.copy_((v.cpu() * (1 + 0.1 * noise)).to(v.device))
        elif m.form == lista.COUPLED:                       # W_k = A / L (1 + noise): stable, not the initial A
            v.copy_((v.cpu() / L * (1 + 0.2 * noise)).to(v.device))
        else:
            v.copy_((v.cpu() + 0.02 * noise / np.sqrt(N)).to(v.device))
    if m.W_const is not None:
        m.W_const.mul_(1.0 / L)
    return m


def n_slots(form, K, share_W):
    return 1 if share_W else (K if form == lista.COUPLED else K - 1)


def slot_birth(form, g, share_W):
    """The layer that creates W slot g (its gradient multiplier's index)."""
    first = 0 if form == lista.COUPLED else 1
    return first if share_W else g + first


# ------------------------------------------------------------------------------------------------ problem builders
def exact_problem(form, M, N, B, ranks, theta, share_W, seed, step=True, gscale=None, dW=True, dstep=True):
    """Inputs whose every product and partial sum is an exact fp32 integer (lo.abs_sum_bound checks it): A, B1 and W
    in {-1, 0, 1} with a few nonzeros per row and column, small integer y and x_in (zeros stored as -0.0), s_k in
    {1, -1, 2}, integer theta and d_xk, power-of-two gscale.  |z| then ties heavily, and |z| == theta and z == 0 are
    common."""
    g = torch.Generator().manual_seed(seed)

    def sparse(*shape):
        rows, cols = shape[-2], shape[-1]
        # one nonzero in every row and one in every column, at random places
        pick = torch.zeros(shape, dtype=torch.bool)
        pick[..., torch.arange(rows), torch.randint(0, cols, (rows,), generator=g)] = True
        pick[..., torch.randint(0, rows, (cols,), generator=g), torch.arange(cols)] = True
        sign = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0)
        return (pick * sign).float()

    def ints(lo_, hi, *shape):
        v = torch.randint(lo_, hi + 1, shape, generator=g).float()
        return torch.where(v == 0, torch.tensor(-0.0), v)

    S = n_slots(form, K, share_W)
    P = dict(form=form, M=M, N=N, B=B, share_W=share_W, dW=dW, dstep=dstep)
    P["A"] = sparse(M, N)      # read by the coupled form only
    P["B1"] = sparse(N, M) if form == lista.LISTA else None
    P["W"] = sparse(S, M, N) if form == lista.COUPLED else sparse(S, N, N)
    P["theta"] = torch.tensor(theta, dtype=torch.float32)
    P["step"] = torch.tensor([-1.0, 1.0, 2.0, -1.0]) if step else None
    P["ranks"] = None if ranks is None else torch.tensor(ranks, dtype=torch.int32)
    P["y"] = ints(-3, 3, B, M)
    P["x_in"] = ints(-2, 2, B, N)
    P["d_xk"] = ints(-1, 1, B, N)
    P["gscale"] = None if gscale is None else torch.tensor(gscale, dtype=torch.float32)
    return P


def generic_problem(form, M, N, B, share_W, seed=0, ranks=None):
    """generic_model's weights (K = 4), make_data rows, a gscale with a zero and the SC loss gradient as d_xk."""
    m = generic_model("lista" if form == lista.LISTA else "lista_cp", M, N, share_W, seed=seed, T=K)
    W, _, B1, _, step, _ = m._weights()
    S = n_slots(form, K, share_W)
    wshape = (S, M, N) if form == lista.COUPLED else (S, N, N)
    # p = 0.1 would leave most rows of y zero at the smallest N, and with them every gradient
    d = lista.make_data(M, N, B, p=min(1.0, max(0.1, 3.0 / N)), seed=seed + 7)["train"]
    P = dict(form=form, M=M, N=N, B=B, share_W=share_W, dW=True, dstep=step is not None)
    P["A"] = m.A.cpu()
    P["B1"] = None if B1 is None else B1.detach().cpu().clone()
    P["W"] = W.detach().cpu().reshape(wshape).clone()
    P["theta"] = m._block(m.name + "_theta1", K).detach().cpu().clone()
    P["step"] = None if step is None else step.detach().cpu().clone()
    P["ranks"] = None if ranks is None else torch.tensor(ranks, dtype=torch.int32)
    P["y"] = torch.as_tensor(d[:, :M]).clone()
    P["x_in"] = None
    P["gscale"] = torch.tensor([1.0, 0.3, 0.0, 0.09])
    # dL/dx_K of the sparse-coding loss against the rows' x, as the models pass it: random d_xk would make dtheta_k
    # and ds_k cancel far below fp32 reach (at (3, 2046) ds_k fell to 2.5e-8 of the sum of its terms' magnitudes)
    P["d_xk"] = None
    x_K = oracle(P, d_xk=None)["xs"][-1]
    P["d_xk"] = (x_K - torch.as_tensor(d[:, M:]).double()).float()
    return P


def sub_rows(P, rows):
    """The same problem on a gather of its rows."""
    Q = dict(P)
    Q["B"] = len(rows)
    for key in ("y", "x_in", "d_xk"):
        if P[key] is not None:
            Q[key] = P[key][rows].clone()
    return Q


# ------------------------------------------------------------------------------------------------ oracle
def oracle(P, k0=0, k1=K, x_in="P", d_xk="P", sels=None, lives=None):
    """fp64 forward over [k0, k1) from x_in, records (z_k, r_k, masks) and, with d_xk, the gradients of
    sum(d_xk * x_k1) times gscale[birth layer], as the kernel lays them out."""
    f64 = lambda t: None if t is None else t.double()
    x_in = P["x_in"] if isinstance(x_in, str) else x_in
    d_xk = P["d_xk"] if isinstance(d_xk, str) else d_xk
    form, N, B = P["form"], P["N"], P["B"]
    leaf = lambda t: None if t is None else t.double().clone().requires_grad_(True)
    W, B1, theta = leaf(P["W"]), leaf(P["B1"]), leaf(P["theta"])
    step = leaf(P["step"] if P["step"] is not None else torch.ones(K))
    x0 = leaf(x_in if x_in is not None else torch.zeros(B, N))
    y, A = f64(P["y"]), f64(P["A"])
    ranks = None if P["ranks"] is None else P["ranks"].tolist()
    zs = []
    xs, used = lo.forward(form, A, B1, W, theta, step, y, k1, P["share_W"], ranks, sels, lives, zs, k0=k0, x0=x0)
    ins = [x0] + xs[:-1]
    out = {"xs": torch.stack(xs).detach(), "zs": torch.stack(zs).detach(),
           "rs": torch.stack([y - x @ A.T for x in ins]).detach() if form == lista.COUPLED else None,
           "sel": torch.stack([torch.zeros(B, N, dtype=torch.bool) if m is None else m for m in used]).to(torch.uint8)}
    if d_xk is not None:
        for x in xs:
            x.retain_grad()
        (f64(d_xk) * xs[-1]).sum().backward()
        gs = torch.ones(K, dtype=torch.float64) if P["gscale"] is None else P["gscale"].double()
        grad = lambda t: torch.zeros_like(t) if t.grad is None else t.grad.detach()
        bscale = lambda j: float(gs[j]) if j < K else 1.0
        dW = grad(W).clone()
        for s in range(dW.shape[0]):
            dW[s] *= bscale(slot_birth(form, s, P["share_W"]))
        out.update(d_x_in=grad(x0), dW=dW, dtheta=grad(theta) * gs, dstep=grad(step) * gs,
                   dB1=None if B1 is None else grad(B1) * gs[0])
        # The sum of the magnitudes of each per-layer scalar's terms: dtheta_k adds dz_k over the live entries that
        # support selection did not pass through, ds_k adds dz_k times the W term of z_k.
        sth, sds = torch.zeros(K, dtype=torch.float64), torch.zeros(K, dtype=torch.float64)
        for l, k in enumerate(range(k0, k1)):
            z, x, Wk = zs[l].detach(), ins[l].detach(), lo.w_slot(form, W.detach(), k, P["share_W"])
            picked = torch.zeros_like(z, dtype=torch.bool) if used[l] is None else used[l]
            live = ((z.abs() > theta[k]) & (z != 0)) if lives is None else lives[l]
            dz = xs[l].grad * (picked | live)      # (LISTA's z_0 is y B1^T itself, whose grad sums every layer's)
            sth[k] = dz.abs()[~picked].sum()
            if form == lista.COUPLED:
                sds[k] = (dz * ((y - x @ A.T) @ Wk)).abs().sum()
            elif k > 0:
                sds[k] = (dz * (x @ Wk.T)).abs().sum()
        out.update(scale_dtheta=sth * gs.abs(), scale_dstep=sds * gs.abs())
    return out


# ------------------------------------------------------------------------------------------------ parametrizations
# (form, (M, N, B), rank set, option set): N = 1, M > N, M < N and batches that leave a partial cluster of rows
EXACT_SHAPES = [(5, 1, 3), (12, 16, 13), (24, 16, 9), (40, 64, 17)]
# ranks per layer with the theta that goes with them: soft layers among support-selection layers, rank 0, N - 1 and
# ranks past N (read as N - 1); theta = 0 where the clamp matters, so that a mask at rank N - 2 would differ
RANK_SETS = {"clamp": (lambda N: [-1, 0, N - 1, N + 3], [1.0, 2.0, 0.0, 0.0]),
             "mixed": (lambda N: [3, -1, 7, 0], [0.0, 1.0, 2.0, 1.0]),
             "soft": (lambda N: None, [2.0, 0.0, 3.0, 1.0])}
# share_W, step given, dW given, dstep given, gscale
OPTIONS = {"perlayer": (False, True, True, True, [1.0, 0.5, 0.0, 4.0]),
           "shared": (True, False, True, True, None),
           "constW": (True, True, False, False, [0.25, 2.0, 1.0, 0.0])}
EXACT_CASES = [(form, shape, rk, opt) for form in (lista.LISTA, lista.COUPLED) for shape in EXACT_SHAPES
               for rk in ("clamp", "mixed") for opt in OPTIONS] + \
              [(form, (24, 16, 9), "soft", opt) for form in (lista.LISTA, lista.COUPLED) for opt in ("perlayer",)]


def exact_case(form, shape, rk, opt, seed=0):
    M, N, B = shape
    share_W, step, dW, dstep, gscale = OPTIONS[opt]
    ranks, theta = RANK_SETS[rk]
    return exact_problem(form, M, N, B, ranks(N), theta, share_W, seed, step=step, gscale=gscale, dW=dW, dstep=dstep)


def exact_bound(P, k0=0, k1=K):
    f = lambda t: None if t is None else t.double()
    return lo.abs_sum_bound(P["form"], f(P["A"]), f(P["B1"]), f(P["W"]), P["step"], f(P["y"]), k1, P["share_W"],
                            k0, f(P["x_in"]), f(P["d_xk"]))


RANGES = [(1, 4), (2, 4), (3, 4), (0, 2), (1, 3)]


def generic_ranks(N):
    """Per-layer ranks of the generic problems: two percentiles, a soft layer and a rank past N."""
    return [lo.ss_rank(N, 5.0), -1, lo.ss_rank(N, 13.0), N + 5]
