"""What the problem-zoo kernel tests share: the launch rule's cluster threshold, the boundary sizes, points where the
objectives are not smooth (built exactly, in fp32 and fp64 alike), the 2-D functions' evaluation points, and fp64
autograd of a Problem's torch restatement as the reference for l2o_zoo_value_grad, l2o_zoo_hvp and l2o_zoo_hess_form."""
import numpy as np
import torch

from open_l2o_b200 import scale_zoo as Z

CLUSTER_WORK = 65536   # rows * n from which the matrix and data families run on a cluster of CL CTAs (l2o_zoo.cu)
CL = 8
TILE = 4               # pairs whose row dots the Hessian form takes at once (l2o_zoo.cu's kTile)

# Matrix and elementwise families at the cluster switch (Quadratic 255 | 256, and 257 with a ragged last row block and
# column block) and at L2O_ZOO_MAX_N = 4096, the largest shared-memory plan
BOUNDARY_CASES = ([("Quadratic", (n,), {}) for n in (255, 256, 257, 4096)]
                  + [("Norm", (n,), {"norm_power": 1.5}) for n in (257, 4096)]
                  + [("Lasso", (4096,), {"lambda_": 0.7}), ("Rastrigin", (256,), {})]
                  + [("IsotropicQuadratic", ([(4096,)],), {}), ("DependencyChain", (4095,), {}),
                     ("MinMaxWell", (4096,), {})])
# Data families (n, batch): one CTA at 4096 x 15 and 64 x 1023, the cluster at 4096 x 16 (2 rows per CTA), 64 x 1024
# and 2 x 32768 (CTAs 2 .. 7 own no columns)
BOUNDARY_DATA = [(4096, 15), (4096, 16), (64, 1023), (64, 1024), (2, 32768)]
DATA_FAMILIES = ("ProjectionQuadratic", "SumOfQuadratics", "OutwardSnake")
PLANE_FAMILIES = ("Rosenbrock", "Saddle", "LogSumExp", "Ackley", "Beale", "Booth", "StyblinskiTang", "Matyas", "Branin",
                  "Michalewicz")


def on_cluster(rows, n):
    return rows * n >= CLUSTER_WORK


def make(cls, args=(), kwargs=None, seed=0):
    if cls == "IsotropicQuadratic":
        return Z.IsotropicQuadratic(*args, random_seed=seed)
    return getattr(Z, cls)(*args, random_seed=seed, **(kwargs or {}))


def data_batch(cls, n, batch, seed):
    """The data batch [batch, n] the data-family tests use (fp32, CPU): batch rows of the family's dataset in a seeded
    random order.  random_symmetric makes rows in +- pairs, so an odd batch leaves one of the last pair out."""
    gen = np.random.RandomState(seed)
    ds = Z.random_binary(n, batch, random_seed=seed) if cls == "OutwardSnake" else \
        Z.random_symmetric(n, batch + batch % 2, random_seed=seed)
    return torch.as_tensor(ds.data[gen.permutation(len(ds.data))[:batch]]).float()


def reference(problem, x, v=None, U=None, V=None, data=None):
    """fp64 autograd of problem.torch_objective at the fp32 point x [n]: f and g, H v with v, and q = sum_k u_k^T H v_k
    with dq/dx with U, V [k, n]."""
    xd = x.detach().double().cpu().requires_grad_(True)
    d = None if data is None else data.double().cpu()
    f = problem.torch_objective([xd.view(problem.param_shapes[0])], d)
    (g,) = torch.autograd.grad(f, xd, create_graph=True)
    out = {"f": f.detach(), "g": g.detach()}
    if v is not None:
        (hv,) = torch.autograd.grad(g, xd, grad_outputs=v.double().cpu(), retain_graph=True)
        out["hv"] = hv
    if U is not None:
        q = 0.0
        for u, w in zip(U.double().cpu(), V.double().cpu()):
            (hw,) = torch.autograd.grad(g, xd, grad_outputs=w, create_graph=True)
            q = q + (hw * u).sum()
        (dq,) = torch.autograd.grad(q, xd)
        out["q"], out["dq"] = q.detach(), dq
    return out


# ---- constructed non-smooth points -----------------------------------------------------------------------------------
def zero_residual(cls, n, seed, p=2.0):
    """A Norm or Rastrigin problem and an fp32 point x [n] with residual r_i = 0 exactly for one row i: that row of the
    matrix is e_a - e_b, x_b = x_a and y_i = 0, so A_i.x - y_i = x_a - x_b = 0 in any precision and summation order.
    A nonzero row keeps A_i v != 0, so the row's curvature weight shows in H v.  On the cluster (n >= 256) the row
    and the two columns sit in different CTAs' blocks.  Returns (problem, x, i, a, b)."""
    problem = make(cls, (n,), {"norm_power": p} if cls == "Norm" else {}, seed)
    i, a, b = (200, 7, 250) if n >= 256 else (n // 2 + 7, 3, n - 10)
    mat, rhs = ("w", "y") if cls == "Norm" else ("a", "b")
    A, y = getattr(problem, mat).copy(), getattr(problem, rhs).copy()
    A[i] = 0.0
    A[i, a], A[i, b] = 1.0, -1.0
    y[i] = 0.0
    setattr(problem, mat, A)   # before the first const() call, which caches the device copy
    setattr(problem, rhs, y)
    x = problem.init_tensors(seed, "cpu")[0].reshape(-1).clone()
    x[b] = x[a]
    return problem, x, i, a, b


def residuals(problem, x, dtype):
    """A x - y of a matrix problem's constants in dtype."""
    mat, rhs = ("w", "y") if isinstance(problem, Z.Norm) else ("a", "b")
    A = torch.as_tensor(getattr(problem, mat)).to(dtype)
    return (A @ x.to(dtype).reshape(-1, 1) - torch.as_tensor(getattr(problem, rhs)).to(dtype)).reshape(-1)


def lasso_zeros(n, seed):
    """A Lasso problem and a point with every third coordinate +0 or -0, where |.|'s gradient is sign(0) = 0."""
    problem = make("Lasso", (n,), {"lambda_": 0.7}, seed)
    x = problem.init_tensors(seed, "cpu")[0].reshape(-1).clone()
    x[0::6] = 0.0
    x[3::6] = -0.0
    return problem, x


MMW_MAX, MMW_MIN = (3, 3000), (1000, 2500)   # thread j % 512, pass j // 512: warps 0 / 13 and 15 / 14, passes 0 / 5, 1 / 4


def min_max_ties(n, seed, all_equal=False):
    """A MinMaxWell point of n coordinates with exactly tied extremes: x_3 = 2.5, x_3000 = -2.5 (the two maxima of x^2)
    and x_1000 = 0.25, x_2500 = -0.25 (the two minima), every other |x_j| in [0.5, 2); or, all_equal, every x_j = +-0.75,
    where the max and the min both tie over all n."""
    g = torch.Generator().manual_seed(seed)
    sgn = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
    if all_equal:
        return 0.75 * sgn
    x = (0.5 + 1.5 * torch.rand(n, generator=g)) * sgn
    x[MMW_MAX[0]], x[MMW_MAX[1]] = 2.5, -2.5
    x[MMW_MIN[0]], x[MMW_MIN[1]] = 0.25, -0.25
    return x


# ---- the 2-D functions -----------------------------------------------------------------------------------------------
MINIMA = {"Rosenbrock": [(1.0, 1.0)], "Beale": [(3.0, 0.5)], "Booth": [(1.0, 3.0)]}


def plane_points(cls, m=8):
    """An m x m grid over the function's init range (Branin: x in [-5, 10], y in [0, 15]; the normal-init functions:
    [-3, 3]^2) and its known minima, as fp32 [points, 2]."""
    rng = getattr(Z, cls).init_range
    if cls == "Branin":
        gx, gy = np.linspace(-5.0, 10.0, m), np.linspace(0.0, 15.0, m)
    else:
        lo, hi = rng if rng is not None else (-3.0, 3.0)
        gx = gy = np.linspace(lo, hi, m)
    pts = [(a, b) for a in gx for b in gy] + MINIMA.get(cls, [])
    return torch.tensor(pts, dtype=torch.float32)
