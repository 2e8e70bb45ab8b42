"""L2O-Scale's synthetic problem zoo: the training problems that ``metarun.py``'s ``--include_*_problems`` flags select
(SC/problems/problem_spec.py, datasets.py, problem_generator.py and problem_sets.py; SC/ =
Model_Free_L2O/L2O-Scale/L2O-Scale-Training/).

* ``Spec`` and ``Dataset``, and the synthetic datasets with the reference's shapes, labels and seed use.
* The problem classes with the reference's ``param_shapes``, ``init_tensors`` distributions and
  ``objective(params, data, labels)``.  The analytic families evaluate their objective with ONE launch of
  ``l2o_zoo_value_grad`` (``csrc/l2o_zoo.cu``) through an autograd Function whose gradient is the kernel's, and whose
  gradient's own backward is ``l2o_zoo_hvp``; ``torch_objective`` is the same objective as torch ops (any dtype and
  device), the restatement the tests and the profile compare against.  The dataset-backed families are torch ops on the
  device; the wrappers compose their inner problem's objective, so an analytic problem inside still runs the kernel.
* Every problem set of problem_sets.py, as a list of ``(Spec, dataset or None, batch_size or None)`` in the reference's
  order, and ``training_objective``, which adds the reference's gradient noise (``Problem.gradients``) and
  ``SparseProblem``'s gradient dropout in the backward.
"""
from __future__ import annotations

import ctypes as C
import math
from collections import namedtuple
from typing import Callable, Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from ._lib import ZOO, ZooArgs
from .engine import _ptr, _stream

EPSILON = 1e-6
MAX_SEED = 4294967295


class Spec(namedtuple("Spec", "callable args kwargs")):
    """A problem class (or any callable) with its arguments (problem_spec.py)."""
    __slots__ = ()

    def build(self):
        return self.callable(*self.args, **self.kwargs)


# ---- datasets (datasets.py:35-218) ------------------------------------------------------------------------------------
class Dataset(namedtuple("Dataset", "data labels")):
    """N samples: ``data`` float32 [N, ...], ``labels`` int32 [N] (or [N, 1])."""
    __slots__ = ()

    @property
    def size(self):
        return len(self.data)

    def batch_indices(self, num_batches, batch_size, rng=None):
        """Shuffled mini-batches that cover the dataset epoch by epoch (datasets.py:53-92)."""
        if len(self.data) != len(self.labels):
            raise ValueError("Labels and data must have the same number of samples.")
        rng = np.random if rng is None else rng
        out, index_in_epoch, size = [], 0, len(self.data)
        order = np.arange(size)
        rng.shuffle(order)
        for _ in range(num_batches):
            start = index_in_epoch
            index_in_epoch += batch_size
            if index_in_epoch > size:
                rng.shuffle(order)
                start, index_in_epoch = 0, batch_size
            out.append(order[start:index_in_epoch].tolist())
        return out


EMPTY_DATASET = Dataset(np.array([[0]], dtype="float32"), np.array([0], dtype="int32"))


def _rng(random_seed):
    """The reference seeds numpy's global generator (a None seed draws one from it); a RandomState with that seed
    draws the same numbers."""
    return np.random.RandomState(np.random.randint(MAX_SEED) if random_seed is None else random_seed)


def noisy_parity_class(n_samples, n_classes=2, n_context_ids=5, noise_prob=0.25, random_seed=None):
    """Sparse-to-sparse data: the label is the parity of the context ids, corrupted with ``noise_prob``."""
    rng = np.random.RandomState(random_seed)
    x = rng.randint(0, n_classes, [n_samples, n_context_ids])
    noise = rng.binomial(1, noise_prob, [n_samples])
    y = (np.sum(x, 1) + noise) % n_classes
    return Dataset(x.astype("float32"), y.astype("int32"))


def random(n_features, n_samples, n_classes=2, sep=1.0, random_seed=None):
    """sklearn's ``make_classification`` with every feature informative."""
    from sklearn.datasets import make_classification
    x, y = make_classification(n_samples=n_samples, n_features=n_features, n_informative=n_features, n_redundant=0,
                               n_classes=n_classes, class_sep=sep, random_state=random_seed)
    return Dataset(x.astype("float32"), y.astype("int32"))


def random_binary(n_features, n_samples, random_seed=None):
    """{0, 1} features, labels all 0 [N, 1]."""
    rng = _rng(random_seed)
    x = rng.randint(2, size=(n_samples, n_features))
    return Dataset(x.astype("float32"), np.zeros((n_samples, 1)).astype("int32"))


def random_symmetric(n_features, n_samples, random_seed=None):
    """N(0, 1) rows followed by their negatives, labels all 0 [N, 1]."""
    rng = _rng(random_seed)
    x1 = rng.normal(size=(int(n_samples / 2), n_features))
    x = np.concatenate((x1, -x1), axis=0)
    return Dataset(x.astype("float32"), np.zeros((n_samples, 1)).astype("int32"))


def random_mlp(n_features, n_samples, random_seed=None, n_layers=6, width=20):
    """Labels from the first output of a random ReLU MLP: 1 where it is positive, else 0."""
    rng = _rng(random_seed)
    x = rng.normal(size=(n_samples, n_features))
    y, n_in = x, n_features
    scale_factor = np.sqrt(2.) / np.sqrt(n_features)
    for _ in range(n_layers):
        y = np.dot(y, rng.normal(size=(n_in, width)) * scale_factor).clip(min=0)
        n_in = width
    y = y[:, 0]
    y[y > 0] = 1
    return Dataset(x.astype("float32"), y.astype("int32"))


def mnist(train=True):
    raise NotImplementedError("mnist needs a download; the zoo has the synthetic datasets only")


def cifar10(train=True):
    raise NotImplementedError("cifar10 needs a download; the zoo has the synthetic datasets only")


# ---- the kernel path of the analytic families -----------------------------------------------------------------------
class ZooKernel(object):
    """The ``l2o_zoo_*`` arguments of one problem other than x: family name, n, rows of ``A``, ``p0`` and the device
    constants ``A``, ``y``, ``c`` (fp32, contiguous)."""

    def __init__(self, family, n, rows=0, p0=0.0, A=None, y=None, c=None):
        self.family, self.n, self.rows, self.p0 = family, int(n), int(rows), float(p0)
        self.A, self.y, self.c = A, y, c

    def args(self, x, out, f=None, v=None) -> ZooArgs:
        a = ZooArgs()
        a.family, a.n, a.rows, a.p0 = ZOO[self.family], self.n, self.rows, self.p0
        a.x, a.v, a.out, a.f = _ptr(x, name="x"), _ptr(v, name="v"), _ptr(out, name="out"), _ptr(f, name="f")
        a.A, a.y, a.c = _ptr(self.A, name="A"), _ptr(self.y, name="y"), _ptr(self.c, name="c")
        return a

    def value_grad(self, x):
        """(f, df/dx) at the flat fp32 x: one ``l2o_zoo_value_grad`` launch."""
        f, g = torch.empty((), device=x.device), torch.empty_like(x)
        _lib.check(_lib.lib().l2o_zoo_value_grad(C.byref(self.args(x, g, f=f)), _stream()), "l2o_zoo_value_grad")
        return f, g

    def hvp(self, x, v):
        """H(x) v: one ``l2o_zoo_hvp`` launch."""
        out = torch.empty_like(x)
        _lib.check(_lib.lib().l2o_zoo_hvp(C.byref(self.args(x, out, v=v)), _stream()), "l2o_zoo_hvp")
        return out

    def hess_form(self, x, U, V=None):
        """(q, dq/dx) with q = sum_k u_k^T H(x) v_k over the rows of U, V [k, n] (V None: V = U): one
        ``l2o_zoo_hess_form`` launch per ``ZOO_MAX_PAIRS`` rows; the chunks' results are added."""
        V = U if V is None else V
        k, m = int(U.shape[0]), _lib.ZOO_MAX_PAIRS
        q, out = None, None
        for lo in range(0, k, m):
            u = U[lo:lo + m].contiguous()
            v = u if V is U else V[lo:lo + m].contiguous()
            qc, oc = torch.empty((), device=x.device), torch.empty_like(x)
            a = _lib.ZooFormArgs()
            a.base = self.args(x, oc)
            a.k, a.U, a.V, a.q = int(u.shape[0]), _ptr(u, name="U"), _ptr(v, name="V"), _ptr(qc, name="q")
            _lib.check(_lib.lib().l2o_zoo_hess_form(C.byref(a), _stream()), "l2o_zoo_hess_form")
            q, out = (qc, oc) if q is None else (q + qc, out + oc)
        return q, out


class _ZooValue(torch.autograd.Function):
    """f(x) from the kernel; backward: grad_out * g, with g a function of x whose backward is the kernel's H v."""

    @staticmethod
    def forward(ctx, x, z):
        f, g = z.value_grad(x.detach().contiguous())
        ctx.save_for_backward(x, g)
        ctx.z = z
        return f

    @staticmethod
    def backward(ctx, df):
        x, g = ctx.saved_tensors
        return df * _ZooGrad.apply(x, g, ctx.z), None


class _ZooGrad(torch.autograd.Function):
    """g(x) = df/dx; backward: H(x) dg, itself differentiable in x and dg (``_ZooHvp``)."""

    @staticmethod
    def forward(ctx, x, g, z):
        ctx.save_for_backward(x)
        ctx.z = z
        return g

    @staticmethod
    def backward(ctx, dg):
        (x,) = ctx.saved_tensors
        return _ZooHvp.apply(x, dg, ctx.z), None, None


class _ZooHvp(torch.autograd.Function):
    """H(x) v from ``l2o_zoo_hvp``; backward: the x-adjoint d(u^T H v)/dx from ``l2o_zoo_hess_form`` (u = the
    adjoint of H v) and the v-adjoint H u."""

    @staticmethod
    def forward(ctx, x, v, z):
        ctx.save_for_backward(x, v)
        ctx.z = z
        return z.hvp(x.detach().contiguous(), v.detach().contiguous())

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, u):
        x, v = ctx.saved_tensors
        x, u = x.detach().contiguous(), u.contiguous()
        dx = ctx.z.hess_form(x, u.view(1, -1), v.detach().contiguous().view(1, -1))[1] \
            if ctx.needs_input_grad[0] else None
        dv = ctx.z.hvp(x, u) if ctx.needs_input_grad[1] else None
        return dx, dv, None


def _flat(params):
    return params[0].reshape(-1) if len(params) == 1 else torch.cat([p.reshape(-1) for p in params])


def _rand_uniform(shape, lo, hi, g, device):
    return (torch.rand(shape, generator=g) * (hi - lo) + lo).to(device)


def _gen(seed):
    g = torch.Generator()
    if seed is not None:
        g.manual_seed(int(seed))
    else:
        g.seed()
    return g


# ---- problems (problem_generator.py) ---------------------------------------------------------------------------------
class Problem(object):
    """Base class (problem_generator.py:49-368): ``param_shapes``, ``random_seed`` (drawn when None) and the numpy
    generator the problem's constants come from, ``noise_stdev``.  ``objective`` is the product path;
    ``torch_objective`` the same objective as torch ops.  Analytic subclasses set ``family`` and ``kernel``."""
    family: Optional[str] = None
    zero_probability = 0.0   # SparseProblem's gradient dropout

    def __init__(self, param_shapes, random_seed=None, noise_stdev=0.0):
        if random_seed is not None and not isinstance(random_seed, int):
            raise ValueError("random_seed must be an integer or None")
        self.random_seed = np.random.randint(MAX_SEED) if random_seed is None else random_seed
        self.noise_stdev = noise_stdev
        self.rng = np.random.RandomState(self.random_seed)
        self.param_shapes = [tuple(s) for s in param_shapes]
        self._consts = {}

    def init_tensors(self, seed=None, device="cuda"):
        """tf.random_normal per parameter."""
        g = _gen(seed)
        return [torch.randn(s, generator=g).to(device) for s in self.param_shapes]

    # constants: numpy arrays, converted once per (device, dtype)
    def const(self, name, like):
        key = (name, like.device, like.dtype)
        if key not in self._consts:
            self._consts[key] = torch.as_tensor(getattr(self, name)).to(device=like.device, dtype=like.dtype)
        return self._consts[key]

    def kernel(self, x, data=None):
        raise NotImplementedError

    def objective(self, params, data=None, labels=None):
        if self.family is None:
            return self.torch_objective(params, data, labels)
        x = _flat(params)
        return _ZooValue.apply(x, self.kernel(x, data))

    def torch_objective(self, params, data=None, labels=None):
        raise NotImplementedError


class _MatrixProblem(Problem):
    """r = W x - y with W [ndim, ndim], y [ndim, 1] drawn in that order."""

    def __init__(self, ndim, random_seed=None, noise_stdev=0.0):
        super().__init__([(ndim, 1)], random_seed, noise_stdev)
        self.w = self.rng.randn(ndim, ndim).astype("float32")
        self.y = self.rng.randn(ndim, 1).astype("float32")

    def residual(self, params):
        return self.const("w", params[0]) @ params[0] - self.const("y", params[0])

    def kernel(self, x, data=None):
        n = x.numel()
        return ZooKernel(self.family, n, n, self.p0, self.const("w", x), self.const("y", x))

    p0 = 0.0


class Quadratic(_MatrixProblem):
    """f = 0.5 ||W x - y||^2."""
    family = "QUADRATIC"

    def torch_objective(self, params, data=None, labels=None):
        return 0.5 * (self.residual(params) ** 2).sum()


class Lasso(_MatrixProblem):
    """f = 0.5 ||W x - y||^2 + lambda ||x||_1."""
    family = "LASSO"

    def __init__(self, ndim, lambda_=1, random_seed=None, noise_stdev=0.0):
        super().__init__(ndim, random_seed, noise_stdev)
        self.lambda_ = lambda_
        self.p0 = float(lambda_)

    def torch_objective(self, params, data=None, labels=None):
        return 0.5 * (self.residual(params) ** 2).sum() + self.lambda_ * params[0].abs().sum()


class Norm(_MatrixProblem):
    """f = (sum (|W x - y| + 1e-6)^p)^(1/p)."""
    family = "NORM"

    def __init__(self, ndim, random_seed=None, noise_stdev=0.0, norm_power=2.):
        super().__init__(ndim, random_seed, noise_stdev)
        self.norm_power = norm_power
        self.p0 = float(norm_power)

    def torch_objective(self, params, data=None, labels=None):
        return ((self.residual(params).abs() + EPSILON) ** self.norm_power).sum() ** (1. / self.norm_power)


class Rastrigin(Problem):
    """f = mean_i(0.5 |(a x - b)_i|^2 - alpha c^T cos(2 pi x) + alpha ndim^2), a, b, c drawn in that order."""
    family = "RASTRIGIN"

    def __init__(self, ndim, alpha=10, random_seed=None, noise_stdev=0.0):
        super().__init__([(ndim, 1)], random_seed, noise_stdev)
        self.a = self.rng.randn(ndim, ndim).astype("float32")
        self.b = self.rng.randn(ndim, 1).astype("float32")
        self.c = self.rng.randn(ndim, 1).astype("float32")
        self.alpha, self.ndim = alpha, ndim

    def kernel(self, x, data=None):
        n = x.numel()
        return ZooKernel(self.family, n, n, self.alpha, self.const("a", x), self.const("b", x), self.const("c", x))

    def torch_objective(self, params, data=None, labels=None):
        x = params[0]
        norm = torch.linalg.vector_norm(self.const("a", x) @ x - self.const("b", x), dim=-1)
        cq = (self.const("c", x).T @ torch.cos(2 * np.pi * x)).squeeze()
        return (0.5 * norm ** 2 - self.alpha * cq + self.alpha * self.ndim * self.ndim).mean()


class Bowl(Problem):
    """f = 0.5 ||M x||^2, M = sqrt(diag(condition_number, 1)) R(angle)."""
    family = "BOWL"

    def __init__(self, condition_number, angle=0.0, random_seed=None, noise_stdev=0.0):
        assert condition_number > 0, "Condition number must be positive."
        super().__init__([(2, 1)], random_seed, noise_stdev)
        self.condition_number, self.angle = condition_number, angle
        hessian = np.array([[condition_number, 0.], [0., 1.]], dtype="float32")
        rotation = np.array([[np.cos(angle), -np.sin(angle)], [np.sin(angle), np.cos(angle)]])
        self.matrix = np.sqrt(hessian).dot(rotation).astype("float32")   # tf.constant(dtype=tf.float32)

    def kernel(self, x, data=None):
        return ZooKernel(self.family, 2, 2, 0.0, self.const("matrix", x))

    def torch_objective(self, params, data=None, labels=None):
        return 0.5 * ((self.const("matrix", params[0]) @ params[0]) ** 2).sum()


class Problem2D(Problem):
    """One parameter of shape (2,)."""
    init_range = None   # tf.random_uniform(minval, maxval) per parameter; None: tf.random_normal

    def __init__(self, random_seed=None, noise_stdev=0.0):
        super().__init__([(2,)], random_seed, noise_stdev)

    def init_tensors(self, seed=None, device="cuda"):
        if self.init_range is None:
            return super().init_tensors(seed, device)
        return [_rand_uniform(s, *self.init_range, _gen(seed), device) for s in self.param_shapes]

    def kernel(self, x, data=None):
        return ZooKernel(self.family, 2)

    def torch_objective(self, params, data=None, labels=None):
        return self.f2(params[0][0], params[0][1])


class Rosenbrock(Problem2D):
    family, init_range = "ROSENBROCK", (-5., 10.)

    def f2(self, x, y):
        return (1 - x) ** 2 + 100 * (y - x ** 2) ** 2


class Saddle(Problem2D):
    family = "SADDLE"

    def f2(self, x, y):
        return x ** 2 - y ** 2


class LogSumExp(Problem2D):
    family = "LOGSUMEXP"

    def f2(self, x, y):
        return torch.log(torch.exp(x + 3. * y - 0.1) + torch.exp(x - 3. * y - 0.1) + torch.exp(-x - 0.1) + 1.0)


class Ackley(Problem2D):
    family, init_range = "ACKLEY", (-32.768, 32.768)

    def f2(self, x, y):
        return (-20 * torch.exp(-0.2 * torch.sqrt(0.5 * (x ** 2 + y ** 2)))
                - torch.exp(0.5 * (torch.cos(2 * np.pi * x) + torch.cos(2 * np.pi * y))) + math.exp(1.0) + 20.)


class Beale(Problem2D):
    family, init_range = "BEALE", (-4.5, 4.5)

    def f2(self, x, y):
        return (1.5 - x + x * y) ** 2 + (2.25 - x + x * y ** 2) ** 2 + (2.625 - x + x * y ** 3) ** 2


class Booth(Problem2D):
    family, init_range = "BOOTH", (-10., 10.)

    def f2(self, x, y):
        return (x + 2 * y - 7) ** 2 + (2 * x + y - 5) ** 2


class StyblinskiTang(Problem2D):
    family, init_range = "STYBLINSKI_TANG", (-5., 5.)

    def f2(self, x, y):
        return 0.5 * sum(z ** 4 - 16 * z ** 2 + 5 * z for z in (x, y)) + 80.


class Matyas(Problem2D):
    family, init_range = "MATYAS", (-10., 10.)

    def f2(self, x, y):
        return 0.26 * (x ** 2 + y ** 2) - 0.48 * x * y


class Branin(Problem2D):
    family = "BRANIN"

    def init_tensors(self, seed=None, device="cuda"):
        g = _gen(seed)   # x1 ~ U(-5, 10), x2 ~ U(0, 15)
        return [torch.cat([_rand_uniform((1,), -5., 10., g, device), _rand_uniform((1,), 0., 15., g, device)])]

    def f2(self, x, y):
        a, b, c, r, s, t = 1., 5.1 / (4. * np.pi ** 2), 5 / np.pi, 6., 10., 1 / (8. * np.pi)
        return a * (y - b * x ** 2 + c * x - r) ** 2 + s * (1 - t) * torch.cos(x) + s


class Michalewicz(Problem2D):
    family, init_range = "MICHALEWICZ", (0., np.pi)

    def f2(self, x, y):
        m = 5
        return 2. - (torch.sin(x) * torch.sin(x ** 2 / np.pi) ** (2 * m)
                     + torch.sin(y) * torch.sin(2 * y ** 2 / np.pi) ** (2 * m))


class IsotropicQuadratic(Problem):
    """f = sum_p sum p^2 over any parameter shapes."""
    family = "ISOTROPIC_QUADRATIC"

    def kernel(self, x, data=None):
        return ZooKernel(self.family, x.numel())

    def torch_objective(self, params, data=None, labels=None):
        return sum((p ** 2).sum() for p in params)


class DependencyChain(Problem):
    """f = sum_i (x_0^2 + x_i^2 / (x_(i-1)^2 + 1e-6)), i = 1 .. ndim (x_0^2 broadcast into every term)."""
    family = "DEPENDENCY_CHAIN"

    def __init__(self, ndim, random_seed=None, noise_stdev=0.):
        super().__init__([(ndim + 1,)], random_seed, noise_stdev)
        self.ndim = ndim

    def kernel(self, x, data=None):
        return ZooKernel(self.family, x.numel())

    def torch_objective(self, params, data=None, labels=None):
        p = params[0]
        return (p[0] ** 2 + p[1:] ** 2 / (p[:-1] ** 2 + EPSILON)).sum()


class MinMaxWell(Problem):
    """f = max x^2 + 1 / min x^2 - 2 + 1e-12."""
    family = "MIN_MAX_WELL"

    def __init__(self, ndim, random_seed=None, noise_stdev=0.):
        super().__init__([(ndim,)], random_seed, noise_stdev)
        self.ndim = ndim

    def kernel(self, x, data=None):
        return ZooKernel(self.family, x.numel())

    def torch_objective(self, params, data=None, labels=None):
        sq = params[0] ** 2
        return sq.amax() + 1. / sq.amin() - 2. + 1e-12


class _DataProblem(Problem):
    """The analytic families whose objective reads the data batch [batch, ndim]."""

    def __init__(self, shape, ndim, random_seed=None, noise_stdev=0.):
        super().__init__([shape], random_seed, noise_stdev)
        self.ndim = ndim

    def kernel(self, x, data=None):
        d = data.reshape(-1, x.numel()).to(dtype=torch.float32).contiguous()
        return ZooKernel(self.family, x.numel(), d.shape[0], 0.0, d)


class OutwardSnake(_DataProblem):
    """f = sum_b d_b0 / (|x| + 1e-6) + sum_b,i>=1 ((x_i - pi cos x_(i-1)) d_bi)^2."""
    family = "OUTWARD_SNAKE"

    def __init__(self, ndim, random_seed=None, noise_stdev=0.):
        super().__init__((ndim,), ndim, random_seed, noise_stdev)

    def torch_objective(self, params, data=None, labels=None):
        p = params[0]
        radius = torch.sqrt((p ** 2).sum())
        rad_loss = (1. / (radius + 1e-6) * data[:, 0]).sum()
        sin_dist = p[1:] - torch.cos(p[:-1]) * np.pi
        return rad_loss + ((sin_dist * data[:, 1:]) ** 2).sum()


class ProjectionQuadratic(_DataProblem):
    """f = sum_b,i (x_i d_bi)^2, params [1, ndim]."""
    family = "PROJECTION_QUADRATIC"

    def __init__(self, ndim, random_seed=None, noise_stdev=0.):
        super().__init__((1, ndim), ndim, random_seed, noise_stdev)

    def torch_objective(self, params, data=None, labels=None):
        return ((params[0] * data) ** 2).sum()


class SumOfQuadratics(_DataProblem):
    """f = sum_b,i (x_i - d_bi)^2 - sum d^2 + 1e-12, params [1, ndim]."""
    family = "SUM_OF_QUADRATICS"

    def __init__(self, ndim, random_seed=None, noise_stdev=0.):
        super().__init__((1, ndim), ndim, random_seed, noise_stdev)

    def torch_objective(self, params, data=None, labels=None):
        return ((params[0] - data) ** 2).sum() - (data ** 2).sum() + 1e-12


# ---- dataset-backed families: torch ops on the device ------------------------------------------------------------------
class SoftmaxClassifier(Problem):
    """Cross entropy averaged over the batch (problem_generator.py:429-503): with two logits, the sigmoid cross entropy
    of logit 0 against the 0/1 label, as the reference computes it; otherwise softmax cross entropy with the labels as
    class indices."""

    def init_tensors(self, seed=None, device="cuda"):
        g = _gen(seed)
        return [(torch.randn(s, generator=g) * 0.01 * 1.2 / np.sqrt(s[0])).to(device) for s in self.param_shapes]

    def torch_objective(self, params, data, labels):
        logits = self.inference(params, data)
        labels = labels.reshape(-1)
        if logits.shape[1] == 2:
            return F.binary_cross_entropy_with_logits(logits[:, 0], labels.to(logits.dtype))
        return F.cross_entropy(logits, labels.long())


class SoftmaxRegression(SoftmaxClassifier):
    def __init__(self, n_features, n_classes, activation=None, random_seed=None, noise_stdev=0.0):
        self.activation, self.n_features = activation, n_features
        super().__init__([(n_features, n_classes), (n_classes,)], random_seed, noise_stdev)

    def inference(self, params, data):
        return data.reshape(-1, self.n_features) @ params[0] + params[1]


class SparseSoftmaxRegression(SoftmaxClassifier):
    """Embeddings [n_classes, n_features] looked up by the integer data, summed over the context ids."""

    def __init__(self, n_features, n_classes, activation=None, random_seed=None, noise_stdev=0.0):
        self.activation, self.n_features, self.n_classes = activation, n_features, n_classes
        super().__init__([(n_classes, n_features), (n_features, n_classes), (n_classes,)], random_seed, noise_stdev)

    def inference(self, params, data):
        emb, w, b = params
        return emb[data.long()].sum(1) @ w + b


class OneHotSparseSoftmaxRegression(SparseSoftmaxRegression):
    """SparseSoftmaxRegression through a one-hot matmul instead of a lookup."""

    def inference(self, params, data):
        emb, w, b = params
        one_hot = F.one_hot(data.long(), self.n_classes).to(emb.dtype).reshape(-1, self.n_classes)
        e = (one_hot @ emb).reshape(-1, data.shape[1], self.n_features).sum(1)
        return e @ w + b


class FullyConnected(SoftmaxClassifier):
    """MLP classifier: activation between layers, none after the last."""

    def __init__(self, n_features, n_classes, hidden_sizes=(32, 64), activation=torch.sigmoid, random_seed=None,
                 noise_stdev=0.0):
        self.n_features, self.activation = n_features, activation
        shapes, sizes = [], tuple(hidden_sizes) + (n_classes,)
        for ix, sz in enumerate(sizes):
            shapes += [(n_features if ix == 0 else hidden_sizes[ix - 1], sz), (sz,)]
        super().__init__(shapes, random_seed, noise_stdev)

    def init_tensors(self, seed=None, device="cuda"):
        g = _gen(seed)
        return [(torch.randn(s, generator=g) * 0.01).to(device) for s in self.param_shapes]

    def inference(self, params, data):
        pre = data.reshape(-1, self.n_features) @ params[0] + params[1]
        for layer in range(2, len(self.param_shapes), 2):
            pre = self.activation(pre) @ params[layer] + params[layer + 1]
        return pre


class MatMulAlgorithm(Problem):
    """theta_a, theta_b [n^2, k]; the least-squares theta_c and the squared error of the one-hot products."""

    def __init__(self, n, k):
        assert isinstance(n, int) and isinstance(k, int) and n >= 2 and n ** 2 <= k <= n ** 3
        super().__init__([(n ** 2, k), (n ** 2, k)], random_seed=None, noise_stdev=0.0)
        self.n, self.k = n, k
        onehots = np.identity(n ** 2).reshape(n ** 2, n, n)
        a3, b3 = np.repeat(onehots, n ** 2, axis=0), np.tile(onehots, [n ** 2, 1, 1])
        self.a = a3.reshape(n ** 4, n ** 2).astype("float32")
        self.b = b3.reshape(n ** 4, n ** 2).astype("float32")
        self.c = np.matmul(a3, b3).reshape(n ** 4, n ** 2).astype("float32")

    def init_tensors(self, seed=None, device="cuda"):
        g = _gen(seed)   # columns of unit L2 norm
        return [F.normalize(torch.randn(s, generator=g), dim=0).to(device) for s in self.param_shapes]

    def torch_objective(self, params, data=None, labels=None):
        ta, tb = params
        c = self.const("c", ta)
        p = (self.const("a", ta) @ ta) * (self.const("b", ta) @ tb)
        theta_c = torch.linalg.inv(p.T @ p) @ p.T @ c
        return ((p @ theta_c - c) ** 2).sum()


# ---- wrappers --------------------------------------------------------------------------------------------------------
class Rescale(Problem):
    """The inner problem in coordinates multiplied by ``scale``."""

    def __init__(self, problem_spec, scale=10., noise_stdev=0.0):
        self.problem = problem_spec.build()
        self.scale = scale
        super().__init__(self.problem.param_shapes, random_seed=None, noise_stdev=noise_stdev)

    def init_tensors(self, seed=None, device="cuda"):
        return [t * self.scale for t in self.problem.init_tensors(seed, device)]

    def objective(self, params, data=None, labels=None):
        return self.problem.objective([t / self.scale for t in params], data, labels)

    def torch_objective(self, params, data=None, labels=None):
        return self.problem.torch_objective([t / self.scale for t in params], data, labels)


class SumTask(Problem):
    """The sum of the inner problems' objectives, each over its own parameters (no data)."""

    def __init__(self, problem_specs, noise_stdev=0.0):
        self.problems = [ps.build() for ps in problem_specs]
        super().__init__([s for p in self.problems for s in p.param_shapes], random_seed=None,
                         noise_stdev=noise_stdev)

    def init_tensors(self, seed=None, device="cuda"):
        return [t for p in self.problems for t in p.init_tensors(seed, device)]

    def _sum(self, params, which):
        obj, i = 0., 0
        for p in self.problems:
            k = len(p.param_shapes)
            obj = obj + getattr(p, which)(params[i:i + k])
            i += k
        return obj

    def objective(self, params, data=None, labels=None):
        return self._sum(params, "objective")

    def torch_objective(self, params, data=None, labels=None):
        return self._sum(params, "torch_objective")


class LogObjective(Problem):
    """log(f + 1e-6) - log(1e-6) of the inner problem."""

    def __init__(self, problem_spec):
        self.problem = problem_spec.build()
        super().__init__(self.problem.param_shapes, random_seed=None, noise_stdev=0.0)

    def init_tensors(self, seed=None, device="cuda"):
        return Problem.init_tensors(self, seed, device)   # the base class's normal draw, as in the reference

    def objective(self, params, data=None, labels=None):
        return torch.log(self.problem.objective(params, data, labels) + EPSILON) - math.log(EPSILON)

    def torch_objective(self, params, data=None, labels=None):
        return torch.log(self.problem.torch_objective(params, data, labels) + EPSILON) - math.log(EPSILON)


class SparseProblem(Problem):
    """The inner objective; each gradient coordinate is set to 0 with probability ``zero_probability``
    (``training_objective`` applies it)."""

    def __init__(self, problem_spec, zero_probability=0.99, random_seed=None, noise_stdev=0.0):
        self.problem = problem_spec.build()
        self.zero_probability = self.zero_prob = zero_probability
        super().__init__(self.problem.param_shapes, random_seed=random_seed, noise_stdev=noise_stdev)

    def objective(self, params, data=None, labels=None):
        return self.problem.objective(params, data, labels)

    def torch_objective(self, params, data=None, labels=None):
        return self.problem.torch_objective(params, data, labels)


# ---- gradient noise and dropout (Problem.gradients, SparseProblem.gradients) --------------------------------------------
class _GradNoise(torch.autograd.Function):
    """Identity forward; backward g + noise_stdev N(0, 1), then zeroed where U(0, 1) < zero_probability.  The draws use
    ``gen`` (a device generator); the result is linear in g, so second-order meta-gradients pass through it."""

    @staticmethod
    def forward(ctx, p, noise_stdev, zero_probability, gen):
        ctx.conf = (noise_stdev, zero_probability, gen)
        return p

    @staticmethod
    def backward(ctx, g):
        noise_stdev, zero_probability, gen = ctx.conf
        out = g
        if noise_stdev:
            out = out + noise_stdev * torch.randn(g.shape, generator=gen, device=g.device, dtype=g.dtype)
        if zero_probability:
            mask = torch.rand(g.shape, generator=gen, device=g.device) < zero_probability
            out = torch.where(mask, torch.zeros_like(out), out)
        return out, None, None, None


def training_objective(problem: Problem, batch: Optional[Callable] = None, generator: Optional[torch.Generator] = None):
    """``objective(list of tensors) -> scalar`` for ``scale_base.train_optimizer``: the problem's objective at the
    batch ``batch()`` returns ((data, labels), or None for problems without data), with the problem's gradient noise
    and dropout drawn from ``generator`` in the backward.

    For the regularisers (``scale_reg``), which need the noise-free gradient on the batch the step's objective saw, the
    function also carries ``objective.problem``, ``objective.batch()`` (the last evaluation's (data, labels)) and
    ``objective.clean(params)`` (the objective at a fresh batch without gradient noise or dropout)."""
    noisy = bool(problem.noise_stdev) or bool(problem.zero_probability)
    if noisy and generator is None:
        raise ValueError("a noisy or sparse-gradient problem needs a generator for its gradient noise")
    last = [(None, None)]

    def evaluate(params, with_noise):
        if with_noise:
            params = [_GradNoise.apply(p, float(problem.noise_stdev), float(problem.zero_probability), generator)
                      for p in params]
        data, labels = batch() if batch is not None else (None, None)
        last[0] = (data, labels)
        return problem.objective(params, data, labels)

    def objective(params):
        return evaluate(params, noisy)
    objective.problem = problem
    objective.batch = lambda: last[0]
    objective.clean = lambda params: evaluate(params, False)
    return objective


# ---- problem sets (problem_sets.py) ----------------------------------------------------------------------------------
_S = Spec


def quadratic_problems():
    return [(_S(Quadratic, (n,), {}), None, None) for n in (20, 25, 50, 100)]


def mnist_conv_problems():
    raise NotImplementedError("mnist_conv_problems needs MNIST (a download)")


def cifar10_conv_problems():
    raise NotImplementedError("cifar10_conv_problems needs CIFAR-10 (a download)")


def mnist_mlp_problems():
    raise NotImplementedError("mnist_mlp_problems needs MNIST (a download)")


def quadratic_problems_noisy():
    return [(_S(Quadratic, (n,), {"noise_stdev": s}), None, None) for n, s in ((20, 0.5), (25, 0.0), (50, 1.0),
                                                                                (100, 2.0))]


def quadratic_problems_large():
    return [(_S(Quadratic, (n,), {}), None, None) for n in (784, 1024, 2048)]


def bowl_problems():
    return [(_S(Bowl, (0.1,), {"noise_stdev": 0.0}), None, None), (_S(Bowl, (1.0,), {"noise_stdev": 0.0}), None, None),
            (_S(Bowl, (5.0,), {"noise_stdev": 0.0}), None, None),
            (_S(Bowl, (5.0,), {"noise_stdev": 0.0, "angle": np.pi / 4.}), None, None)]


def bowl_problems_noisy():
    return [(_S(Bowl, (0.1,), {"noise_stdev": 0.1}), None, None), (_S(Bowl, (1.0,), {"noise_stdev": 0.1}), None, None),
            (_S(Bowl, (5.0,), {"noise_stdev": 0.1}), None, None),
            (_S(Bowl, (5.0,), {"noise_stdev": 0.1, "angle": np.pi / 4.}), None, None)]


def sparse_softmax_2_class_sparse_problems():
    return [(_S(SparseSoftmaxRegression, (5, 2), {"noise_stdev": 0.0}), noisy_parity_class(5, random_seed=123), 23)]


def one_hot_sparse_softmax_2_class_sparse_problems():
    return [(_S(OneHotSparseSoftmaxRegression, (5, 2), {"noise_stdev": 0.0}), noisy_parity_class(5, random_seed=123),
             23)]


def softmax_2_class_problems():
    return [(_S(SoftmaxRegression, (10, 2), {}), random(10, 1000, random_seed=123, sep=2.0), 100),
            (_S(SoftmaxRegression, (100, 2), {}), random(100, 1000, random_seed=123), 50),
            (_S(SoftmaxRegression, (200, 2), {}), random(200, 1000, random_seed=123, sep=1.5), 20),
            (_S(SoftmaxRegression, (256, 2), {}), random(256, 1000, random_seed=123, sep=1.5), 100)]


def softmax_2_class_problems_noisy():
    return [(_S(SoftmaxRegression, (10, 2), {"noise_stdev": 0.5}), random(10, 1000, random_seed=123, sep=2.0), 100),
            (_S(SoftmaxRegression, (100, 2), {"noise_stdev": 0.1}), random(100, 1000, random_seed=123), 50),
            (_S(SoftmaxRegression, (200, 2), {"noise_stdev": 0.1}), random(200, 1000, random_seed=123, sep=1.5), 20),
            (_S(SoftmaxRegression, (256, 2), {"noise_stdev": 0.5}), random(256, 1000, random_seed=123, sep=1.5), 100)]


_TEST_FUNCTIONS = (Ackley, Beale, Booth, Branin, LogSumExp, Matyas, Michalewicz, Rosenbrock, StyblinskiTang)


def optimization_test_problems():
    return [(_S(c, (), {}), None, None) for c in _TEST_FUNCTIONS]


def optimization_test_problems_noisy():
    return [(_S(c, (), {"noise_stdev": 1.}), None, None) for c in _TEST_FUNCTIONS]


_FC_RANDOM = [((8, 2), (8, 5), 8, 10), ((12, 2), (8, 5, 3), 12, 200), ((5, 2), (4, 4, 4, 4), 5, 100),
              ((11, 2), (4, 5, 6), 11, 64), ((9, 2), (8,), 9, 128), ((7, 2), (8, 5), 7, 16),
              ((8, 2), (32, 64), 8, 10), ((12, 2), (16, 8, 3), 12, 200), ((5, 2), (8, 8, 8, 8), 5, 100),
              ((11, 2), (10, 12, 12), 11, 64), ((9, 2), (32,), 9, 128), ((7, 2), (32, 64), 7, 16)]


def fully_connected_random_2_class_problems():
    return [(_S(FullyConnected, args, {"hidden_sizes": h, "activation": torch.sigmoid}), random_mlp(nf, 1000), bs)
            for args, h, nf, bs in _FC_RANDOM]


def matmul_problem_sequence(n, k_min, k_max):
    return [(_S(MatMulAlgorithm, (n, k), {}), None, None) for k in range(k_min, k_max + 1)]


def matmul_problems():
    return matmul_problem_sequence(2, 5, 8) + matmul_problem_sequence(3, 19, 24)


def log_objective_problems():
    return ([(_S(LogObjective, [_S(Quadratic, (n,), {})], {}), None, None) for n in (20, 50, 100)]
            + [(_S(LogObjective, [_S(Bowl, (c,), {})], {}), None, None) for c in (0.1, 1.0, 5.0)])


def sparse_gradient_problems():
    return ([(_S(SparseProblem, [_S(Quadratic, (n,), {})], {}), None, None) for n in (20, 50, 100)]
            + [(_S(SparseProblem, [_S(Bowl, (c,), {})], {}), None, None) for c in (0.1, 1.0, 5.0)])


def sparse_gradient_problems_mlp():
    return [(_S(SparseProblem, [_S(FullyConnected, args, {"hidden_sizes": h, "activation": torch.sigmoid})], {}),
             random_mlp(nf, 1000), bs) for args, h, nf, bs in _FC_RANDOM[:3]]


def rescale_problems():
    return ([(_S(Rescale, [_S(Norm, (18,), {"norm_power": p})], {"scale": s}), None, None)
             for p, s in ((2.5, 0.123), (1.5, 8), (2., 50), (3., 200), (1., 1000))]
            + [(_S(Rescale, [_S(Quadratic, (n,), {})], {"scale": s}), None, None)
               for n, s in ((20, 0.1), (25, 10.), (50, 350.), (100, 132))])


def norm_problems():
    return [(_S(Norm, (n,), {"norm_power": p}), None, None) for n, p in ((27, 1.), (25, 2.), (22, 3.))]


def norm_problems_noisy():
    return [(_S(Norm, (n,), {"noise_stdev": .1, "norm_power": p}), None, None) for n, p in ((19, 1.), (26, 2.),
                                                                                             (23, 3.))]


_NINE = (Rosenbrock, LogSumExp, Ackley, Beale, Booth, StyblinskiTang, Matyas, Branin, Michalewicz)


def sum_problems():
    return [(_S(SumTask, [[_S(Quadratic, (n,), {}) for n in (11, 3, 9, 7, 5, 13, 12)]], {}), None, None),
            (_S(SumTask, [[_S(Norm, (18,), {"norm_power": 3}), _S(Quadratic, (25,), {}), _S(Rosenbrock, (), {})]], {}),
             None, None),
            (_S(SumTask, [[_S(c, (), {}) for c in _NINE]], {}), None, None),
            (_S(SumTask, [[_S(c, (), {}) for c in _NINE] + [_S(Quadratic, (5,), {}), _S(Quadratic, (13,), {})]], {}),
             None, None),
            (_S(SumTask, [[_S(Quadratic, (11,), {}), _S(Quadratic, (3,), {})]], {}), None, None),
            (_S(SumTask, [[_S(Rosenbrock, (), {}), _S(LogSumExp, (), {}), _S(Ackley, (), {})]], {}), None, None)]


def sum_problems_noisy():
    return [(_S(SumTask, [[_S(Quadratic, (n,), {"noise_stdev": 0.1}) for n in (11, 3, 9, 7, 5, 13, 12)]], {}),
             None, None),
            (_S(SumTask, [[_S(c, (), {}) for c in _NINE]
                          + [_S(Quadratic, (5,), {}), _S(Quadratic, (13,), {"noise_stdev": 0.5})]], {}), None, None)]


_DATA_SIZES = [(20, 1000, 100), (12, 200, 10), (56, 5000, 100), (64, 1000, 50), (13, 10000, 50), (20, 1000, 128),
               (12, 300, 16), (56, 5000, 128), (64, 1000, 64), (13, 10000, 32)]
_SYMMETRIC_SIZES = [(20, 1000, 100), (12, 100, 10), (56, 5000, 100), (64, 1000, 50), (13, 10000, 50),
                    (20, 1000, 128), (12, 100, 16), (56, 5000, 128), (64, 1000, 64), (13, 10000, 32)]


def dependency_chain_problems():
    return [(_S(DependencyChain, (n,), {}), random_binary(n, m), bs) for n, m, bs in _DATA_SIZES]


def outward_snake_problems():
    return [(_S(OutwardSnake, (n,), {}), random_binary(n, m), bs) for n, m, bs in _DATA_SIZES]


def min_max_well_problems():
    return [(_S(MinMaxWell, (n,), {}), None, None) for n in (20, 12, 56, 64, 13)]


def sum_of_quadratics_problems():
    return [(_S(SumOfQuadratics, (n,), {}), random_symmetric(n, m), bs) for n, m, bs in _SYMMETRIC_SIZES]


def projection_quadratic_problems():
    return [(_S(ProjectionQuadratic, (n,), {}), random_symmetric(n, m), bs) for n, m, bs in _SYMMETRIC_SIZES]


def adapter_rosenbrock_local():
    raise NotImplementedError("the model_adapter problems wrap TensorFlow variables")


def adapter_rosenbrock_worker():
    raise NotImplementedError("the model_adapter problems wrap TensorFlow variables")


def lasso_problems():
    return [(_S(Lasso, (20,), {}), None, None)]


def rastrigin_problems():
    return [(_S(Rastrigin, (2,), {}), None, None)]


# metarun's --include_<flag>_problems and the set each adds, in metarun's order (SC/metarun.py:267-358)
INCLUDE_FLAGS = [
    ("sparse_softmax", sparse_softmax_2_class_sparse_problems),
    ("mnist_conv", mnist_conv_problems),
    ("cifar10_conv", cifar10_conv_problems),
    ("mnist_mlp", mnist_mlp_problems),
    ("one_hot_sparse_softmax", one_hot_sparse_softmax_2_class_sparse_problems),
    ("quadratic", quadratic_problems),
    ("noisy_quadratic", quadratic_problems_noisy),
    ("large_quadratic", quadratic_problems_large),
    ("bowl", bowl_problems),
    ("noisy_bowl", bowl_problems_noisy),
    ("softmax_2_class", softmax_2_class_problems),
    ("noisy_softmax_2_class", softmax_2_class_problems_noisy),
    ("optimization_test", optimization_test_problems),
    ("noisy_optimization_test", optimization_test_problems_noisy),
    ("fully_connected_random_2_class", fully_connected_random_2_class_problems),
    ("matmul", matmul_problems),
    ("log_objective", log_objective_problems),
    ("rescale", rescale_problems),
    ("norm", norm_problems),
    ("noisy_norm", norm_problems_noisy),
    ("sum", sum_problems),
    ("noisy_sum", sum_problems_noisy),
    ("sparse_gradient", sparse_gradient_problems),
    ("min_max_well", min_max_well_problems),
    ("sum_of_quadratics", sum_of_quadratics_problems),
    ("projection_quadratic", projection_quadratic_problems),
    ("outward_snake", outward_snake_problems),
    ("dependency_chain", dependency_chain_problems),
    ("lasso", lasso_problems),
    ("rastrigin", rastrigin_problems),
]


def problems_and_data(include) -> list:
    """metarun's ``problems_and_data`` for the set of included flag names (``"quadratic"`` for
    ``--include_quadratic_problems``): the sets in metarun's order, ``sparse_gradient_problems_mlp`` after
    ``sparse_gradient_problems`` when ``fully_connected_random_2_class`` is included too."""
    include = set(include)
    unknown = include - {name for name, _ in INCLUDE_FLAGS}
    if unknown:
        raise ValueError("unknown problem sets: %s" % sorted(unknown))
    out = []
    for name, fn in INCLUDE_FLAGS:
        if name in include:
            out.extend(fn())
            if name == "sparse_gradient" and "fully_connected_random_2_class" in include:
                out.extend(sparse_gradient_problems_mlp())
    return out
