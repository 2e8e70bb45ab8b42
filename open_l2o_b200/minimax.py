"""L2O-Minimax's Twin-L2O optimizer pair (MM = Model_Free_L2O/L2O-Minimax/Twin-L2O.py).

Two coordinate-wise optimizers, net 0 (min, updates u) and net 1 (max, updates v), each
LSTMCell(2, H) -> LSTMCell(H, H) -> Linear(H, 1) (MM Optimizer, :676), held in one device arena [2][theta_count] with
fp64 gradients.  The unroll and its meta-gradient run in the l2o_minimax_* kernels (include/l2o_b200.h); this module
holds the weights, the problem batches, the per-batch buffers and the host logic around them (learning-rate schedule,
curriculum selection, reward coefficients).  There is no PyTorch fallback for the unroll.
"""
from __future__ import annotations

import ctypes as C
import math
from collections import OrderedDict

import numpy as np
import torch

from . import _lib

LOSSES = (1, 2, 3, 4)


def param_spec(hidden: int):
    """(name, shape) of one net's parameters in state_dict order (the kernels' theta layout)."""
    G = 4 * hidden
    return [("recurs.weight_ih", (G, 2)), ("recurs.weight_hh", (G, hidden)), ("recurs.bias_ih", (G,)),
            ("recurs.bias_hh", (G,)), ("recurs2.weight_ih", (G, hidden)), ("recurs2.weight_hh", (G, hidden)),
            ("recurs2.bias_ih", (G,)), ("recurs2.bias_hh", (G,)), ("output.weight", (1, hidden)),
            ("output.bias", (1,))]


def theta_count(hidden: int) -> int:
    return int(_lib.lib().l2o_minimax_theta_count(hidden))


def sche_lr(optim_it: int) -> np.ndarray:
    """The warm-up sign-step sizes (MM do_fit :94), indexed by iteration - 1."""
    return np.arange(1e-4, 1e-1, (1e-1 - 1e-4) / int(0.2 * optim_it))


def warm_end(optim_it: int) -> int:
    """The first iteration that is not a sign step (MM :201: iteration < 0.2 optim_it is)."""
    t = 1
    while t < 0.2 * optim_it:
        t += 1
    return t


def sche_ratio(epoch: int) -> float:
    """The curriculum's kept fraction at an epoch (MM :84)."""
    return 0.2 + epoch / 100 if 0 <= epoch <= 80 else 1


def get_index(traj_u: np.ndarray, a, b, iteration: int, unroll_unit: int, ratio: float) -> list:
    """MM utils/metrics.py get_index: the problems kept by the curriculum at boundary `iteration`.  traj_u [B][T] is
    u after each iteration (iteration t at column t-1).  Each problem scores sum_t (b sin(a pi u_t))^2 over the first
    (iteration // 10) 2 unroll_unit - 1 columns, and the int(ratio B) lowest scores are kept (all when that is 0)."""
    B = traj_u.shape[0]
    k = int(ratio * B)
    flag = iteration // 10
    curve = traj_u[:, 0:flag * 2 * unroll_unit - 1]
    result = []
    for i in range(B):
        result.append(sum(((-1) * b[i] * math.sin(a[i] * math.pi * x)) ** 2 for x in curve[i]))
    return sorted(range(B), key=lambda i: result[i], reverse=True)[-k:]


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


def make_matrix_game_data(dim: int, p: float, low: float, high: float, n: int, seed: int) -> np.ndarray:
    """Matrix-game problems as MM dataset/matrix_game/create_dataset.py makes them: entries uniform in [low, high),
    each kept with probability p, one row of dim * dim values per problem ([n][dim * dim])."""
    rng = np.random.RandomState(seed)
    data = rng.uniform(low=low, high=high, size=(n, dim, dim))
    mask = rng.binomial(n=1, p=p, size=(n, dim, dim))
    return np.reshape(data * mask, (n, dim * dim))


def read_toy(path: str, n: int) -> np.ndarray:
    """A problem file, the first n lines as float32: a toy file (MM dataset/toy/*.txt) gives [n][2] `a b` pairs, a
    matrix-game file [n][dim * dim] (problem_tensor shapes either for the kernels)."""
    return np.loadtxt(path).astype(np.float32)[0:n]


def problem_tensor(data, loss: int, dim: int, device) -> torch.Tensor:
    """ToyLoss data of a batch as the kernels read it: [B][2] (a, b) for losses 1-3, [B][dim][dim] A for loss 4."""
    d = torch.as_tensor(np.asarray(data, dtype=np.float32))
    d = d.reshape(-1, dim, dim) if loss == 4 else d.reshape(-1, 2)
    return d.to(device).contiguous()


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


class TwinOptimizer:
    """The min/max optimizer pair: theta [2][theta_count] fp32, grad [2][theta_count] fp64, and the forward's
    weight image (rebuilt by refresh() whenever theta changes)."""

    def __init__(self, hidden: int, device="cuda", seed: int | None = None):
        if hidden <= 0 or hidden > 128:
            raise ValueError("hidden must be in [1, 128]")
        self.hidden = hidden
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.n_theta = theta_count(hidden)
        self.theta = torch.zeros(2, self.n_theta, dtype=torch.float32, device=self.device)
        self.grad = torch.zeros(2, self.n_theta, dtype=torch.float64, device=self.device)
        self.image = torch.zeros(2, int(_lib.lib().l2o_minimax_image_floats(hidden)), dtype=torch.float32,
                                 device=self.device)
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        for n in (0, 1):
            self.load_state_dict(n, self.default_init(hidden, gen))

    @staticmethod
    def default_init(hidden: int, gen=None) -> "OrderedDict[str, torch.Tensor]":
        """torch's own initialisation of LSTMCell and Linear: every entry U(-1/sqrt(H), 1/sqrt(H))."""
        k = 1.0 / math.sqrt(hidden)
        sd = OrderedDict()
        for name, shape in param_spec(hidden):
            sd[name] = (torch.rand(shape, generator=gen) * 2 - 1) * k
        return sd

    def _views(self, n):
        out, off = OrderedDict(), 0
        for name, shape in param_spec(self.hidden):
            cnt = int(np.prod(shape))
            out[name] = (off, cnt, shape)
            off += cnt
        return out

    def state_dict(self, n: int) -> "OrderedDict[str, torch.Tensor]":
        """Net n's parameters under the reference's names and shapes (loadable into MM's Optimizer)."""
        return OrderedDict((name, self.theta[n, off:off + cnt].detach().cpu().clone().reshape(shape))
                           for name, (off, cnt, shape) in self._views(n).items())

    def load_state_dict(self, n: int, sd) -> None:
        views = self._views(n)
        if set(sd.keys()) != set(views.keys()):
            raise KeyError("state_dict keys %s do not match %s" % (sorted(sd.keys()), sorted(views.keys())))
        for name, (off, cnt, shape) in views.items():
            val = torch.as_tensor(sd[name])
            if tuple(val.shape) != tuple(shape):
                raise ValueError("%s: shape %s, expected %s" % (name, tuple(val.shape), shape))
            self.theta[n, off:off + cnt].copy_(val.reshape(-1).to(self.theta))
        self.refresh()

    def refresh(self) -> None:
        _lib.check(_lib.lib().l2o_minimax_image(_ptr(self.theta), _ptr(self.image), self.hidden,
                                                C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)),
                   "l2o_minimax_image")


class Unroll:
    """The buffers of one batch of B problems of dim coordinates under a TwinOptimizer: u, v [R], the states
    [2][4][R][H] and, for training, one segment's checkpoints and backward workspace."""

    def __init__(self, twin: TwinOptimizer, loss: int, data: torch.Tensor, dim: int = 1, rescale: float = 1e-4,
                 out_mul: float = 1.0):
        if loss not in LOSSES:
            raise ValueError("loss must be 1, 2, 3 or 4")
        if dim <= 0 or (loss != 4 and dim != 1):
            raise ValueError("losses 1-3 take dim = 1, loss 4 dim >= 1")
        want = (dim, dim) if loss == 4 else (2,)
        if (not isinstance(data, torch.Tensor) or data.dtype != torch.float32 or data.device != twin.device or
                data.dim() != 1 + len(want) or tuple(data.shape[1:]) != want or data.shape[0] <= 0 or
                not data.is_contiguous()):
            raise ValueError("data must be a contiguous float32 tensor [B]%s on %s (minimax.problem_tensor)"
                             % ("".join("[%d]" % d for d in want), twin.device))
        self.twin, self.loss, self.dim = twin, loss, dim
        self.data = data
        self.batch = int(data.shape[0])
        self.rows = self.batch * dim
        self.rescale, self.out_mul = rescale, out_mul
        dev = twin.device
        self.u = torch.zeros(self.rows, device=dev)
        self.v = torch.zeros(self.rows, device=dev)
        self.state = torch.zeros(2, 4, self.rows, twin.hidden, device=dev)
        self._seg = {}

    def reset(self, gen: torch.Generator | None = None) -> None:
        """MM do_fit's starting point: u, v ~ 0.5 (2 U(0, 1) - 1) (DualOptimizee :660), every h and c ~ N(0, 0.01^2)
        (:114-124), one state row per coordinate."""
        R, H = self.rows, self.twin.hidden
        self.u.copy_(0.5 * ((-1) + 2 * torch.rand(R, generator=gen)))
        self.v.copy_(0.5 * ((-1) + 2 * torch.rand(R, generator=gen)))
        self.state.copy_(torch.randn(2, 4, R, H, generator=gen) * 0.01)

    def _args(self, t0, t1, optim_it, lr, traj=None, ckpt=None, dl=None, lval=None):
        a = _lib.MinimaxArgs()
        a.loss, a.batch, a.dim, a.hidden = self.loss, self.batch, self.dim, self.twin.hidden
        a.t0, a.t1, a.warm_end = t0, t1, warm_end(optim_it)
        a.out_mul, a.rescale = self.out_mul, self.rescale
        a.lr, a.theta, a.image, a.data = _ptr(lr), _ptr(self.twin.theta), _ptr(self.twin.image), _ptr(self.data)
        a.u, a.v, a.state = _ptr(self.u), _ptr(self.v), _ptr(self.state)
        a.traj, a.ckpt, a.dl, a.lval = _ptr(traj), _ptr(ckpt), _ptr(dl), _ptr(lval)
        return a

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.twin.device).cuda_stream)

    def _lr(self, optim_it):
        key = ("lr", optim_it)
        if key not in self._seg:
            self._seg[key] = torch.as_tensor(sche_lr(optim_it), dtype=torch.float32).to(self.twin.device)
        return self._seg[key]

    def buffers(self, n_iter: int):
        """traj [n][R][2], ckpt [n][R][4H+2], dl [n][R], lval [n][B] for a launch of n iterations (cached)."""
        key = ("buf", n_iter)
        if key not in self._seg:
            dev, R, H = self.twin.device, self.rows, self.twin.hidden
            self._seg[key] = dict(traj=torch.zeros(n_iter, R, 2, device=dev),
                                  ckpt=torch.zeros(n_iter, R, 4 * H + 2, device=dev),
                                  dl=torch.zeros(n_iter, R, device=dev),
                                  lval=torch.zeros(n_iter, self.batch, device=dev))
        return self._seg[key]

    def forward(self, t0: int, t1: int, optim_it: int, traj=None, ckpt=None, dl=None, lval=None) -> None:
        """Iterations [t0, t1) of a do_fit of optim_it iterations, one launch."""
        a = self._args(t0, t1, optim_it, self._lr(optim_it), traj, ckpt, dl, lval)
        _lib.check(_lib.lib().l2o_minimax_fwd(C.byref(a), self._stream()), "l2o_minimax_fwd")

    def backward(self, t0: int, t1: int, optim_it: int, ckpt, dl, coef, weight=None) -> torch.Tensor:
        """Meta-gradient of sum_t coef[t - t0] weight[p] l_t over [t0, t1) into twin.grad (two launches)."""
        a = self._args(t0, t1, optim_it, self._lr(optim_it), None, ckpt, dl, None)
        nbytes = C.c_size_t()
        _lib.check(_lib.lib().l2o_minimax_workspace_bytes(C.byref(a), C.byref(nbytes)), "l2o_minimax_workspace_bytes")
        key = ("ws", nbytes.value)
        if key not in self._seg:
            self._seg[key] = torch.empty((nbytes.value + 7) // 8, dtype=torch.float64, device=self.twin.device)
        g = _lib.MinimaxGrads()
        g.coef, g.weight, g.dtheta, g.scratch = _ptr(coef), _ptr(weight), _ptr(self.twin.grad), _ptr(self._seg[key])
        _lib.check(_lib.lib().l2o_minimax_bwd(C.byref(a), C.byref(g), self._stream()), "l2o_minimax_bwd")
        return self.twin.grad


def reward_coefs(t0: int, boundary: int, batch: int) -> torch.Tensor:
    """The weight of each l_t, t in [t0, boundary), in the sum of rewards (l_t + l_{t-1}) / B back-propagated at the
    boundary: l_t enters reward_t and, unless t + 1 is the boundary (whose reward is not yet formed), reward_{t+1}."""
    return torch.tensor([(2.0 if t + 1 < boundary else 1.0) / batch for t in range(t0, boundary)], dtype=torch.float32)
