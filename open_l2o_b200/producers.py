"""Gradient producers (SURVEY.md 8(f) row 4): f and df/dx in ONE library call per evaluation instead of torch autograd.
A problem's builder attaches one as ``build.producer``; MetaOptimizer runs it when it ``accepts`` the program's
variables, arena slices and constants, calling what ``bind(program)`` returns as ``bound(x, scale, t) -> (f, g)`` with
x the flat arena, scale the random-scaling factors or None and t the evaluation (0..T-1 the steps, T the final loss).
The producer on the builder is shared by every program made from the problem; only the bound copy holds device state."""
from __future__ import annotations

import copy
from dataclasses import dataclass

import numpy as np
import torch

from . import cifar_data, mnist_data
from . import engine as _engine


def _names(records):
    return [r["name"] for r in records]


def _creation_order(variables, var_slices):
    """The arena holds the variables back to back in creation order."""
    ends = np.cumsum([0] + [int(np.prod(v["shape"])) for v in variables])
    return [s.start for s in var_slices] == ends[:-1].tolist()


def _mlp_names(n_layers):
    return [n for i in range(n_layers) for n in ("mlp/linear_{}/w".format(i), "mlp/linear_{}/b".format(i))]


def _outputs(x):
    return torch.empty_like(x), torch.zeros((), dtype=torch.float64, device=x.device)


class _Producer(object):
    kind = None   # the name bench.py reports

    def bind(self, prog):
        bound = copy.copy(self)
        bound.prog = prog
        return bound


@dataclass
class Lasso(_Producer):
    """problems.lasso / lasso_fixed: l2o_lasso_grad of the one variable ``var``, A = ``a``, y = ``b``, l1 ``alpha``."""
    var: str
    a: str
    b: str
    alpha: float
    kind = "lasso_batch"

    def accepts(self, variables, var_slices, constants):
        return _names(variables) == [self.var] and {self.a, self.b} <= set(_names(constants))

    def __call__(self, x, scale, t):
        g, fx = _outputs(x)
        _engine.lasso_grad(self.prog.const_vals[self.a], self.prog.const_vals[self.b], x, self.alpha, g, f=fx,
                           scale=scale)
        return fx, g


@dataclass
class MlpXent(_Producer):
    """problems.mlp: problems.mlp_value_and_grad.  It works on the variables' views, so any arena order will do."""
    activation: str
    n_layers: int
    kind = "mlp_xent"

    def accepts(self, variables, var_slices, constants):
        return _names(variables) == _mlp_names(self.n_layers) and _names(constants) == ["data", "labels"]

    def __call__(self, x, scale, t):
        from .problems import mlp_value_and_grad   # problems imports this module
        p, g = self.prog, torch.empty_like(x)
        with torch.no_grad():
            xs = x * scale if scale is not None else x    # f(x (.) scale), DM/meta_dm_train.py:384
            fx = mlp_value_and_grad(p._var_views(xs), p.const_vals["data"], p.const_vals["labels"], self.activation,
                                    p._var_views(g)).double()
            if scale is not None:
                g.mul_(scale)
        return fx, g


@dataclass
class Confocal(_Producer):
    """problems.confocal_microscopy_3d: l2o_confocal_grad, when its shared memory holds the shape and the arena and
    the constants are its [6P+1][B] rows: ``variables`` and ``constants`` in its row order."""
    num_points: int
    roi: tuple
    variables: list
    constants: list
    kind = "confocal_psf"

    def accepts(self, variables, var_slices, constants):
        return (_engine.confocal_fits(self.num_points, self.roi) and _names(variables) == self.variables and
                _names(constants) == self.constants and _creation_order(variables, var_slices) and
                all(tuple(r["shape"]) == (variables[0]["shape"][0], 1) for r in variables + constants))

    def bind(self, prog):
        # the simulated constants as row views of ONE [6P+1][B] buffer: reset_x refills them in place, so the kernel
        # reads them with no packing launch per step and captured graphs stay valid
        bound = super().bind(prog)
        bound.sim = torch.zeros(len(self.constants), prog.variables[0]["shape"][0], device=prog.device)
        shapes = {c["name"]: c["shape"] for c in prog.constants}
        for row, name in zip(bound.sim, self.constants):
            prog.const_vals[name] = row.view(shapes[name])
        return bound

    def __call__(self, x, scale, t):
        g, fx = _outputs(x)
        _engine.confocal_grad(x, self.sim, g, self.sim.shape[1], self.num_points, self.roi, f=fx, scale=scale)
        return fx, g


@dataclass
class _Minibatch(_Producer):
    """A fresh batch of ``batch_size`` from split ``mode`` of ``data_dir``, drawn in the kernel at every evaluation
    (l2o_philox.cuh).  ``device_split(data_dir, mode, device) -> (images, labels)`` is the dataset's loader."""
    batch_size: int
    mode: str
    data_dir: str
    device_split = None

    def bind(self, prog):
        # the split on the device (uploaded once per process, never reset), the seed and the device counter of the
        # draws, and the indices each evaluation drew: row t of idx for step t, row T for the final loss
        bound = super().bind(prog)
        bound.images, bound.labels = self.device_split(self.data_dir, self.mode, prog.device)
        bound.seed = prog.opt.seed
        bound.counter = torch.zeros(1, dtype=torch.int64, device=prog.device)
        bound.idx = torch.zeros(prog.T + 1, self.batch_size, dtype=torch.int32, device=prog.device)
        return bound


class _Mnist(_Minibatch):
    device_split = staticmethod(mnist_data.device_split)


@dataclass
class MnistMlp(_Mnist):
    """problems.mnist: l2o_mnist_grad, when it takes the MLP and the arena holds w0, b0, w1, ... in creation order."""
    layers: tuple
    activation: str
    kind = "mnist_mlp"

    def accepts(self, variables, var_slices, constants):
        return (_engine.mnist_fits(self.layers, self.batch_size) and
                _names(variables) == _mlp_names(len(self.layers) + 1) and _creation_order(variables, var_slices))

    def __call__(self, x, scale, t):
        g, fx = _outputs(x)
        _engine.mnist_grad(self.images, self.labels, x, g, self.layers, self.batch_size, self.activation, self.seed,
                           self.counter, f=fx, scale=scale, idx_out=self.idx[t])
        return fx, g


@dataclass
class MnistConv(_Mnist):
    """problems.mnist_conv: l2o_mnist_conv_grad, when batch norm is on, it takes the batch, and the arena holds
    ``variables`` (name, shape) in creation order."""
    batch_norm: bool
    variables: tuple
    kind = "mnist_conv"

    def accepts(self, variables, var_slices, constants):
        return (self.batch_norm and _engine.mnist_conv_fits(self.batch_size) and _creation_order(variables, var_slices)
                and [(v["name"], tuple(v["shape"])) for v in variables] == list(self.variables))

    def bind(self, prog):
        bound = super().bind(prog)
        bound.ws = torch.empty(_engine.mnist_conv_workspace_bytes(self.batch_size), dtype=torch.uint8,
                               device=prog.device)
        return bound

    def __call__(self, x, scale, t):
        g, fx = _outputs(x)
        _engine.mnist_conv_grad(self.images, self.labels, x, g, self.batch_size, self.seed, self.counter, self.ws,
                                f=fx, scale=scale, idx_out=self.idx[t])
        return fx, g


@dataclass
class CifarConv(_Minibatch):
    """problems.cifar10: l2o_cifar_conv_grad, when batch norm is on, it takes the batch, and the arena holds
    ``variables`` (name, shape) in creation order."""
    batch_norm: bool
    variables: tuple
    kind = "cifar_conv"
    device_split = staticmethod(cifar_data.device_split)

    def accepts(self, variables, var_slices, constants):
        return (self.batch_norm and _engine.cifar_conv_fits(self.batch_size) and _creation_order(variables, var_slices)
                and [(v["name"], tuple(v["shape"])) for v in variables] == list(self.variables))

    def bind(self, prog):
        bound = super().bind(prog)
        bound.ws = torch.empty(_engine.cifar_conv_workspace_bytes(self.batch_size), dtype=torch.uint8,
                               device=prog.device)
        return bound

    def __call__(self, x, scale, t):
        g, fx = _outputs(x)
        _engine.cifar_conv_grad(self.images, self.labels, x, g, self.batch_size, self.seed, self.counter, self.ws,
                                f=fx, scale=scale, idx_out=self.idx[t])
        return fx, g


@dataclass
class Nas(CifarConv):
    """problems.nas: l2o_nas_grad, under the same conditions as CifarConv."""
    kind = "nas"

    def accepts(self, variables, var_slices, constants):
        return (self.batch_norm and _engine.nas_fits(self.batch_size) and _creation_order(variables, var_slices)
                and [(v["name"], tuple(v["shape"])) for v in variables] == list(self.variables))

    def bind(self, prog):
        bound = _Minibatch.bind(self, prog)
        bound.ws = torch.empty(_engine.nas_workspace_bytes(self.batch_size), dtype=torch.uint8, device=prog.device)
        return bound

    def __call__(self, x, scale, t):
        g, fx = _outputs(x)
        _engine.nas_grad(self.images, self.labels, x, g, self.batch_size, self.seed, self.counter, self.ws,
                         f=fx, scale=scale, idx_out=self.idx[t])
        return fx, g
