"""Meta-training of the L2O-Scale ``CoordinatewiseRNN``: BPTT through the unrolled optimizer, with the meta-objective,
the clipped RMSProp meta-step and the training loops of ``hrnn_train`` (``MetaTrainerBase``, ``train_optimizer``).

Mirrors ``TrainableOptimizer.train`` (SC/optimizer/trainable_optimizer.py:200-470) for this optimizer.  The optimizee's
gradients are constants of the meta-gradient unless ``use_second_derivatives=True`` (the reference's default; it
stop_gradient's them only with the flag off, :330-338): then ``l2o_crnn_bwd`` also returns the adjoint of g and torch
autograd carries it on through the optimizee's Hessian-vector product.  The trainer's default stays ``False``.  Each
optimizer step is one ``torch.autograd.Function`` around two CUDA entry points: ``l2o_crnn_step`` forward,
``l2o_crnn_bwd`` backward (recompute from the planes before the step, then the adjoints).  The only torch ops on N
coordinates are the optimizee's own and ``x - update``.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Callable, Optional, Sequence

import torch

from . import _lib
from ._lib import CrnnBwdArgs, L2OError
from .coordinatewise_rnn import RNN_FLOATS, THETA_SPEC, _init_theta, _p, step_launch
from .hrnn_train import MetaTrainerBase, train_optimizer  # noqa: F401  (train_optimizer serves both trainers)


def unpack_theta(theta: torch.Tensor):
    """Differentiable views of the flat theta (layout: coordinatewise_rnn.THETA_SPEC)."""
    out, off = {}, 0
    for name, shape in THETA_SPEC:
        n = int(math.prod(shape))
        out[name] = theta[off:off + n].reshape(shape)
        off += n
    return out


class _Step(torch.autograd.Function):
    """One optimizer step over all coordinates as an autograd node: (theta, planes [103, N], g) -> (planes', update).
    The adjoint of g is computed only when autograd asks for it (second-order meta-gradients)."""

    @staticmethod
    def forward(ctx, theta, planes, g):
        theta, planes = theta.detach().contiguous(), planes.detach().contiguous()
        new = torch.empty_like(planes)
        upd = torch.empty_like(g)
        step_launch(theta, g, planes, new, update=upd)
        ctx.save_for_backward(theta, planes, g)
        return new, upd

    @staticmethod
    def backward(ctx, d_new, d_upd):
        theta, planes, g = ctx.saved_tensors
        d_new = torch.zeros_like(planes) if d_new is None else d_new.contiguous()
        d_upd = torch.zeros_like(g) if d_upd is None else d_upd.contiguous()
        d_old = torch.empty_like(planes)
        d_theta = torch.zeros(theta.numel(), dtype=torch.float64, device=theta.device)
        d_g = torch.empty_like(g) if ctx.needs_input_grad[2] else None
        a = CrnnBwdArgs()
        a.n = int(g.numel())
        a.theta, a.g, a.state_old = _p(theta), _p(g), _p(planes)
        a.d_state_new, a.d_update, a.d_state_old = _p(d_new), _p(d_upd), _p(d_old)
        a.d_theta = d_theta.data_ptr()
        a.d_g = _p(d_g)
        _lib.check(_lib.lib().l2o_crnn_bwd(C.byref(a), torch.cuda.current_stream().cuda_stream), "l2o_crnn_bwd")
        return d_theta.to(torch.float32), d_old, d_g


class OptimizerState(object):
    """The optimizer's state between unrolls: planes [103, N] (rnn c1 h1 c2 h2 c3 h3 | rms | decay | learning_rate) and
    the optimizee coordinates x [N]."""

    def __init__(self, planes, x):
        self.planes, self.x = planes, x


class MetaTrainer(MetaTrainerBase):
    """``TrainableOptimizer.train`` + the RMSProp block of ``metaopt.train_optimizer`` for the CoordinatewiseRNN.

    objective(list of tensors shaped like ``shapes``) -> scalar.  ``theta`` is the optimizer's flat weight vector
    (``CoordinatewiseRNN.theta`` layout); it is updated in place by ``train_step``.

    ``use_second_derivatives``: differentiate through the optimizee's gradients (the reference's default is ``True``;
    this trainer's default stays ``False``, the first-order meta-gradient).  See ``hrnn_train.MetaTrainer``."""

    def __init__(self, shapes: Sequence[Sequence[int]], theta: Optional[torch.Tensor] = None, device="cuda:0",
                 learning_rate=1e-6, rms_decay=0.9, rms_epsilon=1e-20, gradient_clip=1e4, l2_reg=0.0,
                 use_log_objective=True, use_numerator_epsilon=False, init_lr_range=(1e-6, 1e-2), random_seed=None,
                 zero_init_lr_weights=True, use_second_derivatives=False):
        if not torch.cuda.is_available():
            raise L2OError("CoordinatewiseRNN meta-training needs a CUDA device (no CPU path)")
        self._setup(shapes, device)
        self._setup_meta(_init_theta(random_seed, zero_init_lr_weights) if theta is None
                         else theta.detach().clone().float(), learning_rate, rms_decay, rms_epsilon, gradient_clip,
                         l2_reg, use_log_objective, use_numerator_epsilon, init_lr_range, random_seed,
                         use_second_derivatives)

    def initial_state(self, params: Sequence[torch.Tensor], theta: torch.Tensor,
                      learning_rate: Optional[torch.Tensor] = None) -> OptimizerState:
        """_initialize_state (CR:151-173); the learnable init vector keeps its graph.  The learning rates are drawn
        per coordinate as exp(U(log min, log max)) unless given ([N])."""
        dev = self.device
        x = torch.cat([p.detach().reshape(-1).float() for p in params]).to(dev)
        N = x.numel()
        if learning_rate is None:
            lo, hi = self.init_lr_range
            if lo == hi:
                learning_rate = torch.full((N,), float(lo))
            else:
                learning_rate = torch.exp(torch.rand(N, generator=self._gen, dtype=torch.float64)
                                          * (math.log(hi) - math.log(lo)) + math.log(lo))
        rnn = unpack_theta(theta)["LOL/init_vector"].reshape(RNN_FLOATS, 1).expand(RNN_FLOATS, N)
        ones = torch.ones(2, N, device=dev)
        lr = learning_rate.to(dev).float().reshape(1, N)
        return OptimizerState(torch.cat([rnn, ones, lr], 0), x)

    def unroll(self, objective: Callable, state: OptimizerState, num_steps: int, theta: Optional[torch.Tensor] = None,
               obj_weights: Optional[Sequence[float]] = None, initial_obj: Optional[torch.Tensor] = None):
        """``loop_body`` x num_steps (trainable_optimizer.py:263-401).  Returns (meta objective with its graph, the list
        of objective values, the final OptimizerState with its graph)."""
        if num_steps < 1:
            raise ValueError("an unroll needs at least one step")
        theta = self.theta if theta is None else theta
        planes, x = state.planes, state.x
        objs, total = [], 0.0
        w = [1.0] * num_steps if obj_weights is None else list(obj_weights)
        for t in range(num_steps):
            obj, g = self._objective_and_gradient(objective, x)   # g keeps its graph only for second derivatives
            objs.append(obj)
            total = total + w[t] * obj
            planes, upd = _Step.apply(theta, planes, g)
            x = x - upd                                                                     # CR:240
        initial = objs[0].detach() if initial_obj is None else initial_obj
        meta = self.scale_objective(total, torch.stack([o.reshape(()) for o in objs]), initial)
        return meta, objs, OptimizerState(planes, x)

