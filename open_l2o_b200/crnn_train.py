"""Meta-training of the L2O-Scale ``CoordinatewiseRNN``: BPTT through the unrolled optimizer, with the meta-objective,
the clipped RMSProp meta-step and the training loops of ``scale_base`` (``MetaTrainerBase``, ``train_optimizer``).

Mirrors ``TrainableOptimizer.train`` (SC/optimizer/trainable_optimizer.py:200-470) for this optimizer.  The optimizee's
gradients are constants of the meta-gradient unless ``use_second_derivatives=True`` (the reference's default; it
stop_gradient's them only with the flag off, :330-338): then ``l2o_crnn_bwd`` also returns the adjoint of g and torch
autograd carries it on through the optimizee's Hessian-vector product.  The trainer's default stays ``False``.  Each
optimizer step is one ``torch.autograd.Function`` around two CUDA entry points: ``l2o_crnn_step`` forward,
``l2o_crnn_bwd`` backward (recompute from the planes before the step, then the adjoints).  The only torch ops on N
coordinates are the optimizee's own and ``x - update``.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch

from ._lib import CrnnBwdArgs
from .coordinatewise_rnn import RNN_FLOATS, THETA_SPEC, _init_theta, step_launch
from .scale_base import MetaTrainerBase, planes_step, theta_views, train_optimizer  # noqa: F401  (public name)

# One optimizer step over all coordinates as an autograd node: (theta, planes [103, N], g) -> (planes', update)
_Step = planes_step(step_launch, CrnnBwdArgs, "l2o_crnn_bwd")


class OptimizerState(object):
    """The optimizer's state between unrolls: planes [103, N] (rnn c1 h1 c2 h2 c3 h3 | rms | decay | learning_rate) and
    the optimizee coordinates x [N]."""

    def __init__(self, planes, x):
        self.planes, self.x = planes, x


class MetaTrainer(MetaTrainerBase):
    """``TrainableOptimizer.train`` + the RMSProp block of ``metaopt.train_optimizer`` for the CoordinatewiseRNN.

    ``theta`` is the optimizer's flat weight vector (``CoordinatewiseRNN.theta`` layout).  ``use_second_derivatives``
    (default ``False``, the first-order meta-gradient): see ``MetaTrainerBase``."""
    what = "CoordinatewiseRNN"
    theta_spec = THETA_SPEC

    def __init__(self, shapes: Sequence[Sequence[int]], theta: Optional[torch.Tensor] = None, device="cuda:0",
                 learning_rate=1e-6, rms_decay=0.9, rms_epsilon=1e-20, gradient_clip=1e4, l2_reg=0.0,
                 use_log_objective=True, use_numerator_epsilon=False, init_lr_range=(1e-6, 1e-2), random_seed=None,
                 zero_init_lr_weights=True, use_second_derivatives=False, **regularizer):
        super().__init__(shapes, _init_theta(random_seed, zero_init_lr_weights) if theta is None else theta, device,
                         learning_rate, rms_decay, rms_epsilon, gradient_clip, l2_reg, use_log_objective,
                         use_numerator_epsilon, init_lr_range, random_seed, use_second_derivatives, **regularizer)

    def initial_state(self, params: Sequence[torch.Tensor], theta: torch.Tensor,
                      learning_rate: Optional[torch.Tensor] = None) -> OptimizerState:
        """_initialize_state (CR:151-173); the learnable init vector keeps its graph.  The learning rates are drawn
        per coordinate as exp(U(log min, log max)) unless given ([N])."""
        dev = self.device
        x = self._x0(params)
        N = x.numel()
        if learning_rate is None:
            lo, hi = self.init_lr_range
            if lo == hi:
                learning_rate = torch.full((N,), float(lo))
            else:
                learning_rate = torch.exp(torch.rand(N, generator=self._gen, dtype=torch.float64)
                                          * (math.log(hi) - math.log(lo)) + math.log(lo))
        rnn = theta_views(theta, THETA_SPEC)["LOL/init_vector"].reshape(RNN_FLOATS, 1).expand(RNN_FLOATS, N)
        ones = torch.ones(2, N, device=dev)
        lr = learning_rate.to(dev).float().reshape(1, N)
        return OptimizerState(torch.cat([rnn, ones, lr], 0), x)

    def _stepper(self, theta: torch.Tensor):
        def step(state: OptimizerState, g: torch.Tensor):
            planes, upd = _Step.apply(theta, state.planes, g)
            return upd, OptimizerState(planes, None)                                       # x - upd: CR:240
        return step
