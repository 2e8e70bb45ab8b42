"""Meta-training of L2O-Scale's baselines (``TrainableAdam``, ``LearningRateSchedule``, ``GlobalLearningRate``): BPTT
through the unrolled optimizer, with the meta-objective, the clipped RMSProp meta-step and the training loops of
``scale_base`` (``MetaTrainerBase``, ``train_optimizer``).

The loop these classes run in the reference is the Evaluation copy's ``TrainableOptimizer.train``
(SCE/optimizer/trainable_optimizer.py:283-310; the Training copy calls ``_compute_updates`` with six arguments, and the
method these classes inherit takes four).  The optimizee's gradients are constants of the meta-gradient unless
``use_second_derivatives=True`` (the reference's default, :330-338 of the Training copy); then the backward kernels also
return the adjoint of g.  The trainers' default stays ``False``, as for the other two trainers.  Each optimizer step is
one ``torch.autograd.Function`` around two CUDA entry points (``l2o_tadam_step`` / ``l2o_tadam_bwd`` or
``l2o_lrsgd_step`` / ``l2o_lrsgd_bwd``); the only torch op on N coordinates besides the optimizee's own is
``x - update``.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib
from ._lib import LrsgdBwdArgs, TadamBwdArgs
from .engine import _ptr, _stream
from .scale_base import MetaTrainerBase, planes_step, train_optimizer  # noqa: F401  (public names)
from .trainable_baselines import TADAM_THETA_SPEC, _tadam_theta, lrsgd_step_launch, tadam_step_launch

# (theta [4], planes [3, N], g) -> (planes', update)
_TadamStep = planes_step(tadam_step_launch, TadamBwdArgs, "l2o_tadam_bwd")


class _LrsStep(torch.autograd.Function):
    """(rates [n_steps], g) -> update = rates[min(itr, n_steps - 1)] g.  ``itr_new`` is a copy of ``itr_old`` that the
    kernel advances in place; ``itr_old`` (None: index 0, GlobalLearningRate) tells the backward which rate was used."""

    @staticmethod
    def forward(ctx, rates, g, itr_old, itr_new):
        rates = rates.detach().contiguous()
        upd = torch.empty_like(g)
        lrsgd_step_launch(rates, g, itr=itr_new, update=upd)
        ctx.save_for_backward(rates, g)
        ctx.itr = itr_old
        return upd

    @staticmethod
    def backward(ctx, d_upd):
        rates, g = ctx.saved_tensors
        d_rates = torch.zeros(rates.numel(), dtype=torch.float64, device=rates.device)
        d_g = torch.empty_like(g) if ctx.needs_input_grad[1] else None
        a = LrsgdBwdArgs()
        a.n, a.n_steps = int(g.numel()), int(rates.numel())
        a.rates, a.itr, a.g, a.d_update = _ptr(rates), _ptr(ctx.itr, torch.int32), _ptr(g), _ptr(d_upd.contiguous())
        a.d_rates, a.d_g = d_rates.data_ptr(), _ptr(d_g)
        _lib.check(_lib.lib().l2o_lrsgd_bwd(C.byref(a), _stream()), "l2o_lrsgd_bwd")
        return d_rates.to(torch.float32), d_g, None, None


class OptimizerState(object):
    """The optimizer's state between unrolls and the optimizee coordinates x [N].  TrainableAdam: planes [3, N]
    (m | t | v).  LearningRateSchedule: itr, the int32 [2] step counter (None for GlobalLearningRate)."""

    def __init__(self, x, planes=None, itr=None):
        self.x, self.planes, self.itr = x, planes, itr


class _BaselineTrainer(MetaTrainerBase):
    """``TrainableOptimizer.train`` + the RMSProp block of ``metaopt.train_optimizer`` for one of the baselines.

    ``theta`` is the optimizer's flat variable vector.  ``use_second_derivatives`` (default ``False``, the first-order
    meta-gradient): see ``MetaTrainerBase``."""

    def __init__(self, shapes: Sequence[Sequence[int]], theta: torch.Tensor, device="cuda:0", learning_rate=1e-6,
                 rms_decay=0.9, rms_epsilon=1e-20, gradient_clip=1e4, l2_reg=0.0, use_log_objective=True,
                 use_numerator_epsilon=False, random_seed=None, use_second_derivatives=False, **regularizer):
        super().__init__(shapes, theta, device, learning_rate, rms_decay, rms_epsilon, gradient_clip, l2_reg,
                         use_log_objective, use_numerator_epsilon, None, random_seed, use_second_derivatives,
                         **regularizer)


class TrainableAdamTrainer(_BaselineTrainer):
    """Meta-trains TrainableAdam's four scalars (theta = log_learning_rate, beta1_logit, beta2_logit, log_epsilon)."""
    what = "TrainableAdam"
    theta_spec = TADAM_THETA_SPEC

    def __init__(self, shapes, theta: Optional[torch.Tensor] = None, device="cuda:0", **kwargs):
        super().__init__(shapes, _tadam_theta(1e-3, 0.9, 0.999, 1e-8) if theta is None else theta, device, **kwargs)

    def initial_state(self, params, theta, _unused=None) -> OptimizerState:
        x = self._x0(params)
        return OptimizerState(x, planes=torch.zeros(3, x.numel(), device=self.device))   # TA:89-93

    def _stepper(self, theta):
        def step(state, g):
            planes, upd = _TadamStep.apply(theta, state.planes, g)
            return upd, OptimizerState(None, planes=planes)
        return step


class LearningRateScheduleTrainer(_BaselineTrainer):
    """Meta-trains the schedule (theta = learning_rates [n_steps])."""
    what = "LearningRateSchedule"
    counter = True

    def __init__(self, shapes, theta: Optional[torch.Tensor] = None, device="cuda:0", **kwargs):
        super().__init__(shapes, torch.zeros(1000) if theta is None else theta, device, **kwargs)

    def initial_state(self, params, theta, _unused=None) -> OptimizerState:
        itr = torch.zeros(2, dtype=torch.int32, device=self.device) if self.counter else None   # LRS:42-46
        return OptimizerState(self._x0(params), itr=itr)

    def _stepper(self, theta):
        def step(state, g):
            itr_new = None if state.itr is None else state.itr.clone()
            return _LrsStep.apply(theta, g, state.itr, itr_new), OptimizerState(None, itr=itr_new)
        return step


class GlobalLearningRateTrainer(LearningRateScheduleTrainer):
    """Meta-trains the one global learning rate (theta [1]): the schedule trainer with a one-entry table and no
    counter."""
    what = "GlobalLearningRate"
    counter = False

    def __init__(self, shapes, theta: Optional[torch.Tensor] = None, device="cuda:0", **kwargs):
        super().__init__(shapes, torch.full((1,), 1e-3) if theta is None else theta.reshape(1), device, **kwargs)
