"""L2O-Scale's meta-trained hand-designed baselines — ``TrainableAdam``, ``GlobalLearningRate`` and
``LearningRateSchedule`` — on the H100 engine, and ``register_optimizers``, the name table of the reference's drivers.

Mirrors the reference classes of SC/optimizer/ (SC/ = Model_Free_L2O/L2O-Scale/L2O-Scale-Training/): trainable_adam.py
("TA"), global_learning_rate.py ("GLR") and learning_rate_schedule.py ("LRS"): the same constructor arguments, defaults
and checks, ``apply_gradients`` as the ``tf.train.Optimizer`` entry, the reference's slot keys.  Every update is
coordinate-wise, so one optimizer step over all optimizee tensors is ONE launch (``l2o_tadam_step`` or
``l2o_lrsgd_step``) over their concatenated coordinates; there is no PyTorch arithmetic on the step path and no CPU
fallback.  The optimizer's variables stay on the device, and so does the schedule's step counter: ``minimize`` replays a
captured CUDA graph without a host synchronisation per step, and the schedule still advances.  Meta-training lives in
``baselines_train.py``.

TrainableAdam computes the reference's second moment as written (TA:133-134): v' = v / (1 - pow(g^2, b2)).  From its
zero initial state v stays 0, so the update is lr m^ / (1e-5 + eps): bias-corrected momentum SGD with an effective rate
of about 1e5 lr; and a coordinate whose gradient is exactly +-1 gets v = 0/0 = NaN, and with it a NaN update, from then
on.  See DESIGN §3.10.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from . import _lib
from ._lib import LrsgdStepArgs, TadamStepArgs
from .engine import _ptr, _stream
from .scale_base import ScaleOptimizer

TADAM_THETA_SPEC = [("LOL/log_learning_rate", ()), ("LOL/beta1_logit", ()), ("LOL/beta2_logit", ()),
                    ("LOL/log_epsilon", ())]                           # TA:63-82, creation order
TADAM_KEYS = ("m", "t", "v")                                           # TA:86, in sorted order (the planes' order)


def tadam_step_launch(theta, g, state_in, state_out, x=None, update=None):
    """One ``l2o_tadam_step`` launch on the current stream."""
    a = TadamStepArgs()
    a.n = int(g.numel())
    a.theta, a.g, a.state_in, a.state_out = _ptr(theta), _ptr(g), _ptr(state_in), _ptr(state_out)
    a.x, a.update = _ptr(x), _ptr(update)
    _lib.check(_lib.lib().l2o_tadam_step(C.byref(a), _stream()), "l2o_tadam_step")


def lrsgd_step_launch(rates, g, itr=None, x=None, update=None):
    """One ``l2o_lrsgd_step`` launch: update = rates[min(itr[0], n_steps - 1)] g (index 0 without a counter); the
    counter (int32 [2]) is advanced in place on the device."""
    a = LrsgdStepArgs()
    a.n, a.n_steps = int(g.numel()), int(rates.numel())
    a.rates, a.g, a.itr, a.x, a.update = _ptr(rates), _ptr(g), _ptr(itr, torch.int32), _ptr(x), _ptr(update)
    _lib.check(_lib.lib().l2o_lrsgd_step(C.byref(a), _stream()), "l2o_lrsgd_step")


def _tadam_theta(learning_rate, beta1, beta2, epsilon) -> torch.Tensor:
    """TA:64-82: the initial values in float64 (numpy), stored as fp32."""
    def inv_sigmoid(x):
        return np.log(x / (1.0 - x))
    v = np.array([np.log(learning_rate), inv_sigmoid(beta1), inv_sigmoid(beta2), np.log(epsilon)], dtype=np.float64)
    return torch.from_numpy(v).float()


class TrainableAdam(ScaleOptimizer):
    """Adam with learnable scalar parameters (TA:29-175), including the reference's second-moment expression."""
    theta_spec = TADAM_THETA_SPEC
    trainer = "baselines_train.TrainableAdamTrainer"

    def __init__(self, learning_rate=1e-3, beta1=0.9, beta2=0.999, epsilon=1e-8, device="cuda", **kwargs):
        # TA:54-59; **kwargs go to TrainableOptimizer, whose training flags the meta-trainer takes
        if learning_rate <= 0:
            raise ValueError("Learning rate must be positive.")
        if epsilon <= 0:
            raise ValueError("Epsilon must be positive.")
        if not 0 < beta1 < 1 or not 0 < beta2 < 1:
            raise ValueError("Beta values must be between 0 and 1, exclusive.")
        self.n_theta = int(_lib.lib().l2o_tadam_theta_count())
        self.n_planes = int(_lib.lib().l2o_tadam_state_floats())
        super().__init__(_tadam_theta(learning_rate, beta1, beta2, epsilon), device)

    def _new_state(self):
        return torch.empty(self.n_planes, self.N, device=self.device)   # m | t | v, zeroed by reset_state (TA:89-93)

    def get_slot(self, var_index: int, key: str) -> torch.Tensor:
        """Slot ``key`` (``m``, ``v`` or ``t``, TA:86) of optimizee tensor ``var_index``, shape [n, 1]."""
        off, n = sum(self.sizes[:var_index]), self.sizes[var_index]
        return self.state[TADAM_KEYS.index(key), off:off + n].view(n, 1)

    def step_flat(self):
        tadam_step_launch(self.theta, self.g, self.state, self.state, x=self.x)


class LearningRateSchedule(ScaleOptimizer):
    """Learns one learning rate per step of a fixed-length schedule (LRS:27-60); steps past the end keep the last."""
    trainer = "baselines_train.LearningRateScheduleTrainer"

    def __init__(self, initial_rate=0.0, n_steps=1000, device="cuda", **kwargs):
        self.n_steps = int(n_steps)
        self.theta_spec = [("LOL/learning_rates", (self.n_steps,))]                         # LRS:34-38
        super().__init__(torch.full((self.n_steps,), float(initial_rate), dtype=torch.float32), device)

    def _new_state(self):
        # one counter for all optimizee tensors (they step together): index, then the kernel's arrival count
        return torch.empty(2, dtype=torch.int32, device=self.device)

    def get_slot(self, var_index: int, key: str) -> torch.Tensor:
        """The ``itr`` slot (LRS:42-46): the number of steps taken, an int32 scalar shared by all tensors."""
        if key != "itr":
            raise KeyError(key)
        if not 0 <= var_index < len(self.sizes):
            raise IndexError(var_index)
        return self.state[0]

    def step_flat(self):
        lrsgd_step_launch(self.theta, self.g, itr=self.state, x=self.x)


class GlobalLearningRate(ScaleOptimizer):
    """Learns one global learning rate (GLR:27-39): x' = x - lr g, no state."""
    theta_spec = [("LOL/global_learning_rate", ())]
    trainer = "baselines_train.GlobalLearningRateTrainer"

    def __init__(self, initial_rate=1e-3, device="cuda", **kwargs):
        super().__init__(torch.tensor([float(initial_rate)], dtype=torch.float32), device)

    def _new_state(self):
        return torch.empty(0, device=self.device)   # stateless (GLR:36): a placeholder that marks the slots created

    def get_slot(self, var_index: int, key: str) -> torch.Tensor:
        raise KeyError("GlobalLearningRate has no slots (GLR:36): %r" % (key,))

    def step_flat(self):
        lrsgd_step_launch(self.theta, self.g, x=self.x)


def register_optimizers() -> Dict[str, type]:
    """The optimizer classes by the names of the reference drivers' table (SC/metarun.py:247-254,
    SCE/metatest.py:263-269)."""
    from .coordinatewise_rnn import CoordinatewiseRNN
    from .hierarchical_rnn import HierarchicalRNN
    return {"CoordinatewiseRNN": CoordinatewiseRNN, "GlobalLearningRate": GlobalLearningRate,
            "HierarchicalRNN": HierarchicalRNN, "LearningRateSchedule": LearningRateSchedule,
            "TrainableAdam": TrainableAdam}
