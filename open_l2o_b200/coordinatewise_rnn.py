"""L2O-Scale ``CoordinatewiseRNN`` learned optimizer — the update step (inference path) on the H100 engine.

Mirrors the reference class ``optimizer.coordinatewise_rnn.CoordinatewiseRNN`` (SC/optimizer/coordinatewise_rnn.py,
"CR" below; SC/ = Model_Free_L2O/L2O-Scale/L2O-Scale-Training/): same constructor arguments, ``apply_gradients`` as
the ``tf.train.Optimizer`` entry, slot names of ``_initialize_state`` (CR:151-173).  The update has no per-tensor or
global term, so one optimizer step over all optimizee tensors is ONE launch of ``l2o_crnn_step`` over their
concatenated coordinates; there is no PyTorch arithmetic on the step path and no CPU fallback.  Meta-training of the
optimizer's weights lives in ``crnn_train.py``.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import List, Optional, Tuple

import torch

from . import _lib
from ._lib import CrnnStepArgs
from .engine import _ptr, _stream
from .scale_base import ScaleOptimizer

CELL_SIZES = (10, 20, 20)
RNN_FLOATS = 2 * sum(CELL_SIZES)                      # the "rnn" slot: c1 h1 c2 h2 c3 h3 (CR:306-315)
P_RMS, P_DECAY, P_LR = RNN_FLOATS, RNN_FLOATS + 1, RNN_FLOATS + 2
STATE_PLANES = P_LR + 1
# TF 1.14 names of the LSTM variables; BasicLSTMCell names its layer "basic_lstm_cell".  Not checked against TF (not
# installed here): the flat order below is the contract, the names are documentation.
_CELL_LAYER = {"LSTMCell": "lstm_cell", "BasicLSTMCell": "basic_lstm_cell"}


def theta_spec(cell_cls: str = "LSTMCell") -> List[Tuple[str, Tuple[int, ...]]]:
    """(TF variable name, shape) in creation order = the flat ``theta`` layout of ``l2o_crnn_*``: the readouts and the
    init vector of ``__init__`` (CR:90-102), then each cell's kernel and bias on the first call (CR:206)."""
    top, layer = CELL_SIZES[-1], _CELL_LAYER[cell_cls]
    out = [("LOL/update_weights", (top, 1)), ("LOL/decay_weights", (top, 1)), ("LOL/decay_bias", (1,)),
           ("LOL/learning_rate_weights", (top, 1)), ("LOL/learning_rate_bias", (1,)),
           ("LOL/init_vector", (1, RNN_FLOATS))]
    fan = 1
    for l, h in enumerate(CELL_SIZES):
        pre = "LOL/multi_rnn_cell/cell_%d/%s/" % (l, layer)
        out += [(pre + "kernel", (fan + h, 4 * h)), (pre + "bias", (4 * h,))]
        fan = h
    return out


THETA_SPEC = theta_spec()
READOUT_SCALE, DECAY_BIAS_INIT = 0.5, 2.2     # crnn_rnn_readout_scale, crnn_default_decay_var_init (CR:32-37)


def metarun_args() -> dict:
    """The constructor arguments the reference's drivers pass for ``--optimizer=CoordinatewiseRNN``
    (SC/metarun.py:154-225,243,367-398), with ``--cell_cls=LSTMCell``: the default GRUCell crashes the reference at
    CR:99.  The HierarchicalRNN-only flags ride along, as in the drivers, and are ignored."""
    from .hierarchical_rnn import metarun_flags
    args = metarun_flags()
    args.pop("level_sizes")
    args.update(cell_sizes=list(CELL_SIZES), cell_cls="LSTMCell")
    return args


def _init_theta(seed: Optional[int], zero_init_lr_weights: bool) -> torch.Tensor:
    g = torch.Generator()
    if seed is not None:
        g.manual_seed(int(seed))
    scale = READOUT_SCALE / math.sqrt(CELL_SIZES[-1])                                     # CR:86-87
    out = []
    for name, shape in THETA_SPEC:
        n = int(math.prod(shape))
        short = name.split("/")[-1]
        if short in ("update_weights", "decay_weights") or (short == "learning_rate_weights" and not zero_init_lr_weights):
            v = torch.randn(n, generator=g) * scale
        elif short == "decay_bias":
            v = torch.full((n,), DECAY_BIAS_INIT)
        elif short == "init_vector":
            v = torch.rand(n, generator=g) * 2 - 1                                         # CR:100-102
        elif short == "kernel":                                                            # tf.get_variable default
            v = (torch.rand(n, generator=g) * 2 - 1) * math.sqrt(6.0 / (shape[0] + shape[1]))
        else:                                                                              # lr weights / biases
            v = torch.zeros(n)
        out.append(v.float())
    return torch.cat(out)


def _cell_name(cell_cls) -> str:
    name = cell_cls if isinstance(cell_cls, str) else getattr(cell_cls, "__name__", repr(cell_cls))
    if name == "GRUCell":
        raise TypeError("CoordinatewiseRNN with GRUCell: the reference sums each cell's state_size (CR:99), and a "
                        "GRUCell's state_size is an int, so it raises TypeError there too; use LSTMCell")
    if name not in _CELL_LAYER:
        raise NotImplementedError("this build implements the LSTMCell / BasicLSTMCell network; unsupported cell_cls %r"
                                  % (name,))
    return name


def step_launch(theta, g, state_in, state_out, x=None, update=None):
    """One ``l2o_crnn_step`` launch on the current stream (all tensors fp32, contiguous, on the GPU)."""
    a = CrnnStepArgs()
    a.n = int(g.numel())
    a.theta, a.g, a.state_in, a.state_out = _ptr(theta), _ptr(g), _ptr(state_in), _ptr(state_out)
    a.x, a.update = _ptr(x), _ptr(update)
    _lib.check(_lib.lib().l2o_crnn_step(C.byref(a), _stream()), "l2o_crnn_step")


class CoordinatewiseRNN(ScaleOptimizer):
    """Per-coordinate 3-layer LSTM optimizer (cells 10, 20, 20) with learnable RMS decay and dynamic output scale."""
    trainer = "crnn_train.MetaTrainer"

    def __init__(self, cell_sizes, cell_cls, init_lr_range=(1., 1.), dynamic_output_scale=True, learnable_decay=True,
                 zero_init_lr_weights=False, random_seed=None, device="cuda", **kwargs):
        # signature defaults = the reference's (CR:45-52); **kwargs go to TrainableOptimizer, which ignores the
        # HierarchicalRNN flags the drivers pass along
        if len(init_lr_range) != 2:                                                       # CR:70-74
            raise ValueError("Initial LR range must be len 2, was {}".format(len(init_lr_range)))
        if init_lr_range[0] > init_lr_range[1]:
            raise ValueError("Initial LR range min is greater than max.")
        self.cell_cls = _cell_name(cell_cls)
        self.theta_spec = theta_spec(self.cell_cls)
        built = dict(cell_sizes=CELL_SIZES, learnable_decay=True, dynamic_output_scale=True)
        asked = dict(cell_sizes=tuple(cell_sizes), learnable_decay=learnable_decay,
                     dynamic_output_scale=dynamic_output_scale)
        diff = {k: v for k, v in asked.items() if built[k] != v}
        if diff:
            raise NotImplementedError("this build implements the network the reference's drivers build "
                                      "(SC/metarun.py:154-225,243,367-398); unsupported: %r" % (diff,))
        self.cell_sizes = tuple(cell_sizes)
        self.init_lr_range = tuple(init_lr_range)
        self.zero_init_lr_weights = bool(zero_init_lr_weights)
        self.random_seed = random_seed
        self.n_theta = int(_lib.lib().l2o_crnn_theta_count())
        seed = int(torch.seed() % (2 ** 31)) if random_seed is None else random_seed
        theta = _init_theta(seed, self.zero_init_lr_weights)
        assert theta.numel() == self.n_theta
        super().__init__(theta, device)

    def _new_state(self):
        """103 planes over the arena (trainable_optimizer.py:94-105): rnn c1 h1 c2 h2 c3 h3 | rms | decay | lr."""
        return torch.empty(STATE_PLANES, self.N, device=self.device)

    def reset_state(self, seed: Optional[int] = None, learning_rate: Optional[torch.Tensor] = None):
        """_initialize_state (CR:151-173): rnn = init_vector, rms = decay = 1, learning rates exp(U(log min, log max))
        drawn per coordinate (or ``learning_rate`` [N] when given)."""
        P = self.get_variables()
        self.state[:RNN_FLOATS].copy_(P["LOL/init_vector"].reshape(RNN_FLOATS, 1).expand(RNN_FLOATS, self.N))
        self.state[P_RMS].fill_(1.0)
        self.state[P_DECAY].fill_(1.0)
        if learning_rate is None:
            lo, hi = self.init_lr_range
            if lo == hi:
                learning_rate = torch.full((self.N,), float(lo))
            else:
                gen = torch.Generator()
                s = self.random_seed if seed is None else seed
                gen.manual_seed(int(torch.seed() % (2 ** 31)) if s is None else int(s))
                parts = [torch.exp(torch.rand(n, generator=gen, dtype=torch.float64) * (math.log(hi) - math.log(lo))
                                   + math.log(lo)) for n in self.sizes]
                learning_rate = torch.cat(parts)
        self.state[P_LR].copy_(torch.as_tensor(learning_rate, dtype=torch.float32).reshape(-1))

    def get_slot(self, var_index: int, key: str) -> torch.Tensor:
        """Slot ``key`` of optimizee tensor ``var_index`` (reference slot names, CR:104,168-173): ``rnn`` is [n, 100]
        packed c1 h1 c2 h2 c3 h3; ``rms``, ``decay``, ``learning_rate`` are [n, 1]."""
        off = sum(self.sizes[:var_index])
        n = self.sizes[var_index]
        if key == "rnn":
            return self.state[:RNN_FLOATS, off:off + n].t()
        planes = {"rms": P_RMS, "decay": P_DECAY, "learning_rate": P_LR}
        return self.state[planes[key], off:off + n].view(n, 1)

    def step_flat(self):
        """One step with the gradients already in ``self.g`` (flat arena order); the state is updated in place."""
        step_launch(self.theta, self.g, self.state, self.state, x=self.x)
