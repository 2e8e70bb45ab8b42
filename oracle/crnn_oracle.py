"""TEST INFRASTRUCTURE ONLY — CPU restatement (plain torch ops, any dtype) of the L2O-Scale CoordinatewiseRNN update
step.  Only tests/ and __graft_entry__.smoke() may import this module; the product path (open_l2o_b200/) never does.

Follows, op for op (SC/ = Model_Free_L2O/L2O-Scale/L2O-Scale-Training/, CR = SC/optimizer/coordinatewise_rnn.py):
  __init__ (variables, initialisers)        CR:45-105
  _initialize_state                         CR:151-173
  _compute_update                           CR:175-250
  utils.rms_scaling / new_mean_squared      SC/optimizer/utils.py:108-160, asinh as log(x + sqrt(1 + x^2)) (:31-33)
  utils.project                             utils.py:90-105
  _unpack / _pack_tuples_into_rnn_state     CR:292-315 (per cell: c then h)
  tf.contrib.rnn.LSTMCell                   z = [x | h] K + b, split i | j | f | o, c' = sigmoid(f + 1) c +
                                            sigmoid(i) tanh(j), h' = sigmoid(o) tanh(c')
with the configuration the reference's drivers build (SC/metarun.py:154-225,243,367-398): cell sizes [10, 20, 20],
LSTMCell, learnable_decay, dynamic_output_scale, zero_init_lr_weights.  The per-tensor "decay := 0 if ALL(ms == 0)"
of utils.py:129-130 is kept literally.

PARITY UNPINNED beyond the cell: the LSTM cell is pinned by tests/golden/lstm_cell_hand.json; the reference ships no
test, golden vector or checkpoint for the CoordinatewiseRNN and TensorFlow 1.x cannot run here.
"""
from __future__ import annotations

import math
from typing import Dict, List

import torch

CELL_SIZES = (10, 20, 20)


def theta_spec(cell_sizes=CELL_SIZES):
    """(name, shape) in TF variable creation order: __init__ (CR:90-102), then the cells on the first call (CR:206)."""
    top = cell_sizes[-1]
    out = [("update_weights", (top, 1)), ("decay_weights", (top, 1)), ("decay_bias", (1,)),
           ("learning_rate_weights", (top, 1)), ("learning_rate_bias", (1,)),
           ("init_vector", (1, 2 * sum(cell_sizes)))]
    fan = 1
    for l, h in enumerate(cell_sizes):
        out += [("cell_%d/kernel" % l, (fan + h, 4 * h)), ("cell_%d/bias" % l, (4 * h,))]
        fan = h
    return out


def theta_count(cell_sizes=CELL_SIZES) -> int:
    return sum(int(math.prod(s)) for _, s in theta_spec(cell_sizes))


def unpack_theta(theta: torch.Tensor, cell_sizes=CELL_SIZES) -> Dict[str, torch.Tensor]:
    out, off = {}, 0
    for name, shape in theta_spec(cell_sizes):
        n = int(math.prod(shape))
        out[name] = theta[off:off + n].reshape(shape)
        off += n
    return out


def init_theta(seed: int = 0, cell_sizes=CELL_SIZES, zero_init_lr_weights=True, dtype=torch.float32) -> torch.Tensor:
    """Readouts N(0, 0.5/sqrt(top)) (crnn_rnn_readout_scale, CR:32-33,86-87), decay bias 2.2 (CR:34-37,122-125), lr
    weights zero under zero_init_lr_weights, lr bias 0 (CR:139-146), init vector U(-1, 1) (CR:100-102), LSTM kernels
    glorot-uniform (the tf.get_variable default), LSTM biases zero."""
    g = torch.Generator().manual_seed(seed)
    scale = 0.5 / math.sqrt(cell_sizes[-1])
    out = []
    for name, shape in theta_spec(cell_sizes):
        n = int(math.prod(shape))
        if name in ("update_weights", "decay_weights") or (name == "learning_rate_weights" and not zero_init_lr_weights):
            v = torch.randn(n, generator=g, dtype=torch.float64) * scale
        elif name == "decay_bias":
            v = torch.full((n,), 2.2, dtype=torch.float64)
        elif name == "init_vector":
            v = torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1
        elif name.endswith("/kernel"):
            lim = math.sqrt(6.0 / (shape[0] + shape[1]))
            v = (torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1) * lim
        else:
            v = torch.zeros(n, dtype=torch.float64)
        out.append(v)
    return torch.cat(out).to(dtype)


def lstm_cell(x, h, c, kernel, bias):
    """tf.contrib.rnn.LSTMCell / BasicLSTMCell, forget_bias 1.0, no peepholes or projection."""
    z = torch.cat([x, h], 1) @ kernel + bias
    i, j, f, o = torch.split(z, z.shape[1] // 4, dim=1)
    c_new = torch.sigmoid(f + 1.0) * c + torch.sigmoid(i) * torch.tanh(j)
    return torch.sigmoid(o) * torch.tanh(c_new), c_new


def initial_state(P: Dict[str, torch.Tensor], n: int, gen: torch.Generator, init_lr_range=(1e-6, 1e-2),
                  dtype=torch.float64) -> Dict[str, torch.Tensor]:
    """_initialize_state (CR:151-173): learning rates exp(U(log min, log max)) per coordinate."""
    lo, hi = init_lr_range
    if lo == hi:
        lr = torch.full((n, 1), lo, dtype=dtype)
    else:
        lr = torch.exp(torch.rand(n, 1, generator=gen, dtype=torch.float64) * (math.log(hi) - math.log(lo))
                       + math.log(lo)).to(dtype)
    ones = torch.ones(n, 1, dtype=dtype)
    return {"rms": ones.clone(), "learning_rate": lr, "rnn": ones * P["init_vector"].to(dtype), "decay": ones.clone()}


def asinh(x):
    return torch.log(x + torch.sqrt(1. + x ** 2))   # utils.py:31-33


def rms_scaling(gradient, decay, ms):
    grad_vec = gradient.reshape(-1, 1)
    if bool(torch.all(ms == 0.)):                  # utils.py:129-130 (per tensor)
        decay = torch.zeros_like(decay)
    ms = (1. - decay) * (grad_vec ** 2 + 1e-12) + decay * ms
    return asinh(grad_vec / torch.sqrt(ms + 1e-16)), ms


def compute_update(P, param, grad, state, cell_sizes=CELL_SIZES):
    """_compute_update (CR:175-250) for one tensor.  Returns (new param, new state, update)."""
    grad_scaled, rms = rms_scaling(grad, state["decay"], state["rms"])
    inp, pos, packed = grad_scaled, 0, []
    for l, h in enumerate(cell_sizes):
        c, hh = state["rnn"][:, pos:pos + h], state["rnn"][:, pos + h:pos + 2 * h]
        inp, c_new = lstm_cell(inp, hh, c, P["cell_%d/kernel" % l], P["cell_%d/bias" % l])
        packed += [c_new, inp]
        pos += 2 * h
    out = inp
    delta = out @ P["update_weights"]
    decay = torch.sigmoid(out @ P["decay_weights"] + P["decay_bias"])
    lr_change = 2. * torch.sigmoid(out @ P["learning_rate_weights"] + P["learning_rate_bias"])
    new_lr = lr_change * state["learning_rate"]
    update = (new_lr * delta).reshape(grad.shape)
    return param - update, {"rms": rms, "learning_rate": new_lr, "rnn": torch.cat(packed, 1), "decay": decay}, update


def step(theta, params: List[torch.Tensor], grads: List[torch.Tensor], states: List[Dict[str, torch.Tensor]]):
    """One optimizer step over all tensors: (new params, new states, updates)."""
    P = unpack_theta(theta)
    outs = [compute_update(P, p, g, s) for p, g, s in zip(params, grads, states)]
    return [o[0] for o in outs], [o[1] for o in outs], [o[2] for o in outs]


def state_to_planes(states: List[Dict[str, torch.Tensor]]) -> torch.Tensor:
    """Per-tensor state dicts -> the engine's [103, N] planes (rnn 0..99, rms, decay, learning_rate)."""
    return torch.cat([torch.cat([s["rnn"], s["rms"], s["decay"], s["learning_rate"]], 1) for s in states], 0).t()


def planes_to_states(planes: torch.Tensor, sizes) -> List[Dict[str, torch.Tensor]]:
    out, off = [], 0
    for n in sizes:
        p = planes[:, off:off + n].t()
        out.append({"rnn": p[:, :100], "rms": p[:, 100:101], "decay": p[:, 101:102], "learning_rate": p[:, 102:103]})
        off += n
    return out
