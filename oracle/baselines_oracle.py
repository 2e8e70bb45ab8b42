"""TEST INFRASTRUCTURE ONLY — CPU restatement (plain torch ops, fp32 or fp64) of L2O-Scale's meta-trained baselines.
Only tests/ and __graft_entry__.smoke() may import this module; the product path (open_l2o_b200/) never does.

Follows, op for op (SC/ = Model_Free_L2O/L2O-Scale/L2O-Scale-Training/optimizer/):
  TrainableAdam._compute_update          trainable_adam.py:95-175 (TA)
  LearningRateSchedule._compute_update   learning_rate_schedule.py:48-60
  GlobalLearningRate._compute_update     global_learning_rate.py:38-39
The step works on any tensor shape: every term is coordinate-wise and the scalars are shared, so one call on the
concatenation of all tensors equals one call per tensor.

TrainableAdam's second moment is the reference as written (TA:133-134 passes g^2 as the base and b2 as the exponent of
the debias): v' = v / (1 - pow(g^2, b2)).  From v = 0 it stays 0, except where pow(g^2, b2) == 1 (g = +-1), where it is
0/0 = NaN.  Derivative convention: where v == 0 the pow contributes exactly 0 to every adjoint.  Autograd of the literal
expression would give 0 * inf = NaN there (the base derivative b2 g^(2 b2 - 2) at g = 0, the exponent derivative
q log(g^2) at g = 0); so the value is the literal pow, detached, and the differentiable branch evaluates the pow on the
safe base 1 (derivative 0 through the where).  The b2^t' debias of v' gets the same treatment: its derivative
d v^ = v' d(b2^t') / (1 - b2^t')^2 is 0 where v' is, but in fp32 the adjoint of v^ overflows for |g| >~ 1e19 and
0 * inf would make beta2_logit's gradient NaN.  The CUDA backward forms no v-chain term where v == 0 either.  Where
v != 0 (not reachable from the zero state) the literal derivatives are used, except at g^2 == 0 (g = 0, or a g^2 that
underflows), where pow's derivatives are taken as 0: their limit (in g for b2 > 1/2) instead of inf * 0 = NaN.

Rounding (dtype=fp32): the four scalars and b^t' are computed in fp64 and rounded once, as the kernels do; 1 - b1 and
1 - b1^t' cancel by 1000x at b1 = 0.999, so their last-ulp choice shows at 1e-4 in the update.

PARITY UNPINNED: the reference ships no test, golden vector or checkpoint for these optimizers, and TensorFlow 1.x
cannot run here.  The closed forms (tests/test_baselines_cpu.py) pin the oracle instead.
"""
from __future__ import annotations

from typing import Dict, List

import torch

TADAM_KEYS = ("m", "t", "v")   # sorted key order = the engine's planes


def tadam_scalars(theta: torch.Tensor):
    """theta [4] = (log_learning_rate, beta1_logit, beta2_logit, log_epsilon) -> (lr, b1, b2, eps), differentiable."""
    th, dt = theta.double(), theta.dtype
    lr = torch.exp(th[0]).to(dt)
    b1 = torch.sigmoid(th[1]).to(dt)
    b2 = torch.sigmoid(th[2]).to(dt)
    eps = torch.exp(th[3]).to(dt) + 1e-10
    return lr, b1, b2, eps


def _pow_rounded(b, t):
    """b^t in fp64, rounded once to b's dtype."""
    return torch.pow(b.double(), t.double()).to(b.dtype)


def tadam_initial_state(n: int, dtype=torch.float64) -> Dict[str, torch.Tensor]:
    return {k: torch.zeros(n, 1, dtype=dtype) for k in TADAM_KEYS}   # TA:89-93


def tadam_compute_update(theta, param, grad, state):
    """TA:95-175 for one tensor.  Returns (new param, new state, update)."""
    lr, b1, b2, eps = tadam_scalars(theta)
    g = grad.reshape(-1, 1)
    m, t, v = state["m"], state["t"], state["v"]
    t_new = t + 1
    m_new = b1 * m + (1 - b1) * g                                    # _update_adam_estimate
    gg = g * g                                                       # tf.square
    vz = v == 0
    flat = vz | (gg == 0)                                            # (g^2 == 0: pow's derivatives taken as 0)
    q_safe = torch.pow(torch.where(flat, torch.ones_like(gg), gg), b2)
    q = torch.where(flat, torch.pow(gg, b2).detach(), q_safe)        # = pow(g^2, b2), derivative 0 where v == 0
    v_new = v / (1 - q)                                              # _debias_adam_estimate(v, g^2, b2)
    m_hat = m_new / (1 - _pow_rounded(b1, t_new))
    p2 = _pow_rounded(b2, t_new)
    v_hat = torch.where(vz, v_new / (1 - p2.detach()), v_new / (1 - p2))   # (the b2^t' term: 0 where v == 0 too)
    update = (lr * m_hat / (torch.sqrt(v_hat + 1e-10) + eps)).reshape(grad.shape)
    return param - update, {"m": m_new, "t": t_new, "v": v_new}, update


def tadam_step(theta, params: List[torch.Tensor], grads: List[torch.Tensor], states: List[Dict[str, torch.Tensor]]):
    outs = [tadam_compute_update(theta, p, g, s) for p, g, s in zip(params, grads, states)]
    return [o[0] for o in outs], [o[1] for o in outs], [o[2] for o in outs]


def lrs_compute_update(rates, param, grad, itr: int):
    """learning_rate_schedule.py:48-60: (new param, itr + 1, update).  GlobalLearningRate is rates = [rate] with the
    index pinned at 0 (global_learning_rate.py:38-39)."""
    lr = rates.reshape(-1)[min(int(itr), rates.numel() - 1)]
    update = lr * grad
    return param - update, int(itr) + 1, update


def lrs_step(rates, params: List[torch.Tensor], grads: List[torch.Tensor], itr: int):
    outs = [lrs_compute_update(rates, p, g, itr) for p, g in zip(params, grads)]
    return [o[0] for o in outs], int(itr) + 1, [o[2] for o in outs]


def state_to_planes(states: List[Dict[str, torch.Tensor]]) -> torch.Tensor:
    """Per-tensor TrainableAdam states -> the engine's [3, N] planes m | t | v."""
    return torch.cat([torch.cat([s[k] for k in TADAM_KEYS], 1) for s in states], 0).t()


def planes_to_states(planes: torch.Tensor, sizes) -> List[Dict[str, torch.Tensor]]:
    out, off = [], 0
    for n in sizes:
        p = planes[:, off:off + n].t()
        out.append({k: p[:, j:j + 1] for j, k in enumerate(TADAM_KEYS)})
        off += n
    return out
