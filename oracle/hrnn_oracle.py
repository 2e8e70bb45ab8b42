"""TEST INFRASTRUCTURE ONLY — CPU restatement (plain torch ops, any dtype) of the L2O-Scale HierarchicalRNN update
step, the "next" row 1 of SURVEY.md 8(f) / BASELINE config #4.  Only tests/, __graft_entry__.smoke() and bench.py's
CPU-baseline legs may import this module; the product path (open_l2o_b200/) never does.

Follows, function by function (SC/ = /root/reference/Model_Free_L2O/L2O-Scale/L2O-Scale-Training/):
  _compute_updates                  SC/optimizer/hierarchical_rnn.py:353-430
  _compute_mean_log_lr              :432-442
  _compute_scaled_and_ms_grads      :444-496   (+ utils.rms_scaling / new_mean_squared / asinh, SC/optimizer/utils.py:36-38,108-160)
  _extend_rnn_input                 :498-540
  _update_rnn_cells                 :542-604   (+ BiasGRUCell, SC/optimizer/rnn_cells.py:27-68; utils.affine, utils.py:41-90)
  _compute_rnn_state_projections    :606-661
  _compute_new_learning_rate        :663-706
  _compute_updated_global_state     :708-728
  _initialize_state / _initialize_global_state  :303-350
with the flag set the reference's drivers actually run (SC/metarun.py:154-225,243): level sizes [10, 20, 20],
num_gradient_scales=4, use_grad_products, use_log_means_squared, use_relative_lr, use_problem_lr_mean,
use_gradient_shortcut, dynamic_output_scale, learnable_decay, learnable_inp_decay, learnable_rnn_init = True;
use_attention, use_multiple_scale_decays, use_extreme_indicator, use_lr_shortcut = False.

PARITY UNPINNED: the reference ships no test, golden vector or checkpoint for L2O-Scale, and TensorFlow 1.x cannot
run here; this restatement is anchored on the code as written only (including its quirks: asinh as
log(x + sqrt(1 + x^2)); the global RNN sees the LAST tensor's layer state only, :426-427).
"""
from __future__ import annotations

import math
from typing import Dict, List

import torch

NUM_SCALES = 4
LEVELS = (10, 20, 20)
N_FEAT = 12  # 4 scaled grads + 3 grad products + 4 centred log-ms + 1 relative log-lr

# (name, shape, init) in a fixed order = the flat theta layout of include/l2o_b200.h (l2o_hrnn_*)
def theta_spec(levels=LEVELS):
    h0, h1, h2 = levels
    f = N_FEAT
    return [
        ("Level0_RNN/init_vector", (1, h0)), ("Level1_RNN/init_vector", (1, h1)), ("Level2_RNN/init_vector", (1, h2)),
        ("update_weights", (h0, 1)), ("scl_decay_weights", (h0, 1)), ("scl_decay_bias", (1,)),
        ("inp_decay_weights", (h0, 1)), ("inp_decay_bias", (1,)),
        ("learning_rate_weights", (h0, 1)), ("learning_rate_bias", (1,)),
        ("PerTensor/Layer0_RNN/Param/Affine/Matrix", (h1, 3 * h0)), ("PerTensor/Layer0_RNN/Param/Affine/Bias", (3 * h0,)),
        ("PerTensor/Layer0_RNN/Global/Affine/Matrix", (h2, 3 * h0)), ("PerTensor/Layer0_RNN/Global/Affine/Bias", (3 * h0,)),
        ("PerTensor/Layer0_RNN/BiasGRUCell/gates/Affine/Matrix", (f + h0, 2 * h0)),
        ("PerTensor/Layer0_RNN/BiasGRUCell/gates/Affine/Bias", (2 * h0,)),
        ("PerTensor/Layer0_RNN/BiasGRUCell/candidate/Affine/Matrix", (f + h0, h0)),
        ("PerTensor/Layer0_RNN/BiasGRUCell/candidate/Affine/Bias", (h0,)),
        ("PerTensor/Layer1_RNN/Affine/Matrix", (h2, 3 * h1)), ("PerTensor/Layer1_RNN/Affine/Bias", (3 * h1,)),
        ("PerTensor/Layer1_RNN/BiasGRUCell/gates/Affine/Matrix", (h0 + f + h1, 2 * h1)),
        ("PerTensor/Layer1_RNN/BiasGRUCell/gates/Affine/Bias", (2 * h1,)),
        ("PerTensor/Layer1_RNN/BiasGRUCell/candidate/Affine/Matrix", (h0 + f + h1, h1)),
        ("PerTensor/Layer1_RNN/BiasGRUCell/candidate/Affine/Bias", (h1,)),
        ("PerTensor/GradsToDelta/Matrix", (NUM_SCALES, 1)),
        ("PerTensor/learning_rate_momentum_logit", ()), ("PerTensor/param_stepsize_offset", ()),
        ("Layer2_RNN/BiasGRUCell/gates/Affine/Matrix", (h1 + h2, 2 * h2)),
        ("Layer2_RNN/BiasGRUCell/gates/Affine/Bias", (2 * h2,)),
        ("Layer2_RNN/BiasGRUCell/candidate/Affine/Matrix", (h1 + h2, h2)),
        ("Layer2_RNN/BiasGRUCell/candidate/Affine/Bias", (h2,)),
    ]


def theta_count(levels=LEVELS) -> int:
    return sum(int(math.prod(s)) for _, s in theta_spec(levels))


def init_theta(seed: int = 0, levels=LEVELS, dtype=torch.float32) -> torch.Tensor:
    """Flat theta with the reference's initial distributions (flag values of hierarchical_rnn.py:33-56):
    affine matrices N(0, scale/sqrt(fan_in)) (utils.py:70-76) with scale 0.5 (biasgrucell_scale / hrnn_affine_scale),
    gate bias 2.2, readouts N(0, 0.5/sqrt(10)), lr weights zero, scl bias 3.2, inp bias 2.2, lr momentum logit 3.2,
    stepsize offset -1, GradsToDelta N(0.25, 0.1/sqrt(4)), init vectors U(-1, 1)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    h0 = levels[0]
    for name, shape in theta_spec(levels):
        n = int(math.prod(shape))
        if name.endswith("init_vector"):
            v = torch.rand(n, generator=g, dtype=torch.float64) * 2 - 1
        elif name in ("update_weights", "scl_decay_weights", "inp_decay_weights"):
            v = torch.randn(n, generator=g, dtype=torch.float64) * (0.5 / math.sqrt(h0))
        elif name in ("learning_rate_weights", "learning_rate_bias"):
            v = torch.zeros(n, dtype=torch.float64)
        elif name == "scl_decay_bias":
            v = torch.full((n,), 3.2, dtype=torch.float64)
        elif name == "inp_decay_bias":
            v = torch.full((n,), 2.2, dtype=torch.float64)
        elif name.endswith("learning_rate_momentum_logit"):
            v = torch.full((n,), 3.2, dtype=torch.float64)
        elif name.endswith("param_stepsize_offset"):
            v = torch.full((n,), -1.0, dtype=torch.float64)
        elif name.endswith("GradsToDelta/Matrix"):
            v = 0.25 + torch.randn(n, generator=g, dtype=torch.float64) * (0.1 / math.sqrt(shape[0]))
        elif name.endswith("gates/Affine/Bias"):
            v = torch.full((n,), 2.2, dtype=torch.float64)
        elif name.endswith("Bias"):
            v = torch.zeros(n, dtype=torch.float64)
        elif name.endswith("Matrix"):
            v = torch.randn(n, generator=g, dtype=torch.float64) * (0.5 / math.sqrt(shape[0]))
        else:
            raise AssertionError(name)
        out.append(v)
    return torch.cat(out).to(dtype)


def unpack_theta(theta: torch.Tensor, levels=LEVELS) -> Dict[str, torch.Tensor]:
    out, off = {}, 0
    for name, shape in theta_spec(levels):
        n = int(math.prod(shape))
        out[name] = theta[off:off + n].reshape(shape)
        off += n
    assert off == theta.numel()
    return out


def initial_state(P: Dict[str, torch.Tensor], var: torch.Tensor, gen: torch.Generator,
                  init_lr_range=(1e-6, 1e-2)) -> Dict[str, torch.Tensor]:
    """_initialize_state (:303-343) for one optimizee tensor."""
    n, dt = var.numel(), var.dtype
    st = {"parameter": torch.ones(n, 1, dtype=dt) * P["Level0_RNN/init_vector"],
          "scl_decay": torch.zeros(n, 1, dtype=dt), "inp_decay": torch.zeros(n, 1, dtype=dt),
          "layer": torch.ones(1, 1, dtype=dt) * P["Level1_RNN/init_vector"]}
    lo, hi = math.log(init_lr_range[0]) / 2.0, math.log(init_lr_range[1]) / 2.0
    actual = torch.rand(n, 1, generator=gen, dtype=torch.float64) * (hi - lo) + lo
    offset = torch.rand((), generator=gen, dtype=torch.float64) * (hi - lo) + lo
    st["log_learning_rate"] = torch.clamp(actual + offset, -33.0, 33.0).to(dt)
    for i in range(NUM_SCALES):
        st["grad_accum%d" % (i + 1)] = torch.zeros(n, 1, dtype=dt)
        st["ms%d" % (i + 1)] = torch.zeros(n, 1, dtype=dt)
    return st


def initial_global_state(P, dtype=torch.float32):
    return (torch.ones(1, 1, dtype=dtype) * P["Level2_RNN/init_vector"])


def _affine(x, matrix, bias):  # utils.affine (utils.py:41-90)
    return x @ matrix + bias


def _bias_gru(inputs, state, Wg, bg, Wc, bc, bias):  # BiasGRUCell.__call__ (rnn_cells.py:46-68)
    n = state.shape[1]
    r_b, u_b, c_b = bias[:, :n], bias[:, n:2 * n], bias[:, 2 * n:]
    proj = _affine(torch.cat([inputs, state], 1), Wg, bg)
    r = torch.sigmoid(proj[:, :n] + r_b)
    u = torch.sigmoid(proj[:, n:] + u_b)
    c = torch.tanh(_affine(torch.cat([inputs, r * state], 1), Wc, bc) + c_b)
    return u * state + (1 - u) * c


def _asinh(x):  # utils.asinh (utils.py:36-38) — as written, not torch.asinh
    return torch.log(x + torch.sqrt(1.0 + x ** 2))


def step(theta: torch.Tensor, params: List[torch.Tensor], grads: List[torch.Tensor],
         states: List[Dict[str, torch.Tensor]], global_state: torch.Tensor, levels=LEVELS):
    """One _compute_updates (:353-430).  Returns (new_params, new_states, new_global_state, update_steps)."""
    P = unpack_theta(theta, levels)
    h0 = levels[0]
    # _compute_mean_log_lr (:432-442): problem-wide mean of the PREVIOUS log learning rates
    mean_log_lr = sum(s["log_learning_rate"].sum() for s in states) / sum(s["log_learning_rate"].numel() for s in states)
    new_params, new_states, update_steps = [], [], []
    layer_state = None
    for param, grad_unflat, st in zip(params, grads, states):
        grad = grad_unflat.reshape(-1, 1)
        # ---- _compute_scaled_and_ms_grads (:444-496)
        decays = [st["inp_decay"]]
        for i in range(NUM_SCALES - 1):
            decays.append(torch.sqrt(decays[i]))
        sd = st["scl_decay"]
        accs, scaled, mss = [], [], []
        for i, d in enumerate(decays):
            acc = grad * (1.0 - d) + st["grad_accum%d" % (i + 1)] * d
            ms_old = st["ms%d" % (i + 1)]
            dec = torch.zeros_like(sd) if bool((ms_old == 0).all()) else sd       # utils.py:128-130
            ms = (1.0 - dec) * (acc * acc + 1e-12) + dec * ms_old                   # utils.py:133-134
            accs.append(acc)
            mss.append(ms)
            scaled.append(_asinh(acc / torch.sqrt(ms + 1e-16)))                     # utils.py:157-158
        # ---- _extend_rnn_input (:498-540)
        feats = list(scaled)
        feats += [a * b for a, b in zip(scaled[:-1], scaled[1:])]
        lms = [torch.log(m + 1e-16) for m in mss]
        avg = sum(lms) / float(len(lms))                                           # tf.reduce_mean(list, axis=0)
        feats += [m - avg for m in lms]
        feats.append(st["log_learning_rate"].reshape(-1, 1) - mean_log_lr)
        x_in = torch.cat(feats, 1)
        # ---- _update_rnn_cells (:542-604)
        bias0 = (_affine(st["layer"], P["PerTensor/Layer0_RNN/Param/Affine/Matrix"], P["PerTensor/Layer0_RNN/Param/Affine/Bias"])
                 + _affine(global_state, P["PerTensor/Layer0_RNN/Global/Affine/Matrix"], P["PerTensor/Layer0_RNN/Global/Affine/Bias"]))
        h_new = _bias_gru(x_in, st["parameter"], P["PerTensor/Layer0_RNN/BiasGRUCell/gates/Affine/Matrix"],
                          P["PerTensor/Layer0_RNN/BiasGRUCell/gates/Affine/Bias"],
                          P["PerTensor/Layer0_RNN/BiasGRUCell/candidate/Affine/Matrix"],
                          P["PerTensor/Layer0_RNN/BiasGRUCell/candidate/Affine/Bias"], bias0)
        layer_in = torch.cat([h_new, x_in], 1).mean(0, keepdim=True)
        layer_bias = _affine(global_state, P["PerTensor/Layer1_RNN/Affine/Matrix"], P["PerTensor/Layer1_RNN/Affine/Bias"])
        layer_state = _bias_gru(layer_in, st["layer"], P["PerTensor/Layer1_RNN/BiasGRUCell/gates/Affine/Matrix"],
                                P["PerTensor/Layer1_RNN/BiasGRUCell/gates/Affine/Bias"],
                                P["PerTensor/Layer1_RNN/BiasGRUCell/candidate/Affine/Matrix"],
                                P["PerTensor/Layer1_RNN/BiasGRUCell/candidate/Affine/Bias"], layer_bias)
        # ---- _compute_rnn_state_projections (:606-661)
        delta = h_new @ P["update_weights"] + torch.cat(scaled, 1) @ P["PerTensor/GradsToDelta/Matrix"]
        delta = delta / torch.sqrt((delta ** 2).mean() + 1e-16)
        scl = torch.sigmoid(h_new @ P["scl_decay_weights"] + P["scl_decay_bias"])
        inp = torch.sigmoid(h_new @ P["inp_decay_weights"] + P["inp_decay_bias"])
        # ---- _compute_new_learning_rate (:663-693)
        lr_change = h_new @ P["learning_rate_weights"] + P["learning_rate_bias"]
        # straight-through clip (:674-686): the value is clamped to [-33, max_log_lr], the gradient passes as if unclipped
        pre_log_lr = st["log_learning_rate"] + lr_change
        step_log_lr = pre_log_lr + (torch.clamp(pre_log_lr, -33.0, 33.0) - pre_log_lr).detach()
        lrm = torch.sigmoid(P["PerTensor/learning_rate_momentum_logit"])
        new_log_lr = lrm * st["log_learning_rate"] + (1.0 - lrm) * step_log_lr
        lr_param = torch.exp(step_log_lr + P["PerTensor/param_stepsize_offset"])
        upd = (lr_param * delta).reshape(param.shape)
        update_steps.append(upd)
        new_params.append(param - upd)
        ns = {"parameter": h_new, "scl_decay": scl, "inp_decay": inp, "layer": layer_state,
              "log_learning_rate": new_log_lr}
        for i in range(NUM_SCALES):
            ns["grad_accum%d" % (i + 1)] = accs[i]
            ns["ms%d" % (i + 1)] = mss[i]
        new_states.append(ns)
    # ---- _compute_updated_global_state([layer_state], ...) (:426-427,708-728): the LAST tensor's layer state only
    new_global = _bias_gru(layer_state, global_state, P["Layer2_RNN/BiasGRUCell/gates/Affine/Matrix"],
                           P["Layer2_RNN/BiasGRUCell/gates/Affine/Bias"],
                           P["Layer2_RNN/BiasGRUCell/candidate/Affine/Matrix"],
                           P["Layer2_RNN/BiasGRUCell/candidate/Affine/Bias"],
                           torch.zeros(1, 3 * levels[2], dtype=theta.dtype, device=theta.device))  # bias=None -> zeros
    return new_params, new_states, new_global, update_steps
