"""Meta-training of the L2O-Scale ``HierarchicalRNN``: BPTT through the unrolled optimizer, the log meta-objective and
the clipped RMSProp meta-step.

Mirrors ``TrainableOptimizer.train`` (SC/optimizer/trainable_optimizer.py:200-470; SC/ =
Model_Free_L2O/L2O-Scale/L2O-Scale-Training/), ``scale_objective`` (:586-609) and the meta-optimizer block of
``metaopt.train_optimizer`` (SC/metaopt.py:255-289).

Second derivatives.  The reference differentiates through the optimizee's gradients g by default
(``use_second_derivatives=True``, trainable_optimizer.py:61-84) and wraps them in ``tf.stop_gradient`` only when the flag
is off (:330-338).  ``MetaTrainer(use_second_derivatives=True)`` does the same: ``l2o_hrnn_coord_bwd`` then also returns
the adjoint of g, and torch autograd carries it on to x through the optimizee's Hessian-vector product (the gradient is
taken with ``create_graph=True``).  The trainers' default stays ``False`` (g a constant: the cheaper, first-order
meta-gradient) so that existing training runs keep their meta-gradients.

Where the arithmetic runs.  Everything that touches the N optimizee coordinates is CUDA in ``libl2o_b200.so``: the forward
step of the per-parameter level is the tensor-core kernel of the inference path (``l2o_hrnn_step_local``), its backward is
``l2o_hrnn_coord_bwd`` (csrc/hrnn_bwd.cuh).  The cross-coordinate pieces — per-tensor / global BiasGRU(20), the
1/RMS(delta) normalisation, the problem-wide mean log learning rate, the objective scaling — are ``[n_tensors x 20]``-sized
and are written as torch ops, so ``torch.autograd`` stitches the two CUDA entry points into the BPTT graph.  No CPU path.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional, Sequence

import torch

from . import _lib
from ._lib import HrnnArgs, HrnnBwdArgs
from .engine import _ptr, _stream
from .hierarchical_rnn import B0_STRIDE, N_SUMS, THETA_SPEC, HrnnHandle, _init_theta
from .scale_base import MetaTrainerBase, theta_views, train_optimizer  # noqa: F401  (train_optimizer: public name)

H0, H1, H2, NF, NS = 10, 20, 20, 12, 4
PLANES = 21
P_H, P_SCL, P_INP, P_LLR, P_ACC, P_MS = 0, 10, 11, 12, 13, 17


def _bias_gru(inputs, state, Wg, bg, Wc, bc, bias):
    """BiasGRUCell.__call__ (SC/optimizer/rnn_cells.py:46-68) on [rows, features] tensors."""
    n = state.shape[1]
    proj = torch.cat([inputs, state], 1) @ Wg + bg
    r = torch.sigmoid(proj[:, :n] + bias[:, :n])
    u = torch.sigmoid(proj[:, n:] + bias[:, n:2 * n])
    c = torch.tanh(torch.cat([inputs, r * state], 1) @ Wc + bc + bias[:, 2 * n:])
    return u * state + (1 - u) * c


class _Engine(HrnnHandle):
    """The handle and workspace of one optimizee (a list of tensor sizes); the coordinate kernels share the workspace
    regions with the torch-level pieces through the handle's views."""

    def __init__(self, sizes: Sequence[int], device):
        self.sizes = [int(s) for s in sizes]
        self.nt, self.N, self.device = len(self.sizes), int(sum(self.sizes)), device
        super().__init__(self.sizes, device)
        nt, N = self.nt, self.N
        self._dummy_x = torch.zeros(N, device=device)
        self._dummy_layer = torch.zeros(nt, H1, device=device)
        self._dummy_global = torch.zeros(H2, device=device)
        self.counts = torch.tensor(self.sizes, dtype=torch.float32, device=device)

    def coord_forward(self, theta, planes, bias0, mean_llr, g, zero_flag):
        state = planes.detach().clone()                      # the kernel updates the planes in place
        self.w_bias0.copy_(bias0.detach())
        self.w_mean.copy_(mean_llr.detach().reshape(1))
        self.w_zero.copy_(zero_flag)
        self.w_sums.zero_()
        self.w_any.zero_()
        a = HrnnArgs()
        a.theta = _ptr(theta.detach(), name="theta")
        a.x, a.g = _ptr(self._dummy_x, name="x"), _ptr(g, name="g")
        a.state = _ptr(state, name="state")
        a.layer, a.global_ = _ptr(self._dummy_layer, name="layer"), _ptr(self._dummy_global, name="global")
        a.workspace = self.ptr
        a.update = None
        _lib.check(_lib.lib().l2o_hrnn_step_local(self._h, C.byref(a), _stream()), "l2o_hrnn_step_local")
        return state, self.w_upd.clone(), self.w_sums.to(torch.float32), self.w_any.clone()

    def coord_backward(self, theta, planes_old, bias0, mean_llr, g, zero_flag, d_planes, d_upd, d_sums, want_dg=False):
        """Adjoints of (theta, old planes, bias0, mean log-lr) and, with ``want_dg``, of g (else None)."""
        dev = self.device
        d_old = torch.empty_like(planes_old)
        d_g = torch.empty(self.N, dtype=torch.float32, device=dev) if want_dg else None
        d_theta = torch.zeros(theta.numel(), dtype=torch.float64, device=dev)
        d_bias0 = torch.zeros(self.nt, B0_STRIDE, dtype=torch.float64, device=dev)
        d_mean = torch.zeros(1, dtype=torch.float64, device=dev)
        zf = zero_flag.to(torch.int32).contiguous()
        keep = [t.contiguous() for t in (theta.detach(), planes_old.detach(), g, bias0.detach(),
                                         mean_llr.detach().reshape(1), d_planes, d_upd, d_sums)]
        a = HrnnBwdArgs()
        a.theta, a.state_old, a.g, a.bias0 = (_ptr(keep[0], name="theta"), _ptr(keep[1], name="state_old"),
                                              _ptr(keep[2], name="g"), _ptr(keep[3], name="bias0"))
        a.zero_flag = zf.data_ptr()
        a.mean_log_lr = _ptr(keep[4], name="mean_log_lr")
        a.d_state_new, a.d_upd, a.d_sums = (_ptr(keep[5], name="d_state_new"), _ptr(keep[6], name="d_upd"),
                                            _ptr(keep[7], name="d_sums"))
        a.d_state_old = d_old.data_ptr()
        a.d_theta, a.d_bias0, a.d_mean_log_lr = d_theta.data_ptr(), d_bias0.data_ptr(), d_mean.data_ptr()
        a.d_g = None if d_g is None else d_g.data_ptr()
        _lib.check(_lib.lib().l2o_hrnn_coord_bwd(self._h, C.byref(a), _stream()), "l2o_hrnn_coord_bwd")
        return d_theta.to(torch.float32), d_old, d_bias0.to(torch.float32), d_mean.to(torch.float32), d_g


class _CoordStep(torch.autograd.Function):
    """The per-parameter level of one optimizer step as an autograd node around the two CUDA entry points.  The adjoint
    of g is computed only when autograd asks for it (g carries a graph: second-order meta-gradients)."""

    @staticmethod
    def forward(ctx, eng, theta, planes, bias0, mean_llr, g, zero_flag):
        new, upd, sums, any_nz = eng.coord_forward(theta, planes, bias0, mean_llr, g, zero_flag)
        ctx.eng = eng
        ctx.save_for_backward(theta, planes, bias0, mean_llr, g, zero_flag)
        ctx.mark_non_differentiable(any_nz)
        return new, upd, sums, any_nz

    @staticmethod
    def backward(ctx, d_planes, d_upd, d_sums, _d_any):
        theta, planes, bias0, mean_llr, g, zero_flag = ctx.saved_tensors
        eng = ctx.eng
        z = lambda t, like: torch.zeros_like(like) if t is None else t.contiguous()
        d_theta, d_old, d_bias0, d_mean, d_g = eng.coord_backward(
            theta, planes, bias0, mean_llr, g, zero_flag, z(d_planes, planes),
            z(d_upd, g), z(d_sums, torch.empty(eng.nt, N_SUMS, device=planes.device)), want_dg=ctx.needs_input_grad[5])
        return None, d_theta, d_old, d_bias0, d_mean.reshape(mean_llr.shape), d_g, None


class OptimizerState(object):
    """The optimizer's state between unrolls (all tensors detached): planes [21, N], layer [n_tensors, 20], global [1, 20]
    and the first-step flags of the mean-square accumulators."""

    def __init__(self, planes, layer, global_state, zero_flag, x):
        self.planes, self.layer, self.global_state, self.zero_flag, self.x = planes, layer, global_state, zero_flag, x


class MetaTrainer(MetaTrainerBase):
    """``TrainableOptimizer.train`` + the RMSProp block of ``metaopt.train_optimizer`` for the HierarchicalRNN.

    ``theta`` is the optimizer's flat weight vector (``HierarchicalRNN.theta`` layout).  ``use_second_derivatives``
    (default ``False``, the first-order meta-gradient): see ``MetaTrainerBase``."""
    what = "HierarchicalRNN"
    theta_spec = THETA_SPEC

    def __init__(self, shapes: Sequence[Sequence[int]], theta: Optional[torch.Tensor] = None, device="cuda:0",
                 learning_rate=1e-6, rms_decay=0.9, rms_epsilon=1e-20, gradient_clip=1e4, l2_reg=0.0,
                 use_log_objective=True, use_numerator_epsilon=False, init_lr_range=(1e-6, 1e-2), random_seed=None,
                 use_second_derivatives=False, **regularizer):
        super().__init__(shapes, _init_theta(random_seed) if theta is None else theta, device, learning_rate, rms_decay,
                         rms_epsilon, gradient_clip, l2_reg, use_log_objective, use_numerator_epsilon, init_lr_range,
                         random_seed, use_second_derivatives, **regularizer)
        self.engine = _Engine(self.sizes, self.device)

    # ---- state ---------------------------------------------------------------------------------------------------
    def initial_state(self, params: Sequence[torch.Tensor], theta: torch.Tensor,
                      log_learning_rate: Optional[torch.Tensor] = None):
        """_initialize_state / _initialize_global_state (HR:303-350); the learnable init vectors keep their graph."""
        eng, dev = self.engine, self.device
        P = theta_views(theta, THETA_SPEC)
        x = self._x0(params)
        if log_learning_rate is None:
            lo, hi = math.log(self.init_lr_range[0]) / 2.0, math.log(self.init_lr_range[1]) / 2.0
            parts = []
            for n in self.sizes:
                actual = torch.rand(n, generator=self._gen, dtype=torch.float64) * (hi - lo) + lo
                offset = torch.rand((), generator=self._gen, dtype=torch.float64) * (hi - lo) + lo
                parts.append(torch.clamp(actual + offset, -33.0, 33.0).float())
            log_learning_rate = torch.cat(parts)
        llr = log_learning_rate.to(dev).float().reshape(1, -1)
        h = P["Level0_RNN/init_vector"].reshape(H0, 1).expand(H0, eng.N)
        zeros = torch.zeros(1, eng.N, device=dev)
        planes = torch.cat([h, zeros, zeros, llr] + [zeros] * (2 * NS), 0)
        layer = P["Level1_RNN/init_vector"].reshape(1, H1).expand(eng.nt, H1)
        glob = P["Level2_RNN/init_vector"].reshape(1, H2)
        zero_flag = torch.ones(eng.nt, NS, dtype=torch.int32, device=dev)
        return OptimizerState(planes, layer, glob, zero_flag, x)

    # ---- one step ------------------------------------------------------------------------------------------------
    def _stepper(self, theta: torch.Tensor):
        """``loop_body`` (trainable_optimizer.py:263-401) without the objective: the CUDA per-parameter level, then the
        torch per-tensor and global levels.  The named views of theta are taken once per unroll, so that the backward
        sums each variable's adjoint over the unroll before it reaches theta."""
        eng, dev, cnt = self.engine, self.device, self.engine.counts
        P = theta_views(theta, THETA_SPEC)

        def step(state: OptimizerState, g: torch.Tensor):
            planes, layer, glob = state.planes, state.layer, state.global_state
            # per-tensor gate bias and the problem-wide mean log-lr of the PREVIOUS state (HR:561-575, 432-442)
            bias0 = (layer @ P["PerTensor/Layer0_RNN/Param/Affine/Matrix"] + P["PerTensor/Layer0_RNN/Param/Affine/Bias"]
                     + glob @ P["PerTensor/Layer0_RNN/Global/Affine/Matrix"] + P["PerTensor/Layer0_RNN/Global/Affine/Bias"])
            bias0 = torch.cat([bias0, torch.zeros(eng.nt, B0_STRIDE - 3 * H0, device=dev)], 1)
            mean_llr = planes[P_LLR].mean().reshape(1)
            planes, upd, sums, any_nz = _CoordStep.apply(eng, theta, planes, bias0, mean_llr, g, state.zero_flag)
            means = sums[:, :H0 + NF] / cnt[:, None]                        # mean_coords([h' | feat])  (HR:582-587)
            inv = torch.rsqrt(sums[:, H0 + NF] / cnt + 1e-16)               # 1 / RMS(delta)            (HR:621-626)
            # (per-tensor scalar broadcast as expand + cat: its backward is a handful of segment sums, where the
            # backward of inv[tensor_index] is a 354 K-way scatter-add into six numbers — 30 ms per step)
            inv_coord = torch.cat([inv[j:j + 1].expand(n) for j, n in enumerate(eng.sizes)])
            upd = upd * inv_coord                                           # HR:652-653, 404
            layer_bias = glob @ P["PerTensor/Layer1_RNN/Affine/Matrix"] + P["PerTensor/Layer1_RNN/Affine/Bias"]
            layer = _bias_gru(means, layer, P["PerTensor/Layer1_RNN/BiasGRUCell/gates/Affine/Matrix"],
                              P["PerTensor/Layer1_RNN/BiasGRUCell/gates/Affine/Bias"],
                              P["PerTensor/Layer1_RNN/BiasGRUCell/candidate/Affine/Matrix"],
                              P["PerTensor/Layer1_RNN/BiasGRUCell/candidate/Affine/Bias"], layer_bias.expand(eng.nt, -1))
            glob = _bias_gru(layer[-1:], glob, P["Layer2_RNN/BiasGRUCell/gates/Affine/Matrix"],   # LAST tensor only
                             P["Layer2_RNN/BiasGRUCell/gates/Affine/Bias"],                        # (HR:426-427)
                             P["Layer2_RNN/BiasGRUCell/candidate/Affine/Matrix"],
                             P["Layer2_RNN/BiasGRUCell/candidate/Affine/Bias"],
                             torch.zeros(1, 3 * H2, device=dev))
            return upd, OptimizerState(planes, layer, glob, (any_nz == 0).to(torch.int32), None)
        return step
