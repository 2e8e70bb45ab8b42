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
from typing import Callable, Dict, List, Optional, Sequence

import torch

from . import _lib
from ._lib import HrnnArgs, HrnnBwdArgs, L2OError
from .hierarchical_rnn import THETA_SPEC, _init_theta

H0, H1, H2, NF, NS = 10, 20, 20, 12, 4
PLANES = 21
P_H, P_SCL, P_INP, P_LLR, P_ACC, P_MS = 0, 10, 11, 12, 13, 17
B0_STRIDE, N_SUMS = 32, 24


def unpack_theta(theta: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Differentiable views of the flat theta (layout: hierarchical_rnn.theta_spec)."""
    out, off = {}, 0
    for name, shape in THETA_SPEC:
        n = int(math.prod(shape))
        out[name] = theta[off:off + n].reshape(shape)
        off += n
    return out


def _bias_gru(inputs, state, Wg, bg, Wc, bc, bias):
    """BiasGRUCell.__call__ (SC/optimizer/rnn_cells.py:46-68) on [rows, features] tensors."""
    n = state.shape[1]
    proj = torch.cat([inputs, state], 1) @ Wg + bg
    r = torch.sigmoid(proj[:, :n] + bias[:, :n])
    u = torch.sigmoid(proj[:, n:] + bias[:, n:2 * n])
    c = torch.tanh(torch.cat([inputs, r * state], 1) @ Wc + bc + bias[:, 2 * n:])
    return u * state + (1 - u) * c


class _Engine(object):
    """Owns the C handle and the workspace of one optimizee (a list of tensor sizes)."""

    def __init__(self, sizes: Sequence[int], device):
        self.sizes = [int(s) for s in sizes]
        self.nt, self.N, self.device = len(self.sizes), int(sum(self.sizes)), device
        L = _lib.lib()
        self._h = C.c_void_p()
        arr = (C.c_int64 * self.nt)(*self.sizes)
        _lib.check(L.l2o_hrnn_create(C.byref(self._h), arr, self.nt), "l2o_hrnn_create")
        nbytes = int(L.l2o_hrnn_workspace_bytes(self._h))
        self._ws = torch.zeros((nbytes + 255) // 4 + 64, dtype=torch.float32, device=device)
        self._ws_ptr = (self._ws.data_ptr() + 255) // 256 * 256
        base = self._ws_ptr - self._ws.data_ptr()
        off = (C.c_int64 * 7)()
        _lib.check(L.l2o_hrnn_workspace_layout(self._h, off), "l2o_hrnn_workspace_layout")
        raw = self._ws.view(torch.uint8)
        nt, N = self.nt, self.N
        self.w_sums = raw[base + off[0]:base + off[0] + 8 * nt * N_SUMS].view(torch.float64).view(nt, N_SUMS)
        self.w_any = raw[base + off[1]:base + off[1] + 4 * nt * NS].view(torch.int32).view(nt, NS)
        self.w_zero = raw[base + off[2]:base + off[2] + 4 * nt * NS].view(torch.int32).view(nt, NS)
        self.w_bias0 = raw[base + off[3]:base + off[3] + 4 * nt * B0_STRIDE].view(torch.float32).view(nt, B0_STRIDE)
        self.w_mean = raw[base + off[5]:base + off[5] + 4].view(torch.float32)
        self.w_upd = raw[base + off[6]:base + off[6] + 4 * N].view(torch.float32)
        self._dummy_x = torch.zeros(N, device=device)
        self._dummy_layer = torch.zeros(nt, H1, device=device)
        self._dummy_global = torch.zeros(H2, device=device)
        self.counts = torch.tensor(self.sizes, dtype=torch.float32, device=device)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                _lib.lib().l2o_hrnn_destroy(self._h)
                self._h = None
        except Exception:
            pass

    @staticmethod
    def _f32(t, name):
        if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
            raise L2OError("%s: expected a contiguous fp32 CUDA tensor (this engine has no CPU path)" % name)
        return t.data_ptr()

    def coord_forward(self, theta, planes, bias0, mean_llr, g, zero_flag):
        st = torch.cuda.current_stream().cuda_stream
        state = planes.detach().clone()                      # the kernel updates the planes in place
        self.w_bias0.copy_(bias0.detach())
        self.w_mean.copy_(mean_llr.detach().reshape(1))
        self.w_zero.copy_(zero_flag)
        self.w_sums.zero_()
        self.w_any.zero_()
        a = HrnnArgs()
        a.theta = self._f32(theta.detach(), "theta")
        a.x, a.g = self._f32(self._dummy_x, "x"), self._f32(g, "g")
        a.state = self._f32(state, "state")
        a.layer, a.global_ = self._f32(self._dummy_layer, "layer"), self._f32(self._dummy_global, "global")
        a.workspace = self._ws_ptr
        a.update = None
        _lib.check(_lib.lib().l2o_hrnn_step_local(self._h, C.byref(a), st), "l2o_hrnn_step_local")
        return state, self.w_upd.clone(), self.w_sums.to(torch.float32), self.w_any.clone()

    def coord_backward(self, theta, planes_old, bias0, mean_llr, g, zero_flag, d_planes, d_upd, d_sums, want_dg=False):
        """Adjoints of (theta, old planes, bias0, mean log-lr) and, with ``want_dg``, of g (else None)."""
        st = torch.cuda.current_stream().cuda_stream
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
        a.theta, a.state_old, a.g, a.bias0 = (self._f32(keep[0], "theta"), self._f32(keep[1], "state_old"),
                                              self._f32(keep[2], "g"), self._f32(keep[3], "bias0"))
        a.zero_flag = zf.data_ptr()
        a.mean_log_lr = self._f32(keep[4], "mean_log_lr")
        a.d_state_new, a.d_upd, a.d_sums = (self._f32(keep[5], "d_state_new"), self._f32(keep[6], "d_upd"),
                                            self._f32(keep[7], "d_sums"))
        a.d_state_old = d_old.data_ptr()
        a.d_theta, a.d_bias0, a.d_mean_log_lr = d_theta.data_ptr(), d_bias0.data_ptr(), d_mean.data_ptr()
        a.d_g = None if d_g is None else d_g.data_ptr()
        _lib.check(_lib.lib().l2o_hrnn_coord_bwd(self._h, C.byref(a), st), "l2o_hrnn_coord_bwd")
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


class MetaTrainerBase(object):
    """``TrainableOptimizer.train`` + the RMSProp block of ``metaopt.train_optimizer``, for any learned optimizer whose
    subclass provides ``initial_state(params, theta, lr_init)`` and ``unroll(objective, state, num_steps, theta=None,
    obj_weights=None, initial_obj=None)`` -> (meta objective with its graph, objective values, final state).

    ``theta`` is the optimizer's flat weight vector; it is updated in place by ``train_step``.  A state is any object
    whose tensor attributes carry the optimizer and optimizee state between unrolls."""

    def _setup(self, shapes, device):
        self.device = torch.device(device)
        self.shapes = [tuple(int(d) for d in s) for s in shapes]
        self.sizes = [int(math.prod(s)) if len(s) else 1 for s in self.shapes]

    def _setup_meta(self, theta, learning_rate, rms_decay, rms_epsilon, gradient_clip, l2_reg, use_log_objective,
                    use_numerator_epsilon, init_lr_range, random_seed, use_second_derivatives=False):
        self.theta = theta.to(self.device)
        self.theta.requires_grad_(True)
        self.learning_rate, self.rms_decay, self.rms_epsilon = learning_rate, rms_decay, rms_epsilon
        self.gradient_clip, self.l2_reg = gradient_clip, l2_reg
        self.use_log_objective, self.use_numerator_epsilon = use_log_objective, use_numerator_epsilon
        self.use_second_derivatives = bool(use_second_derivatives)
        self.init_lr_range = init_lr_range
        self.rms = torch.ones_like(self.theta)     # tf.train.RMSPropOptimizer initialises its accumulator to one
        self.global_step = 0
        self._gen = torch.Generator()
        if random_seed is not None:
            self._gen.manual_seed(int(random_seed))

    def _split(self, flat):
        out, off = [], 0
        for s, n in zip(self.shapes, self.sizes):
            out.append(flat[off:off + n].view(s))
            off += n
        return out

    def scale_objective(self, total_obj, all_objs, initial_obj, obj_scale_eps=1e-6):
        """trainable_optimizer.py:586-609."""
        if self.use_log_objective:
            if self.use_numerator_epsilon:
                return torch.log((all_objs + obj_scale_eps) / (initial_obj + obj_scale_eps)).mean()
            return torch.log(all_objs / (initial_obj + obj_scale_eps) + obj_scale_eps).mean()
        return total_obj / (initial_obj + obj_scale_eps)

    # ---- meta step -------------------------------------------------------------------------------------------------
    def meta_gradient(self, objective: Callable, params: Sequence[torch.Tensor], num_steps: int,
                      log_learning_rate: Optional[torch.Tensor] = None, state=None,
                      initial_obj: Optional[torch.Tensor] = None):
        """(meta objective, d meta / d theta, objective values, final state) of one unroll — from ``params`` with a fresh
        optimizer state, or continuing from ``state`` (a detached state: truncated BPTT over partial unrolls).
        ``log_learning_rate``: the initial learning-rate state handed to ``initial_state`` (drawn when None)."""
        if self.theta.grad is not None:
            self.theta.grad = None
        st = state if state is not None else self.initial_state(params, self.theta, log_learning_rate)
        meta, objs, final = self.unroll(objective, st, num_steps, initial_obj=initial_obj)
        loss = meta + self.l2_reg * (self.theta ** 2).sum() if self.l2_reg else meta
        # (a one-step unroll scores only f(x_0): constant, no meta-gradient)
        grad = torch.autograd.grad(loss, self.theta)[0] if loss.requires_grad else torch.zeros_like(self.theta)
        return meta.detach(), grad, [float(o.detach()) for o in objs], final

    def apply_meta_gradient(self, grad: torch.Tensor):
        """make_finite -> clip -> tf.train.RMSPropOptimizer(lr, decay, epsilon) (SC/metaopt.py:255-289)."""
        g = torch.where(torch.isfinite(grad), grad, torch.zeros_like(grad)).clamp(-self.gradient_clip, self.gradient_clip)
        with torch.no_grad():
            self.rms.mul_(self.rms_decay).addcmul_(g, g, value=1.0 - self.rms_decay)
            self.theta.sub_(self.learning_rate * g / torch.sqrt(self.rms + self.rms_epsilon))
        self.global_step += 1
        return g

    @staticmethod
    def detach_state(st):
        """The state handed from one partial unroll to the next is a constant of the next unroll's meta-gradient
        (``init_loop_vars_to_override`` assigned from ``final_loop_vals``, SC/metaopt.py:304,546-563)."""
        out = type(st).__new__(type(st))
        out.__dict__.update({k: v.detach() if torch.is_tensor(v) else v for k, v in vars(st).items()})
        return out

    def train_problem(self, objective: Callable, params: Sequence[torch.Tensor], num_unrolls: int, unroll_len: int,
                      log_learning_rate: Optional[torch.Tensor] = None, obj_train_max_multiplier: float = -1.0):
        """One training problem of ``metaopt.train_optimizer`` (SC/metaopt.py:458-613): ``num_unrolls`` partial unrolls of
        ``unroll_len`` steps, a clipped RMSProp meta-step after each, optimizer and optimizee state carried (detached)
        from unroll to unroll, objectives normalised by the first unroll's initial objective.  Stops early when the
        objective is no longer finite or (``obj_train_max_multiplier`` > 0) has grown past that multiple of the initial
        objective (the reference's loop_cond).  Returns (meta objectives, all objective values,
        final optimizee tensors)."""
        state, initial, metas, values = None, None, [], []
        for u in range(num_unrolls):
            meta, grad, objs, final = self.meta_gradient(objective, params, unroll_len, log_learning_rate, state=state,
                                                         initial_obj=initial)
            if not all(math.isfinite(o) for o in objs):
                break
            if initial is None:
                initial = torch.tensor(objs[0], device=self.device)
            if obj_train_max_multiplier > 0:   # loop_cond's third clause (trainable_optimizer.py:411-418): the run ends
                f0 = float(initial)            # once the objective has grown past a multiple of the initial one
                if max(objs) >= f0 + (obj_train_max_multiplier - 1.0) * abs(f0):
                    break
            self.apply_meta_gradient(grad)
            metas.append(float(meta))
            values.extend(objs)
            state = self.detach_state(final)
        out = self._split(state.x) if state is not None else [p.detach() for p in params]
        return metas, values, out

    def train_step(self, objective: Callable, params: Sequence[torch.Tensor], num_steps: int,
                   log_learning_rate: Optional[torch.Tensor] = None):
        meta, grad, objs, final = self.meta_gradient(objective, params, num_steps, log_learning_rate)
        self.apply_meta_gradient(grad)
        return float(meta), objs, self._split(final.x.detach())

    def _objective_and_gradient(self, objective: Callable, x: torch.Tensor):
        """f(x_t) and g_t = df/dx_t in one evaluation.  g_t is handed to the step detached (a constant of the
        meta-gradient) unless ``use_second_derivatives`` is on and x_t depends on theta; then it keeps its graph, so
        that the meta-gradient includes the optimizee's Hessian-vector product."""
        second = self.use_second_derivatives and x.requires_grad
        with torch.enable_grad():
            xg = x if x.requires_grad else x.detach().requires_grad_(True)
            obj = objective(self._split(xg))
            (g,) = torch.autograd.grad(obj, xg, retain_graph=x.requires_grad, create_graph=second)
        if not x.requires_grad:
            obj = obj.detach()
        return obj, (g if second else g.detach()).contiguous()


class MetaTrainer(MetaTrainerBase):
    """``TrainableOptimizer.train`` + the RMSProp block of ``metaopt.train_optimizer`` for the HierarchicalRNN.

    objective(list of tensors shaped like ``shapes``) -> scalar.  ``theta`` is the optimizer's flat weight vector
    (``HierarchicalRNN.theta`` layout); it is updated in place by ``train_step``.

    ``use_second_derivatives``: differentiate through the optimizee's gradients (the reference's
    ``TrainableOptimizer`` argument, default ``True`` there).  The default here is ``False``, the first-order
    meta-gradient this trainer has always computed; the second-order one keeps the optimizee's double-backward graph of
    every step of an unroll alive until the meta-gradient is taken.
    """

    def __init__(self, shapes: Sequence[Sequence[int]], theta: Optional[torch.Tensor] = None, device="cuda:0",
                 learning_rate=1e-6, rms_decay=0.9, rms_epsilon=1e-20, gradient_clip=1e4, l2_reg=0.0,
                 use_log_objective=True, use_numerator_epsilon=False, init_lr_range=(1e-6, 1e-2), random_seed=None,
                 use_second_derivatives=False):
        if not torch.cuda.is_available():
            raise L2OError("HierarchicalRNN meta-training needs a CUDA device (no CPU path)")
        self._setup(shapes, device)
        self.engine = _Engine(self.sizes, self.device)
        self._setup_meta(_init_theta(random_seed) if theta is None else theta.detach().clone().float(), learning_rate,
                         rms_decay, rms_epsilon, gradient_clip, l2_reg, use_log_objective, use_numerator_epsilon,
                         init_lr_range, random_seed, use_second_derivatives)

    # ---- state ---------------------------------------------------------------------------------------------------
    def initial_state(self, params: Sequence[torch.Tensor], theta: torch.Tensor,
                      log_learning_rate: Optional[torch.Tensor] = None):
        """_initialize_state / _initialize_global_state (HR:303-350); the learnable init vectors keep their graph."""
        eng, dev = self.engine, self.device
        P = unpack_theta(theta)
        x = torch.cat([p.detach().reshape(-1).float() for p in params]).to(dev)
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

    # ---- one unroll ------------------------------------------------------------------------------------------------
    def unroll(self, objective: Callable, state: OptimizerState, num_steps: int, theta: Optional[torch.Tensor] = None,
               obj_weights: Optional[Sequence[float]] = None, initial_obj: Optional[torch.Tensor] = None):
        """``loop_body`` x num_steps (trainable_optimizer.py:263-401).  Returns (meta objective with its graph, the list
        of objective values, the final OptimizerState with its graph)."""
        if num_steps < 1:
            raise ValueError("an unroll needs at least one step")
        theta = self.theta if theta is None else theta
        eng = self.engine
        P = unpack_theta(theta)
        planes, layer, glob, zero_flag, x = state.planes, state.layer, state.global_state, state.zero_flag, state.x
        cnt = eng.counts
        objs, total = [], 0.0
        w = [1.0] * num_steps if obj_weights is None else list(obj_weights)
        for t in range(num_steps):
            # objective at x_t and its gradient: a constant of the meta-gradient (stop_gradient,
            # trainable_optimizer.py:330-338) unless use_second_derivatives
            obj, g = self._objective_and_gradient(objective, x)
            objs.append(obj)
            total = total + w[t] * obj
            # per-tensor gate bias and the problem-wide mean log-lr of the PREVIOUS state (HR:561-575, 432-442)
            bias0 = (layer @ P["PerTensor/Layer0_RNN/Param/Affine/Matrix"] + P["PerTensor/Layer0_RNN/Param/Affine/Bias"]
                     + glob @ P["PerTensor/Layer0_RNN/Global/Affine/Matrix"] + P["PerTensor/Layer0_RNN/Global/Affine/Bias"])
            bias0 = torch.cat([bias0, torch.zeros(eng.nt, B0_STRIDE - 3 * H0, device=self.device)], 1)
            mean_llr = planes[P_LLR].mean().reshape(1)
            planes, upd, sums, any_nz = _CoordStep.apply(eng, theta, planes, bias0, mean_llr, g, zero_flag)
            means = sums[:, :H0 + NF] / cnt[:, None]                        # mean_coords([h' | feat])  (HR:582-587)
            inv = torch.rsqrt(sums[:, H0 + NF] / cnt + 1e-16)               # 1 / RMS(delta)            (HR:621-626)
            # (per-tensor scalar broadcast as expand + cat: its backward is a handful of segment sums, where the backward
            # of inv[tensor_index] is a 354 K-way scatter-add into six numbers — 30 ms per step)
            inv_coord = torch.cat([inv[j:j + 1].expand(n) for j, n in enumerate(eng.sizes)])
            x = x - upd * inv_coord                                         # HR:652-653, 404
            layer_bias = glob @ P["PerTensor/Layer1_RNN/Affine/Matrix"] + P["PerTensor/Layer1_RNN/Affine/Bias"]
            layer = _bias_gru(means, layer, P["PerTensor/Layer1_RNN/BiasGRUCell/gates/Affine/Matrix"],
                              P["PerTensor/Layer1_RNN/BiasGRUCell/gates/Affine/Bias"],
                              P["PerTensor/Layer1_RNN/BiasGRUCell/candidate/Affine/Matrix"],
                              P["PerTensor/Layer1_RNN/BiasGRUCell/candidate/Affine/Bias"], layer_bias.expand(eng.nt, -1))
            glob = _bias_gru(layer[-1:], glob, P["Layer2_RNN/BiasGRUCell/gates/Affine/Matrix"],   # LAST tensor only
                             P["Layer2_RNN/BiasGRUCell/gates/Affine/Bias"],                        # (HR:426-427)
                             P["Layer2_RNN/BiasGRUCell/candidate/Affine/Matrix"],
                             P["Layer2_RNN/BiasGRUCell/candidate/Affine/Bias"],
                             torch.zeros(1, 3 * H2, device=self.device))
            zero_flag = (any_nz == 0).to(torch.int32)
        # normalised by the objective at the start of the SERIES of partial unrolls (trainable_optimizer.py:438-441)
        initial = objs[0].detach() if initial_obj is None else initial_obj
        meta = self.scale_objective(total, torch.stack([o.reshape(()) for o in objs]), initial)
        return meta, objs, OptimizerState(planes, layer, glob, zero_flag, x)


def train_optimizer(make_trainer: Callable, problems: Sequence, num_problems: int, num_meta_iterations: int,
                    num_unroll_func: Callable[[], int], num_partial_unroll_itrs_func: Callable[[], int],
                    select_random_problems: bool = True, callbacks: Optional[Sequence[Callable]] = None,
                    fix_unroll: bool = False, fix_unroll_length: int = 20, fix_num_steps: int = 100, seed: int = 0,
                    out=None):
    """The sampling loop of ``metaopt.train_optimizer`` (SC/metaopt.py:117-613) around ``MetaTrainer``: ``num_problems``
    draws of a training problem; on each, ``num_meta_iterations`` optimizee runs, every run a series of partial unrolls
    (``num_unroll_func()`` unrolls of ``num_partial_unroll_itrs_func()`` steps, or ``fix_num_steps // fix_unroll_length``
    unrolls of ``fix_unroll_length`` steps with ``fix_unroll``) with a clipped RMSProp meta-step after each unroll.

    problems: sequence of ``(objective, init_fn)`` — ``objective(list of tensors) -> scalar``, ``init_fn() -> list of
    tensors`` (fresh optimizee parameters for a run).  make_trainer(shapes, theta) -> MetaTrainer (or anything with
    ``theta`` and ``train_problem``); one trainer per problem shape, theta handed on from problem to problem.
    Returns (theta, log of (problem index, meta objectives)).  The curriculum / evaluation / checkpoint bookkeeping of the
    reference driver (SC/metaopt.py:172-176, 613-700) is host-side policy and stays with the caller."""
    import random
    rng = random.Random(seed)
    theta, rms, log, trainers = None, None, [], {}
    for draw in range(num_problems):
        k = rng.randrange(len(problems)) if select_random_problems else draw % len(problems)
        objective, init_fn = problems[k]
        shapes = tuple(tuple(p.shape) for p in init_fn())
        if shapes not in trainers:
            trainers[shapes] = make_trainer(shapes, theta)
        tr = trainers[shapes]
        if theta is not None and tr.theta is not theta:   # one set of meta-parameters and one RMSProp accumulator
            with torch.no_grad():                         # across all problems (SC/metaopt.py:255-260)
                tr.theta.copy_(theta)
                if rms is not None and getattr(tr, "rms", None) is not None:
                    tr.rms.copy_(rms)
        for _ in range(num_meta_iterations):
            if fix_unroll:
                lens = [fix_unroll_length] * (fix_num_steps // fix_unroll_length)
            else:
                lens = [num_partial_unroll_itrs_func() for _ in range(num_unroll_func())]
            params = init_fn()
            # the reference feeds one unroll length per partial unroll; equal lengths go through train_problem directly
            if len(set(lens)) <= 1:
                metas, _, _ = tr.train_problem(objective, params, len(lens), lens[0] if lens else 0)
            else:
                metas, state, initial = [], None, None
                for ln in lens:
                    meta, grad, objs, final = tr.meta_gradient(objective, params, ln, state=state, initial_obj=initial)
                    if not all(math.isfinite(o) for o in objs):
                        break
                    tr.apply_meta_gradient(grad)
                    metas.append(float(meta))
                    initial = torch.tensor(objs[0], device=tr.device) if initial is None else initial
                    state = tr.detach_state(final)
            log.append((k, metas))
            if out is not None:
                print("problem %d: %d unrolls, meta objective %s" % (k, len(metas), ["%.4f" % m for m in metas]), file=out)
        theta, rms = tr.theta, getattr(tr, "rms", None)
        for cb in callbacks or ():
            cb(draw, k, tr)
    return theta, log

