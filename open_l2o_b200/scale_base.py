"""What the five L2O-Scale optimizers (``HierarchicalRNN``, ``CoordinatewiseRNN``, ``TrainableAdam``,
``LearningRateSchedule``, ``GlobalLearningRate``) and their meta-trainers share.

``ScaleOptimizer`` is the ``tf.train.Optimizer`` surface over one flat optimizee arena: named views of the flat weight
vector ``theta``, slot creation, ``apply_gradients``, graph-replayed ``minimize``, ``meta_trainer`` / ``adopt``.
``MetaTrainerBase`` is ``TrainableOptimizer.train`` (SC/optimizer/trainable_optimizer.py:200-470; SC/ =
Model_Free_L2O/L2O-Scale/L2O-Scale-Training/) with the RMSProp block of ``metaopt.train_optimizer``
(SC/metaopt.py:255-289), and ``train_optimizer`` is that driver's problem-sampling loop.
"""
from __future__ import annotations

import ctypes as C
import importlib
import math
import os
from typing import Callable, Dict, Iterable, List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import L2OError
from .engine import _ptr, _stream
from .scale_reg import Regularizer, check_options, reg_switch


def theta_views(theta: torch.Tensor, spec: Sequence[Tuple[str, Tuple[int, ...]]]) -> Dict[str, torch.Tensor]:
    """Views of the flat ``theta`` by name, in the layout of ``spec`` ((name, shape) in order); differentiable."""
    out, off = {}, 0
    for name, shape in spec:
        n = int(math.prod(shape))
        out[name] = theta[off:off + n].view(shape)
        off += n
    return out


def planes_step(launch: Callable, args_cls, entry: str):
    """The autograd Function of one coordinate-wise optimizer step over all coordinates: (theta, planes [P, N], g) ->
    (planes', update).  Forward: ``launch(theta, g, state_in, state_out, update=)``; backward: the C entry point
    ``entry`` with an ``args_cls`` (n, theta, g, state_old, d_state_new, d_update, d_state_old, d_theta, d_g).  The
    adjoint of g is computed only when autograd asks for it (second-order meta-gradients)."""

    class Step(torch.autograd.Function):
        @staticmethod
        def forward(ctx, theta, planes, g):
            theta, planes = theta.detach().contiguous(), planes.detach().contiguous()
            new, upd = torch.empty_like(planes), torch.empty_like(g)
            launch(theta, g, planes, new, update=upd)
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
            a = args_cls()
            a.n = int(g.numel())
            a.theta, a.g, a.state_old = _ptr(theta), _ptr(g), _ptr(planes)
            a.d_state_new, a.d_update, a.d_state_old = _ptr(d_new), _ptr(d_upd), _ptr(d_old)
            a.d_theta, a.d_g = d_theta.data_ptr(), _ptr(d_g)
            _lib.check(getattr(_lib.lib(), entry)(C.byref(a), _stream()), entry)
            return d_theta.to(torch.float32), d_old, d_g

    return Step


class ScaleOptimizer(object):
    """The optimizer surface the five L2O-Scale optimizers share.  A subclass sets ``theta_spec`` and ``trainer`` (the
    meta-trainer class as "module.Class" of this package) and provides the slot state (``_new_state``,
    ``reset_state``, ``get_slot``) and ``step_flat``, the step over the flat arena."""
    theta_spec: List[Tuple[str, Tuple[int, ...]]]
    trainer = ""
    init_lr_range = None     # handed on to the meta-trainer by the optimizers that draw initial learning rates
    kernels_per_step = 1     # library kernels of one step_flat (the count of a replayed CUDA graph)
    distributed = False      # sharded: this process steps a slice of every tensor's coordinates (HierarchicalRNN)

    def __init__(self, theta: torch.Tensor, device):
        self.device = torch.device(device)
        self.theta = theta.to(self.device)
        self.state = None
        self._vars: List[torch.Tensor] = []

    # ---- variables (the TF variable collection of OPTIMIZER_SCOPE) ---------------------------------------------------
    def get_variables(self) -> Dict[str, torch.Tensor]:
        return theta_views(self.theta, self.theta_spec)

    def load_variables(self, values: Dict[str, torch.Tensor]):
        for name, view in self.get_variables().items():
            if name in values:
                view.copy_(torch.as_tensor(values[name], dtype=torch.float32).reshape(view.shape))
        if self.state is not None:
            self._prepare()

    def _prepare(self):
        """Recompute what the slots derive from theta; called after every change of theta once the slots exist."""

    # ---- meta-training ---------------------------------------------------------------------------------------------
    def meta_trainer(self, var_list: Sequence[torch.Tensor], **kwargs):
        """The meta-trainer for optimizees shaped like ``var_list`` that starts from this optimizer's weights
        (``TrainableOptimizer.train``).  ``adopt(trainer)`` copies the trained weights back."""
        if self.init_lr_range is not None:
            kwargs.setdefault("init_lr_range", self.init_lr_range)
        module, cls = self.trainer.rsplit(".", 1)   # the trainer modules import the optimizer modules
        cls = getattr(importlib.import_module("." + module, __package__), cls)
        tr = cls([tuple(v.shape) for v in var_list], theta=self.theta, device=str(self.device), **kwargs)
        tr.theta_spec = self.theta_spec      # checkpoints of the trainer carry this optimizer's variable names
        return tr

    def adopt(self, trainer):
        self.theta.copy_(trainer.theta.detach())
        if self.state is not None:
            self._prepare()

    # ---- slots ---------------------------------------------------------------------------------------------------------
    def _shard_ranges(self, sizes: Sequence[int]) -> List[Tuple[int, int]]:
        """The (lo, hi) coordinates of each optimizee tensor that this process steps."""
        return [(0, n) for n in sizes]

    def _create_slots(self, var_list: Sequence[torch.Tensor]):
        """One slot set per optimizee tensor (trainable_optimizer.py:94-105) over the concatenation of all tensors (the
        coordinates ``_shard_ranges`` gives this process).  Unsharded, the optimizee tensors become views of the flat
        arena ``x``, so that flattening them for the step and back is free."""
        gsizes = [int(v.numel()) for v in var_list]
        if any(s <= 0 for s in gsizes):
            raise ValueError("empty optimizee variable")
        self.global_sizes = gsizes
        self._ranges = self._shard_ranges(gsizes)
        self.sizes = [hi - lo for lo, hi in self._ranges]
        self.N = sum(self.sizes)
        if self.N <= 0:
            raise ValueError("this rank holds no coordinate (more ranks than coordinates)")
        self.x = torch.empty(self.N, device=self.device)
        self.g = torch.empty(self.N, device=self.device)
        off = 0
        for v, (lo, hi) in zip(var_list, self._ranges):
            n = hi - lo
            self.x[off:off + n].copy_(v.detach().reshape(-1)[lo:hi])
            if not self.distributed:
                v.data = self.x[off:off + n].view(v.shape)
            off += n
        self._vars = list(var_list)
        self.state = self._new_state()
        self.reset_state()

    def _new_state(self):
        """The state buffers over the arena; ``reset_state`` initialises them."""
        raise NotImplementedError

    def reset_state(self):
        """_initialize_state: the optimizer's state as before its first step (zeros unless a subclass draws it).  In
        place: a CUDA graph that ``minimize`` captured keeps the state buffer's address."""
        if self.state is not None:
            self.state.zero_()

    # ---- the step --------------------------------------------------------------------------------------------------------
    def apply_gradients(self, grads_and_vars: Iterable[Tuple[torch.Tensor, torch.Tensor]], global_step=None, name=None):
        """tf.train.Optimizer.apply_gradients: one step over all (grad, var) pairs.  Variables are updated in place;
        returns the list of updated variables ("real_params")."""
        grads_and_vars = tuple(grads_and_vars)
        for g, v in grads_and_vars:
            if g is not None and not torch.is_tensor(g):
                raise TypeError("Gradient must be a Tensor or None: %s" % (g,))
            if not torch.is_tensor(v):
                raise TypeError("Variable must be a Tensor: %s" % (v,))
        pairs = [(g, v) for g, v in grads_and_vars if g is not None]
        if not pairs:
            raise ValueError("No gradients provided for any variable: %s" % (grads_and_vars,))
        if self.state is None:
            self._create_slots([v for _, v in pairs])
        elif len(pairs) != len(self._vars) or any(v is not w for (_, v), w in zip(pairs, self._vars)):
            raise ValueError("apply_gradients must be called with the variables the slots were created for")
        off = 0
        for (g, _), (lo, hi) in zip(pairs, self._ranges):
            self.g[off:off + hi - lo].copy_(g.reshape(-1)[lo:hi])
            off += hi - lo
        self.step_flat()
        return [v for _, v in pairs]

    def step_flat(self):
        """One step with the gradients already in ``self.g`` (flat arena order); state and ``x`` updated in place."""
        raise NotImplementedError

    def minimize(self, objective, var_list: Sequence[torch.Tensor], num_steps: int, cuda_graph: Optional[bool] = None):
        """Convenience loop of the evaluation drivers (SC/metatest.py): num_steps x (objective, gradients, step).
        Returns the list of objective values (one device->host read at the end).

        One iteration is tens of tiny launches (the optimizee's forward/backward, the gradient copies, the step kernels)
        and nothing in it needs the host, so after two eager iterations (slot creation, library warm-up) one iteration
        is captured into a CUDA graph and replayed (``cuda_graph=False`` or ``L2O_CUDA_GRAPH=0`` keeps everything
        eager; a failed capture falls back to the same eager kernels with a warning).  A sharded optimizer stays eager:
        its per-step collectives are not captured."""
        from . import engine as _engine
        var_list = list(var_list)

        def body():
            loss = objective(*var_list)
            grads = torch.autograd.grad(loss, var_list)
            self.apply_gradients(zip(grads, var_list))
            return loss.detach()

        if cuda_graph is None:
            cuda_graph = os.environ.get("L2O_CUDA_GRAPH", "1") != "0"
        if self.distributed:
            cuda_graph = False
        return _engine.replay_loop(self, body, objective, var_list, num_steps, cuda_graph, self.kernels_per_step,
                                   type(self).__name__)


class MetaTrainerBase(object):
    """``TrainableOptimizer.train`` + the RMSProp block of ``metaopt.train_optimizer``, for any learned optimizer whose
    subclass provides ``initial_state(params, theta, lr_init)`` and ``_stepper(theta)``.

    objective(list of tensors shaped like ``shapes``) -> scalar.  ``theta`` is the optimizer's flat weight vector; it is
    updated in place by ``train_step``.  A state is any object whose tensor attributes carry the optimizer and
    optimizee state between unrolls, the optimizee coordinates as ``x``.

    ``use_second_derivatives``: differentiate through the optimizee's gradients (the reference's
    ``TrainableOptimizer`` argument, default ``True`` there).  The trainers' default is ``False``, the first-order
    meta-gradient; the second-order one keeps the optimizee's double-backward graph of every step of an unroll alive
    until the meta-gradient is taken.

    The regularisers (``scale_reg``; all off by default, and off the trainer runs the plain loop):
    ``reg_optimizee`` hands the optimizer the noise-free g~_t = d(f_t + beta reg_t)/dx_t instead of g_t (also in
    ``evaluate``); ``reg_optimizer`` adds alpha sum_t reg_t to the scaled meta objective of the partial unrolls that
    ``regularize_time`` / ``reg_scale`` switch on (``scale_reg.reg_switch``).  reg_t is ``reg_option`` at x_t with its
    graph to x_t; imitation unrolls have no regulariser term."""
    what = ""
    theta_spec = None     # (name, shape) layout of theta for get_variables; None: one flat "theta"
    regularizer = None    # a scale_reg.Regularizer when reg_optimizer or reg_optimizee is on

    def __init__(self, shapes, theta, device, learning_rate, rms_decay, rms_epsilon, gradient_clip, l2_reg,
                 use_log_objective, use_numerator_epsilon, init_lr_range, random_seed, use_second_derivatives,
                 reg_optimizer=False, reg_optimizee=False, reg_option="hessian", hessian_itrs=10, alpha=5e-4,
                 beta=1e-4, regularize_time="posterior", reg_scale=0.5):
        check_options(reg_option, reg_optimizee, use_second_derivatives)
        if not torch.cuda.is_available():
            raise L2OError("%s meta-training needs a CUDA device (no CPU path)" % self.what)
        self.device = torch.device(device)
        self.shapes = [tuple(int(d) for d in s) for s in shapes]
        self.sizes = [int(math.prod(s)) if len(s) else 1 for s in self.shapes]
        self.theta = theta.detach().clone().float().to(self.device)
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
        self.reg_optimizer, self.reg_optimizee = bool(reg_optimizer), bool(reg_optimizee)
        self.alpha, self.beta, self.regularize_time, self.reg_scale = alpha, beta, regularize_time, reg_scale
        self.regularizer = Regularizer(reg_option, hessian_itrs, random_seed) \
            if self.reg_optimizer or self.reg_optimizee else None

    def _split(self, flat):
        out, off = [], 0
        for s, n in zip(self.shapes, self.sizes):
            out.append(flat[off:off + n].view(s))
            off += n
        return out

    def _x0(self, params):
        return torch.cat([p.detach().reshape(-1).float() for p in params]).to(self.device)

    def scale_objective(self, total_obj, all_objs, initial_obj, obj_scale_eps=1e-6):
        """trainable_optimizer.py:586-609."""
        if self.use_log_objective:
            if self.use_numerator_epsilon:
                return torch.log((all_objs + obj_scale_eps) / (initial_obj + obj_scale_eps)).mean()
            return torch.log(all_objs / (initial_obj + obj_scale_eps) + obj_scale_eps).mean()
        return total_obj / (initial_obj + obj_scale_eps)

    # ---- one unroll ------------------------------------------------------------------------------------------------
    def _stepper(self, theta: torch.Tensor):
        """``step(state, g) -> (update, state after the step without x)``: one optimizer step.  What depends on theta
        alone is computed here, once per unroll."""
        raise NotImplementedError

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

    def _regularized_objective_and_gradient(self, objective: Callable, x: torch.Tensor):
        """``_objective_and_gradient`` with the regulariser: (f(x_t), g, reg_t).  g is g~_t = d(f + beta reg)/dx_t
        from the noise-free objective under ``reg_optimizee``, else the objective's own gradient; reg_t keeps its graph
        to x_t when x_t depends on theta."""
        second = self.use_second_derivatives and x.requires_grad
        with torch.enable_grad():
            xg = x if x.requires_grad else x.detach().requires_grad_(True)
            obj = (getattr(objective, "clean", objective) if self.reg_optimizee else objective)(self._split(xg))
            reg = self.regularizer(objective, xg, self._split, self._gen)
            target = obj + self.beta * reg if self.reg_optimizee else obj
            (g,) = torch.autograd.grad(target, xg, retain_graph=x.requires_grad, create_graph=second)
        if not x.requires_grad:
            obj, reg = obj.detach(), reg.detach()
        return obj, (g if second else g.detach()).contiguous(), reg

    def unroll(self, objective: Callable, state, num_steps: int, theta: Optional[torch.Tensor] = None,
               obj_weights: Optional[Sequence[float]] = None, initial_obj: Optional[torch.Tensor] = None,
               labels: Optional[torch.Tensor] = None, grads: Optional[torch.Tensor] = None, regularize: bool = False):
        """``loop_body`` x num_steps (trainable_optimizer.py:263-401).  Returns (meta objective with its graph, the list
        of objective values, the final state with its graph).

        With ``labels`` ([num_steps, N], a teacher's positive steps) the unroll imitates (``mode_mt``): x is
        teacher-forced, ``x_{t+1} = x_t - labels[t]`` (hierarchical_rnn.py:398-404), while the optimizer's own update
        still drives its state, and the meta objective is ``sum_t w_t sum_i (upd_t,i - labels_t,i)^2 / 2 / N`` with
        ``w_t = 1 / num_steps`` by default (trainable_optimizer.py:383-389, SC/metaopt.py:407-408).  ``grads``
        ([num_steps, N]) are the optimizee gradients at the teacher-forced points, recorded by ``teacher_labels``: given,
        the unroll replays them and evaluates no objective; None, it evaluates ``objective`` at each forced point.

        ``regularize``: this unroll adds alpha sum_t reg_t to its meta objective (with ``reg_optimizer``)."""
        if num_steps < 1:
            raise ValueError("an unroll needs at least one step")
        step = self._stepper(self.theta if theta is None else theta)
        x = state.x
        objs, total, reg_total = [], 0.0, 0.0
        regular = self.regularizer is not None and labels is None
        if obj_weights is not None:
            w = list(obj_weights)
        else:
            w = [1.0] * num_steps if labels is None else [1.0 / num_steps] * num_steps
        for t in range(num_steps):
            if grads is None:
                # objective at x_t and its gradient: a constant of the meta-gradient (stop_gradient,
                # trainable_optimizer.py:330-338) unless use_second_derivatives
                if regular:
                    obj, g, reg = self._regularized_objective_and_gradient(objective, x)
                    reg_total = reg_total + reg
                else:
                    obj, g = self._objective_and_gradient(objective, x)
                objs.append(obj)
            else:
                g = grads[t]
            upd, state = step(state, g)
            if labels is None:
                total = total + w[t] * obj
                x = x - upd
            else:
                d = upd - labels[t]
                total = total + (w[t] * 0.5 / d.numel()) * (d * d).sum()
                x = x - labels[t]
        state.x = x
        if labels is not None:
            return total, objs, state
        # normalised by the objective at the start of the SERIES of partial unrolls (trainable_optimizer.py:438-441)
        initial = objs[0].detach() if initial_obj is None else initial_obj
        meta = self.scale_objective(total, torch.stack([o.reshape(()) for o in objs]), initial)
        if regular and regularize and self.reg_optimizer:   # added after scaling (trainable_optimizer.py:439-446)
            meta = meta + self.alpha * reg_total
        return meta, objs, state

    # ---- meta step -------------------------------------------------------------------------------------------------
    def meta_gradient(self, objective: Callable, params: Sequence[torch.Tensor], num_steps: int,
                      log_learning_rate: Optional[torch.Tensor] = None, state=None,
                      initial_obj: Optional[torch.Tensor] = None, regularize: Optional[bool] = None):
        """(meta objective, d meta / d theta, objective values, final state) of one unroll — from ``params`` with a fresh
        optimizer state, or continuing from ``state`` (a detached state: truncated BPTT over partial unrolls).
        ``log_learning_rate``: the initial learning-rate state handed to ``initial_state`` (drawn when None).
        ``regularize``: whether the regulariser term is on for this unroll; None: ``regularize_time``'s rule for a
        run of one unroll."""
        if self.regularizer is None:
            return self._meta_gradient(objective, params, num_steps, log_learning_rate, state, initial_obj=initial_obj)
        if regularize is None:
            regularize = reg_switch(self.regularize_time, 0, 1, self.reg_scale)
        return self._meta_gradient(objective, params, num_steps, log_learning_rate, state, initial_obj=initial_obj,
                                   regularize=regularize)

    def meta_gradient_mt(self, objective: Optional[Callable], params: Sequence[torch.Tensor], labels: torch.Tensor,
                         grads: Optional[torch.Tensor], log_learning_rate: Optional[torch.Tensor] = None, state=None):
        """``meta_gradient`` of one imitation unroll (``metaobjmt``): ``labels.shape[0]`` steps with x teacher-forced
        along ``labels`` and the meta objective the weighted mean-square distance of the optimizer's updates from them
        (``unroll``).  Returns (meta objective, d meta / d theta, objective values, final state).

        Replay, not re-evaluation: on a teacher-forced run x_t is a point where the teacher took its gradient, so the
        unroll consumes the gradient rows ``grads`` that ``teacher_labels`` recorded there and evaluates no objective
        (the objective values are then an empty list; ``objective`` may be None).  ``grads=None`` evaluates
        ``objective`` at the forced points instead.  Either way the gradients are constants of the meta-gradient, also
        under ``use_second_derivatives``: x_t does not depend on theta."""
        return self._meta_gradient(objective, params, int(labels.shape[0]), log_learning_rate, state, labels=labels,
                                   grads=grads)

    def _meta_gradient(self, objective, params, num_steps, log_learning_rate, state, **unroll_kwargs):
        if self.theta.grad is not None:
            self.theta.grad = None
        st = state if state is not None else self.initial_state(params, self.theta, log_learning_rate)
        meta, objs, final = self.unroll(objective, st, num_steps, **unroll_kwargs)
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
        return self._train_unrolls(objective, params, [unroll_len] * num_unrolls, log_learning_rate,
                                   obj_train_max_multiplier)

    def _train_unrolls(self, objective, params, unroll_lens, log_learning_rate=None, obj_train_max_multiplier=-1.0):
        """``train_problem`` with one length per partial unroll."""
        state, initial, metas, values = None, None, [], []
        for i, ln in enumerate(unroll_lens):
            kw = {} if self.regularizer is None else \
                dict(regularize=reg_switch(self.regularize_time, i, len(unroll_lens), self.reg_scale))
            meta, grad, objs, final = self.meta_gradient(objective, params, ln, log_learning_rate, state=state,
                                                         initial_obj=initial, **kw)
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

    def train_problem_mt(self, objective: Optional[Callable], params: Sequence[torch.Tensor], labels: torch.Tensor,
                         grads: Optional[torch.Tensor], unroll_lens: Sequence[int],
                         log_learning_rate: Optional[torch.Tensor] = None):
        """One imitation run (SC/metaopt.py:541-548): the partial unrolls of ``unroll_lens`` over consecutive rows of
        ``labels`` / ``grads`` (``teacher_labels`` of the whole run), each ``meta_gradient_mt`` followed by the clipped
        RMSProp meta-step on the same accumulator, optimizer state carried (detached) from unroll to unroll.  Returns
        (meta objectives, final optimizee tensors)."""
        unroll_lens = [int(n) for n in unroll_lens]
        if sum(unroll_lens) != labels.shape[0] or (grads is not None and grads.shape[0] != labels.shape[0]):
            raise ValueError("labels / grads must have one row per step of the run (%d)" % sum(unroll_lens))
        state, metas, off = None, [], 0
        for ln in unroll_lens:
            rows = slice(off, off + ln)
            meta, grad, _, final = self.meta_gradient_mt(objective, params, labels[rows],
                                                         None if grads is None else grads[rows], log_learning_rate,
                                                         state=state)
            self.apply_meta_gradient(grad)
            metas.append(float(meta))
            state = self.detach_state(final)
            off += ln
        out = self._split(state.x) if state is not None else [p.detach() for p in params]
        return metas, out

    def evaluate(self, objective: Callable, params: Sequence[torch.Tensor], unroll_lens: Sequence[int]) -> float:
        """``validate`` (SC/metaopt.py:741-780): a run of partial unrolls from ``params`` with a fresh optimizer state,
        state carried from unroll to unroll, no meta-gradient and no meta-step.  Returns the objective at the run's
        last step."""
        if not unroll_lens:
            raise ValueError("an evaluation run needs at least one unroll")
        theta = self.theta.detach()
        with torch.no_grad():
            state = self.initial_state(params, theta, None)
            for ln in unroll_lens:
                _, objs, state = self.unroll(objective, state, int(ln), theta=theta)
        return float(objs[-1])

    def get_variables(self) -> Dict[str, torch.Tensor]:
        """Named copies of theta (``ScaleOptimizer.get_variables`` names when ``theta_spec`` is known), for checkpoints
        that ``ScaleOptimizer.load_variables`` and ``load_variables`` read back."""
        return {k: v.clone() for k, v in theta_views(self.theta.detach().cpu(), self._spec()).items()}

    def load_variables(self, values: Dict[str, torch.Tensor]):
        spec = self._spec()
        with torch.no_grad():
            for name, view in theta_views(self.theta, spec).items():
                view.copy_(torch.as_tensor(values[name], dtype=torch.float32).reshape(view.shape))

    def _spec(self):
        return self.theta_spec or [("theta", (self.theta.numel(),))]

    def train_step(self, objective: Callable, params: Sequence[torch.Tensor], num_steps: int,
                   log_learning_rate: Optional[torch.Tensor] = None):
        meta, grad, objs, final = self.meta_gradient(objective, params, num_steps, log_learning_rate)
        self.apply_meta_gradient(grad)
        return float(meta), objs, self._split(final.x.detach())


def teacher_labels(objective: Callable, x0: torch.Tensor, sizes: Sequence, lens: Sequence[int], name: str = "adam",
                   k: int = 1):
    """The imitation targets of one run (``mt_utils.get_mt_labels``, SC/mt_utils.py:55-92): a teacher (``name``:
    "adam", "rmsprop" or "nag", the TF-1.14 rules with lr 0.01 and fresh slots, ``data_generator.teacher_update``)
    starts at the flat coordinates ``x0`` and takes ``k`` steps per label.  ``sizes``: the optimizee tensors' shapes
    (an int is a 1-D tensor), for ``objective(list of tensors) -> scalar``; ``lens``: the run's partial-unroll
    lengths.

    Returns ``(labels, grads)``, both ``[sum(lens), N]`` in run order.  ``labels[t] = x_prev - x_cur`` over the t-th
    group of ``k`` steps (the positive step: ``x - labels[t]`` is the teacher's next point); ``grads[t]`` is the
    gradient at the group's first point, the point a teacher-forced unroll visits at step t.  After each group the
    teacher continues from ``x_prev - labels[t]``, which is what teacher forcing computes, so those points are
    bitwise the ones ``MetaTrainerBase.meta_gradient_mt`` replays.  Both live on x0's device: 8 N bytes per step."""
    from .data_generator import teacher_state, teacher_update
    if k < 1:
        raise ValueError("mt_k must be >= 1")
    shapes = [tuple(int(d) for d in s) if isinstance(s, (tuple, list, torch.Size)) else (int(s),) for s in sizes]
    counts = [int(math.prod(s)) for s in shapes]
    x = x0.detach().reshape(-1).float().clone()
    if sum(counts) != x.numel():
        raise ValueError("sizes cover %d coordinates, x0 has %d" % (sum(counts), x.numel()))

    def gradient(at):
        with torch.enable_grad():
            xg = at.detach().requires_grad_(True)
            (g,) = torch.autograd.grad(objective([v.view(s) for v, s in zip(xg.split(counts), shapes)]), xg)
        return g.detach().contiguous()

    T = int(sum(int(n) for n in lens))
    labels = torch.empty(T, x.numel(), dtype=x.dtype, device=x.device)
    grads = torch.empty_like(labels)
    st = teacher_state(x)
    for t in range(T):
        x_prev = x.clone()
        for j in range(k):
            g = gradient(x)
            if j == 0:
                grads[t] = g
            teacher_update(name, x, g, st)
        torch.sub(x_prev, x, out=labels[t])
        torch.sub(x_prev, labels[t], out=x)
    return labels, grads


SCALE_NUM_STEPS = [100, 200, 500, 1000, 1500, 2000, 2500, 3000, 3500, 4000, 4500, 5000]   # SC/metaopt.py:172


def train_optimizer(make_trainer: Callable, problems: Sequence, num_problems: int, num_meta_iterations: int,
                    num_unroll_func: Callable[[], int], num_partial_unroll_itrs_func: Callable[[], int],
                    select_random_problems: bool = True, callbacks: Optional[Sequence[Callable]] = None,
                    fix_unroll: bool = False, fix_unroll_length: int = 20, fix_num_steps: int = 100, seed: int = 0,
                    out=None, if_mt: bool = False, mt_ratio: float = 0.3, mt_k: int = 1, teacher: str = "adam",
                    if_cl: bool = False, evaluation_period: int = 1, evaluation_epochs: int = 20,
                    fix_num_steps_eval: int = 100, save_path: Optional[str] = None, min_num_eval: int = 3):
    """The sampling loop of ``metaopt.train_optimizer`` (SC/metaopt.py:117-700) around a meta-trainer: ``num_problems``
    draws of a training problem; on each, ``num_meta_iterations`` optimizee runs, every run a series of partial unrolls
    (``num_unroll_func()`` unrolls of ``num_partial_unroll_itrs_func()`` steps, or ``fix_num_steps // fix_unroll_length``
    unrolls of ``fix_unroll_length`` steps with ``fix_unroll``) with a clipped RMSProp meta-step after each unroll.

    problems: sequence of ``(objective, init_fn)`` — ``objective(list of tensors) -> scalar``, ``init_fn() -> list of
    tensors`` (fresh optimizee parameters for a run).  make_trainer(shapes, theta) -> a ``MetaTrainerBase`` (or, when
    every run's partial unrolls have one length and the keywords below are off, anything with ``theta`` and
    ``train_problem``); one trainer per problem shape, theta handed on from problem to problem.  Returns (theta, log of
    (problem index, meta objectives)) with one entry per optimizee run; imitation runs are not logged.

    The enhanced-training recipe (all off by default; off, the loop draws no extra random number and runs exactly the
    plain loop):

    * ``if_mt``: each run is, with probability ``mt_ratio`` (drawn from the seeded generator that also draws the
      problems), an imitation run: ``teacher_labels(name=teacher, k=mt_k)`` from the run's initial tensors, then
      ``train_problem_mt`` over the same partial unrolls (SC/metaopt.py:354-360, 416-431, 541-548).
    * ``if_cl``: the curriculum (SC/metaopt.py:170-176, 613-690) — runs of ``SCALE_NUM_STEPS[idx] // fix_unroll_length``
      unrolls of ``fix_unroll_length`` steps, evaluated at the next stage's length.  The schedule is
      ``train_dm.Curriculum``: a new best saves ``-idx`` and ``-0``; ``min_num_eval`` evaluations after an improvement
      restore ``-idx`` and advance (and re-evaluate); ``min_num_eval`` without one end this problem's runs.  At the
      last stage evaluation runs at that stage's own length.
    * Evaluation (with ``if_cl`` or ``save_path``): every ``evaluation_period`` runs of a problem, the mean over
      ``evaluation_epochs`` fresh starts of the objective at the last step of an evaluation run
      (``MetaTrainerBase.evaluate``); without ``if_cl`` the run has ``fix_num_steps_eval // fix_unroll_length`` unrolls
      and a new best is saved as ``-0``.
    * ``save_path``: checkpoints are ``torch.save`` files of the trainer's ``get_variables()`` at
      ``"<save_path>-<idx>"``.  The restore of an advance reads the in-memory copy of the same snapshot, so the
      curriculum also runs without ``save_path``."""
    import random
    from .train_dm import Curriculum
    rng = random.Random(seed)
    theta, rms, log, trainers = None, None, [], {}
    cl = Curriculum(fix_unroll_length, min_num_eval, SCALE_NUM_STEPS) if if_cl else None
    evaluating = if_cl or save_path is not None
    best, snapshots = float("inf"), {}

    def say(msg):
        if out is not None:
            print(msg, file=out)

    def save(tr, idx):
        snapshots[idx] = tr.get_variables()
        if save_path is not None:
            torch.save(snapshots[idx], "%s-%d" % (save_path, idx))

    def evaluate(tr, objective, init_fn):
        if cl is None:
            n = fix_num_steps_eval // fix_unroll_length
        else:    # the next stage's length; the last stage has no next one
            i = cl.idx if cl.idx >= 0 else len(cl.num_unrolls) - 1
            n = cl.num_unrolls[min(i + 1, len(cl.num_unrolls) - 1)]
        lens = [fix_unroll_length] * n
        return sum(tr.evaluate(objective, init_fn(), lens) for _ in range(evaluation_epochs)) / evaluation_epochs

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
        for it in range(num_meta_iterations):
            mt = if_mt and rng.random() < mt_ratio
            if cl is not None:
                lens = [fix_unroll_length] * cl.train_unrolls()
            elif fix_unroll:
                lens = [fix_unroll_length] * (fix_num_steps // fix_unroll_length)
            else:
                lens = [num_partial_unroll_itrs_func() for _ in range(num_unroll_func())]
            params = init_fn()
            if mt and lens:
                labels, grads = teacher_labels(objective, tr._x0(params), tr.shapes, lens, teacher, mt_k)
                metas, _ = tr.train_problem_mt(None, params, labels, grads, lens)
                del labels, grads
                say("problem %d: imitation (%s), %d unrolls, meta objective %s"
                    % (k, teacher, len(metas), ["%.4g" % m for m in metas]))
            else:
                # the reference feeds one unroll length per partial unroll
                if len(set(lens)) <= 1:
                    metas, _, _ = tr.train_problem(objective, params, len(lens), lens[0] if lens else 0)
                else:
                    metas, _, _ = tr._train_unrolls(objective, params, lens)
                log.append((k, metas))
                say("problem %d: %d unrolls, meta objective %s" % (k, len(metas), ["%.4f" % m for m in metas]))
            if not evaluating or (it + 1) % evaluation_period != 0:
                continue
            cost = evaluate(tr, objective, init_fn)
            say("problem %d: evaluation %.6g" % (k, cost))
            if cl is None:
                if cost < best:
                    best = cost
                    save(tr, 0)
                continue
            action = cl.observe(cost)
            if action[0] == "save":
                save(tr, action[1])
                save(tr, 0)
            elif action[0] == "advance":
                tr.load_variables(snapshots[action[1]])
                cl.rebase(evaluate(tr, objective, init_fn))
                say("curriculum %d -> %d (%d steps), evaluation %.6g" % (action[1], action[2], cl.num_steps[action[2]],
                                                                         cl.best))
            elif action[0] == "stop":
                say("no improvement during curriculum %d: stop" % action[1])
                break
        theta, rms = tr.theta, getattr(tr, "rms", None)
        for cb in callbacks or ():
            cb(draw, k, tr)
    return theta, log
