"""L2O-Scale ``HierarchicalRNN`` learned optimizer — the update step (inference path) on the H100 engine.

Mirrors the reference class ``optimizer.hierarchical_rnn.HierarchicalRNN`` (SC/optimizer/hierarchical_rnn.py:62-218;
SC/ = Model_Free_L2O/L2O-Scale/L2O-Scale-Training/): same constructor arguments, ``apply_gradients`` as the
``tf.train.Optimizer`` entry (HR:730-805), slot names of ``_initialize_state`` (HR:303-343).  Underneath, one
optimizer step over all optimizee tensors is three CUDA launches of ``libl2o_b200.so`` (``l2o_hrnn_step``); there
is no PyTorch arithmetic on the step path and no CPU fallback.

Scope (SURVEY.md 8(f) row 1): the step itself, with the flag set the reference's drivers run
(SC/metarun.py:154-225,243).  Meta-training of the HierarchicalRNN's own weights (``TrainableOptimizer.train``,
SC/optimizer/trainable_optimizer.py:200-470: BPTT through this step + RMSProp) lives in ``hrnn_train.py``.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import HrnnArgs, L2OError

NUM_GRADIENT_SCALES = 4
N_FEATURES = 12
STATE_PLANES = ("parameter",) * 10 + ("scl_decay", "inp_decay", "log_learning_rate", "grad_accum1", "grad_accum2",
                                      "grad_accum3", "grad_accum4", "ms1", "ms2", "ms3", "ms4")


def theta_spec(levels=(10, 20, 20)) -> List[Tuple[str, Tuple[int, ...]]]:
    """(variable name, shape) in TF creation order = the flat ``theta`` layout of ``l2o_hrnn_*``
    (HR:176-204 readouts, HR:220-245 cells, HR:561-600 affines, HR:612-620, HR:684-691, HR:720-727)."""
    h0, h1, h2 = levels
    f = N_FEATURES
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
        ("PerTensor/GradsToDelta/Matrix", (NUM_GRADIENT_SCALES, 1)),
        ("PerTensor/learning_rate_momentum_logit", ()), ("PerTensor/param_stepsize_offset", ()),
        ("Layer2_RNN/BiasGRUCell/gates/Affine/Matrix", (h1 + h2, 2 * h2)),
        ("Layer2_RNN/BiasGRUCell/gates/Affine/Bias", (2 * h2,)),
        ("Layer2_RNN/BiasGRUCell/candidate/Affine/Matrix", (h1 + h2, h2)),
        ("Layer2_RNN/BiasGRUCell/candidate/Affine/Bias", (h2,)),
    ]


THETA_SPEC = theta_spec()

# the reference's initialisation flags (HR:32-56)
FLAGS = dict(biasgrucell_scale=0.5, biasgrucell_gate_bias_init=2.2, hrnn_rnn_readout_scale=0.5,
             hrnn_default_decay_var_init=2.2, scale_decay_bias_init=3.2, learning_rate_momentum_logit_init=3.2,
             hrnn_affine_scale=0.5)


def metarun_flags() -> dict:
    """The constructor arguments the reference's drivers pass (SC/metarun.py:154-225,243) — the configuration this
    build implements."""
    return dict(level_sizes=[10, 20, 20], init_lr_range=(1e-6, 1e-2), learnable_decay=True, dynamic_output_scale=True,
                use_attention=False, use_log_objective=True, num_gradient_scales=4, zero_init_lr_weights=True,
                use_log_means_squared=True, use_relative_lr=True, use_extreme_indicator=False, max_log_lr=33,
                obj_train_max_multiplier=-1, use_problem_lr_mean=True, use_gradient_shortcut=True,
                use_lr_shortcut=False, use_grad_products=True, use_multiple_scale_decays=False,
                learnable_inp_decay=True, learnable_rnn_init=True)


def _init_theta(seed: Optional[int]) -> torch.Tensor:
    g = torch.Generator()
    if seed is not None:
        g.manual_seed(int(seed))
    out = []
    for name, shape in THETA_SPEC:
        n = int(math.prod(shape))
        if name.endswith("init_vector"):
            v = torch.rand(n, generator=g) * 2 - 1                                           # HR:233-236
        elif name in ("update_weights", "scl_decay_weights", "inp_decay_weights"):
            v = torch.randn(n, generator=g) * (FLAGS["hrnn_rnn_readout_scale"] / math.sqrt(10))  # HR:183-186
        elif name in ("learning_rate_weights", "learning_rate_bias"):
            v = torch.zeros(n)                                                               # zero_init_lr_weights
        elif name == "scl_decay_bias":
            v = torch.full((n,), FLAGS["scale_decay_bias_init"])
        elif name == "inp_decay_bias":
            v = torch.full((n,), FLAGS["hrnn_default_decay_var_init"])
        elif name.endswith("learning_rate_momentum_logit"):
            v = torch.full((n,), FLAGS["learning_rate_momentum_logit_init"])
        elif name.endswith("param_stepsize_offset"):
            v = torch.full((n,), -1.0)
        elif name.endswith("GradsToDelta/Matrix"):
            v = 0.25 + torch.randn(n, generator=g) * (0.1 / math.sqrt(shape[0]))            # vec_mean=1/len(grads_scaled)
        elif name.endswith("gates/Affine/Bias"):
            v = torch.full((n,), FLAGS["biasgrucell_gate_bias_init"])
        elif name.endswith("Bias"):
            v = torch.zeros(n)
        else:  # affine matrices: N(0, scale / sqrt(fan_in))  (SC/optimizer/utils.py:70-76)
            v = torch.randn(n, generator=g) * (0.5 / math.sqrt(shape[0]))
        out.append(v.float())
    return torch.cat(out)


def _p(t: Optional[torch.Tensor]):
    if t is None:
        return None
    if not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous():
        raise L2OError("expected a contiguous fp32 CUDA tensor (this engine has no CPU path)")
    return t.data_ptr()


class HierarchicalRNN(object):
    """3-level hierarchical RNN optimizer (per-parameter GRU 10, per-tensor GRU 20, global GRU 20)."""

    def __init__(self, level_sizes=(10, 20, 20), init_lr_range=(1e-6, 1e-2), learnable_decay=True,
                 dynamic_output_scale=True, use_attention=False, use_log_objective=True, num_gradient_scales=4,
                 zero_init_lr_weights=True, use_log_means_squared=True, use_relative_lr=True,
                 use_extreme_indicator=False, max_log_lr=33, obj_train_max_multiplier=-1, use_problem_lr_mean=False,
                 use_gradient_shortcut=False, use_lr_shortcut=False, use_grad_products=False,
                 use_multiple_scale_decays=False, learnable_inp_decay=True, learnable_rnn_init=True,
                 random_seed=None, device="cuda", distributed=False, **kwargs):
        # signature defaults = the reference's (HR:69-82); the drivers override three of them (metarun_flags())
        # argument checks of the reference (HR:132-144)
        if len(level_sizes) not in [1, 2, 3]:
            raise ValueError("HierarchicalRNN only supports 1, 2, or 3 levels in the hierarchy, but {} were "
                             "requested.".format(len(level_sizes)))
        if any(not isinstance(level, int) for level in level_sizes):
            raise ValueError("Level sizes must be integer values, were {}".format(level_sizes))
        if len(init_lr_range) != 2:
            raise ValueError("Initial LR range must be len 2, was {}".format(len(init_lr_range)))
        if init_lr_range[0] > init_lr_range[1]:
            raise ValueError("Initial LR range min is greater than max.")
        built = dict(level_sizes=(10, 20, 20), learnable_decay=True, dynamic_output_scale=True, use_attention=False,
                     num_gradient_scales=4, zero_init_lr_weights=True, use_log_means_squared=True,
                     use_relative_lr=True, use_extreme_indicator=False, max_log_lr=33, use_problem_lr_mean=True,
                     use_gradient_shortcut=True, use_lr_shortcut=False, use_grad_products=True,
                     use_multiple_scale_decays=False, learnable_inp_decay=True, learnable_rnn_init=True)
        asked = dict(level_sizes=tuple(level_sizes), learnable_decay=learnable_decay,
                     dynamic_output_scale=dynamic_output_scale, use_attention=use_attention,
                     num_gradient_scales=num_gradient_scales, zero_init_lr_weights=zero_init_lr_weights,
                     use_log_means_squared=use_log_means_squared, use_relative_lr=use_relative_lr,
                     use_extreme_indicator=use_extreme_indicator, max_log_lr=max_log_lr,
                     use_problem_lr_mean=use_problem_lr_mean, use_gradient_shortcut=use_gradient_shortcut,
                     use_lr_shortcut=use_lr_shortcut, use_grad_products=use_grad_products,
                     use_multiple_scale_decays=use_multiple_scale_decays, learnable_inp_decay=learnable_inp_decay,
                     learnable_rnn_init=learnable_rnn_init)
        diff = {k: v for k, v in asked.items() if built[k] != v}
        if diff:
            raise NotImplementedError("this build implements the flag set the reference's drivers run "
                                      "(SC/metarun.py:154-225,243); unsupported: %r" % (diff,))
        self.level_sizes = tuple(level_sizes)
        self.init_lr_range = tuple(init_lr_range)
        self.random_seed = random_seed
        self.device = torch.device(device)
        L = _lib.lib()
        self.n_theta = int(L.l2o_hrnn_theta_count())
        self.distributed = bool(distributed)
        if random_seed is None:   # unseeded like the reference; the ranks of a sharded optimizer must draw the same theta
            theta_seed = int(torch.seed() % (2 ** 31))
            if self.distributed:
                import torch.distributed as tdist
                box = torch.tensor([theta_seed], dtype=torch.int64, device=self.device)
                tdist.broadcast(box, src=0)
                theta_seed = int(box.item())
        else:
            theta_seed = random_seed
        theta = _init_theta(theta_seed)
        assert theta.numel() == self.n_theta
        self.theta = theta.to(self.device)
        self._h = None
        self._vars: List[torch.Tensor] = []
        # distributed=True: every rank holds a contiguous slice of every optimizee tensor's coordinates (the optimizee
        # itself stays replicated); one small all-reduce of the per-tensor sums per step + an all-gather of the
        # updated parameters (SURVEY.md 8(e)).  Needs an initialised torch.distributed process group.
        self.distributed = bool(distributed)

    # ---- variables (the TF variable collection of OPTIMIZER_SCOPE) ---------------------------------------------------
    def get_variables(self) -> Dict[str, torch.Tensor]:
        out, off = {}, 0
        for name, shape in THETA_SPEC:
            n = int(math.prod(shape))
            out[name] = self.theta[off:off + n].view(shape)
            off += n
        return out

    def load_variables(self, values: Dict[str, torch.Tensor]):
        for name, view in self.get_variables().items():
            if name in values:
                view.copy_(torch.as_tensor(values[name], dtype=torch.float32).reshape(view.shape))
        if self._h is not None:
            self._prepare()

    # ---- meta-training ---------------------------------------------------------------------------------------------
    def meta_trainer(self, var_list: Sequence[torch.Tensor], **kwargs):
        """A ``hrnn_train.MetaTrainer`` for optimizees shaped like ``var_list`` that starts from this optimizer's
        weights (``TrainableOptimizer.train``, SC/optimizer/trainable_optimizer.py:200-470).  ``adopt(trainer)`` copies the
        trained weights back."""
        from .hrnn_train import MetaTrainer
        kwargs.setdefault("init_lr_range", self.init_lr_range)
        return MetaTrainer([tuple(v.shape) for v in var_list], theta=self.theta, device=str(self.device), **kwargs)

    def adopt(self, trainer):
        self.theta.copy_(trainer.theta.detach())
        if self._h is not None:
            self._prepare()

    # ---- slots ---------------------------------------------------------------------------------------------------------
    def _create_slots(self, var_list: Sequence[torch.Tensor]):
        """One slot set per optimizee tensor (trainable_optimizer.py:94-105), laid out as 21 planes over the
        concatenation of all tensors; the optimizee tensors become views of one flat arena."""
        gsizes = [int(v.numel()) for v in var_list]
        if any(s <= 0 for s in gsizes):
            raise ValueError("empty optimizee variable")
        self.global_sizes = gsizes
        if self.distributed:
            import torch.distributed as tdist
            from .dist import shard_range
            self._rank, self._world = tdist.get_rank(), tdist.get_world_size()
            self._ranges = [shard_range(n, self._rank, self._world) for n in gsizes]
        else:
            self._rank, self._world = 0, 1
            self._ranges = [(0, n) for n in gsizes]
        sizes = [hi - lo for lo, hi in self._ranges]
        if sum(sizes) <= 0:
            raise ValueError("this rank holds no coordinate (more ranks than coordinates)")
        arr = (C.c_int64 * len(sizes))(*sizes)
        h = C.c_void_p()
        _lib.check(_lib.lib().l2o_hrnn_create(C.byref(h), arr, len(sizes)), "l2o_hrnn_create")
        self._h, self.sizes, self.N = h, sizes, sum(sizes)
        if self.distributed:
            garr = (C.c_int64 * len(gsizes))(*gsizes)
            _lib.check(_lib.lib().l2o_hrnn_set_global_sizes(h, garr), "l2o_hrnn_set_global_sizes")
        dev = self.device
        self.x = torch.empty(self.N, device=dev)
        self.g = torch.empty(self.N, device=dev)
        off = 0
        for v, (lo, hi) in zip(var_list, self._ranges):
            n = hi - lo
            self.x[off:off + n].copy_(v.detach().reshape(-1)[lo:hi])
            if not self.distributed:   # re-seat the variables on the arena (zero-copy flatten/unflatten afterwards)
                v.data = self.x[off:off + n].view(v.shape)
            off += n
        self._vars = list(var_list)
        self.state = torch.zeros(int(_lib.lib().l2o_hrnn_state_floats()), self.N, device=dev)
        self.layer = torch.zeros(len(sizes), self.level_sizes[1], device=dev)
        self.global_state = torch.zeros(self.level_sizes[2], device=dev)
        nbytes = int(_lib.lib().l2o_hrnn_workspace_bytes(h))
        self.workspace = torch.zeros((nbytes + 255) // 4 + 64, dtype=torch.float32, device=dev)
        self.update = torch.empty(self.N, device=dev)
        if self.distributed:   # views of the workspace head that the ranks all-reduce between the two step phases
            nd, fo, nf = C.c_int64(), C.c_int64(), C.c_int64()
            _lib.check(_lib.lib().l2o_hrnn_reduce_layout(h, C.byref(nd), C.byref(fo), C.byref(nf)), "l2o_hrnn_reduce_layout")
            base = (self.workspace.data_ptr() + 255) // 256 * 256 - self.workspace.data_ptr()
            raw = self.workspace.view(torch.uint8)
            self._red_sums = raw[base:base + 8 * nd.value].view(torch.float64)
            self._red_flags = raw[base + fo.value:base + fo.value + 4 * nf.value].view(torch.int32)
        self.reset_state()

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                _lib.lib().l2o_hrnn_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _args(self, with_xg=True) -> HrnnArgs:
        a = HrnnArgs()
        a.theta = _p(self.theta)
        a.x, a.g = (_p(self.x), _p(self.g)) if with_xg else (None, None)
        a.state, a.layer, a.global_ = _p(self.state), _p(self.layer), _p(self.global_state)
        ws = self.workspace.data_ptr()
        a.workspace = (ws + 255) // 256 * 256
        a.update = _p(self.update)
        return a

    def _allreduce_sums(self):
        import torch.distributed as tdist
        tdist.all_reduce(self._red_sums, op=tdist.ReduceOp.SUM)
        tdist.all_reduce(self._red_flags, op=tdist.ReduceOp.MAX)

    def _prepare(self):
        L, st, a = _lib.lib(), torch.cuda.current_stream().cuda_stream, self._args(False)
        if not self.distributed:
            _lib.check(L.l2o_hrnn_prepare(self._h, C.byref(a), st), "l2o_hrnn_prepare")
            return
        _lib.check(L.l2o_hrnn_prepare_local(self._h, C.byref(a), st), "l2o_hrnn_prepare_local")
        self._allreduce_sums()
        _lib.check(L.l2o_hrnn_prepare_finish(self._h, C.byref(a), st), "l2o_hrnn_prepare_finish")

    def reset_state(self, seed: Optional[int] = None, log_learning_rate: Optional[torch.Tensor] = None):
        """_initialize_state / _initialize_global_state (HR:303-350).  The log learning rates are drawn as in the
        reference (per-coordinate U(log(min)/2, log(max)/2) plus one per-tensor offset from the same range, clipped
        to [-33, max_log_lr]) unless given."""
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(_lib.lib().l2o_hrnn_init_state(self._h, C.byref(self._args(False)), st), "l2o_hrnn_init_state")
        if log_learning_rate is None:
            gen = torch.Generator()
            s = self.random_seed if seed is None else seed
            if s is None:   # unseeded like the reference (a fresh draw per call); ranks must agree on it when sharded
                s = int(torch.seed() % (2 ** 31))
                if self.distributed:
                    import torch.distributed as tdist
                    box = torch.tensor([s], dtype=torch.int64, device=self.device)
                    tdist.broadcast(box, src=0)
                    s = int(box.item())
            gen.manual_seed(int(s))
            lo, hi = math.log(self.init_lr_range[0]) / 2.0, math.log(self.init_lr_range[1]) / 2.0
            parts = []
            for n, (slo, shi) in zip(self.global_sizes, self._ranges):   # drawn for the whole tensor, sliced per rank
                actual = torch.rand(n, generator=gen) * (hi - lo) + lo
                offset = torch.rand((), generator=gen) * (hi - lo) + lo
                parts.append(torch.clamp(actual + offset, -33.0, 33.0)[slo:shi])
            log_learning_rate = torch.cat(parts)
        self.state[12].copy_(torch.as_tensor(log_learning_rate, dtype=torch.float32).reshape(-1))
        self._prepare()

    def get_slot(self, var_index: int, key: str) -> torch.Tensor:
        """Slot ``key`` of optimizee tensor ``var_index`` (reference slot names, HR:206-213)."""
        off = sum(self.sizes[:var_index])
        n = self.sizes[var_index]
        if key == "parameter":
            return self.state[0:10, off:off + n].t()
        if key == "layer":
            return self.layer[var_index:var_index + 1]
        if key == "true_param":
            return self._vars[var_index]
        planes = {"scl_decay": 10, "inp_decay": 11, "log_learning_rate": 12, "grad_accum1": 13, "grad_accum2": 14,
                  "grad_accum3": 15, "grad_accum4": 16, "ms1": 17, "ms2": 18, "ms3": 19, "ms4": 20}
        return self.state[planes[key], off:off + n].view(n, 1)

    # ---- the step --------------------------------------------------------------------------------------------------------
    def apply_gradients(self, grads_and_vars: Iterable[Tuple[torch.Tensor, torch.Tensor]], global_step=None, name=None):
        """tf.train.Optimizer.apply_gradients (HR:730-805): one HierarchicalRNN step over all (grad, var) pairs.
        Variables are updated in place; returns the list of updated variables ("real_params")."""
        grads_and_vars = tuple(grads_and_vars)
        for g, v in grads_and_vars:
            if g is not None and not torch.is_tensor(g):
                raise TypeError("Gradient must be a Tensor or None: %s" % (g,))
            if not torch.is_tensor(v):
                raise TypeError("Variable must be a Tensor: %s" % (v,))
        pairs = [(g, v) for g, v in grads_and_vars if g is not None]
        if not pairs:
            raise ValueError("No gradients provided for any variable: %s" % (grads_and_vars,))
        if self._h is None:
            self._create_slots([v for _, v in pairs])
        elif len(pairs) != len(self._vars) or any(v is not w for (_, v), w in zip(pairs, self._vars)):
            raise ValueError("apply_gradients must be called with the variables the slots were created for")
        off = 0
        for (g, v), (lo, hi) in zip(pairs, self._ranges):
            n = hi - lo
            self.g[off:off + n].copy_(g.reshape(-1)[lo:hi])
            off += n
        self.step_flat()
        if self.distributed:   # republish the updated parameters to the replicated optimizee
            from .dist import allgather_shards
            off = 0
            for (_, v), (lo, hi), n in zip(pairs, self._ranges, self.global_sizes):
                v.data.copy_(allgather_shards(self.x[off:off + hi - lo], n).view(v.shape))
                off += hi - lo
        return [v for _, v in pairs]

    def step_flat(self):
        """One step with the gradients already in ``self.g`` (flat arena order)."""
        L, st, a = _lib.lib(), torch.cuda.current_stream().cuda_stream, self._args(True)
        if not self.distributed:
            _lib.check(L.l2o_hrnn_step(self._h, C.byref(a), st), "l2o_hrnn_step")
            return
        _lib.check(L.l2o_hrnn_step_local(self._h, C.byref(a), st), "l2o_hrnn_step_local")
        self._allreduce_sums()
        _lib.check(L.l2o_hrnn_step_finish(self._h, C.byref(a), st), "l2o_hrnn_step_finish")

    def minimize(self, objective, var_list: Sequence[torch.Tensor], num_steps: int, cuda_graph: Optional[bool] = None):
        """Convenience loop of the evaluation drivers (SC/metatest.py): num_steps x (objective, gradients, step).
        Returns the list of objective values (one device->host read at the end).

        One iteration is ~50 tiny launches (the optimizee's forward/backward, the gradient copies, the three step
        kernels) and nothing in it needs the host, so after two eager iterations (slot creation, library warm-up) one
        iteration is captured into a CUDA graph and replayed (``cuda_graph=False`` or ``L2O_CUDA_GRAPH=0`` keeps
        everything eager; a failed capture falls back to the same eager kernels with a warning)."""
        import os
        var_list = list(var_list)

        def body():
            loss = objective(*var_list)
            grads = torch.autograd.grad(loss, var_list)
            self.apply_gradients(zip(grads, var_list))
            return loss.detach()

        if cuda_graph is None:
            cuda_graph = os.environ.get("L2O_CUDA_GRAPH", "1") != "0"
        if self.distributed:
            cuda_graph = False   # the per-step collectives stay outside graph capture
        from . import engine as _engine
        # 3: the three l2o_hrnn_step kernels inside the graph
        return _engine.replay_loop(self, body, objective, var_list, num_steps, cuda_graph, 3, "HierarchicalRNN")
