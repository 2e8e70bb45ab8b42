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
from typing import Iterable, List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import HrnnArgs
from .engine import _ptr, _stream
from .scale_base import ScaleOptimizer

NUM_GRADIENT_SCALES = 4
N_FEATURES = 12
N_SUMS, B0_STRIDE = 24, 32   # per-tensor fp64 sums [h'(10) | features(12) | delta^2 | log-lr'], gate-bias row stride
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


class HrnnHandle(object):
    """An ``l2o_hrnn`` handle (``_h``) for optimizee tensors of ``sizes`` coordinates and the workspace it needs,
    aligned to the 256 B the library requires (``ptr``), with views of the workspace regions that
    ``l2o_hrnn_workspace_layout`` places: ``w_sums`` [n_tensors, 24] fp64 per-tensor sums, ``w_any`` / ``w_zero``
    [n_tensors, 4] int32 flags any(ms != 0) seen this step / all(ms == 0) before the next, ``w_bias0`` [n_tensors, 32]
    per-tensor gate bias, ``w_mean`` [1] problem-wide mean log learning rate, ``w_upd`` [N] raw update lr * delta.
    The handle is destroyed with this object."""

    def __init__(self, sizes: Sequence[int], device):
        L = _lib.lib()
        self._h = C.c_void_p()
        _lib.check(L.l2o_hrnn_create(C.byref(self._h), (C.c_int64 * len(sizes))(*sizes), len(sizes)), "l2o_hrnn_create")
        nbytes = int(L.l2o_hrnn_workspace_bytes(self._h))
        self._buf = torch.zeros((nbytes + 255) // 4 + 64, dtype=torch.float32, device=device)
        self.ptr = (self._buf.data_ptr() + 255) // 256 * 256
        ws = self._buf.view(torch.uint8)[self.ptr - self._buf.data_ptr():]
        off = (C.c_int64 * 7)()
        _lib.check(L.l2o_hrnn_workspace_layout(self._h, off), "l2o_hrnn_workspace_layout")

        def region(k, dtype, *shape):
            return ws[off[k]:off[k] + dtype.itemsize * math.prod(shape)].view(dtype).view(*shape)
        nt, n = len(sizes), int(sum(sizes))
        self.w_sums = region(0, torch.float64, nt, N_SUMS)
        self.w_any = region(1, torch.int32, nt, NUM_GRADIENT_SCALES)
        self.w_zero = region(2, torch.int32, nt, NUM_GRADIENT_SCALES)
        self.w_bias0 = region(3, torch.float32, nt, B0_STRIDE)
        self.w_mean = region(5, torch.float32, 1)
        self.w_upd = region(6, torch.float32, n)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                _lib.lib().l2o_hrnn_destroy(self._h)
                self._h = None
        except Exception:
            pass


class HierarchicalRNN(ScaleOptimizer):
    """3-level hierarchical RNN optimizer (per-parameter GRU 10, per-tensor GRU 20, global GRU 20).

    ``distributed=True``: every rank holds a contiguous slice of every optimizee tensor's coordinates (the optimizee
    itself stays replicated); one small all-reduce of the per-tensor sums per step + an all-gather of the updated
    parameters (SURVEY.md 8(e)).  Needs an initialised torch.distributed process group."""
    theta_spec = THETA_SPEC
    trainer = "hrnn_train.MetaTrainer"
    kernels_per_step = 3

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
        self.n_theta = int(_lib.lib().l2o_hrnn_theta_count())
        self.distributed = bool(distributed)
        # unseeded like the reference; the ranks of a sharded optimizer must draw the same theta
        theta = _init_theta(self._fresh_seed() if random_seed is None else random_seed)
        assert theta.numel() == self.n_theta
        super().__init__(theta, device)

    def _fresh_seed(self) -> int:
        """A fresh seed for an unseeded draw, the same on every rank of a sharded optimizer."""
        s = int(torch.seed() % (2 ** 31))
        if self.distributed:
            import torch.distributed as tdist
            box = torch.tensor([s], dtype=torch.int64, device=self.device)
            tdist.broadcast(box, src=0)
            s = int(box.item())
        return s

    # ---- slots ---------------------------------------------------------------------------------------------------------
    def _shard_ranges(self, sizes):
        if not self.distributed:
            return super()._shard_ranges(sizes)
        import torch.distributed as tdist
        from .dist import shard_range
        rank, world = tdist.get_rank(), tdist.get_world_size()
        return [shard_range(n, rank, world) for n in sizes]

    def _new_state(self):
        """21 planes over the arena (trainable_optimizer.py:94-105), the per-tensor and global GRU states, the handle
        and its workspace."""
        dev = self.device
        self._hrnn = HrnnHandle(self.sizes, dev)
        if self.distributed:
            garr = (C.c_int64 * len(self.global_sizes))(*self.global_sizes)
            _lib.check(_lib.lib().l2o_hrnn_set_global_sizes(self._hrnn._h, garr), "l2o_hrnn_set_global_sizes")
        self.layer = torch.zeros(len(self.sizes), self.level_sizes[1], device=dev)
        self.global_state = torch.zeros(self.level_sizes[2], device=dev)
        self.update = torch.empty(self.N, device=dev)
        return torch.zeros(int(_lib.lib().l2o_hrnn_state_floats()), self.N, device=dev)

    def _args(self, with_xg=True) -> HrnnArgs:
        a = HrnnArgs()
        a.theta = _ptr(self.theta)
        a.x, a.g = (_ptr(self.x), _ptr(self.g)) if with_xg else (None, None)
        a.state, a.layer, a.global_ = _ptr(self.state), _ptr(self.layer), _ptr(self.global_state)
        a.workspace = self._hrnn.ptr
        a.update = _ptr(self.update)
        return a

    def _allreduce_sums(self):
        import torch.distributed as tdist
        tdist.all_reduce(self._hrnn.w_sums, op=tdist.ReduceOp.SUM)
        tdist.all_reduce(self._hrnn.w_any, op=tdist.ReduceOp.MAX)

    def _prepare(self):
        L, h, a = _lib.lib(), self._hrnn._h, self._args(False)
        if not self.distributed:
            _lib.check(L.l2o_hrnn_prepare(h, C.byref(a), _stream()), "l2o_hrnn_prepare")
            return
        _lib.check(L.l2o_hrnn_prepare_local(h, C.byref(a), _stream()), "l2o_hrnn_prepare_local")
        self._allreduce_sums()
        _lib.check(L.l2o_hrnn_prepare_finish(h, C.byref(a), _stream()), "l2o_hrnn_prepare_finish")

    def reset_state(self, seed: Optional[int] = None, log_learning_rate: Optional[torch.Tensor] = None):
        """_initialize_state / _initialize_global_state (HR:303-350).  The log learning rates are drawn as in the
        reference (per-coordinate U(log(min)/2, log(max)/2) plus one per-tensor offset from the same range, clipped
        to [-33, max_log_lr]) unless given."""
        _lib.check(_lib.lib().l2o_hrnn_init_state(self._hrnn._h, C.byref(self._args(False)), _stream()),
                   "l2o_hrnn_init_state")
        if log_learning_rate is None:
            gen = torch.Generator()
            s = self.random_seed if seed is None else seed
            gen.manual_seed(int(self._fresh_seed() if s is None else s))   # unseeded: a fresh draw per call
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
        updated = super().apply_gradients(grads_and_vars, global_step, name)
        if self.distributed:   # republish the updated parameters to the replicated optimizee
            from .dist import allgather_shards
            off = 0
            for v, (lo, hi), n in zip(updated, self._ranges, self.global_sizes):
                v.data.copy_(allgather_shards(self.x[off:off + hi - lo], n).view(v.shape))
                off += hi - lo
        return updated

    def step_flat(self):
        """One step with the gradients already in ``self.g`` (flat arena order)."""
        L, h, a = _lib.lib(), self._hrnn._h, self._args(True)
        if not self.distributed:
            _lib.check(L.l2o_hrnn_step(h, C.byref(a), _stream()), "l2o_hrnn_step")
            return
        _lib.check(L.l2o_hrnn_step_local(h, C.byref(a), _stream()), "l2o_hrnn_step_local")
        self._allreduce_sums()
        _lib.check(L.l2o_hrnn_step_finish(h, C.byref(a), _stream()), "l2o_hrnn_step_finish")
