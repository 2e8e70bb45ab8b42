"""Thin torch-tensor front end of the C-ABI (``include/l2o_b200.h``).  PyTorch is used only as the
owner of device memory and streams; all arithmetic happens in the CUDA library."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import torch

from . import _lib
from ._lib import (BwdArgs, NetDesc, StepArgs, UnrollArgs, L2OError, PRE_FC, PRE_IDENTITY, PRE_LOGSIGN,
                   OPT_NONE, OPT_QUADRATIC_DIAG, OPT_RASTRIGIN_SEP, OPT_QUADRATIC_BATCH, ENGINE_AUTO, ENGINE_FFMA, ENGINE_TC)

_PRE = {"identity": PRE_IDENTITY, "LogAndSign": PRE_LOGSIGN, "fc": PRE_FC}
OPT_KINDS = {"rastrigin_sep": OPT_RASTRIGIN_SEP, "quadratic_diag": OPT_QUADRATIC_DIAG,
             "quadratic_batch": OPT_QUADRATIC_BATCH}


def _ptr(t: Optional[torch.Tensor], dtype=torch.float32, name="tensor"):
    if t is None:
        return None
    if not t.is_cuda:
        raise L2OError(f"{name}: expected a CUDA tensor (this engine has no CPU path)")
    if t.dtype != dtype:
        raise L2OError(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise L2OError(f"{name}: expected a contiguous tensor")
    return t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


class _Handle:
    """What the coordinate-wise and the dense net handles share, and the surface the meta-optimizer uses on either:
    ``n_in``, ``layers``, ``n_theta``, the state arena (``state_size`` / ``new_state`` / ``state_views``), ``step`` and
    ``unroll_bwd``.  The state is kept per row: a row is one coordinate here, K elements for a dense net."""

    n_in = 1
    _destroy = None   # name of the C destructor

    @staticmethod
    def _layers(layers):
        layers = tuple(int(h) for h in layers)
        if len(layers) > 2:
            raise L2OError("at most two LSTM layers are supported")
        return layers

    def _open(self, desc, create, theta_count, state_floats, what):
        """Fill the descriptor's layers, create the C handle and read its sizes."""
        desc.n_layers = len(self.layers)
        desc.hidden[0], desc.hidden[1] = (self.layers + (0, 0))[:2]
        self._h = C.c_void_p()
        _lib.check(create(C.byref(self._h), C.byref(desc)), what)
        self.n_theta = int(theta_count(self._h))
        self.state_floats = int(state_floats(self._h))   # per row

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                getattr(_lib.lib(), self._destroy)(self._h)
                self._h = None
        except Exception:
            pass

    def rows(self, n: int) -> int:
        return n

    def state_size(self, n: int) -> int:
        """Floats of one state arena for n elements."""
        return self.state_floats * self.rows(n)

    def new_state(self, n: int, device) -> torch.Tensor:
        return torch.zeros(max(self.state_size(n), 1), dtype=torch.float32, device=device)

    def state_views(self, arena: torch.Tensor, n: int):
        """Arena -> tuple over layers of (hidden, cell) views [rows, H] (the reference's state structure)."""
        out, off, r = [], 0, self.rows(n)
        for h in self.layers:
            out.append((arena[off:off + r * h].view(r, h), arena[off + r * h:off + 2 * r * h].view(r, h)))
            off += 2 * r * h
        return tuple(out)

    def _check_theta(self, theta):
        if theta.numel() != self.n_theta:
            raise L2OError(f"theta has {theta.numel()} elements, net needs {self.n_theta}")


class NetHandle(_Handle):
    """One optimizer net: shape + run-time scalars (DM/networks.py:157-205)."""

    _destroy = "l2o_net_destroy"

    def __init__(self, layers: Sequence[int] = (20, 20), preprocess_name: str = "identity",
                 preprocess_options: Optional[dict] = None, scale: float = 1.0, tanh_output: bool = False,
                 n_in: int = 1):
        self.layers = self._layers(layers)
        if preprocess_name not in _PRE:
            raise L2OError(f"unsupported preprocess_name {preprocess_name!r}")
        opts = dict(preprocess_options or {})
        d = NetDesc()
        d.preprocess = _PRE[preprocess_name]
        d.n_in = n_in
        d.fc_dim = int(opts.get("dim", 0))
        d.logsign_k = float(opts.get("k", 0.0))
        d.scale = float(scale)
        d.tanh_output = 1 if tanh_output else 0
        self.desc = d
        self.n_in = n_in
        L = _lib.lib()
        self._open(d, L.l2o_net_create, L.l2o_theta_count, L.l2o_state_floats,
                   f"l2o_net_create(layers={self.layers}, preprocess={preprocess_name}, n_in={n_in})")

    def workspace_bytes(self, n: int, T: int):
        """(forward, backward) caller-owned buffer bytes for n coordinates and a T-step unroll."""
        f, b = C.c_size_t(), C.c_size_t()
        _lib.check(_lib.lib().l2o_workspace_bytes(self._h, n, T, C.byref(f), C.byref(b)), "l2o_workspace_bytes")
        return int(f.value), int(b.value)

    def set_engine(self, engine: int):
        _lib.check(_lib.lib().l2o_net_set_engine(self._h, engine), "l2o_net_set_engine")

    # ---- kernels -------------------------------------------------------------------------
    def step(self, theta, in0, state_in, state_out, *, in1=None, m=None, v=None, beta1=0.95, beta2=0.95, p=1.0,
             x=None, delta=None, feat_out=None, step_ptr=None, t_offset=0, reuse_weights=False):
        a = StepArgs()
        a.reuse_weights = 1 if reuse_weights else 0
        a.n = in0.numel()
        a.theta = _ptr(theta, name="theta")
        a.in0, a.in1 = _ptr(in0, name="in0"), _ptr(in1, name="in1")
        a.m, a.v = _ptr(m, name="m"), _ptr(v, name="v")
        a.beta1, a.beta2, a.p = beta1, beta2, p
        a.state_in, a.state_out = _ptr(state_in, name="state_in"), _ptr(state_out, name="state_out")
        a.x, a.delta, a.feat_out = _ptr(x, name="x"), _ptr(delta, name="delta"), _ptr(feat_out, name="feat_out")
        a.step_ptr, a.t_offset = _ptr(step_ptr, torch.int32, "step_ptr"), t_offset
        self._check_theta(theta)
        _lib.check(_lib.lib().l2o_step(self._h, C.byref(a), _stream()), "l2o_step")

    def unroll_fwd(self, theta, n, T, state, *, in_seq=None, opt_kind=OPT_NONE, opt_a=None, opt_b=None,
                   opt_alpha=10.0, opt_fscale=1.0, x=None, ckpt=None, m=None, v=None, beta1=0.95, beta2=0.95,
                   step0=1, g_rec=None, feat_rec=None, fx=None, delta_seq=None, labels=None, imit_loss=None,
                   n_total=0, opt_group=0):
        a = UnrollArgs()
        a.n, a.T = n, T
        a.theta = _ptr(theta, name="theta")
        a.in_seq = _ptr(in_seq, name="in_seq")
        a.opt_kind = opt_kind
        a.opt_a, a.opt_b = _ptr(opt_a, name="opt_a"), _ptr(opt_b, name="opt_b")
        a.opt_alpha, a.opt_fscale = opt_alpha, opt_fscale
        a.x, a.state, a.ckpt = _ptr(x, name="x"), _ptr(state, name="state"), _ptr(ckpt, name="ckpt")
        a.m, a.v = _ptr(m, name="m"), _ptr(v, name="v")
        a.beta1, a.beta2, a.step0 = beta1, beta2, step0
        a.g_rec, a.feat_rec = _ptr(g_rec, name="g_rec"), _ptr(feat_rec, name="feat_rec")
        a.fx = _ptr(fx, torch.float64, "fx")
        a.delta_seq, a.labels = _ptr(delta_seq, name="delta_seq"), _ptr(labels, name="labels")
        a.imit_loss = _ptr(imit_loss, torch.float64, "imit_loss")
        a.n_total = n_total
        a.opt_group = opt_group
        _lib.check(_lib.lib().l2o_unroll_fwd(self._h, C.byref(a), _stream()), "l2o_unroll_fwd")

    def unroll_bwd(self, theta, n, T, in_seq, ckpt, dtheta, *, g_rec=None, labels=None, n_total=0, delta_seq=None,
                   scratch=None):
        """BPTT over the T checkpoint slots.  ``scratch`` ([T, n, 20] floats) lets fc(20) nets (RNNProp) run on the
        tensor-core engine; ``delta_seq`` (the deltas the forward pass recorded) is what a tanh-output net's
        tensor-core BPTT differentiates the output layer with."""
        a = self._bwd_args(theta, n, T, in_seq, ckpt, dtheta, g_rec, labels, n_total, delta_seq, scratch)
        _lib.check(_lib.lib().l2o_unroll_bwd(self._h, C.byref(a), _stream()), "l2o_unroll_bwd")

    def unroll_bwd_carry(self, theta, n, T, in_seq, ckpt, dtheta, d_state, lam, *, g_rec, delta_seq=None,
                         scratch=None):
        """BPTT over one T-step segment of a longer unroll: ``ckpt`` holds the segment's T + 1 slots and ``g_rec`` its
        rows t0..t1.  ``d_state`` (a state arena, the adjoint of the state after the segment) and ``lam`` ([n],
        sum_{tau > t1} g_tau) are updated in place to the adjoint of the state before it and sum_{tau > t0} g_tau."""
        a = self._bwd_args(theta, n, T, in_seq, ckpt, dtheta, g_rec, None, 0, delta_seq, scratch)
        c = _lib.BwdCarry()
        c.d_state, c.lam = _ptr(d_state, name="d_state"), _ptr(lam, name="lam")
        _lib.check(_lib.lib().l2o_unroll_bwd_carry(self._h, C.byref(a), C.byref(c), _stream()), "l2o_unroll_bwd_carry")

    @staticmethod
    def _bwd_args(theta, n, T, in_seq, ckpt, dtheta, g_rec, labels, n_total, delta_seq, scratch):
        a = BwdArgs()
        a.n, a.T = n, T
        a.theta = _ptr(theta, name="theta")
        a.in_seq, a.ckpt = _ptr(in_seq, name="in_seq"), _ptr(ckpt, name="ckpt")
        a.g_rec, a.labels = _ptr(g_rec, name="g_rec"), _ptr(labels, name="labels")
        a.n_total = n_total
        a.dtheta = _ptr(dtheta, torch.float64, "dtheta")
        a.delta_seq = _ptr(delta_seq, name="delta_seq")
        if scratch is not None and scratch.numel() < T * n * 20:
            raise L2OError(f"scratch has {scratch.numel()} floats, the fc-net BPTT needs T*n*20 = {T * n * 20}")
        a.scratch = _ptr(scratch, name="scratch")
        return a


class DenseNetHandle(_Handle):
    """Row-wise dense LSTM net with run-time shapes (StandardDeepLSTM with output_size > 1 = the reference's
    KernelDeepLSTM, DM/networks.py:154-236,303-351).  A variable of n = K * R elements in [kw, kh, cin, cout] order is
    R rows of K inputs (element (k, r) at k * R + r); state per ROW."""

    _destroy = "l2o_dense_destroy"

    def __init__(self, layers: Sequence[int], k_in: int, k_out: int, preprocess_name: str = "identity",
                 preprocess_options: Optional[dict] = None, scale: float = 1.0, tanh_output: bool = False):
        self.layers = self._layers(layers)
        if preprocess_name not in ("identity", "LogAndSign"):
            raise L2OError(f"unsupported preprocess_name {preprocess_name!r} for a dense net")
        d = _lib.DenseDesc()
        d.n_in, d.n_out = int(k_in), int(k_out)
        d.preprocess = _PRE[preprocess_name]
        d.logsign_k = float((preprocess_options or {}).get("k", 0.0))
        d.scale, d.tanh_output = float(scale), 1 if tanh_output else 0
        self.k_in, self.k_out = int(k_in), int(k_out)
        L = _lib.lib()
        self._open(d, L.l2o_dense_create, L.l2o_dense_theta_count, L.l2o_dense_state_floats,
                   f"l2o_dense_create(layers={self.layers}, k_in={k_in}, k_out={k_out}, preprocess={preprocess_name})")

    def rows(self, n: int) -> int:
        if n % self.k_in:
            raise L2OError(f"{n} elements are not a whole number of rows of {self.k_in}")
        return n // self.k_in

    def set_engine(self, engine: int):
        if engine == ENGINE_TC:
            raise L2OError("dense nets run on the CUDA-core engine only")

    def step(self, theta, in0, state_in, state_out, *, x=None, delta=None, reuse_weights=False, **unused):
        a = _lib.DenseStepArgs()
        a.rows = self.rows(in0.numel())
        a.theta, a.in_ = _ptr(theta, name="theta"), _ptr(in0, name="in0")
        a.state_in, a.state_out = _ptr(state_in, name="state_in"), _ptr(state_out, name="state_out")
        a.x, a.delta = _ptr(x, name="x"), _ptr(delta, name="delta")
        self._check_theta(theta)
        _lib.check(_lib.lib().l2o_dense_step(self._h, C.byref(a), _stream()), "l2o_dense_step")

    def unroll_bwd(self, theta, n, T, in_seq, ckpt, dtheta, *, g_rec=None, labels=None, n_total=0, delta_seq=None):
        a = _lib.DenseBwdArgs()
        a.rows, a.T = self.rows(n), T
        a.theta = _ptr(theta, name="theta")
        a.in_seq, a.ckpt = _ptr(in_seq, name="in_seq"), _ptr(ckpt, name="ckpt")
        a.g_rec, a.labels = _ptr(g_rec, name="g_rec"), _ptr(labels, name="labels")
        a.n_total = n_total
        a.dtheta = _ptr(dtheta, torch.float64, "dtheta")
        _lib.check(_lib.lib().l2o_dense_unroll_bwd(self._h, C.byref(a), _stream()), "l2o_dense_unroll_bwd")


def adam_step(theta, dtheta, m, v, k: int, lr=0.01, beta1=0.9, beta2=0.999, eps=1e-8):
    """tf.train.AdamOptimizer update of theta in place (DM/meta.py:411-413)."""
    _lib.check(_lib.lib().l2o_adam_step(_ptr(theta, name="theta"), _ptr(dtheta, torch.float64, "dtheta"),
                                        _ptr(m, name="m"), _ptr(v, name="v"), theta.numel(), k, lr, beta1, beta2,
                                        eps, _stream()), "l2o_adam_step")


def log_and_sign(g: torch.Tensor, k: float) -> torch.Tensor:
    """preprocess.LogAndSign on a flat tensor; returns [2, n] (log row, sign row)."""
    out = torch.empty(2, g.numel(), dtype=torch.float32, device=g.device)
    _lib.check(_lib.lib().l2o_log_and_sign(_ptr(g, name="g"), _ptr(out), g.numel(), k, _stream()), "l2o_log_and_sign")
    return out


def lasso_grad(A, y, x, l1, g, f=None, scale=None):
    """f and df/dx of problems.lasso / lasso_fixed in one launch (DM/problems.py:103-175): A [B,m,n], y [B,m(,1)],
    x [B*n] flat; writes g [B*n] and accumulates the scalar loss into the fp64 tensor ``f`` (if given)."""
    a = _lib.LassoArgs()
    a.batch, a.m, a.n = int(A.shape[0]), int(A.shape[1]), int(A.shape[2])
    if x.numel() != a.batch * a.n or g.numel() != a.batch * a.n or y.numel() != a.batch * a.m:
        raise L2OError("lasso_grad: shape mismatch")
    a.A, a.y, a.x = _ptr(A, name="A"), _ptr(y, name="y"), _ptr(x, name="x")
    a.scale = _ptr(scale, name="scale")
    a.l1 = float(l1)
    a.g = _ptr(g, name="g")
    a.f = _ptr(f, torch.float64, "f")
    _lib.check(_lib.lib().l2o_lasso_grad(C.byref(a), _stream()), "l2o_lasso_grad")


CONFOCAL_SMEM_LIMIT = 200 * 1024   # l2o_producers.cu kConfSmemLimit


def confocal_fits(num_points, roi) -> bool:
    """Whether l2o_confocal_grad takes this shape: one CTA holds the image and its per-axis tables in shared memory,
    4 (V + 4 P (nx+ny+nz) + 2P) bytes (include/l2o_b200.h)."""
    nx, ny, nz = (int(r) for r in roi)
    P = int(num_points)
    return max(nx, ny, nz) <= 65536 and 4 * (nx * ny * nz + 4 * P * (nx + ny + nz) + 2 * P) <= CONFOCAL_SMEM_LIMIT


def confocal_grad(x, sim, g, batch, num_points, roi, f=None, scale=None):
    """f and df/dx of problems.confocal_microscopy_3d (DM/problems.py:701-956, inference=False) in one launch.  x, sim,
    g and scale are [6P+1][batch] (rows I, x0, y0, z0, sigma_xy, sigma_z of each point, then bg); writes g and
    accumulates the scalar loss into the fp64 tensor ``f`` (if given)."""
    a = _lib.ConfocalArgs()
    a.batch, a.num_points = int(batch), int(num_points)
    if len(roi) != 3:
        raise L2OError("confocal_grad: roi must have three sizes")
    for k in range(3):
        a.roi[k] = int(roi[k])
    rows = 6 * a.num_points + 1
    for name, t in (("x", x), ("sim", sim), ("g", g), ("scale", scale)):
        if t is not None and t.numel() != rows * a.batch:
            raise L2OError(f"confocal_grad: {name} has {t.numel()} elements, [6P+1][batch] = {rows * a.batch}")
    a.x, a.sim, a.scale = _ptr(x, name="x"), _ptr(sim, name="sim"), _ptr(scale, name="scale")
    a.g = _ptr(g, name="g")
    a.f = _ptr(f, torch.float64, "f")
    _lib.check(_lib.lib().l2o_confocal_grad(C.byref(a), _stream()), "l2o_confocal_grad")


def mnist_fits(layers, batch) -> bool:
    """Whether l2o_mnist_grad takes this MLP: 1..4 hidden layers of width 1..64 and a batch of 1..1024."""
    layers = tuple(int(w) for w in layers)
    return (1 <= len(layers) <= _lib.MNIST_MAX_HIDDEN and all(1 <= w <= _lib.MNIST_MAX_WIDTH for w in layers)
            and 1 <= int(batch) <= _lib.MNIST_MAX_BATCH)


def mnist_grad(images, labels, x, g, layers, batch, activation, seed, counter, f=None, scale=None, idx_out=None):
    """f and df/dx of problems.mnist (DM/problems.py:254-288) at a fresh batch in one launch.  images [N, 784] and
    labels [N] uint8; x, g and scale the flat arena of the MLP's variables in creation order (w0, b0, w1, b1, ...);
    ``counter`` a one-element int64 device tensor the call reads and advances; writes f (fp64 scalar) and the indices
    drawn into ``idx_out`` (int32 [batch]) if given."""
    a = _lib.MnistArgs()
    layers = tuple(int(w) for w in layers)
    a.batch, a.num_examples, a.n_layers = int(batch), int(images.shape[0]), len(layers) + 1
    for k, w in enumerate(layers[:_lib.MNIST_MAX_HIDDEN]):
        a.hidden[k] = w
    a.activation = {"sigmoid": _lib.MNIST_SIGMOID, "relu": _lib.MNIST_RELU}[activation]
    a.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    if images.numel() != a.num_examples * _lib.MNIST_INPUT or labels.numel() != a.num_examples:
        raise L2OError("mnist_grad: images must be [N, 784] and labels [N]")
    n = 0
    k = _lib.MNIST_INPUT
    for w in layers + (_lib.MNIST_CLASSES,):
        n, k = n + (k + 1) * w, w
    for name, t in (("x", x), ("g", g), ("scale", scale)):
        if t is not None and t.numel() != n:
            raise L2OError(f"mnist_grad: {name} has {t.numel()} elements, the MLP has {n}")
    if idx_out is not None and idx_out.numel() != a.batch:
        raise L2OError(f"mnist_grad: idx_out has {idx_out.numel()} elements, batch is {a.batch}")
    if counter.numel() != 1:
        raise L2OError("mnist_grad: counter must be one int64 element")
    a.counter = _ptr(counter, torch.int64, "counter")
    a.images, a.labels = _ptr(images, torch.uint8, "images"), _ptr(labels, torch.uint8, "labels")
    a.x, a.scale, a.g = _ptr(x, name="x"), _ptr(scale, name="scale"), _ptr(g, name="g")
    a.f = _ptr(f, torch.float64, "f")
    a.idx_out = _ptr(idx_out, torch.int32, "idx_out")
    _lib.check(_lib.lib().l2o_mnist_grad(C.byref(a), _stream()), "l2o_mnist_grad")


def mnist_conv_fits(batch) -> bool:
    """Whether l2o_mnist_conv_grad takes this batch size: 1..1024."""
    return 1 <= int(batch) <= _lib.MNIST_CONV_MAX_BATCH


def mnist_conv_workspace_bytes(batch) -> int:
    """Bytes of device workspace l2o_mnist_conv_grad needs at this batch size (the library allocates nothing)."""
    n = int(_lib.lib().l2o_mnist_conv_workspace_bytes(int(batch)))
    if n < 0:
        raise L2OError(f"mnist_conv_workspace_bytes: batch {batch} is outside 1..{_lib.MNIST_CONV_MAX_BATCH}")
    return n


def mnist_conv_workspace_layout(batch) -> dict:
    """Byte offsets in the l2o_mnist_conv_grad workspace of z1, z2, the batch-norm constants and dlogits, the values
    its ReLU and max-pool decisions come from (include/l2o_b200.h)."""
    off = (C.c_int64 * _lib.MNIST_CONV_LAYOUT)()
    _lib.check(_lib.lib().l2o_mnist_conv_workspace_layout(int(batch), off), "l2o_mnist_conv_workspace_layout")
    return dict(zip(("z1", "z2", "bn", "dl"), (int(v) for v in off)))


def mnist_conv_grad(images, labels, x, g, batch, seed, counter, workspace, f=None, scale=None, idx_out=None):
    """f and df/dx of problems.mnist_conv (DM/problems.py:291-347, batch norm on) at a fresh batch in one launch.
    images [N, 784] and labels [N] uint8; x, g and scale the flat 18,122-float arena of the ConvNet's variables in
    creation order; ``counter`` a one-element int64 device tensor the call reads and advances (the batch is drawn as
    mnist_grad draws it); ``workspace`` a uint8 device tensor of at least mnist_conv_workspace_bytes(batch) bytes;
    writes f (fp64 scalar) and the indices drawn into ``idx_out`` (int32 [batch]) if given."""
    a = _lib.MnistConvArgs()
    a.batch, a.num_examples = int(batch), int(images.shape[0])
    a.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    if images.numel() != a.num_examples * _lib.MNIST_INPUT or labels.numel() != a.num_examples:
        raise L2OError("mnist_conv_grad: images must be [N, 784] and labels [N]")
    for name, t in (("x", x), ("g", g), ("scale", scale)):
        if t is not None and t.numel() != _lib.MNIST_CONV_COORDS:
            raise L2OError(f"mnist_conv_grad: {name} has {t.numel()} elements, the ConvNet has {_lib.MNIST_CONV_COORDS}")
    if idx_out is not None and idx_out.numel() != a.batch:
        raise L2OError(f"mnist_conv_grad: idx_out has {idx_out.numel()} elements, batch is {a.batch}")
    if counter.numel() != 1:
        raise L2OError("mnist_conv_grad: counter must be one int64 element")
    a.counter = _ptr(counter, torch.int64, "counter")
    a.images, a.labels = _ptr(images, torch.uint8, "images"), _ptr(labels, torch.uint8, "labels")
    a.x, a.scale, a.g = _ptr(x, name="x"), _ptr(scale, name="scale"), _ptr(g, name="g")
    a.f = _ptr(f, torch.float64, "f")
    a.idx_out = _ptr(idx_out, torch.int32, "idx_out")
    a.workspace = _ptr(workspace, torch.uint8, "workspace")
    a.workspace_bytes = workspace.numel()
    _lib.check(_lib.lib().l2o_mnist_conv_grad(C.byref(a), _stream()), "l2o_mnist_conv_grad")


def cifar_conv_fits(batch) -> bool:
    """Whether l2o_cifar_conv_grad takes this batch size: 1..1024."""
    return 1 <= int(batch) <= _lib.CIFAR_CONV_MAX_BATCH


def cifar_conv_workspace_bytes(batch) -> int:
    """Bytes of device workspace l2o_cifar_conv_grad needs at this batch size (the library allocates nothing)."""
    n = int(_lib.lib().l2o_cifar_conv_workspace_bytes(int(batch)))
    if n < 0:
        raise L2OError(f"cifar_conv_workspace_bytes: batch {batch} is outside 1..{_lib.CIFAR_CONV_MAX_BATCH}")
    return n


def cifar_conv_workspace_layout(batch) -> dict:
    """Byte offsets in the l2o_cifar_conv_grad workspace of z1, z2, the batch-norm constants and dlogits, the values
    its ReLU and max-pool decisions come from (include/l2o_b200.h)."""
    off = (C.c_int64 * _lib.CIFAR_CONV_LAYOUT)()
    _lib.check(_lib.lib().l2o_cifar_conv_workspace_layout(int(batch), off), "l2o_cifar_conv_workspace_layout")
    return dict(zip(("z1", "z2", "bn", "dl"), (int(v) for v in off)))


def _cifar_args(cls, name, coords, images, labels, x, g, batch, seed, counter, workspace, f, scale, idx_out):
    """The checked argument struct of a CIFAR-10 producer (l2o_cifar_conv_grad, l2o_nas_grad)."""
    a = cls()
    a.batch, a.num_examples = int(batch), int(images.shape[0])
    a.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    if images.numel() != a.num_examples * _lib.CIFAR_INPUT or labels.numel() != a.num_examples:
        raise L2OError(f"{name}: images must be [N, 3072] and labels [N]")
    for what, t in (("x", x), ("g", g), ("scale", scale)):
        if t is not None and t.numel() != coords:
            raise L2OError(f"{name}: {what} has {t.numel()} elements, the network has {coords}")
    if idx_out is not None and idx_out.numel() != a.batch:
        raise L2OError(f"{name}: idx_out has {idx_out.numel()} elements, batch is {a.batch}")
    if counter.numel() != 1:
        raise L2OError(f"{name}: counter must be one int64 element")
    a.counter = _ptr(counter, torch.int64, "counter")
    a.images, a.labels = _ptr(images, torch.uint8, "images"), _ptr(labels, torch.uint8, "labels")
    a.x, a.scale, a.g = _ptr(x, name="x"), _ptr(scale, name="scale"), _ptr(g, name="g")
    a.f = _ptr(f, torch.float64, "f")
    a.idx_out = _ptr(idx_out, torch.int32, "idx_out")
    a.workspace = _ptr(workspace, torch.uint8, "workspace")
    a.workspace_bytes = workspace.numel()
    return a


def cifar_conv_grad(images, labels, x, g, batch, seed, counter, workspace, f=None, scale=None, idx_out=None):
    """f and df/dx of problems.cifar10 (DM/problems.py:369-458, batch norm on) at a fresh batch in one launch.
    images [N, 3072] (each row the record's [3][32][32] planes) and labels [N] uint8; x, g and scale the flat
    13,610-float arena of the ConvNet's variables in creation order; ``counter`` a one-element int64 device tensor the
    call reads and advances (the batch is drawn as mnist_grad draws it); ``workspace`` a uint8 device tensor of at
    least cifar_conv_workspace_bytes(batch) bytes; writes f (fp64 scalar) and the indices drawn into ``idx_out``
    (int32 [batch]) if given."""
    a = _cifar_args(_lib.CifarConvArgs, "cifar_conv_grad", _lib.CIFAR_CONV_COORDS, images, labels, x, g, batch, seed,
                    counter, workspace, f, scale, idx_out)
    _lib.check(_lib.lib().l2o_cifar_conv_grad(C.byref(a), _stream()), "l2o_cifar_conv_grad")


def nas_fits(batch) -> bool:
    """Whether l2o_nas_grad takes this batch size: 1..1024."""
    return 1 <= int(batch) <= _lib.NAS_MAX_BATCH


def nas_workspace_bytes(batch) -> int:
    """Bytes of device workspace l2o_nas_grad needs at this batch size (the library allocates nothing)."""
    n = int(_lib.lib().l2o_nas_workspace_bytes(int(batch)))
    if n < 0:
        raise L2OError(f"nas_workspace_bytes: batch {batch} is outside 1..{_lib.NAS_MAX_BATCH}")
    return n


def nas_workspace_layout(batch) -> dict:
    """Byte offsets in the l2o_nas_grad workspace of the four pre-batch-norm maps, the batch-norm constants and
    dlogits, the values its ReLU decisions come from (include/l2o_b200.h)."""
    off = (C.c_int64 * _lib.NAS_LAYOUT)()
    _lib.check(_lib.lib().l2o_nas_workspace_layout(int(batch), off), "l2o_nas_workspace_layout")
    return dict(zip(("z0", "za", "z1", "zb", "bn", "dl"), (int(v) for v in off)))


def nas_grad(images, labels, x, g, batch, seed, counter, workspace, f=None, scale=None, idx_out=None):
    """f and df/dx of problems.nas (DM/problems.py:540-634, batch norm on) at a fresh batch in one launch; the
    arguments as cifar_conv_grad's, x, g and scale the flat 7,578-float arena of the cell's variables in creation
    order, ``workspace`` at least nas_workspace_bytes(batch) bytes."""
    a = _cifar_args(_lib.NasArgs, "nas_grad", _lib.NAS_COORDS, images, labels, x, g, batch, seed, counter, workspace,
                    f, scale, idx_out)
    _lib.check(_lib.lib().l2o_nas_grad(C.byref(a), _stream()), "l2o_nas_grad")


_graph_replayed = 0  # kernels of this library launched through CUDA-graph replays (not visible to the C-side counter)


def note_graph_replay(kernels_in_graph: int):
    global _graph_replayed
    _graph_replayed += int(kernels_in_graph)


def launch_count() -> int:
    """Kernels of this library launched so far: direct C-ABI launches + kernels replayed inside captured graphs."""
    return int(_lib.lib().l2o_launch_count()) + _graph_replayed


def replay_loop(owner, body, objective, var_list, num_steps: int, cuda_graph: bool, kernels_per_step: int, what: str):
    """The ``minimize`` loop of the learned optimizers: ``num_steps`` calls of ``body()`` (objective, gradients, one
    optimizer step; returns the detached objective).  Returns the objective values as floats (one device->host read).

    With ``cuda_graph`` and at least 4 steps, two eager iterations (slot creation, library warm-up) are followed by one
    iteration captured into a CUDA graph and replayed; the graph is cached on ``owner`` for the same objective and
    variables.  A failed capture falls back to the same kernels, eagerly, with a warning."""
    objs = []
    n_eager = num_steps if (not cuda_graph or num_steps < 4) else 2
    for _ in range(n_eager):
        objs.append(body())
    remaining = num_steps - n_eager
    if remaining > 0:
        # The cache holds STRONG references to the objective and the variables and compares by identity: an id()
        # recycled by the allocator after the old closure died can never alias a new objective.  Tensors the
        # objective closes over are baked into the graph by address - update them in place between calls.
        key = (objective, tuple(var_list))
        old = getattr(owner, "_graph_key", None)
        same = (old is not None and old[0] is objective and len(old[1]) == len(var_list)
                and all(a is b for a, b in zip(old[1], var_list)))
        if not same:
            try:
                import gc
                gc.collect()   # no finaliser (old CUDAGraph pools, handles) may run inside the capture
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    static_loss = body()
                owner._graph, owner._graph_loss, owner._graph_key = graph, static_loss, key
            except Exception as e:   # capture not possible for this objective: same kernels, eagerly
                import warnings
                warnings.warn("CUDA-graph capture of the %s step failed (%r); staying eager" % (what, e))
                torch.cuda.synchronize()
                owner._graph_key = None
                for _ in range(remaining):
                    objs.append(body())
                remaining = 0
        for _ in range(remaining):
            owner._graph.replay()
            note_graph_replay(kernels_per_step)
            objs.append(owner._graph_loss.clone())
    return [float(o) for o in torch.stack(objs).cpu()]
