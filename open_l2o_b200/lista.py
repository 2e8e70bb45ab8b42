"""Model-based L2O's LISTA family on the sm_90a kernels of ``csrc/l2o_ista.cu`` (MB/ = Model_Base_L2O/ of the
reference): ``Lista``, ``ListaCp``, ``ListaCpss``, ``Alista``, ``Lfista`` and ``Lamp``, grown layer by layer with
``create_cell``.

Every variable of a model lives in one fp32 arena on the device (its gradient in a matching fp64 arena), so one
forward, one loss, one backward and one Adam launch train all layers at once; ``variables`` maps the reference's
variable names to views of the arena.  There is no CPU path: a missing kernel or library is an error.

Deviation: with ``share_W`` the reference's ListaCell scales x_k by ``step_size[layer_id - 1]`` of the scalar it was
handed (MB/models/lista.py:41-42), which raises in TensorFlow; here layer k uses its own s_k, as the coupled cells do.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from typing import Dict, Optional

import numpy as np
import torch

from . import _lib
from .engine import _ptr, _stream

LISTA, COUPLED, LFISTA, LAMP = 0, 1, 2, 3
TASK_SC, TASK_LASSO = 0, 1


def ss_ranks(T: int, n: int, q_per_layer: float, maxq: float) -> np.ndarray:
    """Support-selection rank of each layer: q_k = clip((k+1) q_per_layer, 0, maxq) percent (MB/models/
    lista_cpss.py:65), and tfp.stats.percentile(|z|, 100 - q_k, interpolation='nearest') read as the element at
    index round((n-1) q_k / 100) of |z| sorted in descending order, rounding half to even (MB/models/utils.py:34)."""
    q = np.clip([(t + 1) * q_per_layer for t in range(T)], 0.0, maxq).astype(np.float64)
    return np.clip(np.round((n - 1) * q / 100.0), 0, n - 1).astype(np.int32)


def alista_weight(A: np.ndarray) -> np.ndarray:
    """The analytic ALISTA weight: column i = (A A^T)^-1 a_i / (a_i^T (A A^T)^-1 a_i), the minimiser of ||W^T A||_F
    subject to diag(W^T A) = 1.  The reference loads it from a W.npy it does not ship (MB/train.py:115-118)."""
    A64 = np.asarray(A, np.float64)
    G = np.linalg.solve(A64 @ A64.T, A64)          # (A A^T)^-1 A, [M, N]
    return (G / np.sum(A64 * G, axis=0, keepdims=True)).astype(np.float32)


def make_data(M: int, N: int, n, p: float = 0.1, noise: Optional[float] = None, seed: int = 0,
              out_dir: Optional[str] = None):
    """Synthetic sparse-coding data (the LISTA papers' convention): A ~ N(0, 1/M) with unit-norm columns,
    x = Bernoulli(p) N(0, 1), y = x A^T (+ N(0, noise^2)).  ``n`` = (train, val, test) row counts or one count for all.
    Rows are ``[y | x]``, the reference's data layout.  With ``out_dir`` writes A.npy and {train,val,test}_data.npy."""
    rng = np.random.default_rng(seed)
    n_tr, n_va, n_te = (n, n, n) if np.isscalar(n) else n
    A = rng.normal(0.0, 1.0 / np.sqrt(M), (M, N))
    A = (A / np.linalg.norm(A, axis=0, keepdims=True)).astype(np.float32)
    out = {"A": A}
    for split, rows in (("train", n_tr), ("val", n_va), ("test", n_te)):
        x = (rng.random((rows, N)) < p) * rng.normal(0.0, 1.0, (rows, N))
        y = x @ A.T.astype(np.float64)
        if noise:
            y = y + rng.normal(0.0, noise, y.shape)
        out[split] = np.concatenate([y, x], axis=1).astype(np.float32)
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        np.save(os.path.join(out_dir, "A.npy"), A)
        for split in ("train", "val", "test"):
            np.save(os.path.join(out_dir, split + "_data.npy"), out[split])
    return out


class _IstaModel:
    """What the models share: the variable arena, layer-wise growth and the kernel calls."""

    form = COUPLED

    def __init__(self, A, T, lam, share_W, D, name, device, step_trainable, ss=None, W_const=None):
        if D is not None:
            raise NotImplementedError("the cs task (dictionary D) is not supported")
        A = np.asarray(A, np.float32)
        self.name, self.device = name, torch.device(device)
        self.M, self.N = A.shape
        self.T, self.share_W = int(T), bool(share_W)
        self.lam = lam
        self.scale = 1.001 * np.linalg.norm(A.astype(np.float64), ord=2) ** 2
        self.A = torch.from_numpy(A).to(self.device)
        self.ss_rank = None if ss is None else torch.from_numpy(ss_ranks(self.T, self.N, *ss)).to(self.device)
        self.num_cells = 0
        self._specs = []      # (name, shape, birth layer, initial value)
        self._layout(A, W_const, step_trainable)
        self.one_W = self.share_W or self.W_const is not None   # every layer reads one W matrix
        n = sum(int(np.prod(s)) for _, s, _, _ in self._specs)
        self.params = torch.empty(n, dtype=torch.float32, device=self.device)
        self.grads = torch.zeros(n, dtype=torch.float64, device=self.device)
        self.variables: Dict[str, torch.Tensor] = {}
        self.births: Dict[str, int] = {}
        off = 0
        for vname, shape, birth, init in self._specs:
            k = int(np.prod(shape))
            view = self.params[off:off + k].view(shape)
            view.copy_(torch.as_tensor(np.broadcast_to(init, shape).copy(), dtype=torch.float32))
            self.variables[vname], self.births[vname] = view, birth
            off += k
        self._bufs = {}

    # -- layout --------------------------------------------------------------------------------------------------
    def _w_slots(self):
        return 1 if self.share_W else self.T

    def _layout(self, A, W_const, step_trainable):
        nm, T = self.name, self.T
        self.W_const = None if W_const is None else torch.as_tensor(np.asarray(W_const, np.float32)).to(self.device)
        if W_const is None:
            self._layout_W(A)
        theta0 = np.float32(self.lam / self.scale)
        self._specs += [(nm + "_theta%d" % (i + 1), (1,), i, theta0) for i in range(T)]
        if step_trainable:
            self._specs += [(nm + "_step_size%d" % (i + 1), (1,), i, np.float32(1.0)) for i in range(T)]

    def _layout_W(self, A):
        """The coupled cells' W: one per layer, or one shared, each A initially (MB/models/lista_cpss.py:68-74)."""
        if self.share_W:
            self._specs.append((self.name + "_W", A.shape, 0, A))
        else:
            self._specs += [(self.name + "_W%d" % (i + 1), A.shape, i, A) for i in range(self.T)]

    def _theta_block(self):
        """theta_1 .. theta_T (LAMP: lam_1 .. lam_T) as one span of the arena."""
        return self._block(self.name + "_theta1", self.T)

    def _theta_grad(self):
        return self._grad_span(self.name + "_theta1", self.T)

    def _span(self, arena, vname, count):
        """The arena span of `count` consecutive variables starting at the one named `vname`."""
        v = self.variables[vname]
        off = (v.data_ptr() - self.params.data_ptr()) // 4
        return arena[off:off + count * v.numel()]

    def _block(self, vname, count):
        return self._span(self.params, vname, count)

    def _grad_span(self, vname, count):
        return self._span(self.grads, vname, count)

    def _second(self):
        """(W2, dW2) for the kernel arguments: LFISTA's Wm slots."""
        return None, None

    def _weights(self):
        """(W pointer, dW span or None, B1, dB1, step, dstep) for the kernel arguments."""
        nm = self.name
        if self.W_const is not None:
            W, dW = self.W_const, None
        else:
            first = nm + ("_W" if self.share_W else "_W1")
            W, dW = self._block(first, self._w_slots()), self._grad_span(first, self._w_slots())
        if nm + "_step_size1" in self.variables:
            step, dstep = self._block(nm + "_step_size1", self.T), self._grad_span(nm + "_step_size1", self.T)
        else:
            step = dstep = None
        return W, dW, None, None, step, dstep

    # -- reference surface ---------------------------------------------------------------------------------------
    def create_cell(self, layer_id: int):
        if layer_id != self.num_cells or layer_id >= self.T:
            raise ValueError("cells are created in order 0..T-1 (got %d after %d)" % (layer_id, self.num_cells))
        self.num_cells += 1

    def layer_variables(self, layer_id: int):
        """Names of the trainable variables created with layer `layer_id` (Keras' layer.trainable_variables that
        are new at that layer, MB/train.py:268-270)."""
        return [n for n, b in self.births.items() if b == layer_id]

    def __call__(self, inputs: torch.Tensor) -> torch.Tensor:
        """The Keras model's output: [y, x_1, ..., x_k] for the k cells created so far (MB/train.py:249-252)."""
        y = inputs[:, :self.M].contiguous()
        xs = self.forward(y, self.num_cells)
        return torch.cat([y] + [xs[i] for i in range(self.num_cells)], dim=1)

    # -- kernels -------------------------------------------------------------------------------------------------
    def _bufs_for(self, B, record):
        key = (B, record)
        if key not in self._bufs:
            z = lambda *s, dt=torch.float32: torch.empty(*s, dtype=dt, device=self.device)
            b = {"xs": z(self.T, B, self.N)}
            if record:
                b["zs"] = z(self.T, B, self.N)
                b["rs"] = z(self.T, B, self.M) if self.form in (COUPLED, LAMP) else None
                b["rowrec"] = z(self.T, B, 2) if self.form == LAMP else None
                b["sel"] = z(self.T, B, self.N, dt=torch.uint8) if self.ss_rank is not None else None
                b["d_xk"] = z(B, self.N)
                b["loss"] = z(B, dt=torch.float64)
            self._bufs[key] = b
        return self._bufs[key]

    def _args(self, y, ldy, B, k1, bufs, record):
        W, _, B1, _, step, _ = self._weights()
        a = _lib.IstaArgs()
        a.form, a.batch, a.m, a.n, a.num_layers, a.k0, a.k1 = self.form, B, self.M, self.N, self.T, 0, k1
        a.share_W = int(self.one_W)
        a.A, a.B1, a.W, a.W2 = _ptr(self.A), _ptr(B1), _ptr(W), _ptr(self._second()[0])
        a.theta = _ptr(self._theta_block())
        a.step = _ptr(step)
        a.ss_rank = None if self.ss_rank is None else _ptr(self.ss_rank, torch.int32, "ss_rank")
        a.y, a.ldy = y.data_ptr(), ldy
        a.xs = _ptr(bufs["xs"])
        if record:
            a.zs, a.rs, a.rowrec = _ptr(bufs["zs"]), _ptr(bufs["rs"]), _ptr(bufs["rowrec"])
            a.sel = _ptr(bufs["sel"], torch.uint8, "sel")
        return a

    def _rows(self, data):
        if not (data.is_cuda and data.dtype == torch.float32 and data.dim() == 2 and data.stride(1) == 1):
            raise _lib.L2OError("expected a float32 CUDA matrix with unit column stride")
        return data.shape[0], data.stride(0)

    def forward(self, data: torch.Tensor, k1: Optional[int] = None, record: bool = False) -> torch.Tensor:
        """x_1 .. x_k1 as [k1, B, N] (a view of a reused buffer) from rows whose first M columns are y."""
        k1 = self.num_cells if k1 is None else k1
        B, ld = self._rows(data)
        bufs = self._bufs_for(B, record)
        a = self._args(data, ld, B, k1, bufs, record)
        _lib.check(_lib.lib().l2o_ista_fwd(C.byref(a), _stream()), "l2o_ista_fwd")
        return bufs["xs"][:k1]

    def loss_and_grad(self, data: torch.Tensor, task: int, lasso_lam: float = 0.0, gscale=None,
                      k1: Optional[int] = None) -> torch.Tensor:
        """Forward over layers [0, k1), the loss of x_k1 against the rows [y | x_true], and the gradient of every
        variable into ``grads`` (times gscale[birth layer]).  Returns the per-row losses [B] (fp64)."""
        k1 = self.num_cells if k1 is None else k1
        B, ld = self._rows(data)
        bufs = self._bufs_for(B, True)
        a = self._args(data, ld, B, k1, bufs, True)
        L = _lib.lib()
        _lib.check(L.l2o_ista_fwd(C.byref(a), _stream()), "l2o_ista_fwd")
        la = _lib.IstaLossArgs()
        la.task, la.batch, la.m, la.n = task, B, self.M, self.N
        la.A, la.y, la.ldy = _ptr(self.A), data.data_ptr(), ld
        la.x_true, la.ldx = data.data_ptr() + 4 * self.M, ld
        la.x, la.lam = _ptr(bufs["xs"][k1 - 1]), float(lasso_lam)
        la.d_x, la.loss = _ptr(bufs["d_xk"]), _ptr(bufs["loss"], torch.float64, "loss")
        _lib.check(L.l2o_ista_loss_grad(C.byref(la), _stream()), "l2o_ista_loss_grad")
        self.backward(a, bufs["d_xk"], gscale)
        return bufs["loss"]

    def backward(self, a, d_xk, gscale=None, d_x_in=None):
        _, dW, _, dB1, _, dstep = self._weights()
        nbytes = C.c_size_t()
        L = _lib.lib()
        _lib.check(L.l2o_ista_workspace_bytes(C.byref(a), C.byref(nbytes)), "l2o_ista_workspace_bytes")
        key = ("scratch", nbytes.value)
        if key not in self._bufs:
            self._bufs[key] = torch.empty((nbytes.value + 3) // 4, dtype=torch.float32, device=self.device)
        g = _lib.IstaGrads()
        g.d_xk, g.d_x_in = _ptr(d_xk), _ptr(d_x_in)
        g.dW, g.dB1 = _ptr(dW, torch.float64, "dW"), _ptr(dB1, torch.float64, "dB1")
        g.dW2 = _ptr(self._second()[1], torch.float64, "dW2")
        g.dtheta = _ptr(self._theta_grad(), torch.float64, "dtheta")
        g.dstep = _ptr(dstep, torch.float64, "dstep")
        g.gscale = _ptr(gscale)
        g.scratch = _ptr(self._bufs[key])
        _lib.check(L.l2o_ista_bwd(C.byref(a), C.byref(g), _stream()), "l2o_ista_bwd")

    def state_dict(self):
        return {n: v.detach().cpu().numpy().copy() for n, v in self.variables.items()}

    def load_state_dict(self, d):
        for n, v in self.variables.items():
            v.copy_(torch.as_tensor(d[n]).reshape(v.shape))


class Lista(_IstaModel):
    """LISTA (MB/models/lista.py): z_k = y B1^T + s_k x_k W_k^T, B1 = A^T / L, W = I - B1 A, theta = lam / L."""

    form = LISTA

    def __init__(self, A, T, lam, share_W=False, D=None, name="Lista", device="cuda"):
        super().__init__(A, T, lam, share_W, D, name, device, step_trainable=share_W)

    def _w_slots(self):
        return 1 if self.share_W else self.T - 1

    def _layout_W(self, A):
        """B1 = A^T / L and W = I - B1 A, shared or one per layer k >= 1 (MB/models/lista.py:66-76, 91)."""
        M, N = A.shape
        B = (A.T.astype(np.float32) / np.float32(self.scale)).astype(np.float32)
        W = (np.eye(N, dtype=np.float32) - B @ A).astype(np.float32)
        nm = self.name
        self._specs.append((nm + "_B", (N, M), 0, B))
        if self.share_W:
            self._specs.append((nm + "_W", (N, N), 1, W))
        else:
            self._specs += [(nm + "_W%d" % (i + 1), (N, N), i, W) for i in range(1, self.T)]

    def _weights(self):
        nm = self.name
        B1, dB1 = self.variables[nm + "_B"], self._grad_span(nm + "_B", 1)
        if self._w_slots() > 0:
            first = nm + ("_W" if self.share_W else "_W2")
            W, dW = self._block(first, self._w_slots()), self._grad_span(first, self._w_slots())
        else:
            W, dW = None, None
        if self.share_W:
            step, dstep = self._block(nm + "_step_size1", self.T), self._grad_span(nm + "_step_size1", self.T)
        else:
            step = dstep = None
        return W, dW, B1, dB1, step, dstep


class ListaCp(_IstaModel):
    """LISTA-CP (MB/models/lista_cp.py): z_k = x_k + s_k (y - x_k A^T) W_k, W_k = A initially."""

    def __init__(self, A, T, lam, share_W=False, D=None, name="ListaCp", device="cuda"):
        super().__init__(A, T, lam, share_W, D, name, device, step_trainable=share_W)


class ListaCpss(_IstaModel):
    """LISTA-CPSS (MB/models/lista_cpss.py): LISTA-CP with support selection."""

    def __init__(self, A, T, lam, q_per_layer, maxq, share_W=False, D=None, name="ListaCpss", device="cuda"):
        super().__init__(A, T, lam, share_W, D, name, device, step_trainable=share_W, ss=(q_per_layer, maxq))


class Alista(_IstaModel):
    """ALISTA (MB/models/alista.py): the coupled cell with a constant analytic W; trains s_k and theta_k."""

    def __init__(self, A, W, T, lam, q_per_layer, maxq, D=None, name="Alista", device="cuda"):
        super().__init__(A, T, lam, False, D, name, device, step_trainable=True, ss=(q_per_layer, maxq), W_const=W)


def fista_momenta(T: int):
    """m_0 .. m_{T-1} of MB/models/lfista.py: t = [1, 1], t_{i+2} = (1 + sqrt(1 + 4 t_{i+1}^2)) / 2,
    m_i = (t_{i+1} - 1) / t_{i+2}."""
    t, m = [1.0, 1.0], []
    for _ in range(T):
        t.append((1 + math.sqrt(1 + 4 * t[-1] ** 2.0)) / 2)
        m.append((t[-2] - 1) / t[-1])
    return m


class Lfista(_IstaModel):
    """LFISTA (MB/models/lfista.py): z_k = y We^T + x_k Wg_k^T + x_{k-1} Wm_k^T (Wg from layer 1, Wm from layer 2).
    We = A^T / L is one variable shared by every layer; Wg_{k+1} = (1 + m_k) W and Wm_{k+1} = -m_k W with
    W = I - We A.  ``Lfista_Wm2`` belongs to layer 1 but no layer reads it: its gradient is 0.  ``share_W`` is
    accepted and ignored, as in the reference."""

    form = LFISTA

    def __init__(self, A, T, lam, share_W=False, D=None, name="Lfista", device="cuda"):
        super().__init__(A, T, lam, False, D, name, device, step_trainable=False)

    def _layout_W(self, A):
        M, N = A.shape
        B = (A.T.astype(np.float32) / np.float32(self.scale)).astype(np.float32)
        W = (np.eye(N, dtype=np.float32) - B @ A).astype(np.float32)
        m, nm = fista_momenta(self.T), self.name
        self._specs.append((nm + "_We1", (N, M), 0, B))
        self._specs += [(nm + "_Wg%d" % (i + 1), (N, N), i, (W * (1 + m[i])).astype(np.float32))
                        for i in range(1, self.T)]
        self._specs += [(nm + "_Wm%d" % (i + 1), (N, N), i, (-m[i] * W).astype(np.float32)) for i in range(1, self.T)]

    def _second(self):
        if self.T < 2:
            return None, None
        nm = self.name
        return self._block(nm + "_Wm2", self.T - 1), self._grad_span(nm + "_Wm2", self.T - 1)

    def _weights(self):
        nm = self.name
        B1, dB1 = self.variables[nm + "_We1"], self._grad_span(nm + "_We1", 1)
        if self.T < 2:
            return None, None, B1, dB1, None, None
        return self._block(nm + "_Wg2", self.T - 1), self._grad_span(nm + "_Wg2", self.T - 1), B1, dB1, None, None


class Lamp(_IstaModel):
    """LAMP (MB/models/lamp.py): v_k = y - x_k A^T + b_k v_{k-1} (v_0 = y), b_k = ||x_k||_0 / M,
    r_k = x_k + s_k v_k W_k, x_{k+1} = shrink(r_k, max(sqrt(||v_k||^2 / M) lam_k, 0)).  W_k = A / L initially, lam_k =
    lam; the step sizes are trainable only with ``share_W`` (otherwise 1)."""

    form = LAMP

    def __init__(self, A, T, lam, share_W=False, D=None, name="Lamp", device="cuda"):
        super().__init__(A, T, lam, share_W, D, name, device, step_trainable=share_W)

    def _layout(self, A, W_const, step_trainable):
        nm, T = self.name, self.T
        self.W_const = None
        W = (A.astype(np.float32) / np.float32(self.scale)).astype(np.float32)
        if self.share_W:
            self._specs.append((nm + "_W", A.shape, 0, W))
        else:
            self._specs += [(nm + "_W%d" % (i + 1), A.shape, i, W) for i in range(T)]
        self._specs += [(nm + "_lam%d" % (i + 1), (1,), i, np.float32(self.lam)) for i in range(T)]
        if step_trainable:
            self._specs += [(nm + "_step_size%d" % (i + 1), (1,), i, np.float32(1.0)) for i in range(T)]

    def _theta_block(self):
        return self._block(self.name + "_lam1", self.T)

    def _theta_grad(self):
        return self._grad_span(self.name + "_lam1", self.T)

    def __call__(self, inputs: torch.Tensor) -> torch.Tensor:
        """The Keras model's output: [y, v_0, x_1, v_1, x_2, ..., v_{k-1}, x_k] (output_interval M + N)."""
        y = inputs[:, :self.M].contiguous()
        k = self.num_cells
        xs = self.forward(y, k, record=True)
        vs = self._bufs_for(y.shape[0], True)["rs"]
        return torch.cat([y] + [t for i in range(k) for t in (vs[i], xs[i])], dim=1)
