"""Second-order meta-gradients (``use_second_derivatives``), CPU side: the oracles' second-order meta-gradient against
central finite differences of the meta-objective, and the C-ABI checks of the new ``d_g`` output.  The oracle
meta-gradient functions here are shared with tests/test_second_order_gpu.py."""
import ctypes
import inspect
import math
import os

import pytest
import torch

from oracle import crnn_oracle as CR
from oracle import hrnn_oracle as H
from open_l2o_b200 import _lib


def _unrolled_objectives(step, objective, params, states, T, second, fresh):
    """The unrolled loop of TrainableOptimizer.train (SC/optimizer/trainable_optimizer.py:263-401) over an oracle's
    step(params, grads, states) -> (params, states).  The optimizee gradient is a constant (stop_gradient) unless
    `second`, where it keeps its graph wherever the parameters depend on theta (every step but the first of a fresh
    unroll).  Returns (objective values, final params, final states)."""
    objs = []
    for t in range(T):
        if second and params[0].requires_grad:
            f = objective(params)
            grads = torch.autograd.grad(f, params, create_graph=True)
        else:
            leaf = [p.detach().requires_grad_(True) for p in params]
            f = objective(leaf)
            grads = [g.detach() for g in torch.autograd.grad(f, leaf)]
            f = objective(params) if (t > 0 or not fresh) else f.detach()
        objs.append(f)
        params, states = step(params, grads, states)
    return objs, params, states


def _meta(objs, f0):
    allo = torch.stack([o.reshape(()) for o in objs])
    return torch.log(allo / (f0 + 1e-6) + 1e-6).mean()


def hrnn_oracle_meta(theta, objective, init, llr, T, second, dtype=torch.float64, carry=None, initial_obj=None,
                     need_grad=True):
    """(meta, d meta / d theta, carry) of one HierarchicalRNN unroll through oracle/hrnn_oracle.py in `dtype`: from
    `init` with the log learning rates `llr`, or from a detached `carry` (truncated BPTT) normalised by `initial_obj`."""
    th = theta.to(dtype).clone().requires_grad_(True)
    P = H.unpack_theta(th)
    if carry is None:
        params = [p.to(dtype) for p in init]
        states, off = [], 0
        for p in params:
            st = H.initial_state(P, p, torch.Generator().manual_seed(0))
            st["log_learning_rate"] = llr[off:off + p.numel()].to(dtype).reshape(-1, 1)
            off += p.numel()
            states.append(st)
        glob = H.initial_global_state(P, dtype)
    else:
        params = [p.detach() for p in carry[0]]
        states = [{k: v.detach() for k, v in st.items()} for st in carry[1]]
        glob = carry[2].detach()
    box = [glob]

    def step(ps, gs, sts):
        ps, sts, box[0], _ = H.step(th, ps, gs, sts, box[0])
        return ps, sts
    objs, params, states = _unrolled_objectives(step, objective, params, states, T, second, carry is None)
    f0 = objs[0].detach() if initial_obj is None else initial_obj
    meta = _meta(objs, f0)
    g = torch.autograd.grad(meta, th)[0] if need_grad else None
    return meta.detach(), g, (params, states, box[0], f0)


def crnn_oracle_meta(theta, objective, init, lr0, T, second, dtype=torch.float64, carry=None, initial_obj=None,
                     need_grad=True):
    """As hrnn_oracle_meta, for the CoordinatewiseRNN (oracle/crnn_oracle.py) with initial learning rates `lr0`."""
    th = theta.to(dtype).clone().requires_grad_(True)
    P = CR.unpack_theta(th)
    if carry is None:
        params = [p.to(dtype) for p in init]
        states, off = [], 0
        for p in params:
            st = CR.initial_state(P, p.numel(), torch.Generator(), dtype=dtype)
            st["learning_rate"] = lr0[off:off + p.numel()].to(dtype).reshape(-1, 1)
            off += p.numel()
            states.append(st)
    else:
        params = [p.detach() for p in carry[0]]
        states = [{k: v.detach() for k, v in st.items()} for st in carry[1]]

    def step(ps, gs, sts):
        ps, sts, _ = CR.step(th, ps, gs, sts)
        return ps, sts
    objs, params, states = _unrolled_objectives(step, objective, params, states, T, second, carry is None)
    f0 = objs[0].detach() if initial_obj is None else initial_obj
    meta = _meta(objs, f0)
    g = torch.autograd.grad(meta, th)[0] if need_grad else None
    return meta.detach(), g, (params, states, None, f0)


def curved_problem(shapes, seed, dtype=torch.float64, device="cpu", cos_weight=0.3):
    """sum over tensors of mean((p - target)^2) + cos_weight mean(cos 3p): a Hessian with a strongly varying diagonal,
    so the optimizee's curvature term of the meta-gradient is far from zero."""
    gen = torch.Generator().manual_seed(seed)
    tgt = [torch.randn(s, generator=gen, dtype=torch.float64).to(device=device, dtype=dtype) for s in shapes]

    def objective(params):
        return sum(((p - t) ** 2).mean() + cos_weight * torch.cos(3.0 * p).mean() for p, t in zip(params, tgt))
    init = [torch.randn(s, generator=gen, dtype=torch.float64) * 0.5 for s in shapes]
    return objective, init


TINY = [(3,), (2, 2)]


def _fd_check(meta_fn, theta, n_dirs, seed):
    """Directional derivatives of the second- and first-order oracle meta-gradients against central differences."""
    _, g2, _ = meta_fn(theta, True)
    _, g1, _ = meta_fn(theta, False)
    gen = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n_dirs):
        v = torch.randn(theta.numel(), generator=gen, dtype=torch.float64)
        v = v / v.norm()
        eps = 1e-5
        fp = float(meta_fn(theta.double() + eps * v, False, need_grad=False)[0])
        fm = float(meta_fn(theta.double() - eps * v, False, need_grad=False)[0])
        fd = (fp - fm) / (2 * eps)
        out.append((fd, float(g2 @ v), float(g1 @ v)))
    return out


def _assert_fd(rows):
    for fd, so, fo in rows:
        scale = max(abs(fd), 1e-8)
        err2, err1 = abs(so - fd) / scale, abs(fo - fd) / scale
        assert err2 <= 1e-6, (fd, so, fo)            # second order: the derivative of the meta-objective
        assert err1 >= 1e3 * max(err2, 1e-9), (fd, so, fo)   # first order misses it: the problem exercises the term


def test_hrnn_oracle_second_order_matches_finite_differences():
    """T = 3 on two tiny tensors, generic weights, log learning rates in [-2.5, -1] (well inside the +-33 clip, whose
    straight-through gradient is not the derivative)."""
    from tests.helpers import hrnn_generic_theta
    objective, init = curved_problem(TINY, seed=2)
    n = sum(p.numel() for p in init)
    llr = torch.rand(n, generator=torch.Generator().manual_seed(3), dtype=torch.float64) * 1.5 - 2.5
    theta = hrnn_generic_theta(5, dtype=torch.float64)

    def meta_fn(th, second, need_grad=True):
        return hrnn_oracle_meta(th, objective, init, llr, 3, second, need_grad=need_grad)
    _assert_fd(_fd_check(meta_fn, theta, 3, seed=0))


def test_crnn_oracle_second_order_matches_finite_differences():
    """T = 3 on two tiny tensors, generic weights.  The initial learning rates are large (e^1 .. e^2) because the
    CoordinatewiseRNN's first updates are small: lr' delta with delta = h3 . Wu."""
    from tests.test_crnn_gpu import crnn_generic_theta
    objective, init = curved_problem(TINY, seed=4)
    n = sum(p.numel() for p in init)
    lr0 = torch.exp(torch.rand(n, generator=torch.Generator().manual_seed(5), dtype=torch.float64) + 1.0)
    theta = crnn_generic_theta(7, dtype=torch.float64)

    def meta_fn(th, second, need_grad=True):
        return crnn_oracle_meta(th, objective, init, lr0, 3, second, need_grad=need_grad)
    _assert_fd(_fd_check(meta_fn, theta, 3, seed=1))


def test_trainers_take_use_second_derivatives_default_off():
    """The trainers' argument defaults to the first-order meta-gradient (the reference's default is True)."""
    from open_l2o_b200 import crnn_train, hrnn_train
    for cls in (hrnn_train.MetaTrainer, crnn_train.MetaTrainer):
        assert inspect.signature(cls.__init__).parameters["use_second_derivatives"].default is False


def test_crnn_bwd_rejects_misaligned_or_overlapping_d_g():
    """l2o_crnn_bwd validates d_g before any CUDA call: 4-byte alignment, and no byte shared with another buffer."""
    assert [f[0] for f in _lib.CrnnBwdArgs._fields_][-1] == "d_g"
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    n, planes, n_theta = 4, 103, 6402
    sizes = dict(theta=4 * n_theta, g=4 * n, state_old=4 * planes * n, d_state_new=4 * planes * n, d_update=4 * n,
                 d_state_old=4 * planes * n, d_theta=8 * n_theta)
    bufs = {k: (ctypes.c_double * (b // 8 + 4))() for k, b in sizes.items()}   # host memory: never reaches a kernel
    args = {k: ctypes.addressof(b) for k, b in bufs.items()}
    E = _lib.L2O_E_INVALID
    own = (ctypes.c_double * 4)()
    call = lambda d_g: L.l2o_crnn_bwd(ctypes.byref(_lib.CrnnBwdArgs(n=n, d_g=d_g, **args)), None)
    assert call(ctypes.addressof(own) + 2) == E
    for k, base in args.items():
        for d_g in (base, base + sizes[k] - 4, base - 4 * (n - 1)):   # first byte, last float, straddling the start
            assert call(d_g) == E, (k, d_g - base)
