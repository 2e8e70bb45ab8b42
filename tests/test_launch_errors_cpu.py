"""CPU-only: every launching entry point, called with valid arguments where no CUDA device can be used, returns
L2O_E_CUDA, counts no launch, and leaves an l2o_last_cuda_error() message that starts with its own name.  The device
pointers are placeholder addresses: each call fails at its first CUDA call, before any kernel could read them."""
import ctypes as C
import os

import pytest
import torch

from open_l2o_b200 import _lib

ADDR = [0x100000 * (k + 1) for k in range(16)]   # 256-byte aligned placeholders, one per pointer argument


def _fill(args, names, **scalars):
    for name, addr in zip(names, ADDR):
        setattr(args, name, addr)
    for name, v in scalars.items():
        setattr(args, name, v)
    return C.byref(args)


def _net_call(engine, fn, carry=False):
    def call(L):
        from open_l2o_b200.engine import NetHandle
        h = NetHandle(layers=(20, 20))
        h.set_engine(engine)
        if fn == "l2o_step":
            a = _fill(_lib.StepArgs(), ["theta", "in0", "state_in", "state_out", "x"], n=300)
            return L.l2o_step(h._h, a, None)
        if fn == "l2o_unroll_fwd":
            a = _fill(_lib.UnrollArgs(), ["theta", "in_seq", "state", "x"], n=300, T=5)
            return L.l2o_unroll_fwd(h._h, a, None)
        a = _fill(_lib.BwdArgs(), ["theta", "in_seq", "ckpt", "g_rec", "dtheta"], n=300, T=5)
        if carry:
            return L.l2o_unroll_bwd_carry(h._h, a, _fill(_lib.BwdCarry(), ["d_state", "lam"]), None)
        return L.l2o_unroll_bwd(h._h, a, None)
    return call


def _dense_call(fn):
    def call(L):
        d = _lib.DenseDesc()
        d.n_layers, d.hidden[0], d.n_in, d.n_out, d.preprocess, d.scale = 1, 20, 9, 9, _lib.PRE_IDENTITY, 0.1
        h = C.c_void_p()
        assert L.l2o_dense_create(C.byref(h), C.byref(d)) == _lib.L2O_OK
        try:
            if fn == "l2o_dense_step":
                a = _fill(_lib.DenseStepArgs(), ["theta", "in_", "state_in", "state_out", "x"], rows=300)
                return L.l2o_dense_step(h, a, None)
            a = _fill(_lib.DenseBwdArgs(), ["theta", "in_seq", "ckpt", "g_rec", "dtheta"], rows=300, T=5)
            return L.l2o_dense_unroll_bwd(h, a, None)
        finally:
            L.l2o_dense_destroy(h)
    return call


def _args_call(fn, cls, names, **scalars):
    return lambda L: getattr(L, fn)(_fill(cls(), names, **scalars), None)


def _confocal(L):
    a = _lib.ConfocalArgs()
    a.roi[0] = a.roi[1] = a.roi[2] = 4
    return L.l2o_confocal_grad(_fill(a, ["x", "sim", "g"], batch=2, num_points=3), None)


CASES = {
    "l2o_step[ffma]": ("l2o_step", _net_call(_lib.ENGINE_FFMA, "l2o_step")),
    "l2o_step[tc]": ("l2o_step", _net_call(_lib.ENGINE_TC, "l2o_step")),
    "l2o_unroll_fwd[ffma]": ("l2o_unroll_fwd", _net_call(_lib.ENGINE_FFMA, "l2o_unroll_fwd")),
    "l2o_unroll_fwd[tc]": ("l2o_unroll_fwd", _net_call(_lib.ENGINE_TC, "l2o_unroll_fwd")),
    "l2o_unroll_bwd[ffma]": ("l2o_unroll_bwd", _net_call(_lib.ENGINE_FFMA, "l2o_unroll_bwd")),
    "l2o_unroll_bwd[tc]": ("l2o_unroll_bwd", _net_call(_lib.ENGINE_TC, "l2o_unroll_bwd")),
    "l2o_unroll_bwd_carry[ffma]": ("l2o_unroll_bwd_carry", _net_call(_lib.ENGINE_FFMA, "l2o_unroll_bwd", carry=True)),
    "l2o_unroll_bwd_carry[tc]": ("l2o_unroll_bwd_carry", _net_call(_lib.ENGINE_TC, "l2o_unroll_bwd", carry=True)),
    "l2o_dense_step": ("l2o_dense_step", _dense_call("l2o_dense_step")),
    "l2o_dense_unroll_bwd": ("l2o_dense_unroll_bwd", _dense_call("l2o_dense_unroll_bwd")),
    "l2o_crnn_step": ("l2o_crnn_step", _args_call("l2o_crnn_step", _lib.CrnnStepArgs,
                                                  ["theta", "g", "state_in", "state_out", "x", "update"], n=300)),
    "l2o_crnn_bwd": ("l2o_crnn_bwd", _args_call("l2o_crnn_bwd", _lib.CrnnBwdArgs,
                                                ["theta", "g", "state_old", "d_state_new", "d_update", "d_state_old",
                                                 "d_theta"], n=300)),
    "l2o_tadam_step": ("l2o_tadam_step", _args_call("l2o_tadam_step", _lib.TadamStepArgs,
                                                    ["theta", "g", "state_in", "state_out", "x", "update"], n=300)),
    "l2o_tadam_bwd": ("l2o_tadam_bwd", _args_call("l2o_tadam_bwd", _lib.TadamBwdArgs,
                                                  ["theta", "g", "state_old", "d_state_new", "d_update", "d_state_old",
                                                   "d_theta"], n=300)),
    "l2o_lrsgd_step": ("l2o_lrsgd_step", _args_call("l2o_lrsgd_step", _lib.LrsgdStepArgs,
                                                    ["rates", "g", "itr", "x", "update"], n=300, n_steps=7)),
    "l2o_lrsgd_bwd": ("l2o_lrsgd_bwd", _args_call("l2o_lrsgd_bwd", _lib.LrsgdBwdArgs,
                                                  ["rates", "g", "itr", "d_update", "d_rates"], n=300, n_steps=7)),
    "l2o_lasso_grad": ("l2o_lasso_grad", _args_call("l2o_lasso_grad", _lib.LassoArgs, ["A", "y", "x", "g"],
                                                    batch=2, m=5, n=10)),
    "l2o_confocal_grad": ("l2o_confocal_grad", _confocal),
    "l2o_adam_step": ("l2o_adam_step",
                      lambda L: L.l2o_adam_step(ADDR[0], ADDR[1], ADDR[2], ADDR[3], 300, 1, 1e-3, 0.9, 0.999, 1e-8,
                                                None)),
    "l2o_log_and_sign": ("l2o_log_and_sign", lambda L: L.l2o_log_and_sign(ADDR[0], ADDR[1], 300, 5.0, None)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_failed_call_is_reported_and_not_counted(case):
    if torch.cuda.is_available():
        pytest.skip("needs a machine without a usable CUDA device")
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    name, call = CASES[case]
    # leave another entry point's message behind, so that a call which records nothing cannot pass on a stale one
    CASES["l2o_adam_step" if name == "l2o_log_and_sign" else "l2o_log_and_sign"][1](L)
    before = L.l2o_launch_count()
    assert call(L) == _lib.L2O_E_CUDA
    assert L.l2o_launch_count() == before
    msg = L.l2o_last_cuda_error().decode()
    assert msg.startswith(name + ": "), msg
