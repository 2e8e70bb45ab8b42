"""CPU-only: the dense (KernelDeepLSTM) entry points l2o_dense_create / l2o_dense_step / l2o_dense_unroll_bwd validate
their arguments before any CUDA call.  The step and BPTT calls get placeholder addresses that are never valid device
pointers, so a check that came after a launch would fault instead of returning its status."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import l2o_oracle as orc
from open_l2o_b200 import _lib

PRE_IDENTITY, PRE_LOGSIGN, PRE_FC = 0, 1, 2


@pytest.fixture(scope="module")
def L():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    return _lib.lib()


def _desc(layers=(20,), n_in=9, n_out=9, pre=PRE_IDENTITY, tanh=0):
    d = _lib.DenseDesc()
    d.n_layers = len(layers)
    for i, h in enumerate(layers[:2]):
        d.hidden[i] = h
    d.n_in, d.n_out, d.preprocess = n_in, n_out, pre
    d.logsign_k, d.scale, d.tanh_output = 5.0, 0.1, tanh
    return d


def _create(L, d):
    h = C.c_void_p()
    rc = L.l2o_dense_create(C.byref(h), C.byref(d))
    if rc == _lib.L2O_OK:
        assert h.value
    return rc, h


@pytest.mark.parametrize("kw", [dict(layers=(20, 20, 20)), dict(n_in=0), dict(n_out=0)])
def test_dense_create_rejects_invalid(L, kw):
    assert _create(L, _desc(**kw))[0] == _lib.L2O_E_INVALID, kw


def test_dense_create_rejects_negative_layer_count(L):
    d = _desc()
    d.n_layers = -1
    assert _create(L, d)[0] == _lib.L2O_E_INVALID
    d.n_layers = 3
    assert _create(L, d)[0] == _lib.L2O_E_INVALID
    assert L.l2o_dense_create(None, C.byref(_desc())) == _lib.L2O_E_INVALID
    assert L.l2o_dense_create(C.byref(C.c_void_p()), None) == _lib.L2O_E_INVALID


@pytest.mark.parametrize("kw", [dict(pre=PRE_FC), dict(layers=(0,)), dict(layers=(33,)), dict(layers=(20, 33)),
                                dict(layers=(20, 0)), dict(pre=PRE_LOGSIGN, n_in=65), dict(n_in=129),
                                dict(n_out=65)])
def test_dense_create_rejects_unsupported(L, kw):
    assert _create(L, _desc(**kw))[0] == _lib.L2O_E_UNSUPPORTED, kw


@pytest.mark.parametrize("layers,n_in,n_out,pre", [((32, 32), 64, 64, PRE_LOGSIGN), ((32,), 128, 64, PRE_IDENTITY),
                                                   ((), 16, 16, PRE_LOGSIGN), ((1, 32), 6, 6, PRE_IDENTITY),
                                                   ((20,), 128, 3, PRE_IDENTITY), ((20, 20), 9, 9, PRE_IDENTITY)])
def test_dense_create_edges_and_counts(L, layers, n_in, n_out, pre):
    rc, h = _create(L, _desc(layers, n_in, n_out, pre))
    assert rc == _lib.L2O_OK
    try:
        shapes = orc.kernel_net_shapes([n_in], layers, pre == PRE_LOGSIGN)
        if n_out != n_in:   # the oracle's Linear has K outputs; a dense net may have any n_out
            f_top = shapes[-2][2][0]
            shapes = shapes[:-2] + [("linear", "w", (f_top, n_out)), ("linear", "b", (n_out,))]
        n_theta = sum(int(np.prod(s)) for _, _, s in shapes)
        assert L.l2o_dense_theta_count(h) == n_theta
        assert L.l2o_dense_state_floats(h) == 2 * sum(layers)
    finally:
        L.l2o_dense_destroy(h)


def test_dense_theta_count_null_handle(L):
    assert L.l2o_dense_theta_count(None) == _lib.L2O_E_INVALID
    assert L.l2o_dense_state_floats(None) == _lib.L2O_E_INVALID


def _step_args(**kw):
    a = _lib.DenseStepArgs()
    a.rows = 300
    a.theta, a.in_, a.state_in, a.state_out, a.x, a.delta = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000, 0x60000
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("kw", [dict(rows=-1), dict(theta=None), dict(in_=None), dict(state_in=None),
                                dict(state_out=None)])
def test_dense_step_rejects_invalid(L, kw):
    rc, h = _create(L, _desc((20, 20)))
    assert rc == _lib.L2O_OK
    try:
        assert L.l2o_dense_step(h, C.byref(_step_args(**kw)), None) == _lib.L2O_E_INVALID, kw
        assert L.l2o_dense_step(None, C.byref(_step_args()), None) == _lib.L2O_E_INVALID
        assert L.l2o_dense_step(h, None, None) == _lib.L2O_E_INVALID
    finally:
        L.l2o_dense_destroy(h)


def test_dense_step_rows_zero_launches_nothing(L):
    """rows = 0 is a valid empty call; with no LSTM layer (SF = 0) the state pointers may be null."""
    rc, h = _create(L, _desc((), 16, 16, PRE_LOGSIGN))
    assert rc == _lib.L2O_OK
    try:
        n0 = L.l2o_launch_count()
        assert L.l2o_dense_step(h, C.byref(_step_args(rows=0, state_in=None, state_out=None)), None) == _lib.L2O_OK
        assert L.l2o_launch_count() == n0
    finally:
        L.l2o_dense_destroy(h)


def _bwd_args(**kw):
    a = _lib.DenseBwdArgs()
    a.rows, a.T = 300, 5
    a.theta, a.in_seq, a.ckpt, a.g_rec, a.labels, a.dtheta = 0x10000, 0x20000, 0x30000, 0x40000, None, 0x60000
    a.n_total = 0
    for k, v in kw.items():
        setattr(a, k, v)
    return a


@pytest.mark.parametrize("kw", [dict(T=-1), dict(rows=-1), dict(in_seq=None), dict(ckpt=None), dict(theta=None),
                                dict(dtheta=None), dict(g_rec=None), dict(g_rec=None, labels=0x50000, n_total=0),
                                dict(g_rec=None, labels=0x50000, n_total=-3)])
def test_dense_unroll_bwd_rejects_invalid(L, kw):
    rc, h = _create(L, _desc((20, 20)))
    assert rc == _lib.L2O_OK
    try:
        assert L.l2o_dense_unroll_bwd(h, C.byref(_bwd_args(**kw)), None) == _lib.L2O_E_INVALID, kw
        assert L.l2o_dense_unroll_bwd(None, C.byref(_bwd_args()), None) == _lib.L2O_E_INVALID
        assert L.l2o_dense_unroll_bwd(h, None, None) == _lib.L2O_E_INVALID
    finally:
        L.l2o_dense_destroy(h)


def test_dense_unroll_bwd_empty_calls_launch_nothing(L):
    """T = 0 (with no input sequence) and rows = 0 are valid empty calls; a Linear-only net needs no checkpoints."""
    rc, h = _create(L, _desc((20, 20)))
    rc0, h0 = _create(L, _desc((), 16, 16, PRE_LOGSIGN))
    assert rc == rc0 == _lib.L2O_OK
    try:
        n0 = L.l2o_launch_count()
        assert L.l2o_dense_unroll_bwd(h, C.byref(_bwd_args(T=0, in_seq=None)), None) == _lib.L2O_OK
        assert L.l2o_dense_unroll_bwd(h, C.byref(_bwd_args(rows=0)), None) == _lib.L2O_OK
        assert L.l2o_dense_unroll_bwd(h, C.byref(_bwd_args(rows=0, g_rec=None, labels=0x50000, n_total=7)),
                                      None) == _lib.L2O_OK
        assert L.l2o_dense_unroll_bwd(h0, C.byref(_bwd_args(rows=0, ckpt=None)), None) == _lib.L2O_OK
        assert L.l2o_launch_count() == n0
    finally:
        L.l2o_dense_destroy(h)
        L.l2o_dense_destroy(h0)
