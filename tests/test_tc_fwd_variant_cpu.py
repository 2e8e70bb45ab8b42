"""CPU-only: which tensor-core forward kernel a call runs.  The full-tile instantiation (l2o_tc_fwd_variant == 1) is
for DM nets on an in-kernel Rastrigin or diagonal quadratic with n a multiple of 64, T >= 1, a plain output layer, and
checkpoints and g_rec both recorded or both not; every other call runs the general kernel (0)."""
import ctypes
import os

import pytest

from open_l2o_b200 import _lib

N_FULL = 64 * 601


def _args(**kw):
    # placeholder addresses: the query reads the argument set only, it never touches the device
    a = _lib.UnrollArgs()
    a.n, a.T = N_FULL, 100
    a.theta, a.state, a.x, a.opt_a, a.opt_b = 0x10000, 0x20000, 0x30000, 0x40000, 0x50000
    a.ckpt, a.g_rec, a.fx = 0x60000, 0x70000, 0x80000
    a.opt_kind = _lib.OPT_RASTRIGIN_SEP
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _variant(handle, **kw):
    return _lib.lib().l2o_tc_fwd_variant(handle._h, ctypes.byref(_args(**kw)))


@pytest.fixture(scope="module")
def nets():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    from open_l2o_b200.engine import NetHandle
    return {"identity": NetHandle(layers=(20, 20)),
            "logsign": NetHandle(layers=(20, 20), preprocess_name="LogAndSign", preprocess_options={"k": 5}),
            "tanh": NetHandle(layers=(20, 20), tanh_output=True),
            "rnnprop": NetHandle(layers=(20, 20), preprocess_name="fc", preprocess_options={"dim": 20}, n_in=2,
                                 tanh_output=True)}


@pytest.mark.parametrize("net", ["identity", "logsign"])
@pytest.mark.parametrize("kind", [_lib.OPT_RASTRIGIN_SEP, _lib.OPT_QUADRATIC_DIAG])
@pytest.mark.parametrize("record", [True, False])
def test_full_tile_forward_is_chosen(nets, net, kind, record):
    rec = {} if record else dict(ckpt=None, g_rec=None)
    assert _variant(nets[net], opt_kind=kind, **rec) == 1
    assert _variant(nets[net], opt_kind=kind, fx=None, **rec) == 1


@pytest.mark.parametrize("why,net,kw", [
    ("ragged n", "identity", dict(n=64 * 600 + 20)),
    ("n below one tile", "identity", dict(n=44)),
    ("T = 0", "identity", dict(T=0)),
    ("checkpoints without g_rec", "identity", dict(g_rec=None)),
    ("g_rec without checkpoints", "identity", dict(ckpt=None)),
    ("recorded deltas", "identity", dict(delta_seq=0x90000)),
    ("imitation labels", "identity", dict(labels=0x90000, imit_loss=0xA0000, n_total=N_FULL)),
    ("tanh output layer", "tanh", {}),
    ("gradients from in_seq", "identity", dict(opt_kind=_lib.OPT_NONE, in_seq=0x90000, x=None, opt_a=None, opt_b=None)),
    ("RNNProp", "rnnprop", dict(m=0x90000, v=0xA0000)),
])
def test_general_forward_is_chosen(nets, why, net, kw):
    assert _variant(nets[net], **kw) == 0, why


def test_query_rejects_what_the_tensor_core_engine_does_not_run(nets):
    assert _variant(nets["identity"], opt_kind=_lib.OPT_QUADRATIC_BATCH, opt_group=64) == _lib.L2O_E_UNSUPPORTED
    assert _lib.lib().l2o_tc_fwd_variant(None, None) == _lib.L2O_E_INVALID
