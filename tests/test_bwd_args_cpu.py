"""CPU-only: l2o_unroll_bwd rejects a checkpoint arena that is not 16-byte aligned, on every engine, before it touches
the device.  Both BPTT engines read checkpoint rows 16 bytes at a time (FFMA float4 loads, tensor-core TMA bulk
copies), so an arena at an odd float offset, such as a tensor view, must be refused rather than launched."""
import ctypes
import os

import pytest

from open_l2o_b200 import _lib


@pytest.mark.parametrize("preprocess,options", [("identity", None), ("LogAndSign", {"k": 5})])
def test_unroll_bwd_rejects_misaligned_ckpt(preprocess, options):
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    from open_l2o_b200.engine import ENGINE_AUTO, ENGINE_FFMA, ENGINE_TC, NetHandle
    h = NetHandle(layers=(20, 20), preprocess_name=preprocess, preprocess_options=options)
    L = _lib.lib()
    a = _lib.BwdArgs()
    a.n, a.T = 19_021, 5
    # placeholder addresses: validation must return before any of them is dereferenced
    a.theta, a.in_seq, a.g_rec, a.dtheta = 0x10000, 0x20000, 0x30000, 0x40000
    for engine in (ENGINE_AUTO, ENGINE_FFMA, ENGINE_TC):
        h.set_engine(engine)
        for off in (4, 8, 12):
            a.ckpt = 0x50000 + off
            assert L.l2o_unroll_bwd(h._h, ctypes.byref(a), None) == _lib.L2O_E_INVALID, (engine, off)
