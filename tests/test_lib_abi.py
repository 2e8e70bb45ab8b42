"""CPU-only: the C-ABI library loads and exports every symbol include/l2o_b200.h declares."""
import ctypes
import os
import re

import pytest

from open_l2o_b200 import _lib

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "l2o_b200.h")


def _declared():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(l2o_[a-z_0-9]+)\s*\(", src)))


def test_header_and_binding_agree():
    assert _declared() == sorted(_lib.EXPORTS)


def test_library_exports_every_declared_symbol():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built (run __graft_entry__.build())")
    L = ctypes.CDLL(_lib.LIB_PATH)
    for name in _declared():
        assert hasattr(L, name), name
    L.l2o_version.restype = ctypes.c_char_p
    assert b"sm_90a" in L.l2o_version()
    L.l2o_status_string.restype = ctypes.c_char_p
    assert L.l2o_status_string(-2) and L.l2o_launch_count() >= 0


def test_net_create_validates_without_gpu():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    from open_l2o_b200.engine import NetHandle
    h = NetHandle(layers=(20, 20))
    assert h.n_theta == 5061 and h.state_floats == 80
    assert NetHandle(layers=(20, 20), preprocess_name="LogAndSign", preprocess_options={"k": 5}).n_theta == 5141
    assert NetHandle(layers=(20, 20), preprocess_name="fc", preprocess_options={"dim": 20}, n_in=2).n_theta == 6641
    with pytest.raises(_lib.L2OError):
        NetHandle(layers=(33, 5))
    # caller-owned buffers of BASELINE config #5 on one GPU: 1M coordinates x T=100 (32.3 GB of checkpoints)
    fwd, bwd = h.workspace_bytes(1_000_000, 100)
    assert fwd == 4 * (80 * 1_000_000 * 102 + 101 * 1_000_000)
    assert bwd == 4 * (80 * 1_000_000 * 101 + 101 * 1_000_000) + 8 * 5061


def test_product_package_never_imports_oracle():
    root = os.path.dirname(_lib.__file__)
    for dp, _, fs in os.walk(root):
        for f in fs:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle|import_module\([\"']oracle|oracle[./]l2o_oracle", src, re.M), f


def test_hrnn_abi_without_gpu():
    """HierarchicalRNN entry points: constants and argument validation happen before any CUDA call."""
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    assert L.l2o_hrnn_theta_count() == 8349 and L.l2o_hrnn_state_floats() == 21
    h = ctypes.c_void_p()
    assert L.l2o_hrnn_create(ctypes.byref(h), None, 3) == _lib.L2O_E_INVALID
    sizes = (ctypes.c_int64 * 2)(5, -1)
    assert L.l2o_hrnn_create(ctypes.byref(h), sizes, 2) == _lib.L2O_E_INVALID       # negative size
    sizes = (ctypes.c_int64 * 2)(0, 0)
    assert L.l2o_hrnn_create(ctypes.byref(h), sizes, 2) == _lib.L2O_E_INVALID       # no coordinate at all
    assert L.l2o_hrnn_workspace_bytes(None) == _lib.L2O_E_INVALID
    assert L.l2o_hrnn_step(None, None, None) == _lib.L2O_E_INVALID
    from open_l2o_b200.hierarchical_rnn import THETA_SPEC
    import math
    assert sum(math.prod(s) for _, s in THETA_SPEC) == 8349


def _struct_fields(name):
    """Field names of `typedef struct { ... } name;` in the header, in declaration order."""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"typedef struct\s*\{([^}]*)\}\s*%s\s*;" % name, src)
    assert m, name
    out = []
    for decl in m.group(1).split(";"):
        decl = decl.strip()
        if decl:
            for part in decl.split(","):     # `float beta1, beta2`
                out.append(re.findall(r"[A-Za-z_][A-Za-z_0-9]*", part)[-1])
    return out


def test_ctypes_structs_follow_the_header_field_order():
    pairs = [("l2o_bwd_args", _lib.BwdArgs), ("l2o_hrnn_bwd_args", _lib.HrnnBwdArgs), ("l2o_hrnn_args", _lib.HrnnArgs)]
    for cname, cls in pairs:
        want = _struct_fields(cname)
        got = [f[0].rstrip("_") for f in cls._fields_]
        assert got == want, (cname, got, want)


def test_new_entry_points_validate_without_gpu():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    assert L.l2o_hrnn_coord_bwd(None, None, None) == _lib.L2O_E_INVALID
    assert L.l2o_hrnn_workspace_layout(None, None) == _lib.L2O_E_INVALID
    from open_l2o_b200.engine import NetHandle
    rp = NetHandle(layers=(20, 20), preprocess_name="fc", preprocess_options={"dim": 20}, n_in=2, tanh_output=True)
    n, T = 1000, 20
    fwd, bwd = rp.workspace_bytes(n, T)
    base = 4 * (80 * n * (T + 1) + (T + 1) * n + 2 * T * n) + 8 * rp.n_theta
    assert bwd == base + 4 * T * n * 21          # + recorded deltas and the [T][n][20] hand-over buffer of the two-pass BPTT
