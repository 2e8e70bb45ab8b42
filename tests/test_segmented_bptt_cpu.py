"""CPU-only: the segment planner of MetaOptimizer's BPTT (meta.plan_segments / meta.bptt_buffers) and the argument
checks of l2o_unroll_bwd_carry, which happen before any CUDA call."""
import ctypes
import math
import os
import re

import pytest

from open_l2o_b200 import _lib, meta

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "l2o_b200.h")


@pytest.mark.parametrize("T,S,bounds", [
    (12, 4, [0, 4, 8, 12]),            # S divides T
    (10, 3, [0, 3, 6, 9, 10]),         # ragged last segment
    (5, 1, [0, 1, 2, 3, 4, 5]),        # one step per segment
    (6, 6, [0, 6]),                    # S = T: full checkpoints
    (6, 9, [0, 6]),                    # S > T degenerates to full
    (1, 1, [0, 1]),
])
def test_plan_bounds(T, S, bounds):
    p = meta.plan_segments(T, 80, 10, S=S)
    assert p.bounds == bounds and p.S == min(S, T)
    assert ("boundary" in p.bytes) == (len(bounds) > 2)


def test_plan_bytes():
    slot, n, T, S, bnd, step = 80 * 1000, 1000, 10, 3, 2000, 20000
    p = meta.plan_segments(T, slot, n, S=S, boundary_floats=bnd, step_floats=step)
    assert p.bytes == {"ckpt": 4 * 4 * slot, "handover": 4 * 3 * step, "boundary": 4 * (5 * slot + 4 * bnd),
                       "recompute": 4 * (2 * slot + bnd + n)}
    full = meta.plan_segments(T, slot, n, S=T, boundary_floats=bnd, step_floats=step)
    assert full.bytes == {"ckpt": 4 * 11 * slot, "handover": 4 * 10 * step}


@pytest.mark.parametrize("S", [1, 3, 7, 20])
@pytest.mark.parametrize("fused", [True, False])
def test_plan_bytes_match_the_buffers(S, fused):
    """What _Program allocates (bptt_buffers) is what the planner counted, buffer by buffer."""
    T, N = 20, 7000
    # a DM run, an RNNProp run with the tensor-core hand-over buffer, a small net with a one-float slot
    runs = [(80 * 5000, 5000, False, False), (80 * 1500, 1500, True, True), (1, 500, False, False)]
    p = meta.plan_segments(T, sum(r[0] for r in runs), sum(r[1] for r in runs), S=S,
                           boundary_floats=(N if fused else 0) + sum(2 * r[1] for r in runs if r[2]),
                           step_floats=sum(20 * r[1] for r in runs if r[3]))
    bufs = meta.bptt_buffers(p, runs, N, fused)
    got = {k: 4 * sum(math.prod(shape) for _, _, shape in v) for k, v in bufs.items()}
    assert got == {k: v for k, v in p.bytes.items() if v}
    assert ("bx" in [name for _, name, _ in bufs.get("boundary", [])]) == (fused and S < T)


def test_plan_selection_from_free_memory():
    T, slot, n = 100, 80 * 1_000_000, 1_000_000
    full = 4 * (T + 1) * slot
    assert meta.plan_segments(T, slot, n, 2 * full).S == T                 # fits: full checkpoints
    p = meta.plan_segments(T, slot, n, full)                                # does not fit with headroom
    assert p.S == 10 and p.bounds == list(range(0, 101, 10))               # argmin ceil(T/S) + S
    assert sum(p.bytes.values()) < full / 4
    with pytest.raises(_lib.L2OError, match="segments of 10 steps"):
        meta.plan_segments(T, slot, n, full / 10)
    # what the program allocates either way counts against the free memory
    assert meta.plan_segments(T, slot, n, 2 * full, fixed_bytes=full).S == 10
    assert meta.plan_segments(T, slot, n, S=25).S == 25                     # forced


def test_ctypes_carry_struct_follows_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"typedef struct\s*\{([^}]*)\}\s*l2o_bwd_carry\s*;", src)
    assert m
    want = [re.findall(r"[A-Za-z_][A-Za-z_0-9]*", d)[-1] for d in m.group(1).split(";") if d.strip()]
    assert [f[0] for f in _lib.BwdCarry._fields_] == want == ["d_state", "lam"]
    assert "l2o_unroll_bwd_carry" in _lib.EXPORTS


@pytest.mark.parametrize("preprocess,options,n_in", [("identity", None, 1), ("LogAndSign", {"k": 5}, 1),
                                                    ("fc", {"dim": 20}, 2)])
def test_unroll_bwd_carry_validates_before_the_device(preprocess, options, n_in):
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    from open_l2o_b200.engine import ENGINE_AUTO, ENGINE_FFMA, ENGINE_TC, NetHandle
    h = NetHandle(layers=(20, 20), preprocess_name=preprocess, preprocess_options=options, n_in=n_in)
    L = _lib.lib()
    a = _lib.BwdArgs()
    a.n, a.T = 19_021, 5
    # placeholder addresses: validation must return before any of them is dereferenced
    a.theta, a.in_seq, a.ckpt, a.g_rec, a.dtheta = 0x10000, 0x20000, 0x50000, 0x30000, 0x40000
    c = _lib.BwdCarry()
    c.d_state, c.lam = 0x60000, 0x70000
    call = lambda a, c: L.l2o_unroll_bwd_carry(h._h, ctypes.byref(a), c if c is None else ctypes.byref(c), None)
    for engine in (ENGINE_AUTO, ENGINE_FFMA, ENGINE_TC):
        h.set_engine(engine)
        assert call(a, None) == _lib.L2O_E_INVALID, engine                       # no carry
        for off in (4, 8, 12):
            c.d_state = 0x60000 + off
            assert call(a, c) == _lib.L2O_E_INVALID, (engine, off)             # misaligned adjoint state
            c.d_state = 0x60000
            a.ckpt = 0x50000 + off
            assert call(a, c) == _lib.L2O_E_INVALID, (engine, off)             # misaligned checkpoints
            a.ckpt = 0x50000
        c.lam = None
        assert call(a, c) == _lib.L2O_E_INVALID, engine
        c.lam = 0x70000
        c.d_state = None
        assert call(a, c) == _lib.L2O_E_INVALID, engine
        c.d_state = 0x60000
        a.g_rec, a.labels, a.n_total = None, 0x80000, 100                       # imitation mode
        assert call(a, c) == _lib.L2O_E_UNSUPPORTED, engine
        a.g_rec, a.labels, a.n_total = 0x30000, None, 0
