"""Tensor-core BPTT over many tiles per warpgroup: the DM kernel's full-tile instantiation (n a multiple of 64) and its
predicated one (a ragged last tile).

Each coordinate's backward sweep is its own: the carries a segment hands on (adjoint state, lambda) of coordinate i
depend on coordinate i's inputs only.  So a problem of n = 64 k + 20 coordinates, which runs the predicated kernel,
must hand on bitwise the carries of the same coordinates inside a problem of 64 (k + 1) coordinates, which runs the
full-tile kernel.  dtheta sums over coordinates and is compared with the exact-fp32 engine's."""
import pytest
import torch

from oracle import l2o_oracle as orc
from tests.helpers import SPECS, make_handle, rel_err

pytestmark = pytest.mark.gpu

DTHETA_TOL = 2e-5   # tensor-core dtheta against the exact-fp32 engine's (as in tests/test_segmented_bptt_gpu.py)


def _sweep(spec, engine, n, T, a, b, x0):
    """Fused Rastrigin unroll of the first n coordinates (gradient scale fixed, so each coordinate's inputs do not
    depend on n), then one carried BPTT sweep from a zero carry: dtheta, adjoint state [4][n][20], lambda [n]."""
    from open_l2o_b200.engine import OPT_KINDS
    h = make_handle(spec)
    h.set_engine(engine)
    theta = orc.init_theta(spec, seed=5, out_gain=0.05).cuda()
    state = h.new_state(n, "cuda")
    ckpt = torch.zeros((T + 1) * h.state_size(n), device="cuda")
    g_rec = torch.zeros(T + 1, n, device="cuda")
    h.unroll_fwd(theta, n, T, state, opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=a[:n].clone(), opt_b=b[:n].clone(),
                 opt_alpha=10.0, opt_fscale=1e-4, x=x0[:n].clone(), ckpt=ckpt, g_rec=g_rec)
    dth = torch.zeros(h.n_theta, dtype=torch.float64, device="cuda")
    d_state = torch.zeros(h.state_size(n), device="cuda")
    lam = torch.zeros(n, device="cuda")
    h.unroll_bwd_carry(theta, n, T, g_rec, ckpt, dth, d_state, lam, g_rec=g_rec)
    torch.cuda.synchronize()
    return dth, d_state.view(4, n, 20), lam


@pytest.mark.parametrize("name", ["dm_identity", "dm_logsign"])
def test_tc_bptt_ragged_tile_matches_full_tiles(name):
    from open_l2o_b200.engine import ENGINE_FFMA, ENGINE_TC
    spec, T = SPECS[name], 6
    n_full, n_rag = 64 * 601, 64 * 600 + 20   # several tiles per warpgroup on a 132-SM H100
    g = torch.Generator().manual_seed(5)
    a, b, x0 = (torch.randn(n_full, generator=g).cuda() for _ in range(3))
    full = _sweep(spec, ENGINE_TC, n_full, T, a, b, x0)
    rag = _sweep(spec, ENGINE_TC, n_rag, T, a, b, x0)
    assert float(rag[1][:, -20:].abs().max()) > 0 and float(rag[2][-20:].abs().max()) > 0
    assert torch.equal(rag[1], full[1][:, :n_rag]) and torch.equal(rag[2], full[2][:n_rag])
    for n, out in ((n_full, full), (n_rag, rag)):
        ref = _sweep(spec, ENGINE_FFMA, n, T, a, b, x0)
        assert rel_err(out[0], ref[0]) <= DTHETA_TOL, (n, rel_err(out[0], ref[0]))
