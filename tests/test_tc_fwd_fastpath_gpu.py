"""Tensor-core forward: the DM kernel's full-tile instantiation (n a multiple of 64) against its general, predicated one.

Each coordinate's forward unroll is its own: x, the state, every checkpoint slot and g_rec of coordinate i depend on
coordinate i's inputs only.  So n = 64 * 601 coordinates in one full-tile launch must give bitwise what the same
coordinates give as two ragged launches (64 * 600 + 20 and 44 coordinates, both on the general kernel), with the arenas
split and rejoined by copies.  fx is an fp64 atomic sum over coordinates, so it matches to summation order only."""
import ctypes

import pytest
import torch

from oracle import l2o_oracle as orc
from tests.helpers import SPECS, make_handle

pytestmark = pytest.mark.gpu

FX_RTOL = 1e-13


def _unroll(h, theta, T, kind, state, x, a, b, record):
    """One forward launch over len(x) coordinates: (x, state, ckpt [T+1][4][n][20], g_rec [T+1][n], fx [T+1], the
    kernel variant the call ran)."""
    from open_l2o_b200 import _lib
    n = x.numel()
    ckpt = torch.full(((T + 1) * h.state_size(n),), float("nan"), device="cuda") if record else None
    g_rec = torch.full((T + 1, n), float("nan"), device="cuda") if record else None
    fx = torch.zeros(T + 1, dtype=torch.float64, device="cuda")
    kw = dict(opt_kind=kind, opt_a=a.clone(), opt_b=b.clone(), opt_alpha=10.0, opt_fscale=1e-4, x=x.clone(), ckpt=ckpt,
              g_rec=g_rec, fx=fx)
    args = _lib.UnrollArgs()
    args.n, args.T, args.opt_kind, args.theta, args.state = n, T, kind, theta.data_ptr(), state.data_ptr()
    args.x, args.opt_a, args.opt_b = kw["x"].data_ptr(), kw["opt_a"].data_ptr(), kw["opt_b"].data_ptr()
    if record:
        args.ckpt, args.g_rec = ckpt.data_ptr(), g_rec.data_ptr()
    variant = _lib.lib().l2o_tc_fwd_variant(h._h, ctypes.byref(args))
    h.unroll_fwd(theta, n, T, state, **kw)
    torch.cuda.synchronize()
    return (kw["x"], state.view(4, n, 20), ckpt.view(T + 1, 4, n, 20) if record else None, g_rec, fx, variant)


@pytest.mark.parametrize("record", [True, False], ids=["ckpt", "infer"])
@pytest.mark.parametrize("opt", ["rastrigin_sep", "quadratic_diag"])
@pytest.mark.parametrize("name", ["dm_identity", "dm_logsign"])
def test_tc_fwd_full_tiles_match_ragged_launches(name, opt, record):
    from open_l2o_b200.engine import ENGINE_TC, OPT_KINDS
    spec, T, kind = SPECS[name], 7, OPT_KINDS[opt]
    n, n1 = 64 * 601, 64 * 600 + 20   # several tiles per warpgroup on a 132-SM H100
    h = make_handle(spec)
    h.set_engine(ENGINE_TC)
    theta = orc.init_theta(spec, seed=11, out_gain=0.1).cuda()
    g = torch.Generator().manual_seed(11)
    state = (0.5 * torch.randn(4, n, 20, generator=g)).cuda()
    a, b, x0 = (torch.randn(n, generator=g).cuda() for _ in range(3))

    full = _unroll(h, theta, T, kind, state.clone().reshape(-1), x0, a, b, record)
    parts = [_unroll(h, theta, T, kind, state[:, sl].contiguous().reshape(-1), x0[sl], a[sl], b[sl], record)
             for sl in (slice(0, n1), slice(n1, n))]
    assert full[5] == 1 and parts[0][5] == 0 and parts[1][5] == 0

    assert torch.equal(full[0], torch.cat([parts[0][0], parts[1][0]]))
    assert torch.equal(full[1], torch.cat([parts[0][1], parts[1][1]], dim=1))
    assert not torch.equal(full[1], state)
    if record:
        assert torch.equal(full[2], torch.cat([parts[0][2], parts[1][2]], dim=2))
        assert torch.equal(full[3], torch.cat([parts[0][3], parts[1][3]], dim=1))
        assert not full[2].isnan().any() and not full[3].isnan().any()
    fx_sum = parts[0][4] + parts[1][4]
    assert float((full[4] - fx_sum).abs().max() / fx_sum.abs().max()) <= FX_RTOL
