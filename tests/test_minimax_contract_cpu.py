"""CPU: the l2o_minimax_* contract reference (tests/minimax_contract.py) against the Twin-L2O oracle, and the oracle's
dtype argument."""
import copy

import numpy as np
import pytest
import torch

from oracle import minimax_oracle as MO
from tests import minimax_contract as MC

OPTIM_IT, UNROLL = 30, 3   # sign steps t < 6, boundaries at 6, 12, 18, 24, 30


def _case(loss, dim, H, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    nets = [MO.Net(H).double() for _ in (0, 1)]
    if loss == 4:
        from open_l2o_b200.minimax import make_matrix_game_data
        data = torch.tensor(make_matrix_game_data(dim, 0.5, 0.5, 1.0, B, seed), dtype=torch.float64).view(B, dim, dim)
    else:
        data = torch.stack([0.5 + torch.rand(B, generator=g, dtype=torch.float64),
                            0.5 + 0.5 * torch.rand(B, generator=g, dtype=torch.float64)], 1)
    u0 = torch.rand(B, dim, generator=g, dtype=torch.float64) - 0.5
    v0 = torch.rand(B, dim, generator=g, dtype=torch.float64) - 0.5
    state = torch.randn(2, 4, B * dim, H, generator=g, dtype=torch.float64) * 0.01
    return nets, data, u0, v0, state


def _do_fit_args(loss, data, u0, v0, state, rescale):
    B = data.shape[0]
    st = {n: ([state[n, 0], state[n, 2]], [state[n, 1], state[n, 3]]) for n in (0, 1)}
    return (loss, [data[p] for p in range(B)], list(u0), list(v0), st, UNROLL, OPTIM_IT, rescale)


def _rel(got, want):
    got, want = got.reshape(-1), want.reshape(-1)
    scale = float(want.abs().max())
    err = float((got - want).abs().max())
    return err if scale == 0.0 else err / scale


@pytest.mark.parametrize("rescale", [1e-4, 1.0])
@pytest.mark.parametrize("loss,dim,H,B", [(3, 1, 9, 7), (4, 3, 6, 5)])
def test_contract_reference_chained_over_boundaries_is_do_fit(loss, dim, H, B, rescale):
    # do_fit back-propagates the rewards at every boundary T, before iteration T's own reward: the segment [t, T]
    # weighs l_t 2/B, l_{T-1} 1/B and l_T 0 (it reaches the next segment as a constant), and the curriculum's
    # choice is a 0/1 problem weight
    nets, data, u0, v0, state = _case(loss, dim, H, B)
    seg = 2 * UNROLL
    picks = {T: sorted(np.random.RandomState(T).choice(B, (B + 1) // 2, replace=False).tolist())
             for T in range(seg, OPTIM_IT + 1, seg)}
    recs, grads = MO.do_fit(nets, *_do_fit_args(loss, data, u0, v0, state, rescale), train=True,
                            select=lambda T, _traj: picks[T])
    u, v, st = u0.reshape(-1), v0.reshape(-1), state
    t, k = 1, 0
    while t <= OPTIM_IT:
        T = ((t - 1) // seg + 1) * seg
        coef = [(2.0 if s + 1 < T else 1.0) / B for s in range(t, T)] + [0.0]
        weight = torch.zeros(B, dtype=torch.float64)
        weight[picks[T]] = 1.0
        out = MC.segment(nets, loss, data, u, v, st, t, T + 1, 6, MO.sche_lr(OPTIM_IT), rescale, coef=coef,
                         weight=weight)
        for i, s in enumerate(range(t, T + 1)):
            r = recs[s - 1]
            assert _rel(out["u"][i], r["u"]) <= 1e-13 and _rel(out["v"][i], r["v"]) <= 1e-13, (s, "u, v")
            assert _rel(out["l"][i], torch.tensor(r["l"], dtype=torch.float64)) <= 1e-13, (s, "l")
            for m in (0, 1):
                for j in range(4):
                    assert _rel(out["state"][i][m][j], r["state"][m][j]) <= 1e-13, (s, m, j)
        for n in (0, 1):
            for name, got, want in zip([p for p, _ in nets[n].named_parameters()], out["grads"][n], grads[k][n]):
                if want is None:   # only sign steps in the segment: no path to the nets
                    assert float(got.abs().max()) == 0.0, (k, n, name)
                else:
                    assert _rel(got, want) <= 1e-11, (k, n, name, _rel(got, want))
        u, v, st = out["u"][-1], out["v"][-1], out["state"][-1]
        t, k = T + 1, k + 1
    assert k == len(grads)


def test_contract_reference_weight_hh_blocks_carry_weight_at_rescale_one():
    # the premise of the block-by-block GPU tests: at rescale 1 the recurrent blocks are a visible part of the
    # gradient, and cutting the recurrence (rescale 0) moves every net's gradient well past 1e-5
    nets, data, u0, v0, state = _case(4, 3, 6, 5)
    coef = [1.0] * 10
    kw = dict(t0=3, t1=13, warm_end=6, lr=MO.sche_lr(OPTIM_IT), coef=coef)
    one = MC.segment(nets, 4, data, u0.reshape(-1), v0.reshape(-1), state, rescale=1.0, **kw)["grads"]
    cut = MC.segment(nets, 4, data, u0.reshape(-1), v0.reshape(-1), state, rescale=0.0, **kw)["grads"]
    names = [p for p, _ in nets[0].named_parameters()]
    for n in (0, 1):
        whole = torch.cat([g.reshape(-1) for g in one[n]])
        for name, g in zip(names, one[n]):
            if "weight_hh" in name:
                assert float(g.abs().max()) >= 1e-3 * float(whole.abs().max()), (n, name)
        assert _rel(torch.cat([g.reshape(-1) for g in cut[n]]), whole) >= 1e-2, n


@pytest.mark.parametrize("loss,dim", [(2, 1), (4, 3)])
def test_do_fit_float64_is_the_default_bit_for_bit(loss, dim):
    nets, data, u0, v0, state = _case(loss, dim, 6, 4, seed=1)
    args = _do_fit_args(loss, data, u0, v0, state, 0.5)
    r0, g0 = MO.do_fit(nets, *args, train=True)
    r1, g1 = MO.do_fit(nets, *args, train=True, dtype=torch.float64)
    # inputs given in fp32 are widened exactly: the same run as their fp64 values
    r2, g2 = MO.do_fit(nets, *_do_fit_args(loss, data.float(), u0.float(), v0.float(), state.float(), 0.5),
                       train=True, dtype=torch.float64)
    r3, g3 = MO.do_fit(nets, *_do_fit_args(loss, data.float().double(), u0.float().double(), v0.float().double(),
                                           state.float().double(), 0.5), train=True)
    for (ra, ga), (rb, gb) in (((r0, g0), (r1, g1)), ((r3, g3), (r2, g2))):
        assert len(ra) == len(rb) == OPTIM_IT and len(ga) == len(gb)
        for a, b in zip(ra, rb):
            assert a["u"].dtype == torch.float64 and torch.equal(a["u"], b["u"]) and torch.equal(a["v"], b["v"])
            assert a["l"] == b["l"]
            assert all(torch.equal(a["state"][m], b["state"][m]) for m in (0, 1))
        for a, b in zip(ga, gb):
            for n in (0, 1):
                assert all((x is None and y is None) or torch.equal(x, y) for x, y in zip(a[n], b[n]))


def test_do_fit_float32_runs_in_float32_close_to_float64():
    nets, data, u0, v0, state = _case(4, 3, 6, 4, seed=2)
    args = _do_fit_args(4, data, u0, v0, state, 1.0)
    r64, g64 = MO.do_fit(nets, *args, train=True)
    r32, g32 = MO.do_fit([copy.deepcopy(n).float() for n in nets], *args, train=True, dtype=torch.float32)
    for a, b in zip(r32, r64):
        assert a["u"].dtype == torch.float32 and a["state"][0].dtype == torch.float32
        assert _rel(a["u"].double(), b["u"]) <= 1e-5 and _rel(a["v"].double(), b["v"]) <= 1e-5
    for a, b in zip(g32[1:], g64[1:]):
        for n in (0, 1):
            for x, y in zip(a[n], b[n]):
                assert x.dtype == torch.float32 and _rel(x.double(), y) <= 1e-4
