"""GPU: the l2o_minimax_* kernels and the Twin-L2O trainer against the fp64 oracle (oracle/minimax_oracle.py)."""
import numpy as np
import pytest
import torch

from oracle import minimax_oracle as MO

pytestmark = pytest.mark.gpu

DEV = "cuda"
# (loss, dim, H, B)
SETTINGS = [(1, 1, 50, 128), (2, 1, 50, 37), (3, 1, 80, 37), (4, 1, 50, 37), (4, 5, 80, 128), (4, 5, 50, 37),
            (4, 12, 50, 37)]   # dim > 8 takes the forward's 32-row CTAs
OPTIM_IT, UNROLL = 30, 3   # sign steps t < 6, boundaries at 6, 12, 18, 24, 30


def _rel(got, want):
    got, want = got.double().cpu().reshape(-1), want.double().cpu().reshape(-1)
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-300))


def _problems(loss, dim, B, seed):
    g = np.random.RandomState(seed)
    if loss == 4:
        from open_l2o_b200.minimax import make_matrix_game_data
        return make_matrix_game_data(dim, 0.5 if dim > 1 else 1.0, 0.5, 1.0, B, seed).astype(np.float32)
    return np.stack([g.uniform(0.5, 1.5, B), g.uniform(0.5, 1.0, B)], 1).astype(np.float32)


def _setup(loss, dim, H, B, seed=0):
    from open_l2o_b200 import minimax as mm
    twin = mm.TwinOptimizer(H, DEV, seed=seed)
    data = mm.problem_tensor(_problems(loss, dim, B, seed), loss, dim, DEV)
    un = mm.Unroll(twin, loss, data, dim)
    un.reset(torch.Generator().manual_seed(seed + 1))
    nets = []
    for n in (0, 1):
        net = MO.Net(H).double()
        net.load_state_dict({k: v.double() for k, v in twin.state_dict(n).items()})
        nets.append(net)
    dcpu = data.double().cpu()
    pdata = [dcpu[p] for p in range(B)]
    u0 = list(un.u.double().cpu().view(B, dim))
    v0 = list(un.v.double().cpu().view(B, dim))
    st = un.state.double().cpu()
    state0 = {n: ([st[n, 0], st[n, 2]], [st[n, 1], st[n, 3]]) for n in (0, 1)}
    return twin, un, nets, pdata, u0, v0, state0


@pytest.mark.parametrize("loss,dim,H,B", SETTINGS)
def test_every_iteration_matches_oracle(loss, dim, H, B):
    twin, un, nets, pdata, u0, v0, state0 = _setup(loss, dim, H, B)
    recs, _ = MO.do_fit(nets, loss, pdata, u0, v0, state0, UNROLL, OPTIM_IT, 1e-4, train=False)
    lval = torch.zeros(1, B, device=DEV)
    worst = 0.0
    for t in range(1, OPTIM_IT + 1):
        un.forward(t, t + 1, OPTIM_IT, lval=lval)
        r = recs[t - 1]
        e = dict(u=_rel(un.u, r["u"]), v=_rel(un.v, r["v"]), l=_rel(lval[0], torch.tensor(r["l"])),
                 s0=_rel(un.state[0], r["state"][0]), s1=_rel(un.state[1], r["state"][1]))
        worst = max(worst, max(e.values()))
        assert max(e.values()) <= 1e-5, (t, e)
    print("max rel err over all iterations", worst)


def _segment_grads(twin, un, B, select=None):
    from open_l2o_b200 import minimax as mm
    out, seg, t = [], 2 * UNROLL, 1
    traj = torch.zeros(OPTIM_IT, un.rows, 2, device=DEV)
    while t <= OPTIM_IT:
        T = ((t - 1) // seg + 1) * seg
        bufs = un.buffers(T + 1 - t)
        un.forward(t, T + 1, OPTIM_IT, traj=traj[t - 1:T], ckpt=bufs["ckpt"], dl=bufs["dl"])
        weight = None
        if select is not None:
            weight = torch.zeros(B, device=DEV)
            weight[list(select(T, None))] = 1.0
        un.backward(t, T, OPTIM_IT, bufs["ckpt"], bufs["dl"], mm.reward_coefs(t, T, B).to(DEV), weight)
        out.append(twin.grad.clone())
        t = T + 1
    return out


@pytest.mark.parametrize("loss,dim,H,B", SETTINGS)
@pytest.mark.parametrize("cl", [False, True])
def test_segment_meta_gradients_match_oracle(loss, dim, H, B, cl):
    twin, un, nets, pdata, u0, v0, state0 = _setup(loss, dim, H, B)
    select = None
    if cl:
        picks = {T: sorted(np.random.RandomState(T).choice(B, B // 2, replace=False).tolist())
                 for T in range(2 * UNROLL, OPTIM_IT + 1, 2 * UNROLL)}
        select = lambda T, _traj: picks[T]   # noqa: E731
    _, seg_ref = MO.do_fit(nets, loss, pdata, u0, v0, state0, UNROLL, OPTIM_IT, 1e-4, train=True, select=select)
    got = _segment_grads(twin, un, B, select)
    assert len(got) == len(seg_ref)
    for k, (g, ref) in enumerate(zip(got, seg_ref)):
        for n in (0, 1):
            want = torch.cat([x.reshape(-1) for x in ref[n]])
            if float(want.abs().max()) == 0.0:   # sign steps only: sign passes zeros
                assert float(g[n].abs().max()) == 0.0, (k, n)
            else:
                assert _rel(g[n], want) <= 1e-5, (k, n, _rel(g[n], want))


def test_training_follows_oracle_with_torch_adam():
    from open_l2o_b200 import minimax_train as tr
    loss, dim, H, B = 3, 1, 50, 37
    twin, un, nets, pdata, u0, v0, state0 = _setup(loss, dim, H, B)
    # eps = 1e-3 keeps Adam's step linear in components whose gradient is within fp32 noise of zero, where the
    # normalised step would otherwise turn that noise into +-lr
    opts_ref = [torch.optim.Adam(n.parameters(), lr=1e-3, eps=1e-3) for n in nets]
    before = twin.theta.clone()
    MO.do_fit(nets, loss, pdata, u0, v0, state0, UNROLL, OPTIM_IT, 1e-4, train=True, meta_opts=opts_ref)
    opts = tr.make_meta_opts(twin, 1e-3, eps=1e-3)
    tr.do_fit(twin, opts, loss, un.data, dim, UNROLL, OPTIM_IT, True, unroll=un)
    for n in (0, 1):
        want = torch.cat([p.detach().reshape(-1) for p in nets[n].parameters()])
        step = want - before[n].double().cpu()
        assert float(step.abs().max()) > 0.0
        assert _rel(twin.theta[n] - before[n], step) <= 1e-3, (n, _rel(twin.theta[n] - before[n], step))


def test_evaluation_score_matches_oracle():
    from open_l2o_b200 import minimax_train as tr
    for loss in (3, 4):
        dim = 5 if loss == 4 else 1
        twin, un, nets, pdata, u0, v0, state0 = _setup(loss, dim, 50, 20)
        it = 40
        recs, _ = MO.do_fit(nets, loss, pdata, u0, v0, state0, UNROLL, it, 1e-4, train=False)
        traj, _ = tr.do_fit(twin, None, loss, un.data, dim, UNROLL, it, False, unroll=un)
        want = MO.eval_score(loss, pdata, recs, it // 2)
        got = tr.eval_score(loss, un.data, traj, dim, it // 2)
        assert abs(got - want) <= 1e-5 * abs(want), (loss, got, want)


def test_backward_is_bit_identical_run_to_run():
    from open_l2o_b200 import minimax as mm
    twin, un, *_ = _setup(4, 5, 80, 128)
    bufs = un.buffers(12)
    un.forward(1, 13, 30, ckpt=bufs["ckpt"], dl=bufs["dl"])
    coef = mm.reward_coefs(1, 12, 128).to(DEV)
    a = un.backward(1, 12, 30, bufs["ckpt"], bufs["dl"], coef).clone()
    b = un.backward(1, 12, 30, bufs["ckpt"], bufs["dl"], coef).clone()
    assert torch.equal(a, b)


def test_cuda_graph_replay_equals_eager():
    from open_l2o_b200 import minimax as mm
    twin, un, *_ = _setup(2, 1, 50, 37)
    bufs = un.buffers(7)
    coef = mm.reward_coefs(1, 6, 37).to(DEV)
    u0, v0, s0 = un.u.clone(), un.v.clone(), un.state.clone()

    def seg():
        un.forward(1, 7, 30, ckpt=bufs["ckpt"], dl=bufs["dl"])
        un.backward(1, 6, 30, bufs["ckpt"], bufs["dl"], coef)

    seg()   # warm-up allocates the workspace
    torch.cuda.synchronize()
    eager = (un.u.clone(), un.state.clone(), twin.grad.clone())
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        un.u.copy_(u0), un.v.copy_(v0), un.state.copy_(s0)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            seg()
    un.u.copy_(u0), un.v.copy_(v0), un.state.copy_(s0)
    twin.grad.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(un.u, eager[0]) and torch.equal(un.state, eager[1]) and torch.equal(twin.grad, eager[2])


def test_launches_per_segment_do_not_grow_with_batch():
    from open_l2o_b200 import minimax_train as tr
    from open_l2o_b200.engine import launch_count
    counts = []
    for B in (8, 128):
        twin, un, *_ = _setup(1, 1, 50, B)
        opts = tr.make_meta_opts(twin, 1e-3)
        before = launch_count()
        tr.do_fit(twin, opts, 1, un.data, 1, UNROLL, OPTIM_IT, True)
        torch.cuda.synchronize()
        counts.append(launch_count() - before)
    assert counts[0] == counts[1], counts
    assert counts[0] <= 4 * (OPTIM_IT // (2 * UNROLL)), counts   # forward, 2 backward, weight image per segment


def test_torch_state_dict_round_trips():
    from open_l2o_b200 import minimax as mm
    twin = mm.TwinOptimizer(80, DEV, seed=3)
    ref = MO.Net(80)
    ref.load_state_dict(twin.state_dict(1))
    other = mm.TwinOptimizer(80, DEV, seed=4)
    other.load_state_dict(0, ref.state_dict())
    for k, v in ref.state_dict().items():
        assert torch.equal(other.state_dict(0)[k], v)
    assert torch.equal(other.theta[0], twin.theta[1])
