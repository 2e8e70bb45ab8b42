"""GPU: the Twin-L2O kernels (l2o_minimax_fwd, l2o_minimax_bwd's chain and weight-gradient kernels) output by output
and parameter block by parameter block against the contract reference (tests/minimax_contract.py).

At the reference's rescale of 1e-4 the active net's h and c enter its cells scaled by 1e-4, so the recurrent half of
both nets hardly moves what a whole-vector comparison sees: the weight_hh gradients are 1e-8..1e-6 of a net's largest
entry.  Here every quantity is held to its own scale (each iteration's u, v, l, dl, checkpoint columns and eight state
planes; each of a net's ten parameter blocks), at rescales 0.5 and 1 where the recurrence carries weight, across the
kernels' shape limits and over segment ranges MO.do_fit never produces.  The reference runs in fp64; where its fp32 run
is further from fp64 than REL_TOL on a quantity, three times that distance is the bar instead.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import minimax_oracle as MO
from tests import minimax_contract as MC

pytestmark = pytest.mark.gpu

DEV = "cuda"
REL_TOL = 1e-5
OPTIM_IT = 30          # warm_end 6: iterations 1..5 take the sign step
SIGN_MARGIN = 1e-5     # every sign-phase delta of the reference is at least this far from zero

# (loss, dim, H, B, seed); each seed keeps every sign-phase delta clear of zero (SIGN_MARGIN)
SHAPES = [
    (1, 1, 7, 3, 0),      # G = 28, far below the 128 threads; B smaller than one chain CTA
    (2, 1, 33, 130, 0),   # ragged 32x32 weight-gradient tiles (4H = 132, 2H + 1 = 67); many CTAs
    (3, 1, 128, 37, 1),   # H at its limit: 512 threads, 115 KB of chain shared memory; R mod 4 = 1
    (4, 8, 64, 13, 0),    # the largest dim on the forward's 8-row path (one problem per CTA)
    (4, 9, 50, 11, 0),    # the smallest dim on the 32-row path: 3 problems, 27 of 32 rows, last CTA partial
    (4, 32, 128, 5, 1),   # dim and H both at their limits
]


def _rel(got, want):
    """Max-norm error relative to want's largest entry; an all-zero want must be matched exactly."""
    got, want = got.double().cpu().reshape(-1), want.double().cpu().reshape(-1)
    scale = float(want.abs().max())
    err = float((got - want).abs().max())
    if scale == 0.0:
        return 0.0 if err == 0.0 else float("inf")
    return err / scale if err == err else float("inf")


def _problems(loss, dim, B, seed):
    g = np.random.RandomState(seed)
    if loss == 4:
        from open_l2o_b200.minimax import make_matrix_game_data
        return make_matrix_game_data(dim, 0.5 if dim > 1 else 1.0, 0.5, 1.0, B, seed).astype(np.float32)
    return np.stack([g.uniform(0.5, 1.5, B), g.uniform(0.5, 1.0, B)], 1).astype(np.float32)


def _setup(loss, dim, H, B, rescale=1.0, out_mul=1.0, seed=0):
    from open_l2o_b200 import minimax as mm
    twin = mm.TwinOptimizer(H, DEV, seed=seed)
    data = mm.problem_tensor(_problems(loss, dim, B, seed), loss, dim, DEV)
    un = mm.Unroll(twin, loss, data, dim, rescale=rescale, out_mul=out_mul)
    un.reset(torch.Generator().manual_seed(seed + 1))
    nets = []
    for n in (0, 1):
        net = MO.Net(H).double()
        net.load_state_dict({k: v.double() for k, v in twin.state_dict(n).items()})
        nets.append(net)
    return twin, un, nets


def _weights(B, T, seed):
    """Non-uniform reward coefficients [T] and per-problem weights [B] (every fourth problem 0, as a curriculum
    drops it), fp32 on the device."""
    g = torch.Generator().manual_seed(seed)
    coef = (0.5 + 1.5 * torch.rand(T, generator=g)) / B
    weight = 0.25 + 1.5 * torch.rand(B, generator=g)
    weight[::4] = 0.0
    return coef.to(DEV), weight.to(DEV)


def _buffers(un, n):
    R, H = un.rows, un.twin.hidden
    return dict(traj=torch.zeros(n, R, 2, device=DEV), ckpt=torch.zeros(n, R, 4 * H + 2, device=DEV),
                dl=torch.zeros(n, R, device=DEV), lval=torch.zeros(n, un.batch, device=DEV))


def _forward(un, t0, t1, bufs, null_lr=False):
    """One l2o_minimax_fwd launch over [t0, t1); null_lr passes lr = NULL, which the ABI allows from warm_end on."""
    if not null_lr:
        un.forward(t0, t1, OPTIM_IT, **bufs)
        return
    from open_l2o_b200 import _lib
    a = un._args(t0, t1, OPTIM_IT, None, bufs["traj"], bufs["ckpt"], bufs["dl"], bufs["lval"])
    _lib.check(_lib.lib().l2o_minimax_fwd(C.byref(a), un._stream()), "l2o_minimax_fwd")


def _backward(un, t0, t1, bufs, coef, weight, null_lr=False):
    """l2o_minimax_bwd over [t0, t1) into twin.grad, filled with NaN first so an entry no tile writes shows."""
    un.twin.grad.fill_(float("nan"))
    if not null_lr:
        un.backward(t0, t1, OPTIM_IT, bufs["ckpt"], bufs["dl"], coef, weight)
        return
    from open_l2o_b200 import _lib
    a = un._args(t0, t1, OPTIM_IT, None, None, bufs["ckpt"], bufs["dl"], None)
    nbytes = C.c_size_t()
    _lib.check(_lib.lib().l2o_minimax_workspace_bytes(C.byref(a), C.byref(nbytes)), "l2o_minimax_workspace_bytes")
    scratch = torch.empty((nbytes.value + 7) // 8, dtype=torch.float64, device=DEV)
    g = _lib.MinimaxGrads()
    g.coef, g.weight = C.c_void_p(coef.data_ptr()), C.c_void_p(weight.data_ptr())
    g.dtheta, g.scratch = C.c_void_p(un.twin.grad.data_ptr()), C.c_void_p(scratch.data_ptr())
    _lib.check(_lib.lib().l2o_minimax_bwd(C.byref(a), C.byref(g), un._stream()), "l2o_minimax_bwd")


def _held(got, want64, want32, what):
    """Assert got is within REL_TOL of want64 on want64's own scale, or 3x the fp32 reference's distance if larger;
    returns (error, bar)."""
    err, bar = _rel(got, want64), max(REL_TOL, 3.0 * _rel(want32, want64))
    assert err <= bar, (what, err, bar)
    return err, bar


def _held_blocks(grad, ref64, ref32, H, what):
    """Hold each of both nets' ten parameter blocks of grad [2][theta_count] to its own scale (ref[n][i] None: no
    path reaches the block, so it must be 0).  Every entry must have been written, and each layer's bias_ih and
    bias_hh gradients are one value written twice.  Returns the worst (error, bar, block)."""
    from open_l2o_b200 import minimax as mm
    got, worst = grad.cpu(), (0.0, REL_TOL, "")
    for n in (0, 1):
        off, blocks = 0, {}
        for (name, shape), a64, a32 in zip(mm.param_spec(H), ref64[n], ref32[n]):
            cnt = int(np.prod(shape))
            blocks[name] = got[n, off:off + cnt]
            off += cnt
            assert bool(torch.isfinite(blocks[name]).all()), (what, n, name, "entries left unwritten")
            a64 = torch.zeros(cnt, dtype=torch.float64) if a64 is None else a64
            a32 = torch.zeros(cnt, dtype=torch.float32) if a32 is None else a32
            worst = max(worst, _held(blocks[name], a64, a32, (what, n, name)) + (name,))
        for layer in ("recurs", "recurs2"):
            assert torch.equal(blocks[layer + ".bias_ih"], blocks[layer + ".bias_hh"]), (what, n, layer)
    return worst


def _check_segment(twin, un, nets, t0, t1, coef, weight, null_lr=False, label=""):
    """Run [t0, t1) forward and backward from un's current point and hold every output to the contract reference run
    from the same point.  The forward runs once as one launch and once as one launch per iteration, which must agree
    bitwise; the second gives the state after every iteration.  Returns the worst forward and backward (error, bar)."""
    from open_l2o_b200 import minimax as mm
    H, n_it, we = twin.hidden, t1 - t0, mm.warm_end(OPTIM_IT)
    start = (un.u.clone(), un.v.clone(), un.state.clone())
    kw = dict(loss=un.loss, data=un.data.cpu(), u=start[0].cpu(), v=start[1].cpu(), state=start[2].cpu(), t0=t0,
              t1=t1, warm_end=we, lr=[float(x) for x in un._lr(OPTIM_IT).cpu()],
              rescale=float(np.float32(un.rescale)), out_mul=float(np.float32(un.out_mul)),
              coef=[float(c) for c in coef.cpu()], weight=weight.cpu())
    r64 = MC.segment(nets, dtype=torch.float64, **kw)
    r32 = MC.segment(nets, dtype=torch.float32, **kw)
    n_sign = max(0, min(t1, we) - t0)
    if n_sign:   # a sign that fp32 rounding could flip would make the comparison ill-posed, not the kernel wrong
        closest = float(r64["delta"][:n_sign].abs().min())
        assert closest >= SIGN_MARGIN, (label, closest)

    one = _buffers(un, n_it)
    _forward(un, t0, t1, one, null_lr)
    end = (un.u.clone(), un.v.clone(), un.state.clone())
    un.u.copy_(start[0]), un.v.copy_(start[1]), un.state.copy_(start[2])
    steps, states = _buffers(un, n_it), []
    for i, t in enumerate(range(t0, t1)):
        _forward(un, t, t + 1, {k: b[i:i + 1] for k, b in steps.items()}, null_lr)
        states.append(un.state.clone())
    for k in one:
        assert torch.equal(one[k], steps[k]), (label, k)
    assert torch.equal(un.u, end[0]) and torch.equal(un.v, end[1]) and torch.equal(un.state, end[2]), label

    worst_f = (0.0, REL_TOL)
    cols = dict(in0=slice(0, 1), in1=slice(1, 2), h1=slice(2, 2 + H), c1=slice(2 + H, 2 + 2 * H),
                h2=slice(2 + 2 * H, 2 + 3 * H), c2=slice(2 + 3 * H, 2 + 4 * H))
    for i, t in enumerate(range(t0, t1)):
        got = dict(u=one["traj"][i, :, 0], v=one["traj"][i, :, 1], l=one["lval"][i], dl=one["dl"][i])
        for name in got:
            e = _held(got[name], r64[name][i], r32[name][i], (label, t, name))
            worst_f = max(worst_f, e)
        for name, cs in cols.items():
            e = _held(one["ckpt"][i, :, cs], r64["ckpt"][i][:, cs], r32["ckpt"][i][:, cs], (label, t, "ckpt", name))
            worst_f = max(worst_f, e)
        for m in (0, 1):
            for j, plane in enumerate(("h1", "c1", "h2", "c2")):
                e = _held(states[i][m, j], r64["state"][i][m][j], r32["state"][i][m][j], (label, t, m, plane))
                worst_f = max(worst_f, e)

    _backward(un, t0, t1, one, coef, weight, null_lr)
    return worst_f, _held_blocks(twin.grad, r64["grads"], r32["grads"], H, label)


@pytest.mark.parametrize("out_mul", [1.0, 0.3])
@pytest.mark.parametrize("rescale", [1e-4, 0.5, 1.0])
@pytest.mark.parametrize("loss,dim,H,B,seed", SHAPES)
def test_shape_limits_block_by_block(loss, dim, H, B, seed, rescale, out_mul):
    # one segment from iteration 1 through the sign phase and 9 iterations after it: the carried adjoints cross
    # from the updates that get a gradient into the sign steps before them
    twin, un, nets = _setup(loss, dim, H, B, rescale, out_mul, seed)
    coef, weight = _weights(B, 14, seed=loss * 100 + dim)
    label = "loss %d dim %d H %d B %d rescale %g out_mul %g" % (loss, dim, H, B, rescale, out_mul)
    wf, wb = _check_segment(twin, un, nets, 1, 15, coef, weight, label=label)
    print("%s: forward worst %.1e (bar %.1e), backward worst %.1e (bar %.1e) on %s" % (label, *wf, *wb))


# (t0, t1, null_lr): ranges the trainer's segments never take
SEGMENTS = [
    (8, 13, False),   # even t0, so net 1 goes first; odd length
    (3, 10, False),   # starts inside the sign phase, ends after warm_end; odd t0, odd length
    (2, 11, False),   # starts inside the sign phase with net 1 first
    (9, 10, False),   # one iteration of net 0: net 1's dtheta must come back all zero
    (10, 11, False),  # one iteration of net 1: net 0's dtheta must come back all zero
    (6, 13, True),    # t0 = warm_end with lr = NULL
    (11, 14, True),   # t0 > warm_end with lr = NULL, net 0 both first and last
]


@pytest.mark.parametrize("loss,dim,H,B", [(3, 1, 50, 37), (4, 5, 40, 9)])
@pytest.mark.parametrize("t0,t1,null_lr", SEGMENTS)
def test_segment_ranges_block_by_block(loss, dim, H, B, t0, t1, null_lr):
    twin, un, nets = _setup(loss, dim, H, B, rescale=1.0, out_mul=0.3, seed=2)
    if t0 > 1:   # reach t0 on the GPU; the reference starts from where the kernels are
        un.forward(1, t0, OPTIM_IT)
    coef, weight = _weights(B, t1 - t0, seed=t0)
    label = "loss %d dim %d [%d, %d)%s" % (loss, dim, t0, t1, " lr NULL" if null_lr else "")
    wf, wb = _check_segment(twin, un, nets, t0, t1, coef, weight, null_lr, label)
    if t1 == t0 + 1:
        idle = 1 if t0 % 2 else 0
        assert bool((twin.grad[idle] == 0).all()), label
        assert float(twin.grad[1 - idle].abs().max()) > 0.0, label
    print("%s: forward worst %.1e (bar %.1e), backward worst %.1e (bar %.1e) on %s" % (label, *wf, *wb))


@pytest.mark.parametrize("loss,dim,H,B", [(4, 5, 40, 9), (4, 12, 24, 7)])   # the 8-row and the 32-row forward
def test_forward_split_is_bitwise_one_launch(loss, dim, H, B):
    twin, un, _ = _setup(loss, dim, H, B, rescale=1.0, out_mul=0.3, seed=4)
    t0, m, t1 = 4, 7, 15   # even t0 in the sign phase; m is the first update after it
    start = (un.u.clone(), un.v.clone(), un.state.clone())
    whole = _buffers(un, t1 - t0)
    un.forward(t0, t1, OPTIM_IT, **whole)
    end = (un.u.clone(), un.v.clone(), un.state.clone())
    un.u.copy_(start[0]), un.v.copy_(start[1]), un.state.copy_(start[2])
    split = _buffers(un, t1 - t0)
    un.forward(t0, m, OPTIM_IT, **{k: b[:m - t0] for k, b in split.items()})
    un.forward(m, t1, OPTIM_IT, **{k: b[m - t0:] for k, b in split.items()})
    assert torch.equal(un.u, end[0]) and torch.equal(un.v, end[1]) and torch.equal(un.state, end[2])
    for k in whole:
        assert torch.equal(whole[k], split[k]), k


@pytest.mark.parametrize("loss,dim,H,B", [(3, 1, 50, 37), (4, 5, 80, 37)])
def test_do_fit_segments_block_by_block_at_rescale_one(loss, dim, H, B):
    # the trainer's own segments and curriculum weights, each block against MO.do_fit in fp64 with its fp32 run as
    # the slack
    from open_l2o_b200 import minimax as mm
    unroll = 3
    twin, un, nets = _setup(loss, dim, H, B, rescale=1.0, seed=5)
    picks = {T: sorted(np.random.RandomState(T).choice(B, B // 2, replace=False).tolist())
             for T in range(2 * unroll, OPTIM_IT + 1, 2 * unroll)}
    dcpu = un.data.double().cpu()
    pdata = [dcpu[p] for p in range(B)]
    st = un.state.double().cpu()
    args = (loss, pdata, list(un.u.double().cpu().view(B, dim)), list(un.v.double().cpu().view(B, dim)),
            {n: ([st[n, 0], st[n, 2]], [st[n, 1], st[n, 3]]) for n in (0, 1)}, unroll, OPTIM_IT, 1.0)
    warm = MC.segment(nets, loss, un.data.cpu(), un.u.cpu(), un.v.cpu(), un.state.cpu(), 1, mm.warm_end(OPTIM_IT),
                      mm.warm_end(OPTIM_IT), MO.sche_lr(OPTIM_IT), 1.0)
    assert float(warm["delta"].abs().min()) >= SIGN_MARGIN
    _, g64 = MO.do_fit(nets, *args, train=True, select=lambda T, _t: picks[T])
    _, g32 = MO.do_fit([copy.deepcopy(n).float() for n in nets], *args, train=True, select=lambda T, _t: picks[T],
                       dtype=torch.float32)
    seg, t, k = 2 * unroll, 1, 0
    worst = (0.0, REL_TOL, "")
    while t <= OPTIM_IT:
        T = ((t - 1) // seg + 1) * seg
        bufs = un.buffers(T + 1 - t)
        un.forward(t, T + 1, OPTIM_IT, ckpt=bufs["ckpt"], dl=bufs["dl"])
        weight = torch.zeros(B, device=DEV)
        weight[picks[T]] = 1.0
        twin.grad.fill_(float("nan"))
        un.backward(t, T, OPTIM_IT, bufs["ckpt"], bufs["dl"], mm.reward_coefs(t, T, B).to(DEV), weight)
        worst = max(worst, _held_blocks(twin.grad, g64[k], g32[k], H, "segment %d" % k))
        t, k = T + 1, k + 1
    assert k == len(g64)
    print("loss %d dim %d H %d: worst block %.1e (bar %.1e) on %s" % (loss, dim, H, *worst))

