"""L2O-Scale HierarchicalRNN step (SURVEY.md 8(f) row 1): CUDA path through the C-ABI vs the CPU oracle."""
import math

import pytest
import torch

from oracle import hrnn_oracle as H
from tests.helpers import HRNN_CONVNET, HRNN_TILE, REL_TOL, hrnn_generic_theta, hrnn_ragged_shapes, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FLUSH_TILES, CTAS_PER_SM = 8, 2   # coord_tc_kernel flushes its per-tensor sums every 8 tiles; grid = 2 CTAs per SM


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def ragged_grad_scales(n, seed=0):
    """Per-tensor gradient magnitudes spread log-uniformly over [1e-6, 10]; tensor 7's gradient is zero on every step."""
    s = 10.0 ** (torch.rand(n, generator=torch.Generator().manual_seed(seed + 1), dtype=torch.float64) * 7.0 - 6.0)
    s[7] = 0.0
    return s


def _problem(problem, seed):
    """(shapes, initial params, grad_fn(t, gvars) -> list of CPU gradients, also handed to the engine)."""
    gen = torch.Generator().manual_seed(seed + 1)
    if problem == "convnet":
        from open_l2o_b200.scale_problems import ConvNet
        prob = ConvNet(*HRNN_CONVNET)
        shapes = [tuple(s) for s in prob.param_shapes]
        params = [p.detach() for p in prob.init_tensors(seed=0, device="cpu")]
        data = torch.randn(128, 32, 32, 3, generator=gen).to(DEV)
        labels = torch.nn.functional.one_hot(torch.randint(0, 10, (128,), generator=gen), 10).float().to(DEV)

        def grad_fn(t, gvars):
            ps = [v.detach().clone().requires_grad_(True) for v in gvars]
            return [g.detach().cpu() for g in torch.autograd.grad(prob.objective(ps, data, labels), ps)]
        return shapes, params, grad_fn
    if problem == "ragged":
        shapes = hrnn_ragged_shapes()
        scales = ragged_grad_scales(len(shapes))
        params = [torch.randn(s, generator=gen) for s in shapes]

        def grad_fn(t, gvars):
            out = []
            for s, sc in zip(shapes, scales):
                g = (torch.randn(s, generator=gen, dtype=torch.float64) * sc).float()
                g.view(-1)[t % 5::5] = 0.0          # exact zeros at coordinates that move from step to step
                out.append(g)
            return out
        return shapes, params, grad_fn
    shapes = problem
    params = [torch.randn(s, generator=gen) for s in shapes]
    return shapes, params, lambda t, gvars: [torch.randn(s, generator=gen) * (0.3 if t % 2 == 0 else 3e-3) for s in shapes]


def _ids(*parts):
    return "-".join(str(p) for p in parts)


_SMALL = [[(3, 3, 3, 8), (8,), (40, 5), (5,)],   # ragged, tiny tensors
          [(700, 300), (1,), (257,)],           # multi-block tensor + size 1
          [(64,)]]
STEP_CASES = ([pytest.param(s, n, "init", False, id=_ids("shapes%d" % k, n)) for k, (s, n) in enumerate(zip(_SMALL, (6, 4, 3)))]
              + [pytest.param(_SMALL[0], 6, "generic", False, id="shapes0-6-generic"),
                 pytest.param(_SMALL[1], 4, "generic", True, id="shapes1-4-clip")]
              + [pytest.param(p, 3, th, clip, id=_ids(p, th if not clip else "clip"))
                 for p in ("convnet", "ragged") for th, clip in (("init", False), ("generic", False), ("generic", True))])


@pytest.mark.parametrize("shapes,steps,theta_kind,clip", STEP_CASES)
def test_hrnn_steps_match_oracle(shapes, steps, theta_kind, clip):
    """One engine step after another against the fp32 and fp64 oracle steps fed the same gradients.  theta_kind
    "generic" (tests/helpers.hrnn_generic_theta) makes every zero / repeated-constant block of the initial weights
    distinct; clip starts a third of the coordinates at log-lr = -33 so that the step log-lr is clipped.  "convnet"
    (BASELINE #4, its own gradients) has one tensor long enough for coord_tc_kernel's periodic flush of the per-tensor
    sums; "ragged" has > 300 tensors at tile-edge sizes, gradients from 1e-6 to 10, exact zeros and one all-zero
    gradient.  Each tensor is held to 3x its own fp32-oracle distance from fp64 (at least 1e-5)."""
    from open_l2o_b200 import hierarchical_rnn as hr
    problem = shapes
    shapes, params, grad_fn = _problem(problem, 3)
    tiles = [math.ceil(math.prod(s) / HRNN_TILE) for s in shapes]
    if problem == "convnet":   # some CTA must see more than FLUSH_TILES tiles of one tensor, or the flush never runs
        assert max(tiles) > FLUSH_TILES * CTAS_PER_SM * _sms(), (max(tiles), _sms())
    if problem == "ragged":    # tensor_kernel (64 threads) walks the [tensors x 4] flags with a stride: it must wrap
        assert len(shapes) * 4 > 64 and sum(tiles) > CTAS_PER_SM * _sms(), (len(shapes), sum(tiles), _sms())
    opt = hr.HierarchicalRNN(random_seed=3, **hr.metarun_flags())
    if theta_kind == "generic":
        opt.theta.copy_(hrnn_generic_theta(5).to(DEV))
    theta = opt.theta.detach().cpu().clone()
    assert theta.numel() == H.theta_count()
    gvars = [p.clone().to(DEV) for p in params]
    grads0 = grad_fn(0, gvars)
    opt.apply_gradients(zip([g.to(DEV) for g in grads0], gvars))          # creates the slots, then steps
    # rebuild the oracle's initial state from the engine's own initial draw (log-lr is random): re-run from scratch
    P = H.unpack_theta(theta)
    opt.reset_state(seed=11)
    if clip:
        llr = opt.state[12].clone()
        llr[::3] = -33.0
        opt.reset_state(log_learning_rate=llr)
    for v, p in zip(gvars, params):
        v.data.copy_(p.to(DEV))
    llr = opt.state[12].detach().cpu().clone()
    states32, states64 = [], []
    off = 0
    for p in params:
        n = p.numel()
        st = H.initial_state(P, p, torch.Generator().manual_seed(0))
        st["log_learning_rate"] = llr[off:off + n].reshape(n, 1).clone()
        states32.append(st)
        states64.append({k: v.double() for k, v in st.items()})
        off += n
    g32, g64 = H.initial_global_state(P), H.initial_global_state(P).double()
    p32, p64 = [p.clone() for p in params], [p.double() for p in params]
    th64 = theta.double()
    P64 = H.unpack_theta(th64)
    clipped = inside = 0
    for t in range(steps):
        llr_old = [st["log_learning_rate"] for st in states64]
        grads = grad_fn(t, gvars)
        opt.apply_gradients(zip([g.to(DEV) for g in grads], gvars))
        p32, states32, g32, u32 = H.step(theta, p32, grads, states32, g32)
        p64, states64, g64, u64 = H.step(th64, p64, [g.double() for g in grads], states64, g64)
        torch.cuda.synchronize()
        # per tensor: 3x the fp32 oracle's own distance from fp64 on that tensor, at least REL_TOL; a state plane that
        # is worse conditioned than the hidden state (the gradient accumulators of a one-coordinate tensor, where
        # acc = g (1 - d) + acc_old d can cancel) is held to 3x its own fp32 distance
        slacks = [max(REL_TOL, 3.0 * rel_err(states32[j]["parameter"], states64[j]["parameter"]),
                      3.0 * rel_err(p32[j], p64[j])) for j in range(len(shapes))]
        off = 0
        for j, p in enumerate(params):
            n, slack = p.numel(), slacks[j]
            assert rel_err(gvars[j], p64[j]) <= slack, (problem, t, j, "x")
            e_u = rel_err(opt.update[off:off + n], u64[j])
            tol = max(3 * slack, 3.0 * rel_err(u32[j], u64[j]))
            assert e_u <= tol, (problem, t, j, "update", e_u, tol)
            for key in ("parameter", "scl_decay", "inp_decay", "log_learning_rate", "grad_accum1", "grad_accum4",
                        "ms1", "ms4", "layer"):
                e_k = rel_err(opt.get_slot(j, key), states64[j][key])
                tol = max(3 * slack, 3.0 * rel_err(states32[j][key], states64[j][key]))
                assert e_k <= tol, (problem, t, j, key, e_k, tol)
            off += n
        slack = max(slacks)
        assert rel_err(opt.global_state, g64) <= 3 * slack, (t, "global", rel_err(opt.global_state, g64), slack)
        if clip:   # count the coordinates whose step log-lr l + lr_change fell below the clip
            for o, st in zip(llr_old, states64):
                pre = o + (st["parameter"] @ P64["learning_rate_weights"] + P64["learning_rate_bias"])
                clipped += int((pre < -33.0).sum())
                inside += int(((o == -33.0) & (pre > -33.0)).sum())
    if clip:   # the case must reach what it is meant to: the clip active at some coordinates and not at others
        assert clipped > 0 and inside > 0, (clipped, inside)


def test_hrnn_argument_errors():
    from open_l2o_b200 import hierarchical_rnn as hr
    with pytest.raises(ValueError):
        hr.HierarchicalRNN(level_sizes=[10, 20, 20, 5])
    with pytest.raises(ValueError):
        hr.HierarchicalRNN(level_sizes=[10, 20, 20], init_lr_range=(1e-2, 1e-6))
    with pytest.raises(NotImplementedError):
        hr.HierarchicalRNN(level_sizes=[10, 20, 20])      # the reference's signature defaults are not the built flag set
    opt = hr.HierarchicalRNN(**hr.metarun_flags())
    with pytest.raises(ValueError):
        opt.apply_gradients([(None, torch.zeros(3, device=DEV))])


def test_hrnn_minimizes_a_quadratic():
    """Smoke-level behaviour check: with random-init weights the optimizer still moves downhill on a bowl
    (the update direction is the RMS-normalised gradient shortcut, HR:612-626)."""
    from open_l2o_b200 import hierarchical_rnn as hr
    opt = hr.HierarchicalRNN(random_seed=0, **hr.metarun_flags())
    w = torch.randn(300, 30, device=DEV).requires_grad_(True)
    b = torch.randn(30, device=DEV).requires_grad_(True)
    objs = opt.minimize(lambda w, b: (w ** 2).sum() + (b ** 2).sum(), [w, b], 60)
    assert objs[-1] < objs[0]


def test_hrnn_minimize_graph_replay_matches_eager():
    """HierarchicalRNN.minimize captures one (objective, gradients, step) iteration as a CUDA graph; the objective
    trajectory must equal the eager one."""
    from open_l2o_b200 import hierarchical_rnn as hr
    out = []
    for use_graph in (False, True):
        opt = hr.HierarchicalRNN(random_seed=0, **hr.metarun_flags())
        gen = torch.Generator().manual_seed(5)
        w = torch.randn(200, 20, generator=gen).to(DEV).requires_grad_(True)
        b = torch.randn(20, generator=gen).to(DEV).requires_grad_(True)
        t = torch.randn(64, 200, generator=gen).to(DEV)
        out.append(opt.minimize(lambda w, b: ((t @ w + b) ** 2).mean(), [w, b], 12, cuda_graph=use_graph))
    assert len(out[0]) == len(out[1]) == 12
    assert max(abs(a - c) / (abs(a) + 1e-30) for a, c in zip(out[0], out[1])) <= 1e-6


def test_hrnn_sharded_step_matches_single_gpu():
    """Coordinates of every tensor split over 2 ranks (one all-reduce of the per-tensor sums per step + an all-gather of
    the updated parameters, scripts/hrnn_dist_check.py under torchrun) against the single-GPU optimizer."""
    import os
    import subprocess
    import sys
    # < 2 GPUs: both ranks share cuda:0 and the collectives go through gloo (see the script) - never skipped
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29541",
                        os.path.join(root, "scripts", "hrnn_dist_check.py")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "PASS" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
