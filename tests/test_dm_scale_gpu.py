"""The L2O-DM LSTM engines at the benchmark's scale: T = 100 unrolls over 270K coordinates through the C ABI, and the
benchmark workload (1M coordinates) through MetaOptimizer, output by output and theta block by theta block against the
chunked fp64 oracle of tests/dm_scale_reference.py.

At these sizes every tensor-core BPTT warpgroup walks at least 16 tiles of 100 steps, so its dW drains and the
checkpoint ring's hand-over to the next tile run many times, and each exact-fp32 CTA walks many 128-coordinate tiles.  The checkpoint holds more than 2^31 floats, so slot T and every slot the backward reads near it sit past 2^31.

Every comparison is a max-norm relative error against the fp64 reference, with a bar of max(floor, 3 x the error of the
same oracle run in fp32): the fp32 run measures how far round-off alone carries each quantity over 100 steps."""
import types

import pytest
import torch

from oracle import l2o_oracle as orc
from tests.dm_scale_reference import BUDGET_BYTES, chunked_meta_grad
from tests.helpers import REL_TOL, SPECS, assert_theta_close, make_handle
from tests.test_kernels_gpu import _fused_problem
from tests.test_tc_bwd_blocks_gpu import BLOCK_TOL, theta_blocks

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
T = 100
N_FULL = 64 * 4224          # whole 64-coordinate tiles: the tensor-core kernels' FULL instantiations
N_RAG = N_FULL + 37         # a ragged last tile: the predicated instantiations
SLOT = 80                   # checkpoint floats per coordinate of an LSTM-20x2 (h1, c1, h2, c2)
# output-layer gains: the identity net (scale 1) moves x by O(0.1) per step at 0.05; the LogAndSign and RNNProp nets
# (scale 0.01) need the full Sonnet init to leave every theta block's meta-gradient clear of zero
GAIN = {"dm_identity": 0.05, "dm_logsign": 1.0, "rnnprop": 1.0}


def _tc_bptt_tiles_per_warpgroup(n):
    """Tiles the busiest and the least busy tensor-core BPTT warpgroup walk: 64-coordinate tiles, two warpgroups per
    CTA, grid = min(CTAs, SMs) (cwlstm_tc_bwd.cuh tc_launch_bwd)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ntiles = -(-n // 64)
    wgs = 2 * min(-(-ntiles // 2), sms)
    return -(-ntiles // wgs), ntiles // wgs


@pytest.mark.parametrize("n", [N_FULL, N_RAG])
def test_sizes_reach_the_regime(n):
    """Both sizes cross 2^31 checkpoint floats with slot T, and make every warpgroup walk at least 16 tiles."""
    assert (n % 64 == 0) == (n == N_FULL)
    assert SLOT * n * T >= 2 ** 31
    assert _tc_bptt_tiles_per_warpgroup(n)[1] >= 16, _tc_bptt_tiles_per_warpgroup(n)


def rel(a, b):
    """max-norm relative error of a against b, on the device."""
    a, b = a.reshape(-1).double(), b.reshape(-1).double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def bar(floor, r32, r64):
    return max(floor, 3.0 * rel(r32, r64))


# ---------------------------------------------------------------------------------------------------------------
# one fp64 and one fp32 reference per (net, problem, n); the cases of one key run next to each other
# ---------------------------------------------------------------------------------------------------------------
_REF = {}


def _reference(name, kind, n):
    key = (name, kind, n)
    if key not in _REF:
        _REF.clear()
        torch.cuda.empty_cache()
        spec = SPECS[name]
        prob, x0 = _fused_problem(kind, n, torch.Generator().manual_seed(7))
        theta = orc.init_theta(spec, seed=1, out_gain=GAIN[name])
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        r64 = chunked_meta_grad(spec, theta, prob, x0.to(DEV), T, torch.float64)
        peak = torch.cuda.max_memory_allocated() - base
        outputs = 8 * n * (1 + (T + 1) + 2 * sum(spec.layers) + (2 if spec.rnnprop else 0))
        assert peak - outputs <= BUDGET_BYTES, (peak, outputs)
        r32 = chunked_meta_grad(spec, theta, prob, x0.to(DEV), T, torch.float32)
        print(f"\nreference {key}: fp64 chunk peak {(peak - outputs) / 2 ** 30:.2f} GiB")
        _REF[key] = (spec, theta, prob, x0, r64, r32)
    return _REF[key]


def _engine(engine):
    from open_l2o_b200.engine import ENGINE_FFMA, ENGINE_TC
    return {"ffma": ENGINE_FFMA, "tc": ENGINE_TC}[engine]


def _forward(spec, engine, theta, prob, x0, n):
    """The fused T-step unroll on `engine`, recording what a BPTT reads."""
    from open_l2o_b200.engine import OPT_KINDS
    h = make_handle(spec)
    h.set_engine(_engine(engine))
    run = types.SimpleNamespace(h=h, th=theta.to(DEV), arena=h.new_state(n, DEV), x=x0.to(DEV).clone(),
                                ckpt=torch.zeros((T + 1) * h.state_size(n), device=DEV),
                                g_rec=torch.empty(T + 1, n, device=DEV),
                                fx=torch.zeros(T + 1, dtype=torch.float64, device=DEV),
                                delta=torch.empty(T, n, device=DEV), scratch=None)
    kw = {}
    run.in_seq = run.g_rec[:T]
    if spec.rnnprop:
        run.m, run.v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
        run.in_seq = torch.empty(T, 2, n, device=DEV)
        run.scratch = torch.empty(T, n, 20, device=DEV)
        kw = dict(m=run.m, v=run.v, beta1=0.95, beta2=0.95, step0=1, feat_rec=run.in_seq)
    h.unroll_fwd(run.th, n, T, run.arena, opt_kind=OPT_KINDS[prob.kind], opt_a=prob.a.to(DEV), opt_b=prob.b.to(DEV),
                 opt_alpha=prob.alpha, opt_fscale=prob.fscale, x=run.x, ckpt=run.ckpt, g_rec=run.g_rec, fx=run.fx,
                 delta_seq=run.delta, **kw)
    torch.cuda.synchronize()
    return run


def _check_blocks(spec, dtheta, r64, r32, floor, tag):
    """Every theta block against the fp64 reference at max(floor, 3 x the fp32 reference's error on that block);
    returns the worst block as (error / bar, block, error)."""
    worst = (0.0, None, 0.0)
    for block, off, cnt in theta_blocks(spec):
        ref = r64.dtheta[off:off + cnt]
        assert float(ref.abs().max()) > 0, (tag, block)
        b = bar(floor, r32.dtheta[off:off + cnt], ref)
        err = rel(dtheta[off:off + cnt], ref)
        assert err <= b, (tag, block, err, b)
        worst = max(worst, (err / b, block, err))
    print(f"\n{tag}: worst block {worst[1]} {worst[2]:.2e} ({worst[0]:.2f} of its bar)")
    return worst


# (net, problem, n, engine), grouped by reference
CASES = [
    ("dm_identity", "rastrigin_sep", N_RAG, "ffma"),
    ("dm_identity", "rastrigin_sep", N_RAG, "tc"),
    ("dm_identity", "rastrigin_sep", N_FULL, "tc"),
    ("dm_logsign", "rastrigin_sep", N_RAG, "ffma"),
    ("dm_logsign", "rastrigin_sep", N_RAG, "tc"),
    ("dm_logsign", "rastrigin_sep", N_FULL, "tc"),
    ("rnnprop", "rastrigin_sep", N_RAG, "ffma"),
    ("rnnprop", "rastrigin_sep", N_RAG, "tc"),
    ("dm_identity", "quadratic_diag", N_RAG, "ffma"),
    ("dm_identity", "quadratic_diag", N_RAG, "tc"),
]


@pytest.mark.parametrize("engine", ["ffma", "tc"])
def test_carry_segments_every_theta_block(engine):
    """l2o_unroll_bwd_carry as 10 segments of 10 steps, last first, over the whole unroll's checkpoints: each segment
    ends every fp32 dW sum early and hands on the adjoint state and lambda through HBM."""
    spec, theta, prob, x0, r64, r32 = _reference("dm_identity", "rastrigin_sep", N_RAG)
    n = N_RAG
    run = _forward(spec, engine, theta, prob, x0, n)
    h, slot = run.h, run.h.state_size(n)
    dtheta = torch.zeros(h.n_theta, dtype=torch.float64, device=DEV)
    d_state = torch.zeros(slot, device=DEV)
    lam = torch.zeros(n, device=DEV)
    for t0 in range(T - 10, -1, -10):
        h.unroll_bwd_carry(run.th, n, 10, run.in_seq[t0:], run.ckpt[t0 * slot:], dtheta, d_state, lam,
                           g_rec=run.g_rec[t0:], delta_seq=run.delta[t0:])
    torch.cuda.synchronize()
    assert rel(lam, r64.g_rec[1:].sum(0)) <= bar(REL_TOL, r32.g_rec[1:].double().sum(0), r64.g_rec[1:].sum(0))
    _check_blocks(spec, dtheta, r64, r32, REL_TOL if engine == "ffma" else BLOCK_TOL, f"carry {engine}")


@pytest.mark.parametrize("name,kind,n,engine", CASES, ids=[f"{c[0]}-{c[1]}-{c[2]}-{c[3]}" for c in CASES])
def test_engine_unroll_and_bptt_match_chunked_fp64(name, kind, n, engine):
    """Forward: fx, x_T, the final (h, c) of each layer, every g_rec row and RNNProp's m and v.  Checkpoint slot T is
    bitwise the final state.  BPTT: every theta block."""
    spec, theta, prob, x0, r64, r32 = _reference(name, kind, n)
    run = _forward(spec, engine, theta, prob, x0, n)
    tag = f"{name} {kind} n={n} {engine}"

    assert rel(run.fx, r64.fx) <= bar(REL_TOL, r32.fx, r64.fx), tag
    assert rel(run.x, r64.x) <= bar(REL_TOL, r32.x, r64.x), tag
    for li, ((hg, cg), (h64, c64), (h32, c32)) in enumerate(zip(run.h.state_views(run.arena, n), r64.state,
                                                                r32.state)):
        assert rel(hg, h64) <= bar(REL_TOL, h32, h64), (tag, "h", li)
        assert rel(cg, c64) <= bar(REL_TOL, c32, c64), (tag, "c", li)
    if spec.rnnprop:
        assert rel(run.m, r64.mv[0]) <= bar(REL_TOL, r32.mv[0], r64.mv[0]), tag
        assert rel(run.v, r64.mv[1]) <= bar(REL_TOL, r32.mv[1], r64.mv[1]), tag
    # g_rec row by row: a late row is not hidden behind an early, larger one
    g64 = r64.g_rec
    den = g64.abs().amax(1).clamp_min(1e-30)
    row_err = (run.g_rec.double() - g64).abs().amax(1) / den
    row_bar = (3.0 * (r32.g_rec.double() - g64).abs().amax(1) / den).clamp_min(REL_TOL)
    bad = torch.nonzero(row_err > row_bar).flatten().tolist()
    assert not bad, (tag, bad[:5], row_err[bad[:5]].tolist(), row_bar[bad[:5]].tolist())

    slot = run.h.state_size(n)
    assert run.ckpt.numel() > 2 ** 31 and T * slot >= 2 ** 31
    assert torch.equal(run.ckpt[T * slot:], run.arena), tag

    dtheta = torch.zeros(run.h.n_theta, dtype=torch.float64, device=DEV)
    run.h.unroll_bwd(run.th, n, T, run.in_seq, run.ckpt, dtheta, g_rec=run.g_rec, delta_seq=run.delta,
                     scratch=run.scratch)
    torch.cuda.synchronize()
    _check_blocks(spec, dtheta, r64, r32, REL_TOL if engine == "ffma" else BLOCK_TOL, tag)


# ---------------------------------------------------------------------------------------------------------------
# the benchmark workload through MetaOptimizer
# ---------------------------------------------------------------------------------------------------------------
BENCH_N = 1_000_000
BENCH_NET = {"net": "CoordinateWiseDeepLSTM", "net_options": {"layers": (20, 20), "scale": 0.1}}
_BENCH_REF = {}


def _bench_bytes(n):
    """Device memory of the unsegmented benchmark program plus its chunked references: the checkpoints, the recorded
    gradients, x and its copies, the fp64 and fp32 reference outputs, and one chunk's autograd graph."""
    ckpt = 4 * (T + 1) * SLOT * n
    program = 4 * ((T + 1) * n + SLOT * n + 8 * n)
    outputs = 12 * n * (1 + (T + 1) + SLOT // 2)
    return ckpt + program + outputs + BUDGET_BYTES


def _bench_reference(theta, X, b, c):
    """fp64 and fp32 chunked references, shared by the two programs when they start from the same point."""
    inputs = (theta, X, b, c)
    if "in" not in _BENCH_REF or not all(torch.equal(u, v) for u, v in zip(_BENCH_REF["in"], inputs)):
        _BENCH_REF.clear()
        spec = orc.NetSpec(layers=(20, 20), scale=0.1)
        prob = orc.FusedProblem("rastrigin_sep", b, c, alpha=10.0, fscale=1.0 / X.numel())
        r64 = chunked_meta_grad(spec, theta, prob, X, T, torch.float64)
        r32 = chunked_meta_grad(spec, theta, prob, X, T, torch.float32)
        for r in (r64, r32):
            r.g_rec = r.state = None   # not compared here
        _BENCH_REF.update({"in": inputs, "spec": spec, "r64": r64, "r32": r32})
    return _BENCH_REF["spec"], _BENCH_REF["r64"], _BENCH_REF["r32"]


@pytest.mark.parametrize("segment", [None, 10])
def test_benchmark_workload_matches_chunked_fp64(segment):
    """problems.rastrigin_separable(1M) with the LSTM-20x2 net of bench.py, T = 100, learning rate 0.001: one
    sess.run([fx, x, update, step]) against the chunked fp64 oracle from the same x, b, c and theta.  Unsegmented, the
    program holds 32.3 GB of checkpoints; segmented, it recomputes them 10 steps at a time."""
    from open_l2o_b200 import meta, problems
    _REF.clear()
    torch.cuda.empty_cache()
    if segment is None:
        free = torch.cuda.mem_get_info(DEV)[0]
        need = _bench_bytes(BENCH_N)
        if free < need:
            pytest.skip(f"the unsegmented benchmark program and its reference need {need / 1e9:.1f} GB, "
                        f"{free / 1e9:.1f} GB free")
    kw = {} if segment is None else {"_bptt_segment": segment}
    optimizer = meta.MetaOptimizer(cw=BENCH_NET, **kw)
    step, update, reset, fx, x = optimizer.meta_minimize(problems.rastrigin_separable(num_dims=BENCH_N), T,
                                                         learning_rate=0.001)
    prog = optimizer.program
    assert prog.segmented == (segment is not None)
    sess = meta.Session()
    sess.run(reset)
    (key, net), = prog.nets.items()
    theta0, X0 = net.theta.detach().clone(), prog.X.clone()
    b, c = prog.const_vals["b"].clone(), prog.const_vals["c"].clone()
    torch.cuda.reset_peak_memory_stats()
    cost, xs, _, _ = sess.run([fx, x, update, step])
    torch.cuda.synchronize()
    spec, r64, r32 = _bench_reference(theta0, X0, b, c)
    print(f"\nbenchmark workload, segment {segment}: peak {torch.cuda.max_memory_allocated() / 1e9:.1f} GB")

    f64, f32 = r64.fx[-1:], r32.fx[-1:]
    assert rel(torch.tensor([cost], dtype=torch.float64, device=DEV), f64) <= bar(REL_TOL, f32, f64)
    assert rel(torch.as_tensor(xs[0], device=DEV), r64.x) <= bar(REL_TOL, r32.x, r64.x)
    _check_blocks(spec, prog.dtheta[key], r64, r32, BLOCK_TOL, f"benchmark workload, segment {segment}")
    zeros = torch.zeros_like(r64.dtheta)
    theta1, _, _ = orc.tf_adam_step(theta0.double(), r64.dtheta, zeros, zeros, 1, lr=0.001)
    assert_theta_close(net.theta, types.SimpleNamespace(theta=theta1.cpu(), last_grad=r64.dtheta.cpu()), segment)
