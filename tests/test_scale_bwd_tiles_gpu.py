"""GPU: the L2O-Scale backward kernels output by output against fp64 autograd through the oracles, at sizes chosen by
how many tiles each CTA walks.

l2o_crnn_bwd runs one persistent CTA per SM over tiles of 128 coordinates and sums d theta over every tile it walks in a
per-CTA shared-memory image; l2o_tadam_bwd / l2o_lrsgd_bwd run grid-stride loops with per-thread fp64 accumulators over
an occupancy-capped grid; l2o_hrnn_coord_bwd runs up to 2 CTAs per SM over per-tensor tiles with its own image.  A slip
that only shows once a CTA (or a thread) walks a second tile — an image re-zeroed or flushed per tile, an accumulator
that keeps one iteration, a ragged-tile predicate that goes wrong after the first tile — leaves small problems
correct.  So every case states how many tiles its CTAs walk, and checks each output on its own scale: every theta
block, every old-plane adjoint and d g, within 1e-5 max-norm relative of the fp64 reference, or 3x the fp32 oracle's
distance from fp64 where that is larger; an output whose reference is exactly 0 must be exactly 0.

The references are the oracles run by torch on the GPU in fp64 (and fp32, for the round-off scale), over coordinate
chunks for the coordinate-wise optimizers (tests/test_scale_bwd_reference_cpu.py checks the chunking on the CPU)."""
import ctypes
import math
from functools import partial

import pytest
import torch

from oracle import crnn_oracle as CR
from oracle import hrnn_oracle as H
from tests.helpers import HRNN_CONVNET, HRNN_TILE, REL_TOL, hrnn_generic_theta, hrnn_ragged_shapes
from tests.test_baselines_cpu import tadam_theta
from tests.test_crnn_gpu import crnn_generic_theta
from tests.test_scale_bwd_reference_cpu import (TADAM_THETA, chunked_vjp, crnn_generic_planes, crnn_vjp, lrs_vjp,
                                                tadam_generic_planes, tadam_vjp)
from tests.test_second_order_gpu import HRNN_KEYS, _crnn_bwd, _hrnn_planes

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TILE = 128          # coordinates per tile of l2o_crnn_bwd, one CTA per SM (about 150 KB of shared memory each)
BASE_BLOCK = 256    # threads per CTA of l2o_tadam_bwd / l2o_lrsgd_bwd: at most 2048 / 256 = 8 CTAs per SM
CONVNET_N = 354218


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _size(case):
    """Coordinates of a case, from the SM count: "tile" one ragged tile; "tail" SMs x 128 + 77, so CTA 0 walks a full
    tile and then the ragged tail; "convnet" the ConvNet benchmark's 354,218 (21 tiles per CTA on 132 SMs); "large"
    250 tiles per CTA, the last one 77 coordinates short (an odd count, about 4.2 M on 132 SMs)."""
    s = _sms()
    return {"tile": 77, "tail": s * TILE + 77, "convnet": CONVNET_N, "large": s * TILE * 250 - 51}[case]


def _crnn_tiles_per_cta(n):
    """Tiles CTA 0 of l2o_crnn_bwd walks: the grid is min(tiles, SMs) (one CTA per SM)."""
    tiles = -(-n // TILE)
    return -(-tiles // min(tiles, _sms()))


CASES = ["tile", "tail", "convnet", "large"]
CRNN_TILES = {"tile": 1, "tail": 2, "large": 250}   # convnet: 21 on 132 SMs, asserted >= 16


def _assert_tiles(case, n):
    t = _crnn_tiles_per_cta(n)
    if case == "convnet":
        assert n == CONVNET_N and t >= 16, t
    else:
        assert t == CRNN_TILES[case], (case, t)
    if case == "large":   # every thread of the baselines' grid-stride loops runs >= 15 iterations
        assert n % 2 == 1 and n >= 15 * BASE_BLOCK * 8 * _sms()
    return t


@pytest.fixture(autouse=True)
def _exact_fp32_matmul():
    """The fp32 oracle measures the round-off of an exact fp32 evaluation: no TF32 in its matmuls."""
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _both(vjp):
    """`vjp` in fp64 and in fp32 on the same chunk, stacked (fp64 first) for chunked_vjp."""
    def f(theta, planes, g, d_new, d_upd, dtype):
        a = vjp(theta, planes, g, d_new, d_upd, torch.float64)
        b = vjp(theta, planes, g, d_new, d_upd, torch.float32)
        return tuple(None if x is None else torch.stack([x.double(), y.double()]) for x, y in zip(a, b))
    return f


class _Rows(object):
    """Running per-row maxima over coordinate chunks of |got - ref64|, |ref32 - ref64| and |ref64|."""

    def __init__(self, names):
        self.names = list(names)
        z = lambda: torch.zeros(len(self.names), dtype=torch.float64, device=DEV)
        self.err, self.own, self.ref = z(), z(), z()

    def add(self, got, r64, r32):
        got, r64, r32 = (t.double().reshape(len(self.names), -1) for t in (got, r64, r32))
        self.err = torch.maximum(self.err, (got - r64).abs().amax(1))     # (NaN propagates)
        self.own = torch.maximum(self.own, (r32 - r64).abs().amax(1))
        self.ref = torch.maximum(self.ref, r64.abs().amax(1))

    def rows(self):
        return list(zip(self.names, self.err.tolist(), self.own.tolist(), self.ref.tolist()))


def _judge(tag, rows, tol=REL_TOL):
    """rows of (name, max |got - ref64|, max |ref32 - ref64|, max |ref64|): exact 0 where the reference is 0, else
    within max(tol, 3x the fp32 oracle's distance) of the reference's own scale.  Prints the worst relative errors."""
    bad, rel = [], []
    for name, err, own, ref in rows:
        if ref == 0.0:
            if not err == 0.0:
                bad.append((name, "reference 0, got", err))
            continue
        rel.append((err / ref, name))
        if not err / ref <= max(tol, 3.0 * own / ref):
            bad.append((name, err / ref, own / ref))
    rel.sort(reverse=True)
    print("%s: worst rel err %s" % (tag, ", ".join("%s %.2e" % (nm, e) for e, nm in rel[:3])))
    assert not bad, (tag, bad[:10])


def _theta_rows(got, ref, blocks):
    """Per theta block (name, lo, hi): rows for _judge from the kernel's d theta and the stacked fp64 / fp32
    reference."""
    got, r64, r32 = got.double(), ref[0], ref[1]
    return [(name, float((got[lo:hi] - r64[lo:hi]).abs().max()), float((r32[lo:hi] - r64[lo:hi]).abs().max()),
             float(r64[lo:hi].abs().max())) for name, lo, hi in blocks]


def crnn_theta_blocks():
    """(name, lo, hi) of each block of CR.theta_spec(); an LSTM kernel splits into its input rows and recurrent rows."""
    out, off = [], 0
    for name, shape in CR.theta_spec():
        k = int(math.prod(shape))
        if name.endswith("/kernel"):
            k_in = (shape[0] - shape[1] // 4) * shape[1]
            out += [(name + "[inputs]", off, off + k_in), (name + "[h]", off + k_in, off + k)]
        else:
            out.append((name, off, off + k))
        off += k
    return out


def _cuts(n):
    """Two cut points that split [0, n) into three slices, none of them at a multiple of 128."""
    cuts = [n // 3 + 5, (2 * n) // 3 + 77]
    return [c + 1 if c % TILE == 0 else c for c in cuts]


# ---------------------------------------------------------------------------------------------------------------------
# CoordinatewiseRNN: l2o_crnn_bwd

def _crnn_inputs(n):
    theta = crnn_generic_theta(5)
    planes = crnn_generic_planes(theta, n, seed=11, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(12)
    g = torch.randn(n, generator=gen, device=DEV) * 0.3
    d_new = torch.randn(103, n, generator=gen, device=DEV)
    d_upd = torch.randn(n, generator=gen, device=DEV)
    return theta, planes, g, d_new, d_upd


def _crnn_call(theta_d, planes, g, d_new, d_upd):
    d_g = torch.empty_like(g)
    d_old, d_theta = _crnn_bwd(theta_d, planes, g, d_new, d_upd, d_g)
    return d_old, d_theta, d_g


@pytest.mark.parametrize("case", CASES)
def test_crnn_bwd_every_output_matches_oracle(case):
    """One l2o_crnn_bwd from a generic state (two fp64 oracle steps, rounded to fp32) with random adjoints of the 103
    new planes and the update, generic weights: each theta block (LSTM kernels split into input and recurrent rows),
    each of the 103 old-plane adjoints and d g against the chunked fp64 oracle.  init_vector gets exactly 0."""
    n = _size(case)
    tiles = _assert_tiles(case, n)
    torch.cuda.reset_peak_memory_stats()
    theta, planes, g, d_new, d_upd = _crnn_inputs(n)
    d_old, d_theta, d_g = _crnn_call(theta.to(DEV), planes, g, d_new, d_upd)
    rows = _Rows(["plane%d" % k for k in range(103)] + ["g"])

    def each(lo, hi, dp, dg):
        rows.add(torch.cat([d_old[:, lo:hi], d_g[lo:hi].reshape(1, -1)]), torch.cat([dp[0], dg[0:1]]),
                 torch.cat([dp[1], dg[1:2]]))
    ref = chunked_vjp(_both(crnn_vjp), theta.to(DEV), planes, g, d_new, d_upd, None, each=each)
    torch.cuda.synchronize()
    print("crnn %s: n=%d, %d tiles per CTA, peak %.2f GB" % (case, n, tiles, torch.cuda.max_memory_allocated() / 2**30))
    _judge("crnn %s theta" % case, _theta_rows(d_theta, ref, crnn_theta_blocks()))
    _judge("crnn %s planes" % case, rows.rows())


@pytest.mark.parametrize("case", ["tail", "convnet", "large"])
def test_crnn_bwd_does_not_depend_on_placement(case):
    """[0, n) split into three slices at offsets that are not multiples of 128, each run as its own call: every
    coordinate's old-plane adjoints and d g bit-identical to the whole call's, whichever tile and CTA handled it, and
    the slices' d theta summed within 1e-5 of the whole call's per block (each tile's contraction sums in fp32, and the
    slices group the coordinates into other tiles)."""
    n = _size(case)
    _assert_tiles(case, n)
    theta, planes, g, d_new, d_upd = _crnn_inputs(n)
    th = theta.to(DEV)
    d_old, d_theta, d_g = _crnn_call(th, planes, g, d_new, d_upd)
    total = torch.zeros_like(d_theta)
    edges = [0] + _cuts(n) + [n]
    for a, b in zip(edges[:-1], edges[1:]):
        s_old, s_theta, s_g = _crnn_call(th, planes[:, a:b].contiguous(), g[a:b].contiguous(),
                                         d_new[:, a:b].contiguous(), d_upd[a:b].contiguous())
        assert torch.equal(s_old, d_old[:, a:b]) and torch.equal(s_g, d_g[a:b]), (a, b)
        total += s_theta
        del s_old
    worst = []
    for name, lo, hi in crnn_theta_blocks():
        ref = float(d_theta[lo:hi].abs().max())
        err = float((total[lo:hi] - d_theta[lo:hi]).abs().max())
        if ref == 0.0:
            assert err == 0.0, name
            continue
        worst.append((err / ref, name))
    worst.sort(reverse=True)
    print("crnn %s placement: worst d theta rel diff %.2e (%s)" % (case, worst[0][0], worst[0][1]))
    assert worst[0][0] <= REL_TOL, worst[:5]


# ---------------------------------------------------------------------------------------------------------------------
# TrainableAdam: l2o_tadam_bwd; LearningRateSchedule / GlobalLearningRate: l2o_lrsgd_bwd

def _tadam_inputs(n):
    theta = tadam_theta(dtype=torch.float32, **TADAM_THETA).to(DEV)
    planes, g = tadam_generic_planes(n, seed=31, device=DEV)
    gen = torch.Generator(device=DEV).manual_seed(32)
    d_new = torch.randn(3, n, generator=gen, device=DEV)   # (the t row is ignored: t carries no adjoint)
    d_upd = torch.randn(n, generator=gen, device=DEV)
    return theta, planes, g, d_new, d_upd


def _tadam_call(theta, planes, g, d_new, d_upd):
    from open_l2o_b200 import _lib
    from open_l2o_b200.engine import _ptr as _p
    n = g.numel()
    d_old, d_g = torch.empty_like(planes), torch.empty_like(g)
    d_theta = torch.zeros(4, dtype=torch.float64, device=DEV)
    a = _lib.TadamBwdArgs(n=n, theta=_p(theta), g=_p(g), state_old=_p(planes), d_state_new=_p(d_new),
                          d_update=_p(d_upd), d_state_old=_p(d_old), d_theta=d_theta.data_ptr(), d_g=_p(d_g))
    _lib.check(_lib.lib().l2o_tadam_bwd(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "l2o_tadam_bwd")
    return d_old, d_theta, d_g


LRS_TABLES = {"lrs": ([0.3, -0.2, 0.45], [5, 0]),   # index min(5, 3 - 1) = 2: the clamped last entry
              "glr": ([0.37], None)}                # one entry, no counter


def _lrs_call(rates, itr, g, d_upd):
    from open_l2o_b200 import _lib
    from open_l2o_b200.engine import _ptr as _p
    d_rates = torch.zeros(rates.numel(), dtype=torch.float64, device=DEV)
    d_g = torch.empty_like(g)
    a = _lib.LrsgdBwdArgs(n=g.numel(), rates=_p(rates), n_steps=rates.numel(), itr=_p(itr, torch.int32), g=_p(g),
                          d_update=_p(d_upd), d_rates=d_rates.data_ptr(), d_g=_p(d_g))
    _lib.check(_lib.lib().l2o_lrsgd_bwd(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "l2o_lrsgd_bwd")
    return d_rates, d_g


def _lrs_inputs(n, table):
    rates, itr = LRS_TABLES[table]
    gen = torch.Generator(device=DEV).manual_seed(41)
    g, d_upd = (torch.randn(n, generator=gen, device=DEV) for _ in range(2))
    itr_d = None if itr is None else torch.tensor(itr, dtype=torch.int32, device=DEV)
    return torch.tensor(rates, device=DEV), itr_d, (0 if itr is None else itr[0]), g, d_upd


@pytest.mark.parametrize("case", CASES)
def test_tadam_bwd_every_output_matches_oracle(case):
    """One l2o_tadam_bwd from a state with v != 0 on two thirds of the coordinates (some g = 0, some g = 1e-25), with
    random adjoints of m', v' and the update: each of the 4 theta entries, the m and v adjoints and d g against the
    chunked fp64 oracle, and the t plane's adjoint exactly 0."""
    n = _size(case)
    _assert_tiles(case, n)
    theta, planes, g, d_new, d_upd = _tadam_inputs(n)
    d_old, d_theta, d_g = _tadam_call(theta, planes, g, d_new, d_upd)
    rows = _Rows(["m", "t", "v", "g"])

    def each(lo, hi, dp, dg):
        rows.add(torch.cat([d_old[:, lo:hi], d_g[lo:hi].reshape(1, -1)]), torch.cat([dp[0], dg[0:1]]),
                 torch.cat([dp[1], dg[1:2]]))
    ref = chunked_vjp(_both(tadam_vjp), theta, planes, g, d_new, d_upd, None, each=each)
    torch.cuda.synchronize()
    names = ["log_learning_rate", "beta1_logit", "beta2_logit", "log_epsilon"]
    trows = _theta_rows(d_theta, ref, [(nm, j, j + 1) for j, nm in enumerate(names)])
    assert all(r > 0 for _, _, _, r in trows), trows
    _judge("tadam %s theta" % case, trows)
    _judge("tadam %s planes" % case, rows.rows())
    assert float(d_old[1].abs().max()) == 0.0


@pytest.mark.parametrize("table", ["lrs", "glr"])
@pytest.mark.parametrize("case", CASES)
def test_lrsgd_bwd_matches_oracle(case, table):
    """l2o_lrsgd_bwd: d rates against the chunked fp64 oracle (the used entry; every other entry exactly 0) and d g,
    which is one fp32 product rate * d_upd, bit for bit."""
    n = _size(case)
    _assert_tiles(case, n)
    rates, itr_d, itr, g, d_upd = _lrs_inputs(n, table)
    d_rates, d_g = _lrs_call(rates, itr_d, g, d_upd)
    rows = _Rows(["g"])
    ref_g = []

    def each(lo, hi, dp, dg):
        rows.add(d_g[lo:hi], dg[0], dg[1])
        ref_g.append(torch.equal(d_g[lo:hi], dg[0].float()))
    ref = chunked_vjp(_both(partial(lrs_vjp, itr=itr)), rates, None, g, None, d_upd, None, each=each)
    torch.cuda.synchronize()
    _judge("%s %s rates" % (table, case), _theta_rows(d_rates, ref, [("rate%d" % j, j, j + 1)
                                                                      for j in range(rates.numel())]))
    _judge("%s %s g" % (table, case), rows.rows())
    assert all(ref_g)


@pytest.mark.parametrize("case", ["tail", "convnet", "large"])
def test_baselines_bwd_do_not_depend_on_placement(case):
    """As for the CoordinatewiseRNN: three slices at offsets that are not multiples of 128 give the whole call's
    per-coordinate adjoints bit for bit, and their d theta / d rates summed match the whole call's to 1e-12 (each
    coordinate's term is added in fp64)."""
    n = _size(case)
    theta, planes, g, d_new, d_upd = _tadam_inputs(n)
    d_old, d_theta, d_g = _tadam_call(theta, planes, g, d_new, d_upd)
    rates, itr_d, _, gl, d_updl = _lrs_inputs(n, "lrs")
    d_rates, d_gl = _lrs_call(rates, itr_d, gl, d_updl)
    tot_theta, tot_rates = torch.zeros_like(d_theta), torch.zeros_like(d_rates)
    edges = [0] + _cuts(n) + [n]
    for a, b in zip(edges[:-1], edges[1:]):
        s_old, s_theta, s_g = _tadam_call(theta, planes[:, a:b].contiguous(), g[a:b].contiguous(),
                                          d_new[:, a:b].contiguous(), d_upd[a:b].contiguous())
        assert torch.equal(s_old, d_old[:, a:b]) and torch.equal(s_g, d_g[a:b]), (a, b)
        s_rates, s_gl = _lrs_call(rates, itr_d, gl[a:b].contiguous(), d_updl[a:b].contiguous())
        assert torch.equal(s_gl, d_gl[a:b]), (a, b)
        tot_theta += s_theta
        tot_rates += s_rates
    for j in range(4):
        assert float(d_theta[j]) != 0.0
        assert abs(float(tot_theta[j] - d_theta[j])) <= 1e-12 * abs(float(d_theta[j])), (j, tot_theta, d_theta)
    assert float(d_rates[:2].abs().max()) == 0.0 and float(tot_rates[:2].abs().max()) == 0.0
    assert abs(float(tot_rates[2] - d_rates[2])) <= 1e-12 * abs(float(d_rates[2])), (tot_rates, d_rates)


# ---------------------------------------------------------------------------------------------------------------------
# HierarchicalRNN: one step through hrnn_train.MetaTrainer (l2o_hrnn_step_local, l2o_hrnn_coord_bwd, torch levels)

HRNN_COLS = [("parameter", 0, 10), ("scl_decay", 10, 1), ("inp_decay", 11, 1), ("log_learning_rate", 12, 1)] \
    + [("grad_accum%d" % (s + 1), 13 + s, 1) for s in range(4)] + [("ms%d" % (s + 1), 17 + s, 1) for s in range(4)]
assert [k for k, _, _ in HRNN_COLS] == HRNN_KEYS


def _hrnn_states(planes, layer, sizes):
    """The engine's planes [21, N] and per-tensor RNN states [n_tensors, 20] -> the oracle's per-tensor state dicts
    (views: autograd reaches planes and layer)."""
    out, off = [], 0
    for j, n in enumerate(sizes):
        p = planes[:, off:off + n].t()
        st = {k: p[:, c:c + w] for k, c, w in HRNN_COLS}
        st["layer"] = layer[j:j + 1]
        out.append(st)
        off += n
    return out


def _hrnn_shapes(kind):
    if kind == "convnet":
        from open_l2o_b200.scale_problems import ConvNet
        return [tuple(s) for s in ConvNet(*HRNN_CONVNET).param_shapes]
    return hrnn_ragged_shapes()   # 301 tensors


@pytest.mark.parametrize("kind", ["convnet", "ragged"])
def test_hrnn_step_every_adjoint_matches_oracle(kind):
    """One HierarchicalRNN step through MetaTrainer.unroll (second derivatives on) from a generic state two fp64 oracle
    steps in, with generic weights and random adjoints of every output (x, the 21 planes, the per-tensor and global RNN
    states).  Against fp64 autograd through the oracle on the GPU: every theta block, each of the 21 old planes on its
    own (a swapped pair of plane adjoints shows here, where a meta-gradient of theta alone could hide it), the old
    per-tensor and global states, x and the gradients G.  The coordinate kernels' CTAs walk >= 2 tiles each."""
    from open_l2o_b200 import hrnn_train as ht
    shapes = _hrnn_shapes(kind)
    sizes = [int(math.prod(s)) for s in shapes]
    n, nt = sum(sizes), len(sizes)
    tiles = sum(-(-s // HRNN_TILE) for s in sizes)
    assert tiles >= 4 * _sms(), (tiles, _sms())   # grid min(tiles, 2 x SMs): every CTA walks >= 2 tiles
    gen = torch.Generator().manual_seed(21)
    theta = hrnn_generic_theta(5)
    llr = torch.rand(n, generator=gen, dtype=torch.float64) * 3.0 - 6.0
    P64 = H.unpack_theta(theta.double())
    states, off = [], 0
    for s in sizes:
        st = H.initial_state(P64, torch.empty(s, dtype=torch.float64), torch.Generator().manual_seed(0))
        st["log_learning_rate"] = llr[off:off + s].reshape(-1, 1)
        off += s
        states.append({k: v.to(DEV) for k, v in st.items()})
    glob = H.initial_global_state(P64, torch.float64).to(DEV)
    th64 = theta.double().to(DEV)
    rnd = lambda *sh, scale=1.0: (torch.randn(*sh, generator=gen, dtype=torch.float64) * scale).to(DEV)
    params = [rnd(s, scale=0.5) for s in shapes]
    for _ in range(2):
        params, states, glob, _ = H.step(th64, params, [rnd(s, scale=0.3) for s in shapes], states, glob)
    planes = _hrnn_planes(states).float().contiguous()
    assert bool((planes[17:21] > 0).all())   # ms > 0: no tensor's first-step predicate fires
    layer = torch.cat([st["layer"] for st in states], 0).float()
    glob = glob.float()
    x0 = torch.cat([p.reshape(-1) for p in params]).float()
    G = rnd(n, scale=0.3).float()
    R_x, R_planes, R_layer, R_glob = rnd(n), rnd(21, n), rnd(nt, 20), rnd(1, 20)
    split = lambda v: [t.reshape(s) for t, s in zip(torch.split(v, sizes), shapes)]

    def oracle(dtype):
        th, pl, ly, gl, xs, Gl = (t.detach().to(dtype).requires_grad_(True) for t in (theta.to(DEV), planes, layer,
                                                                                       glob, x0, G))
        ps, new, gnew, _ = H.step(th, split(xs), split(Gl), _hrnn_states(pl, ly, sizes), gl)
        L = (R_x.to(dtype) * torch.cat([p.reshape(-1) for p in ps])).sum() \
            + (R_planes.to(dtype) * _hrnn_planes(new)).sum() \
            + (R_layer.to(dtype) * torch.cat([st["layer"] for st in new], 0)).sum() + (R_glob.to(dtype) * gnew).sum()
        return [d.double() for d in torch.autograd.grad(L, (th, pl, ly, gl, xs, Gl))]
    want64, want32 = oracle(torch.float64), oracle(torch.float32)

    tr = ht.MetaTrainer(shapes, theta=theta, device=DEV, use_second_derivatives=True)
    pl, ly, gl, xs, Gd = (t.detach().clone().requires_grad_(True) for t in (planes, layer, glob, x0, G))
    lin = lambda ps: sum((gj * p).sum() for gj, p in zip(tr._split(Gd), ps))   # its gradient is G, kept in the graph
    st0 = ht.OptimizerState(pl, ly, gl, torch.zeros(nt, 4, dtype=torch.int32, device=DEV), xs)
    _, _, fin = tr.unroll(lin, st0, 1)
    f = lambda t: t.float()
    L = (f(R_x) * fin.x).sum() + (f(R_planes) * fin.planes).sum() + (f(R_layer) * fin.layer).sum() \
        + (f(R_glob) * fin.global_state).sum()
    got = [d.double() for d in torch.autograd.grad(L, (tr.theta, pl, ly, gl, xs, Gd))]
    torch.cuda.synchronize()

    def row(name, e, w64, w32):
        return (name, float((e - w64).abs().max()), float((w32 - w64).abs().max()), float(w64.abs().max()))
    blocks, off = [], 0
    for name, shape in H.theta_spec():
        k = int(math.prod(shape))
        blocks.append((name, off, off + k))
        off += k
    _judge("hrnn %s theta" % kind, _theta_rows(got[0], torch.stack([want64[0], want32[0]]), blocks))
    _judge("hrnn %s planes" % kind, [row(HRNN_KEYS[0] + "[%d]" % k if k < 10 else HRNN_KEYS[k - 9], got[1][k],
                                         want64[1][k], want32[1][k]) for k in range(21)])
    _judge("hrnn %s states, x, G" % kind, [row(nm, got[j], want64[j], want32[j])
                                           for j, nm in ((2, "layer"), (3, "global"), (4, "x"), (5, "G"))])
