"""The LFISTA and LAMP kernels through their C ABI (l2o_ista_fwd / l2o_ista_bwd), at what the models never pass:
every layer range [k0, k1) from a given x_{k0} and second state (LFISTA x_{k0-1}, LAMP v_{k0-1}) with the gradients
of both coming in and going out, the largest shared-memory plans, M or N below 8 (CTAs with empty column slices),
optional weight-gradient outputs left NULL, strided y, partial clusters of rows and LAMP rows with rvar = 0.  Every
check is against the fp64 oracle of tests/lfista_lamp_cases.py with autograd for the gradients, or bit for bit
against another launch."""
import ctypes as C

import numpy as np
import pytest
import torch

from open_l2o_b200 import _lib, lista
from tests import lfista_lamp_cases as fc
from tests.lfista_lamp_cases import EXACT2_CASES, K2, RANGES2, SPLITS2

pytestmark = pytest.mark.gpu

GUARD = 37            # sentinel elements past the end of every output
PAD_COLS, PAD_ROWS = 3, 5   # NaN columns past M in every y row, NaN rows past the batch in every input row matrix
SENTINEL = {torch.float32: 1234.5, torch.float64: -4321.25}


# ------------------------------------------------------------------------------------------------ kernel harness
class _Bufs:
    """Output buffers prefilled with NaN, each followed by GUARD sentinels that must stay intact."""

    def __init__(self):
        self.flat = []

    def out(self, shape, dtype):
        n = int(np.prod(shape))
        f = torch.empty(n + GUARD, dtype=dtype, device="cuda")
        f[:n] = float("nan")
        f[n:] = SENTINEL[dtype]
        self.flat.append((f, n))
        return f[:n].view(shape)

    def check_guards(self):
        for f, n in self.flat:
            assert bool((f[n:] == SENTINEL[f.dtype]).all()), "write past the end of an output"


def _cuda(t):
    return None if t is None else t.float().contiguous().cuda()


def _p(t):
    return None if t is None else t.data_ptr()


def _padded(t, cols):
    """A [rows, cols] CUDA tensor: t in the top-left corner, NaN around it (columns past t's, PAD_ROWS rows)."""
    if t is None:
        return None
    buf = torch.full((t.shape[0] + PAD_ROWS, cols), float("nan"), dtype=torch.float32)
    buf[:t.shape[0], :t.shape[1]] = t
    return buf.cuda()


def launch2(P, k0=0, k1=K2, x_in="P", s2_in="P", d_xk="P", d_s2="P", backward=True, pad_cols=PAD_COLS,
            dW=True, dW2=True, dstep=True):
    """l2o_ista_fwd (and l2o_ista_bwd) on P over [k0, k1) with every record; returns the outputs on the CPU.  y has
    row stride M + pad_cols with NaN padding; y, x_in, s2_in, d_xk and d_s2 have NaN rows past the batch.  dW, dW2
    and dstep False pass those outputs as NULL."""
    form, M, N, B = P["form"], P["M"], P["N"], P["B"]
    lamp = form == lista.LAMP
    S2 = M if lamp else N
    x_in, s2_in = fc._arg(P, x_in, "x_in"), fc._arg(P, s2_in, "s2_in")
    d_xk, d_s2 = fc._arg(P, d_xk, "d_xk"), fc._arg(P, d_s2, "d_s2")
    L, bufs = _lib.lib(), _Bufs()
    dev = {k: _cuda(P[k]) for k in ("A", "We", "W", "W2", "theta", "step", "gscale")}
    y = _padded(P["y"], M + pad_cols)
    xi, si = _padded(x_in, N), _padded(s2_in, S2)
    Lp = k1 - k0
    a = _lib.IstaArgs()
    a.form, a.batch, a.m, a.n, a.num_layers, a.k0, a.k1 = form, B, M, N, K2, k0, k1
    a.share_W = int(P["share_W"])
    a.A, a.B1, a.W, a.W2, a.theta, a.step = (_p(dev[k]) for k in ("A", "We", "W", "W2", "theta", "step"))
    a.y, a.ldy, a.x_in, a.s2_in = y.data_ptr(), M + pad_cols, _p(xi), _p(si)
    f32, f64 = torch.float32, torch.float64
    o = {"xs": bufs.out((Lp, B, N), f32), "zs": bufs.out((Lp, B, N), f32),
         "rs": bufs.out((Lp, B, M), f32) if lamp else None, "rowrec": bufs.out((Lp, B, 2), f32) if lamp else None}
    a.xs, a.zs, a.rs, a.rowrec = (_p(o[k]) for k in ("xs", "zs", "rs", "rowrec"))
    _lib.check(L.l2o_ista_fwd(C.byref(a), None), "l2o_ista_fwd")
    if backward:
        nb = C.c_size_t()
        _lib.check(L.l2o_ista_workspace_bytes(C.byref(a), C.byref(nb)), "l2o_ista_workspace_bytes")
        scratch = torch.empty((nb.value + 3) // 4, dtype=f32, device="cuda")
        dx, ds = _padded(d_xk, N), _padded(d_s2, S2)
        o["d_x_in"], o["d_s2_in"] = bufs.out((B, N), f32), bufs.out((B, S2), f32)
        o["dW"] = bufs.out(tuple(P["W"].shape), f64) if dW else None
        o["dW2"] = bufs.out(tuple(P["W2"].shape), f64) if dW2 and not lamp else None
        o["dB1"] = bufs.out((N, M), f64) if not lamp else None
        o["dtheta"] = bufs.out((K2,), f64)
        o["dstep"] = bufs.out((K2,), f64) if dstep and P["step"] is not None else None
        gr = _lib.IstaGrads()
        gr.d_xk, gr.d_s2, gr.scratch, gr.gscale = _p(dx), _p(ds), _p(scratch), _p(dev["gscale"])
        gr.d_x_in, gr.d_s2_in, gr.dW, gr.dW2, gr.dB1, gr.dtheta, gr.dstep = \
            (_p(o[k]) for k in ("d_x_in", "d_s2_in", "dW", "dW2", "dB1", "dtheta", "dstep"))
        _lib.check(L.l2o_ista_bwd(C.byref(a), C.byref(gr), None), "l2o_ista_bwd")
    torch.cuda.synchronize()
    bufs.check_guards()
    return {k: (None if v is None else v.cpu()) for k, v in o.items()}


# ------------------------------------------------------------------------------------------------ comparisons
REC = ("xs", "zs", "rs", "rowrec")
GRADS = ("d_x_in", "d_s2_in", "dW", "dW2", "dB1", "dtheta", "dstep")


def assert_exact(got, ref, keys):
    for k in keys:
        if ref.get(k) is None or got.get(k) is None:
            continue
        g, r = got[k].double(), ref[k].double()
        bad = g != r
        assert int(bad.sum()) == 0, (k, int(bad.sum()), g[bad][:5], r[bad][:5])


def masks(P, zs, rowrec, k0=0):
    """Each layer's classification from records (the kernel's in fp32, or the oracle's): LFISTA |z| > theta_k,
    z != 0; LAMP r != 0 and |r| >= max(sqrt(rvar) lam_k, 0) with the recorded sqrt(rvar)."""
    th = P["theta"].to(zs.dtype)
    out = []
    for l in range(zs.shape[0]):
        z = zs[l]
        if P["form"] == lista.LFISTA:
            out.append((z.abs() > th[k0 + l]) & (z != 0))
        else:
            t = torch.clamp_min(rowrec[l][:, :1] * th[k0 + l], 0.0)
            out.append((z != 0) & (z.abs() >= t))
    return out


def _rel(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _rel_rows(a, b, mag):
    """The worst row's max |a - b| over its max |mag| ([B, N]); a row where mag is all zero must match exactly."""
    err, mag = (a.double() - b.double()).abs().amax(dim=1), mag.double().abs().amax(dim=1)
    return float(torch.where(mag > 0, err / mag.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0)).max())


def _outside(k0, k1):
    return [k for k in range(K2) if not k0 <= k < k1]


def _slot_layers(P):
    """The layer of each W slot (and, for LFISTA, of each Wm slot)."""
    return [fc.slot_birth2(P["form"], g, P["share_W"]) for g in range(P["W"].shape[0])]


# ------------------------------------------------------------------------------------------------ a. exact, every range
@pytest.mark.parametrize("case", EXACT2_CASES, ids=lambda c: "%s-%dx%dx%d-%s" % (
    "lfista" if c[0] == lista.LFISTA else "lamp", *c[1], "shared" if c[2] else "perlayer"))
@pytest.mark.parametrize("k0,k1", RANGES2)
def test_exact_every_layer_range_matches_fp64_bit_for_bit(case, k0, k1):
    """A pass [k0, k1) from x_in and s2_in, with d_xk and d_s2 coming in: every record and gradient is the fp64
    oracle's value bit for bit, except LAMP's sqrt(rvar) and dlam at the lam_k = 0 layers (sqrt is inexact); dlam at
    lam_k < 0, and every W slot, dtheta and ds of a layer outside the pass, are exactly 0."""
    P = fc.exact_case2(case)
    assert fc.exact_bound2(P, k0, k1) < 2 ** 24
    got, ref = launch2(P, k0, k1), fc.oracle2(P, k0, k1)
    assert_exact(got, ref, ("xs", "zs", "rs", "d_x_in", "d_s2_in", "dW", "dW2", "dB1", "dstep"))
    out = _outside(k0, k1)
    assert bool((got["dtheta"][out] == 0).all())
    if got["dstep"] is not None:
        assert bool((got["dstep"][out] == 0).all())
    if not P["share_W"]:
        for g, k in enumerate(_slot_layers(P)):
            if k in out:
                assert not got["dW"][g].any() and (got["dW2"] is None or not got["dW2"][g].any()), g
    if P["form"] == lista.LFISTA:
        assert_exact(got, ref, ("dtheta",))
        assert not got["dW2"][0].any()          # Wm_1 is never read
        return
    assert torch.equal(got["rowrec"][..., 1], ref["rowrec"][..., 1].float())             # b_k = ||x_k||_0 / M
    sq, sq_ref = got["rowrec"][..., 0].double(), ref["rowrec"][..., 0]
    assert bool(((sq - sq_ref).abs() <= 1e-6 * sq_ref).all()), _rel(sq, sq_ref)
    neg = P["theta"] < 0
    assert bool((got["dtheta"][neg] == 0).all())
    err = (got["dtheta"] - ref["dtheta"]).abs()
    assert bool((err <= 1e-6 * ref["scale_dtheta"]).all()), (err, ref["scale_dtheta"])


# ------------------------------------------------------------------------------------------------ b. generic weights
# K = 6 at generic weights and d_xk the sparse-coding loss gradient, the kernel's classification passed to the
# oracle: every row of x_k (and of LFISTA's z_k, LAMP's r_k and v_k) within 1e-5 of that row's max |z_k| (|r_k|,
# |v_k|), sqrt(rvar) within 1e-5 and b_k exact, d_x_in, d_s2_in, dWe and each W / Wm slot within 1e-5 of their own
# magnitude, and each dtheta_k (dlam_k) and ds_k within 1e-5 of the sum of its terms' magnitudes (oracle2's scale_*),
# which it must itself reach to 1e-4: a scalar that cancelled further would measure nothing.  Measured worst cases
# (H100 80GB HBM3, 700 W): x_k and z_k rows 1.5e-6, v_k rows and sqrt(rvar) 2.5e-6, d_x_in 6.1e-7, dWe 4.2e-6, Wm
# slots 2.7e-6, W slots 7.7e-6 (MATRIX_TOL's case aside), dtheta_k / dlam_k and ds_k 2.5e-6 of their terms.
EDGE2 = [(lista.LFISTA, (1, 1), 7), (lista.LFISTA, (3, 17), 129), (lista.LFISTA, (17, 3), 9),
         (lista.LFISTA, (8, 5), 1), (lista.LFISTA, (33, 65), 9), (lista.LFISTA, (64, 8), 129),
         (lista.LAMP, (1, 1), 1), (lista.LAMP, (3, 17), 9), (lista.LAMP, (17, 3), 129),
         (lista.LAMP, (8, 5), 7), (lista.LAMP, (33, 65), 129), (lista.LAMP, (64, 8), 9),
         # the largest shared-memory plans check_args accepts: LFISTA 8 (M + 5N) + 2048 floats, LAMP 8 (2M + 3N)
         # + 2048 floats, <= 200 KB (N = 2046: 256-column slices, one thread per column)
         (lista.LFISTA, (2048, 819), 7), (lista.LFISTA, (4, 1228), 9), (lista.LFISTA, (1144, 1000), 9),
         (lista.LAMP, (2048, 682), 9), (lista.LAMP, (3, 2046), 7), (lista.LAMP, (1024, 1365), 9)]
EDGE2_CASES = [(f, s, b, False) for f, s, b in EDGE2] + [(f, s, b, True) for f, s, b in EDGE2 if f == lista.LAMP]
MAX_FLIPS = 4
# At M = N = B = 1 a shared W is one number, the sum over the six layers of s_k v_k dr_k, and those terms cancel to
# 1/65 of their magnitudes: measured 2.0e-5 of the sum (3e-7 of the terms) on an H100 80GB HBM3 at 700 W.
MATRIX_TOL = {(lista.LAMP, (1, 1), True, "dW"): 1e-4}


def _edge_id(c):
    return "%s-%dx%d-B%d%s" % ("lfista" if c[0] == lista.LFISTA else "lamp", *c[1], c[2], "-shared" if c[3] else "")


@pytest.mark.parametrize("form,shape,B,share_W", EDGE2_CASES, ids=[_edge_id(c) for c in EDGE2_CASES])
def test_generic_weights_at_edge_shapes(form, shape, B, share_W):
    M, N = shape
    P = fc.generic_problem2(form, M, N, B, share_W)
    got = launch2(P)
    lives = masks(P, got["zs"], got["rowrec"])
    ref = fc.oracle2(P, lives=lives)
    own = fc.oracle2(P, d_xk=None)
    for k, (m_own, m_got) in enumerate(zip(masks(P, own["zs"], own["rowrec"]), lives)):
        assert int((m_own != m_got).sum()) <= MAX_FLIPS, k
    for k in range(K2):
        for key in ("xs", "zs"):
            err = _rel_rows(got[key][k], ref[key][k], ref["zs"][k])
            assert err <= 1e-5, (key, k, err)
        if form == lista.LAMP:
            assert _rel_rows(got["rs"][k], ref["rs"][k], ref["rs"][k]) <= 1e-5, k
            assert _rel(got["rowrec"][k][:, 0], ref["rowrec"][k][:, 0]) <= 1e-5, k
            assert torch.equal(got["rowrec"][k][:, 1], ref["rowrec"][k][:, 1].float()), k
    for key in ("dtheta", "dstep"):
        r, g = ref[key], got[key]
        if r is None:
            continue
        scale = ref["scale_" + key]
        assert bool((r.abs() >= 1e-4 * scale).all()), (key, r, scale)      # zero only where every term is
        err = (g - r).abs()
        assert bool((err <= 1e-5 * scale).all()), (key, err / scale)
    for key in ("d_x_in", "d_s2_in", "dB1", "dW", "dW2"):
        r, g = ref[key], got[key]
        if r is None:
            continue
        pairs = list(zip(g, r)) if key in ("dW", "dW2") else [(g, r)]     # each slot against its own magnitude
        for i, (gg, rr) in enumerate(pairs):
            if rr.abs().max() == 0:
                assert gg.abs().max() == 0, (key, i)
            else:
                assert _rel(gg, rr) <= MATRIX_TOL.get((form, shape, share_W, key), 1e-5), (key, i, _rel(gg, rr))


# ------------------------------------------------------------------------------------------------ c. three-way split
FORMS2 = [(lista.LFISTA, False), (lista.LAMP, False), (lista.LAMP, True)]
_form_id = lambda c: ("lfista" if c[0] == lista.LFISTA else "lamp") + ("-shared" if c[1] else "")


@pytest.mark.parametrize("form,share_W", FORMS2, ids=[_form_id(c) for c in FORMS2])
@pytest.mark.parametrize("a,b", SPLITS2)
def test_three_way_split_reproduces_the_full_pass(form, share_W, a, b):
    """fwd [0, a), [a, b), [b, K) chained through x_in / s2_in is the full forward bit for bit; bwd [b, K), [a, b),
    [0, a) chained through d_xk / d_s2 gives the full pass's d_x_in, d_s2_in and per-layer gradients bit for bit (and
    exact zeros for the layers a pass does not run), and a shared W or LFISTA's We once the parts are added in
    fp64."""
    P = fc.generic_problem2(form, 33, 65, 13, share_W, seed=2)
    full = launch2(P)
    lo = launch2(P, 0, a, backward=False)
    mid = launch2(P, a, b, x_in=lo["xs"][-1], s2_in=fc.s2_after(P, lo, P["x_in"]), backward=False)
    x_b, s_b = mid["xs"][-1], fc.s2_after(P, mid, lo["xs"][-1])
    hi = launch2(P, b, K2, x_in=x_b, s2_in=s_b)
    mid = launch2(P, a, b, x_in=lo["xs"][-1], s2_in=fc.s2_after(P, lo, P["x_in"]),
                  d_xk=hi["d_x_in"], d_s2=hi["d_s2_in"])
    lo = launch2(P, 0, a, d_xk=mid["d_x_in"], d_s2=mid["d_s2_in"])
    parts = [(lo, 0, a), (mid, a, b), (hi, b, K2)]
    for key in REC:
        if full[key] is not None:
            assert torch.equal(torch.cat([p[key] for p, _, _ in parts]), full[key]), key
    assert torch.equal(lo["d_x_in"], full["d_x_in"]) and torch.equal(lo["d_s2_in"], full["d_s2_in"])
    for key in ("dtheta", "dstep"):
        if full[key] is None:
            continue
        for p, k0, k1 in parts:
            assert torch.equal(p[key][k0:k1], full[key][k0:k1]), (key, k0)
            assert bool((p[key][_outside(k0, k1)] == 0).all()), (key, k0)
    shared = ["dB1"] if form == lista.LFISTA else []        # LFISTA's We, in every layer
    slotted = ["dW2"] if form == lista.LFISTA else []
    (shared if share_W else slotted).append("dW")
    for key in slotted:
        for g, k in enumerate(_slot_layers(P)):
            for p, k0, k1 in parts:
                if k0 <= k < k1:
                    assert torch.equal(p[key][g], full[key][g]), (key, g)
                else:
                    assert not p[key][g].any(), (key, g, k0)
    for key in shared:
        ps = [p[key] for p, _, _ in parts]
        assert bool(((sum(ps) - full[key]).abs() <= 1e-14 * sum(q.abs() for q in ps).max()).all()), key


# ------------------------------------------------------------------------------------------------ d. optional outputs
@pytest.mark.parametrize("dW,dW2", [(True, True), (True, False), (False, True), (False, False)])
def test_lfista_optional_weight_gradients(dW, dW2):
    """dW (Wg) and dW2 (Wm) NULL or present: the weight-gradient launch places its slots by blockIdx.y from how many
    are present, so every later slot (Wm, then We) moves.  Each present output is the full call's bits; the Wm_1
    slot, which no layer reads, is exactly 0 although x_0 is given (it would hold dz_1^T x_0)."""
    P = fc.exact_case2(EXACT2_CASES[0])
    full = launch2(P)
    assert_exact(full, fc.oracle2(P), GRADS)
    got = launch2(P, dW=dW, dW2=dW2)
    assert (got["dW"] is None) != dW and (got["dW2"] is None) != dW2
    assert_exact(got, full, REC + GRADS)
    for o in (full, got):
        if o["dW2"] is not None:
            assert not o["dW2"][0].any()


@pytest.mark.parametrize("k0,k1", [(0, K2), (2, 5)])
def test_lamp_optional_dstep(k0, k1):
    """LAMP with a shared W and dstep NULL: every other output is the full call's bits."""
    P = fc.exact_case2(EXACT2_CASES[3])
    assert P["share_W"] and P["step"] is not None
    full = launch2(P, k0, k1)
    got = launch2(P, k0, k1, dstep=False)
    assert got["dstep"] is None and full["dstep"] is not None
    assert_exact(got, full, REC + GRADS)


@pytest.mark.parametrize("form", [lista.LFISTA, lista.LAMP], ids=["lfista", "lamp"])
def test_strided_y_padding_and_every_output_written_in_range(form):
    """y with 29 NaN columns past M, and NaN rows past a partial batch in every input; every output starts as NaN
    with a sentinel guard past its end (launch2 checks the guards), and everything in range is written."""
    P = fc.exact_case2(EXACT2_CASES[1] if form == lista.LFISTA else EXACT2_CASES[2])
    got = launch2(P, 1, 5, pad_cols=29)
    for key, v in got.items():
        assert v is None or not bool(v.isnan().any()), key
    assert_exact(got, fc.oracle2(P, 1, 5), ("xs", "zs", "rs", "d_x_in", "d_s2_in", "dW", "dW2", "dB1"))


# ------------------------------------------------------------------------------------------------ e. rows
ZERO_ROW = 12


@pytest.mark.parametrize("form,share_W", FORMS2, ids=[_form_id(c) for c in FORMS2])
def test_rows_are_independent_of_their_batch(form, share_W):
    """A row's records are the same bits alone (B = 1), at each of the 9 positions of a partial cluster, and inside
    B = 129 under a permutation.  For LAMP, row 12 has zero y (and x_in): rvar = 0 in every layer.  Its records are
    finite with sqrt(rvar) exactly 0, alone it gives dlam exactly 0, and its cluster neighbours keep their bits."""
    P = fc.generic_problem2(form, 33, 65, 129, share_W, seed=4)
    if form == lista.LAMP:
        P["y"][ZERO_ROW] = 0.0
    full = launch2(P, backward=False)
    recs = [k for k in REC if full[k] is not None]

    def same(o, rows, what):
        for k in recs:
            assert torch.equal(o[k], full[k][:, rows]), (what, k)

    for r in (0, 77, 128, ZERO_ROW):
        same(launch2(fc.sub_rows2(P, [r]), backward=False), [r], r)
    others = [3, 50, 9, 101, 64, ZERO_ROW, 8, 120]
    for pos in range(9):
        rows = others[:pos] + [77] + others[pos:]
        same(launch2(fc.sub_rows2(P, rows), backward=False), rows, pos)
    perm = torch.randperm(129, generator=torch.Generator().manual_seed(1)).tolist()
    same(launch2(fc.sub_rows2(P, perm), backward=False), perm, "perm")
    if form == lista.LAMP:
        for k in recs:
            assert bool(full[k][:, ZERO_ROW].isfinite().all()), k
        assert not full["rowrec"][:, ZERO_ROW, 0].any() and not full["xs"][:, ZERO_ROW].any()
        alone = fc.sub_rows2(P, [ZERO_ROW])
        alone["d_s2"] = torch.ones(1, P["M"])
        got = launch2(alone)
        assert not got["dtheta"].any()
        for k in GRADS:
            assert got[k] is None or bool(got[k].isfinite().all()), k
        assert_exact(got, fc.oracle2(alone), ("d_x_in", "d_s2_in", "dtheta"))


@pytest.mark.parametrize("form,share_W", FORMS2, ids=[_form_id(c) for c in FORMS2])
def test_backward_is_deterministic_at_a_partial_batch(form, share_W):
    P = fc.generic_problem2(form, 33, 65, 13, share_W, seed=6)
    a, b = launch2(P), launch2(P)
    for key in REC + GRADS:
        if a[key] is not None:
            assert torch.equal(a[key], b[key]), key
