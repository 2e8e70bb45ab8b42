"""The LISTA-family kernels through their C ABI (l2o_ista_fwd / l2o_ista_bwd / l2o_ista_loss_grad), at what the
models never pass: layer ranges [k0, k1) from a given x_{k0} with its gradient, per-layer shrinkage (soft layers among
support-selection layers, ranks clamped at N - 1), strided y, partial clusters of rows, the largest shared-memory plans,
and support selection held to exact agreement on inputs where every fp32 sum is exact.  Every check is against the
fp64 oracle (oracle/lista_oracle.py) with autograd for the gradients."""
import ctypes as C

import numpy as np
import pytest
import torch

from open_l2o_b200 import _lib, lista
from oracle import lista_oracle as lo
from tests.lista_cases import (EXACT_CASES, K, RANGES, exact_bound, exact_case, generic_problem, generic_ranks,
                                n_slots, oracle, sub_rows)

pytestmark = pytest.mark.gpu

GUARD = 37            # sentinel elements past the end of every output
PAD_COLS, PAD_ROWS = 3, 5   # NaN columns past M in every y row, NaN rows past the batch in y and x_in
SENTINEL = {torch.float32: 1234.5, torch.float64: -4321.25, torch.uint8: 0x5A}


# ------------------------------------------------------------------------------------------------ kernel harness
class _Bufs:
    """Output buffers prefilled with NaN (0xFF for bytes), each followed by GUARD sentinels that must stay intact."""

    def __init__(self):
        self.flat = []

    def out(self, shape, dtype):
        n = int(np.prod(shape))
        f = torch.empty(n + GUARD, dtype=dtype, device="cuda")
        f[:n] = 255 if dtype == torch.uint8 else float("nan")
        f[n:] = SENTINEL[dtype]
        self.flat.append((f, n))
        return f[:n].view(shape)

    def check_guards(self):
        for f, n in self.flat:
            assert bool((f[n:] == SENTINEL[f.dtype]).all()), "write past the end of an output"


def _cuda(t, dtype=torch.float32):
    return None if t is None else t.to(dtype).contiguous().cuda()


def _p(t):
    return None if t is None else t.data_ptr()


def _padded(t, cols):
    """A [rows, cols] CUDA tensor: t in the top-left corner, NaN around it (columns past t's, PAD_ROWS rows)."""
    buf = torch.full((t.shape[0] + PAD_ROWS, cols), float("nan"), dtype=torch.float32)
    buf[:t.shape[0], :t.shape[1]] = t
    return buf.cuda()


def launch(P, k0=0, k1=K, x_in="P", d_xk="P", backward=True, pad_cols=PAD_COLS):
    """l2o_ista_fwd (and l2o_ista_bwd) on P over [k0, k1) with every record; returns the outputs on the CPU.  y has
    row stride M + pad_cols with NaN padding and NaN rows past the batch; x_in has NaN rows past the batch."""
    form, M, N, B = P["form"], P["M"], P["N"], P["B"]
    x_in = P["x_in"] if isinstance(x_in, str) else x_in
    d_xk = P["d_xk"] if isinstance(d_xk, str) else d_xk
    L, bufs = _lib.lib(), _Bufs()
    dev = {k: _cuda(P[k]) for k in ("A", "B1", "W", "theta", "step", "gscale")}
    ranks = _cuda(P["ranks"], torch.int32)
    y = _padded(P["y"], M + pad_cols)
    xi = None if x_in is None else _padded(x_in, N)
    L_ = k1 - k0
    a = _lib.IstaArgs()
    a.form, a.batch, a.m, a.n, a.num_layers, a.k0, a.k1 = form, B, M, N, K, k0, k1
    a.share_W = int(P["share_W"])
    a.A, a.B1, a.W, a.theta, a.step = (_p(dev[k]) for k in ("A", "B1", "W", "theta", "step"))
    a.ss_rank, a.y, a.ldy, a.x_in = _p(ranks), y.data_ptr(), M + pad_cols, _p(xi)
    o = {"xs": bufs.out((L_, B, N), torch.float32), "zs": bufs.out((L_, B, N), torch.float32),
         "rs": bufs.out((L_, B, M), torch.float32) if form == lista.COUPLED else None,
         "sel": bufs.out((L_, B, N), torch.uint8) if ranks is not None else None}
    a.xs, a.zs, a.rs, a.sel = (_p(o[k]) for k in ("xs", "zs", "rs", "sel"))
    _lib.check(L.l2o_ista_fwd(C.byref(a), None), "l2o_ista_fwd")
    if backward:
        nb = C.c_size_t()
        _lib.check(L.l2o_ista_workspace_bytes(C.byref(a), C.byref(nb)), "l2o_ista_workspace_bytes")
        scratch = torch.empty((nb.value + 3) // 4, dtype=torch.float32, device="cuda")
        dx = _cuda(d_xk)
        S = n_slots(form, K, P["share_W"])
        wshape = (S, M, N) if form == lista.COUPLED else (S, N, N)
        o["d_x_in"] = bufs.out((B, N), torch.float32)
        o["dW"] = bufs.out(wshape, torch.float64) if P["dW"] else None
        o["dB1"] = bufs.out((N, M), torch.float64) if form == lista.LISTA else None
        o["dtheta"] = bufs.out((K,), torch.float64)
        o["dstep"] = bufs.out((K,), torch.float64) if P["dstep"] else None
        gr = _lib.IstaGrads()
        gr.d_xk, gr.d_x_in, gr.dW, gr.dB1 = dx.data_ptr(), *(_p(o[k]) for k in ("d_x_in", "dW", "dB1"))
        gr.dtheta, gr.dstep, gr.gscale, gr.scratch = _p(o["dtheta"]), _p(o["dstep"]), _p(dev["gscale"]), _p(scratch)
        _lib.check(L.l2o_ista_bwd(C.byref(a), C.byref(gr), None), "l2o_ista_bwd")
    torch.cuda.synchronize()
    bufs.check_guards()
    return {k: (None if v is None else v.cpu()) for k, v in o.items()}


# ------------------------------------------------------------------------------------------------ oracle
def kernel_masks(P, got, k0=0):
    """The kernel's support masks and |z| > theta classification of each layer, for the oracle to follow."""
    th = P["theta"][k0:k0 + got["zs"].shape[0]].view(-1, 1, 1)
    lives = list((got["zs"].abs() > th) & (got["zs"] != 0))
    sels = None if got["sel"] is None else list(got["sel"].bool())
    return sels, lives


def assert_exact(got, ref, keys):
    for k in keys:
        if ref.get(k) is None or got.get(k) is None:
            continue
        g, r = got[k].double(), ref[k].double()
        bad = int((g != r).sum())
        assert bad == 0, (k, bad, g.reshape(-1)[(g != r).reshape(-1)][:5], r.reshape(-1)[(g != r).reshape(-1)][:5])


FWD = ("xs", "zs", "rs", "sel")
BWD = ("d_x_in", "dW", "dB1", "dtheta", "dstep")


def _rel(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _rel_rows(a, b, mag):
    """The worst row's max |a - b| over its max |mag| ([B, N]); a row where mag is all zero must match exactly."""
    err, mag = (a.double() - b.double()).abs().amax(dim=1), mag.double().abs().amax(dim=1)
    return float(torch.where(mag > 0, err / mag.clamp_min(1e-300), torch.where(err > 0, float("inf"), 0.0)).max())


# ------------------------------------------------------------------------------------------------ a. exact arithmetic
@pytest.mark.parametrize("form,shape,rk,opt", EXACT_CASES)
def test_exact_inputs_match_fp64_bit_for_bit(form, shape, rk, opt):
    """No flip allowance: the oracle classifies |z| against theta and the rank threshold itself."""
    P = exact_case(form, shape, rk, opt)
    assert exact_bound(P) < 2 ** 24
    got, ref = launch(P), oracle(P)
    assert_exact(got, ref, FWD + BWD)


@pytest.mark.parametrize("form", [lista.LISTA, lista.COUPLED])
@pytest.mark.parametrize("k0,k1", RANGES)
def test_exact_layer_range_from_x_in(form, k0, k1):
    """A pass [k0, k1) from a given x_{k0}, with dL/dx_{k0}; W slots, dtheta and ds of layers outside the pass are
    exactly 0 (the buffers start as NaN)."""
    P = exact_case(form, (12, 16, 13), "clamp", "perlayer", seed=3)
    assert exact_bound(P, k0, k1) < 2 ** 24
    got, ref = launch(P, k0, k1), oracle(P, k0, k1)
    assert_exact(got, ref, FWD + BWD)
    outside = [k for k in range(K) if not k0 <= k < k1]
    assert bool((got["dtheta"][outside] == 0).all()) and bool((got["dstep"][outside] == 0).all())


# ------------------------------------------------------------------------------------------------ b. generic weights
# K = 4 at generic weights and d_xk the sparse-coding loss gradient, the kernel's masks passed to the oracle: every
# row of x_k within 1e-5 of the row's max |z_k| (x_k = shrink(z_k) carries z_k's rounding: at N = 1 a row is one
# shrunk value |z| - theta that can be 1e-2 of |z|), d_x_in, dB1 and each W slot within 1e-5 of their own magnitude, and each
# dtheta_k and ds_k within SCALAR_TOL of its own value.  That needs the scalar not to cancel far below the sum of its
# terms' magnitudes (oracle's scale_*), and the test asserts it does not: every one is at least 1e-4 of it (the
# lowest, coupled ds_k at (3, 2046), is 2.4e-4).  Measured worst cases (H100 SXM, 700 W): x_k rows 1.2e-6, d_x_in
# 1.1e-6, dB1 1.5e-6, W slots 5.2e-6, dtheta_k 9.9e-7, ds_k 9.0e-7 and 6.1e-6 at (3, 2046).
EDGE = [(lista.COUPLED, (1, 1), 1), (lista.LISTA, (1, 1), 7), (lista.COUPLED, (3, 17), 9), (lista.LISTA, (3, 17), 129),
        (lista.COUPLED, (17, 3), 7), (lista.LISTA, (17, 3), 9), (lista.COUPLED, (33, 65), 129),
        (lista.LISTA, (33, 65), 1), (lista.COUPLED, (64, 8), 9), (lista.LISTA, (64, 8), 7),
        # the largest shared-memory plans check_args accepts (N = 2046: 256-column slices, one thread per column)
        (lista.COUPLED, (1024, 1365), 9), (lista.COUPLED, (2048, 682), 7), (lista.COUPLED, (3, 2046), 129),
        (lista.LISTA, (1024, 1280), 9), (lista.LISTA, (2048, 1024), 7), (lista.LISTA, (4, 1535), 129)]
MAX_FLIPS = 4
# At M = 3, N = 2046 the coupled residual r_k = y - x_k A^T is a small difference of large terms, so ds_k, a sum of
# r_k times dz_k W_k^T, carries its fp32 rounding at about 1e-5 of its value (measured 6.1e-6; an fp32 CPU evaluation misses it by 2e-5).
SCALAR_TOL = {(lista.COUPLED, (3, 2046), "dstep"): 1e-4}


@pytest.mark.parametrize("form,shape,B", EDGE)
@pytest.mark.parametrize("share_W", [False, True])
def test_generic_weights_at_edge_shapes(form, shape, B, share_W):
    M, N = shape
    P = generic_problem(form, M, N, B, share_W, ranks=generic_ranks(N))
    got = launch(P)
    sels, lives = kernel_masks(P, got)
    ref = oracle(P, sels=sels, lives=lives)
    for k in range(K):
        err = _rel_rows(got["xs"][k], ref["xs"][k], ref["zs"][k])
        assert err <= 1e-5, (k, err)
    own = oracle(P, d_xk=None)
    for k in range(K):
        assert int((own["sel"][k] != got["sel"][k]).sum()) <= MAX_FLIPS, k
    for key in BWD:
        r, g = ref[key], got[key]
        if r is None or g is None:
            continue
        if key in ("dtheta", "dstep"):
            scale = ref["scale_" + key]
            assert bool((r.abs() >= 1e-4 * scale).all()), (key, r, scale)      # zero only where every term is
            err = (g - r).abs()
            assert bool((err <= SCALAR_TOL.get((form, shape, key), 1e-5) * r.abs()).all()), (key, err / r.abs())
            continue
        pairs = list(zip(g, r)) if key == "dW" else [(g, r)]   # each W slot against its own magnitude
        for i, (gg, rr) in enumerate(pairs):
            if rr.abs().max() == 0:
                assert gg.abs().max() == 0, (key, i)
            else:
                assert _rel(gg, rr) <= 1e-5, (key, i, _rel(gg, rr))


# ------------------------------------------------------------------------------------------------ c. layer ranges
SPLIT = [(lista.LISTA, False), (lista.LISTA, True), (lista.COUPLED, False), (lista.COUPLED, True)]


@pytest.mark.parametrize("form,share_W", SPLIT)
@pytest.mark.parametrize("j", [1, 2, 3])
def test_split_passes_reproduce_the_full_pass(form, share_W, j):
    """fwd [0, j) then fwd [j, K) from x_j is the full forward bit for bit; bwd [j, K) then bwd [0, j) from its
    d_x_in gives the full pass's per-layer gradients and d_x_in bit for bit, and a shared W or B1 (summed over the
    layers) once the two passes' parts are added in fp64."""
    P = generic_problem(form, 33, 65, 13, share_W, seed=2, ranks=generic_ranks(65))
    full = launch(P)
    lo_pass = launch(P, 0, j, d_xk=None, backward=False)
    hi = launch(P, j, K, x_in=lo_pass["xs"][j - 1])
    lo_pass = launch(P, 0, j, d_xk=hi["d_x_in"])
    for key in FWD:
        if full[key] is not None:
            assert torch.equal(torch.cat([lo_pass[key], hi[key]]), full[key]), key
    assert torch.equal(lo_pass["d_x_in"], full["d_x_in"])
    for key in ("dtheta", "dstep"):
        if full[key] is not None:
            assert torch.equal(lo_pass[key][:j], full[key][:j]) and torch.equal(hi[key][j:], full[key][j:]), key
            assert bool((lo_pass[key][j:] == 0).all()) and bool((hi[key][:j] == 0).all()), key
    shared = [("dB1", full["dB1"], lo_pass["dB1"], hi["dB1"])] if form == lista.LISTA else []
    if share_W:
        shared.append(("dW", full["dW"], lo_pass["dW"], hi["dW"]))
    else:
        first = 0 if form == lista.COUPLED else 1
        for s in range(full["dW"].shape[0]):
            part = lo_pass if s + first < j else hi
            other = hi if part is lo_pass else lo_pass
            assert torch.equal(part["dW"][s], full["dW"][s]), s
            assert bool((other["dW"][s] == 0).all()), s
    for key, f, a, b in shared:
        assert (a + b - f).abs().max() <= 1e-15 * f.abs().max(), key


# ------------------------------------------------------------------------------------------------ d. buffers
@pytest.mark.parametrize("form", [lista.LISTA, lista.COUPLED])
def test_strided_y_padding_and_every_output_written_in_range(form):
    """y with 29 NaN columns past M and NaN rows past a partial batch; every output starts as NaN (0xFF for sel) with
    a sentinel guard past its end (launch checks the guards).  Everything in range is written, and matches the
    oracle."""
    P = exact_case(form, (24, 16, 13), "mixed", "perlayer", seed=5)
    got = launch(P, pad_cols=29)
    for key, v in got.items():
        if v is None:
            continue
        if v.dtype == torch.uint8:
            assert bool((v <= 1).all()), key
        else:
            assert not bool(v.isnan().any()), key
    assert_exact(got, oracle(P), FWD + BWD)


# ------------------------------------------------------------------------------------------------ e. rows
@pytest.mark.parametrize("form", [lista.LISTA, lista.COUPLED])
def test_rows_are_independent_of_their_batch(form):
    """A row's x_k is the same bits alone (B = 1), at each position of a partial cluster (B = 9), inside B = 129 and
    in a permuted gather of the batch."""
    P = generic_problem(form, 33, 65, 129, False, seed=4, ranks=generic_ranks(65))
    full = launch(P, backward=False)["xs"]
    for r in (0, 77, 128):
        assert torch.equal(launch(sub_rows(P, [r]), backward=False)["xs"][:, 0], full[:, r]), r
    others = [3, 50, 9, 101, 64, 12, 8, 120]
    for pos in range(9):
        rows = others[:pos] + [77] + others[pos:]
        xs = launch(sub_rows(P, rows), backward=False)["xs"]
        assert torch.equal(xs, full[:, rows]), pos
    perm = torch.randperm(129, generator=torch.Generator().manual_seed(1)).tolist()
    assert torch.equal(launch(sub_rows(P, perm), backward=False)["xs"], full[:, perm])


@pytest.mark.parametrize("form,share_W", SPLIT)
def test_backward_is_deterministic_at_a_partial_batch(form, share_W):
    P = generic_problem(form, 33, 65, 13, share_W, seed=6, ranks=generic_ranks(65))
    a, b = launch(P), launch(P)
    for key in FWD + BWD:
        if a[key] is not None:
            assert torch.equal(a[key], b[key]), key


# ------------------------------------------------------------------------------------------------ f. loss kernel
def _loss_launch(task, A, y, x, x_true, lam, pad):
    B, N = x.shape
    M = A.shape[0]
    bufs = _Bufs()
    d_x, loss = bufs.out((B, N), torch.float32), bufs.out((B,), torch.float64)
    dA, dx = _cuda(A), _cuda(x)
    ys = _padded(y, M + pad)
    xt = _padded(x_true, N + pad)
    la = _lib.IstaLossArgs()
    la.task, la.batch, la.m, la.n = task, B, M, N
    la.A, la.y, la.ldy, la.x_true, la.ldx = dA.data_ptr(), ys.data_ptr(), M + pad, xt.data_ptr(), N + pad
    la.x, la.lam, la.d_x, la.loss = dx.data_ptr(), float(lam), d_x.data_ptr(), loss.data_ptr()
    _lib.check(_lib.lib().l2o_ista_loss_grad(C.byref(la), None), "l2o_ista_loss_grad")
    torch.cuda.synchronize()
    bufs.check_guards()
    return loss.cpu(), d_x.cpu()


@pytest.mark.parametrize("task,M,N,B", [(lista.TASK_SC, 24, 40, 9), (lista.TASK_LASSO, 64, 24, 9),
                                        (lista.TASK_LASSO, 17, 300, 3)])
def test_loss_kernel_strided_rows_and_zeros_in_x(task, M, N, B):
    """SC with x_true rows of stride > N; Lasso at M > N and M < N; x with exact zeros (sign 0) in every row and
    one all-zero row."""
    g = torch.Generator().manual_seed(M + N)
    A = torch.randn(M, N, generator=g) / np.sqrt(M)
    x = torch.randn(B, N, generator=g) * (torch.rand(B, N, generator=g) < 0.5)
    x[1] = 0.0
    x_true = torch.randn(B, N, generator=g) * (torch.rand(B, N, generator=g) < 0.3)
    y = torch.randn(B, M, generator=g)
    lam = 0.05
    loss, d_x = _loss_launch(task, A, y, x, x_true, lam, pad=7)
    xr = x.double().requires_grad_(True)
    for b in range(B):
        if task == lista.TASK_SC:
            ref = lo.sc_loss(xr[b:b + 1], x_true[b:b + 1].double())
        else:
            ref = lo.lasso_loss(xr[b:b + 1], A.double(), y[b:b + 1].double(), lam)
        ref.backward()
        assert abs(float(loss[b]) - ref.item()) <= 1e-5 * abs(ref.item()), b
    assert _rel(d_x, xr.grad) <= (1e-6 if task == lista.TASK_SC else 1e-5)
    if task == lista.TASK_LASSO:   # where x == 0 only the data term: 0.5 A^T (x A^T - y)
        zero = x == 0
        data_term = 0.5 * (x.double() @ A.double().T - y.double()) @ A.double()
        assert _rel(d_x[zero], data_term[zero]) <= 1e-5
