"""The problem-zoo kernels through their C ABI (l2o_zoo_value_grad, l2o_zoo_hvp, l2o_zoo_hess_form) where the Problem
tests do not reach: points where the objective is not smooth (a residual exactly 0, sign(0), tied extremes, sqrt at
0), every output entry written and nothing past it at the cluster switch and the largest plans, f and q left NULL,
every pair count around the Hessian form's tiles of 4, V = U by pointer and by value, and the 2-D functions point by
point.  The reference is fp64 autograd of the Problem's torch restatement (tests/zoo_cases.py)."""
import ctypes as C
import threading

import pytest
import torch

from open_l2o_b200 import _lib
from tests import zoo_cases as zc

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 37           # sentinel floats past the end of every output
SENTINEL = 1234.5
NAN = float("nan")


# ---- one launch -------------------------------------------------------------------------------------------------------
def _buf(n):
    """n floats prefilled with NaN, followed by GUARD sentinels."""
    b = torch.full((n + GUARD,), NAN, device=DEV)
    b[n:] = SENTINEL
    return b


def launch(mode, problem, x, v=None, U=None, V=None, data=None, scalar=True):
    """One l2o_zoo_<mode> launch ("grad", "hvp" or "form") on the problem's constants at the fp32 point x: returns
    (f or q, or None; out [n]) on the CPU, after checking that nothing was written past out or the scalar.  V is U
    (the same pointer) when V is None."""
    x = x.to(DEV).contiguous()
    n = x.numel()
    z = problem.kernel(x, None if data is None else data.to(DEV))
    out, s = _buf(n), (_buf(1) if scalar else None)
    a = _lib.ZooArgs()
    a.family, a.n, a.rows, a.p0 = _lib.ZOO[z.family], z.n, z.rows, z.p0
    keep = [None if t is None else t.to(DEV).contiguous() for t in (v, U, V)]
    dv, dU, dV = keep
    a.x, a.out = x.data_ptr(), out.data_ptr()
    a.A, a.y, a.c = (None if t is None else t.data_ptr() for t in (z.A, z.y, z.c))
    L = _lib.lib()
    if mode == "form":
        fa = _lib.ZooFormArgs()
        fa.base = a
        fa.k, fa.U = dU.shape[0], dU.data_ptr()
        fa.V = dU.data_ptr() if dV is None else dV.data_ptr()
        fa.q = None if s is None else s.data_ptr()
        _lib.check(L.l2o_zoo_hess_form(C.byref(fa), None), "l2o_zoo_hess_form")
    else:
        a.f = None if s is None or mode == "hvp" else s.data_ptr()
        a.v = None if dv is None else dv.data_ptr()
        fn = L.l2o_zoo_value_grad if mode == "grad" else L.l2o_zoo_hvp
        _lib.check(fn(C.byref(a), None), "l2o_zoo_" + mode)
    torch.cuda.synchronize()
    out, s = out.cpu(), (None if s is None else s.cpu())
    assert bool((out[n:] == SENTINEL).all()), "write past the end of out"
    if s is not None:
        assert bool((s[1:] == SENTINEL).all()), "write past the end of f / q"
        s = None if mode == "hvp" else s[0]
    return s, out[:n]


def _rel(got, ref):
    got, ref = got.double().reshape(-1), ref.double().reshape(-1)
    return float((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


def _close(name, got, ref, tol):
    e = _rel(got, ref)
    assert e <= tol, (name, e)


def _randn(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _all_modes(problem, x, tol=1e-5, form_tol=None, k=3, data=None, seed=0):
    """f, g, H v, (q, dq/dx) against fp64 autograd, V distinct from U; returns the kernel's outputs."""
    n = x.numel()
    v, U, V = _randn(n, seed=seed + 1), _randn(k, n, seed=seed + 2), _randn(k, n, seed=seed + 3)
    ref = zc.reference(problem, x, v, U, V, data)
    f, g = launch("grad", problem, x, data=data)
    _, hv = launch("hvp", problem, x, v=v, data=data)
    q, dq = launch("form", problem, x, U=U, V=V, data=data)
    got = dict(f=f, g=g, hv=hv, q=q, dq=dq)
    err = {k: _rel(got[k], ref[k]) for k in got}
    tols = dict(f=tol, g=tol, hv=tol, q=form_tol or tol, dq=form_tol or tol)
    assert all(err[k] <= tols[k] for k in err), " ".join("%s %.2e" % kv for kv in err.items())
    return got


def _form_tol(p):
    # as in test_scale_reg_gpu: Norm's third derivative at p = 1.5 weights the fp32 rounding of the smallest residuals
    return 1e-4 if p == 1.5 else 1e-5


# ---- constructed non-smooth points -------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [100, 300], ids=["one_cta", "cluster"])
@pytest.mark.parametrize("p", [1.5, 2.0, 3.0])
def test_norm_zero_residual_has_no_curvature(n, p):
    """r_i = 0 exactly on a nonzero row: sign(r_i) = 0 and d sign / dr = 0, so row i adds nothing to g, H v or the
    Hessian form, as autograd of the restatement has it."""
    for seed in (0, 1):
        problem, x, _, _, _ = zc.zero_residual("Norm", n, seed, p)
        assert zc.on_cluster(n, n) == (n == 300)
        _all_modes(problem, x, form_tol=_form_tol(p), seed=seed)


@pytest.mark.parametrize("n", [100, 300], ids=["one_cta", "cluster"])
def test_rastrigin_zero_residual_is_nan_everywhere(n):
    """tf.norm of a single-element row has gradient r / |r|, NaN at r = 0: every entry of g, H v, q and dq/dx is NaN
    (pinned against the header's convention: torch.linalg.vector_norm's subgradient at 0 is 0).  f stays finite."""
    problem, x, _, _, _ = zc.zero_residual("Rastrigin", n, 0)
    ref = zc.reference(problem, x)
    f, g = launch("grad", problem, x)
    _close("f", f, ref["f"], 1e-5)
    assert bool(torch.isnan(g).all()), int(torch.isnan(g).sum())
    _, hv = launch("hvp", problem, x, v=_randn(n, seed=1))
    assert bool(torch.isnan(hv).all()), int(torch.isnan(hv).sum())
    for k in (1, 5):
        q, dq = launch("form", problem, x, U=_randn(k, n, seed=2), V=_randn(k, n, seed=3))
        assert bool(torch.isnan(q)) and bool(torch.isnan(dq).all()), (k, float(q), int(torch.isnan(dq).sum()))


@pytest.mark.parametrize("n", [20, 300])
def test_lasso_sign_of_zero(n):
    problem, x = zc.lasso_zeros(n, 0)
    out = _all_modes(problem, x)
    assert not bool(out["dq"].any())


@pytest.mark.parametrize("all_equal", [False, True], ids=["two_each", "all_equal"])
def test_min_max_well_ties_share_evenly(all_equal):
    """n = 4096 with two maxima and two minima in different warps and passes, or every |x_j| equal: torch's amax / amin
    share the gradient evenly between ties, as the kernel does."""
    problem = zc.make("MinMaxWell", (4096,))
    x = zc.min_max_ties(4096, 0, all_equal)
    sq = x.double() ** 2
    ties = 4096 if all_equal else 2
    assert int((sq == sq.max()).sum()) == ties and int((sq == sq.min()).sum()) == ties
    _all_modes(problem, x)


@pytest.mark.parametrize("case", ["ackley", "snake_one_cta", "snake_cluster"])
def test_sqrt_at_zero_is_nan_where_autograd_is(case):
    """Ackley at the origin and OutwardSnake at x = 0: NaN exactly where fp64 autograd has NaN, the rest close."""
    if case == "ackley":
        problem, x, data = zc.make("Ackley"), torch.zeros(2), None
    else:
        n, batch = (64, 128) if case == "snake_one_cta" else (300, 300)
        problem, x = zc.make("OutwardSnake", (n,)), torch.zeros(n)
        data = zc.data_batch("OutwardSnake", n, batch, 0)
    n = x.numel()
    v, U, V = _randn(n, seed=1), _randn(3, n, seed=2), _randn(3, n, seed=3)
    ref = zc.reference(problem, x, v, U, V, data)
    f, g = launch("grad", problem, x, data=data)
    _, hv = launch("hvp", problem, x, v=v, data=data)
    q, dq = launch("form", problem, x, U=U, V=V, data=data)
    assert abs(float(f) - float(ref["f"])) <= 1e-5 * max(1.0, abs(float(ref["f"])))
    for name, got in (("g", g), ("hv", hv), ("q", q), ("dq", dq)):
        r = ref[name].reshape(-1)
        got = got.reshape(-1)
        assert torch.equal(torch.isnan(got), torch.isnan(r)), (name, got, r)
        fin = ~torch.isnan(r)
        if bool(fin.any()):
            _close(name, got[fin], r[fin], 1e-5)


# ---- the shared-memory limit across host threads ----------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["grad", "hvp", "form"])
def test_shared_memory_limit_holds_across_threads(mode):
    """A kernel's dynamic shared-memory limit is one per process, whichever host thread launches (torch's autograd
    calls the zoo from its device threads).  One CTA each: the largest plan on this thread (ProjectionQuadratic at
    4096 x 15, 160 KB), a small one on another thread (Norm(18)), then a medium one here (Norm(100)); the small launch
    must not lower the limit below what this thread's launches need."""
    def run(problem, n, data=None, seed=0):
        x = problem.init_tensors(seed, "cpu")[0].reshape(-1).contiguous()
        kw = {"grad": {}, "hvp": {"v": _randn(n, seed=1)}, "form": {"U": _randn(2, n, seed=2)}}[mode]
        return launch(mode, problem, x, data=data, **kw)

    run(zc.make("ProjectionQuadratic", (4096,)), 4096, zc.data_batch("ProjectionQuadratic", 4096, 15, 0))
    errors = []

    def other():
        try:
            run(zc.make("Norm", (18,), {"norm_power": 2.5}), 18)
        except Exception as e:   # reported on this thread
            errors.append(e)

    t = threading.Thread(target=other)
    t.start()
    t.join()
    assert not errors, errors
    problem = zc.make("Norm", (100,), {"norm_power": 2.5})
    x = problem.init_tensors(0, "cpu")[0].reshape(-1)
    v, U = _randn(100, seed=1), _randn(2, 100, seed=2)
    ref = zc.reference(problem, x, v, U, U)
    _, out = run(problem, 100)
    key = {"grad": "g", "hvp": "hv", "form": "dq"}[mode]
    _close(key, out, ref[key], 1e-5)


# ---- output coverage at the boundary shapes --------------------------------------------------------------------------
COVERAGE = ([("%s%s" % (c, a), c, a, kw, None) for c, a, kw in zc.BOUNDARY_CASES]
            + [("%s(%d,%d)" % (c, n, b), c, (n,), {}, b) for c in zc.DATA_FAMILIES for n, b in zc.BOUNDARY_DATA])


@pytest.mark.parametrize("name,cls,args,kwargs,batch", COVERAGE, ids=[c[0] for c in COVERAGE])
def test_every_output_written_once_and_nothing_past_it(name, cls, args, kwargs, batch):
    """out prefilled with NaN and followed by sentinels: every entry of [0, n) is written (finite at these points),
    nothing after it; with f or q NULL out has the same bits; a second launch has the same bits."""
    problem = zc.make(cls, args, kwargs, 0)
    data = None if batch is None else zc.data_batch(cls, args[0], batch, 0)
    x = problem.init_tensors(0, "cpu")[0].reshape(-1).contiguous()
    n = x.numel()
    v, U, V = _randn(n, seed=1), _randn(zc.TILE + 1, n, seed=2), _randn(zc.TILE + 1, n, seed=3)
    for mode, kw in (("grad", {}), ("hvp", {"v": v}), ("form", {"U": U, "V": V})):
        s0, o0 = launch(mode, problem, x, data=data, **kw)
        assert bool(torch.isfinite(o0).all()), (mode, int((~torch.isfinite(o0)).sum()))
        if s0 is not None:
            assert bool(torch.isfinite(s0)), mode
        _, o1 = launch(mode, problem, x, data=data, scalar=False, **kw)
        s2, o2 = launch(mode, problem, x, data=data, **kw)
        assert torch.equal(o0, o1), (mode, "out differs with the scalar NULL")
        assert torch.equal(o0, o2) and (s0 is None or torch.equal(s0, s2)), (mode, "second launch differs")


# ---- the Hessian form's pair tiles -----------------------------------------------------------------------------------
TILE_CASES = [("Norm(100)", "Norm", (100,), {"norm_power": 2.5}, None),
              ("Norm(300)", "Norm", (300,), {"norm_power": 2.5}, None),
              ("Rastrigin(300)", "Rastrigin", (300,), {}, None),
              ("OutwardSnake(64,128)", "OutwardSnake", (64,), {}, 128),
              ("OutwardSnake(300,300)", "OutwardSnake", (300,), {}, 300),
              ("DependencyChain(20)", "DependencyChain", (20,), {}, None),
              ("MinMaxWell(64)", "MinMaxWell", (64,), {}, None),
              ("Ackley", "Ackley", (), {}, None)]


@pytest.mark.parametrize("name,cls,args,kwargs,batch", TILE_CASES, ids=[c[0] for c in TILE_CASES])
def test_hess_form_every_pair_count(name, cls, args, kwargs, batch):
    """k = 1 .. 10 (a tile of 4 alone, one past it, two tiles, ...) against fp64 triple autograd, with V distinct from
    U and V = U; V = U by pointer (the kernel's shortcut) and as an equal copy give the same bits."""
    problem = zc.make(cls, args, kwargs, 0)
    data = None if batch is None else zc.data_batch(cls, args[0], batch, 0)
    x = problem.init_tensors(0, "cpu")[0].reshape(-1).contiguous()
    n = x.numel()
    for k in range(1, _lib.ZOO_MAX_PAIRS + 1):
        U, V = _randn(k, n, seed=10 + k), _randn(k, n, seed=30 + k)
        ref = zc.reference(problem, x, U=U, V=V, data=data)
        q, dq = launch("form", problem, x, U=U, V=V, data=data)
        _close(("q", k), q, ref["q"], 1e-5)
        _close(("dq", k), dq, ref["dq"], 1e-5)
        ref = zc.reference(problem, x, U=U, V=U, data=data)
        q1, d1 = launch("form", problem, x, U=U, data=data)
        q2, d2 = launch("form", problem, x, U=U, V=U.clone(), data=data)
        _close(("q, V = U", k), q1, ref["q"], 1e-5)
        _close(("dq, V = U", k), d1, ref["dq"], 1e-5)
        assert torch.equal(q1, q2) and torch.equal(d1, d2), (k, "V = U by pointer and by value differ")


# ---- the 2-D functions, point by point -------------------------------------------------------------------------------
@pytest.mark.parametrize("cls", zc.PLANE_FAMILIES)
def test_plane_function_point_by_point(cls):
    """f, g, H v and (q, dq/dx) at every point of an 8 x 8 grid over the init range and at the known minima, each held
    to 1e-5 relative to its own max norm at that point (a small term at one point is not hidden by a large value at
    another)."""
    problem = zc.make(cls)
    pts = zc.plane_points(cls)
    assert pts.shape[0] >= 64
    for i, x in enumerate(pts):
        v, U, V = _randn(2, seed=i), _randn(2, 2, seed=100 + i), _randn(2, 2, seed=200 + i)
        ref = zc.reference(problem, x, v, U, V)
        f, g = launch("grad", problem, x)
        _, hv = launch("hvp", problem, x, v=v)
        q, dq = launch("form", problem, x, U=U, V=V)
        for name, got in (("f", f), ("g", g), ("hv", hv), ("q", q), ("dq", dq)):
            e = _rel(got, ref[name])
            assert e <= 1e-5, (cls, tuple(x.tolist()), name, e, got, ref[name])
