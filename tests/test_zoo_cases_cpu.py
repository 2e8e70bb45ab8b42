"""CPU: the inputs of the problem-zoo kernel tests are what they claim to be: the constructed non-smooth points are
exact in fp32 and fp64, the boundary sizes straddle the cluster switch as intended, and the fp64 autograd reference
follows the conventions the kernels are held to at those points."""
import math

import pytest
import torch

from open_l2o_b200 import _lib
from tests import zoo_cases as zc


@pytest.mark.parametrize("cls", ["Norm", "Rastrigin"])
@pytest.mark.parametrize("n", [100, 300])
def test_zero_residual_is_exact(cls, n):
    for seed in (0, 1):
        problem, x, i, a, b = zc.zero_residual(cls, n, seed)
        assert a != b and x[a] == x[b] and x[a] != 0
        for dtype in (torch.float32, torch.float64):
            r = zc.residuals(problem, x, dtype)
            assert r[i] == 0, (dtype, float(r[i]))
            assert int((r == 0).sum()) == 1, dtype   # the other rows are generic
        if n >= 256:   # row i, column a and column b in three different CTAs' blocks of the cluster
            blk = math.ceil(n / zc.CL)
            assert len({i // blk, a // blk, b // blk}) == 3
        assert bool(problem.const("w" if cls == "Norm" else "a", x)[i].abs().sum() == 2)   # the cached constant
        ref = zc.reference(problem, x)
        assert bool(torch.isfinite(ref["f"])) and bool(torch.isfinite(ref["g"]).all())   # subgradient 0 at r_i = 0


def test_lasso_zeros_and_min_max_ties_are_exact():
    _, x = zc.lasso_zeros(300, 0)
    assert int((x == 0).sum()) == 100 and int(torch.signbit(x[3::6]).sum()) == 50
    for dtype in (torch.float32, torch.float64):
        sq = zc.min_max_ties(4096, 0).to(dtype) ** 2
        assert [int(j) for j in torch.nonzero(sq == sq.max())] == sorted(zc.MMW_MAX)
        assert [int(j) for j in torch.nonzero(sq == sq.min())] == sorted(zc.MMW_MIN)
        sq = zc.min_max_ties(4096, 0, all_equal=True).to(dtype) ** 2
        assert bool((sq == sq[0]).all())
    # the tied extremes sit in different warps (j % 512 // 32) and different passes of the block loop (j // 512)
    for pair in (zc.MMW_MAX, zc.MMW_MIN):
        assert len({j % 512 // 32 for j in pair}) == 2 and len({j // 512 for j in pair}) == 2


def test_boundary_sizes_straddle_the_cluster_switch():
    sizes = {(c, a[0]): zc.on_cluster(a[0], a[0]) for c, a, _ in zc.BOUNDARY_CASES if c in ("Quadratic", "Norm",
                                                                                              "Lasso", "Rastrigin")}
    assert sizes[("Quadratic", 255)] is False and sizes[("Quadratic", 256)] is True and 256 * 256 == zc.CLUSTER_WORK
    n = 257   # a ragged last row block and column block next to full ones
    blk = math.ceil(n / zc.CL)
    assert sizes[("Quadratic", n)] and sizes[("Norm", n)] and n - (zc.CL - 1) * blk not in (0, blk)
    elementwise = [zc.make(c, a, kw) for c, a, kw in zc.BOUNDARY_CASES[-3:]]   # at the largest plan, n = 4096
    assert [sum(math.prod(s) for s in p.param_shapes) for p in elementwise] == [_lib.ZOO_MAX_N] * 3
    on = {nb: zc.on_cluster(nb[1], nb[0]) for nb in zc.BOUNDARY_DATA}
    assert on == {(4096, 15): False, (4096, 16): True, (64, 1023): False, (64, 1024): True, (2, 32768): True}
    assert math.ceil(16 / zc.CL) == 2   # rows per CTA at (4096, 16)
    owners = [r for r in range(zc.CL) if min(2, r * math.ceil(2 / zc.CL)) < 2]
    assert owners == [0, 1]   # at n = 2 CTAs 2 .. 7 own no columns but still join both cluster barriers
    from tests.test_scale_zoo_gpu import CASES, DATA_CASES
    assert all(c in CASES for c in zc.BOUNDARY_CASES)
    assert all((c, n, b) in DATA_CASES for c in zc.DATA_FAMILIES for n, b in zc.BOUNDARY_DATA)


@pytest.mark.parametrize("p", [1.5, 2.0, 3.0])
def test_autograd_gives_zero_curvature_at_a_zero_residual(p):
    """d sign / dr = 0: row and column i of the Hessian of Norm's (sum (|r| + 1e-6)^p)^(1/p) in r vanish at r_i = 0."""
    r = torch.tensor([0.7, 0.0, -1.3, 0.4], dtype=torch.float64, requires_grad=True)
    f = ((r.abs() + 1e-6) ** p).sum() ** (1.0 / p)
    (g,) = torch.autograd.grad(f, r, create_graph=True)
    H = torch.stack([torch.autograd.grad(g[j], r, retain_graph=True)[0] for j in range(4)])
    assert g[1] == 0 and not bool(H[1].any()) and not bool(H[:, 1].any())
    assert bool((H[[0, 2, 3]][:, [0, 2, 3]].diagonal() != 0).all())


def test_reference_is_nan_at_sqrt_zero():
    """fp64 autograd has NaN in every entry of g, H v and dq/dx at Ackley's origin and at OutwardSnake's x = 0, which
    the GPU test matches entry for entry."""
    cases = [(zc.make("Ackley"), torch.zeros(2), None),
             (zc.make("OutwardSnake", (64,)), torch.zeros(64), zc.data_batch("OutwardSnake", 64, 128, 0))]
    for problem, x, data in cases:
        n = x.numel()
        g = torch.Generator().manual_seed(0)
        ref = zc.reference(problem, x, torch.randn(n, generator=g), torch.randn(3, n, generator=g),
                           torch.randn(3, n, generator=g), data)
        assert bool(torch.isfinite(ref["f"]))
        for k in ("g", "hv", "dq"):
            assert bool(torch.isnan(ref[k]).all()), (type(problem).__name__, k)


def test_plane_points_cover_the_init_range_and_minima():
    for cls in zc.PLANE_FAMILIES:
        pts = zc.plane_points(cls)
        assert pts.shape[0] >= 64 and pts.dtype == torch.float32
        for m in zc.MINIMA.get(cls, []):
            assert any(tuple(p.tolist()) == m for p in pts)
    for cls, m in zc.MINIMA.items():   # the minima are exact in fp32, and the restatement's gradient is 0 there
        x = torch.tensor(m, dtype=torch.float32)
        ref = zc.reference(zc.make(cls), x)
        assert float(ref["f"]) == 0.0 and not bool(ref["g"].any()), cls
