"""CPU-only: the confocal_microscopy_3d and square_cos problems (DM/problems.py:701-995), their registry entries
(DM/util.py:215-230), the oracle's losses and the argument checks of l2o_confocal_grad."""
import ctypes

import torch

from tests import confocal_oracle as co
from tests.helpers import rel_err


def _capture(build, seed=0):
    """Run a builder through variables.variable_getter: (trainables, constants) as lists of (name, shape, tensor)."""
    from open_l2o_b200.variables import variable_getter
    gen = torch.Generator().manual_seed(seed)
    out = ([], [])

    def getter(name, shape, dtype, initializer, trainable):
        t = initializer(shape, gen)
        out[0 if trainable else 1].append((name, tuple(shape), t))
        return t

    with variable_getter(getter):
        loss = build()
    return out[0], out[1], loss


def _rows(entries):
    return torch.stack([t.reshape(-1) for _, _, t in entries])


def test_confocal_names_shapes_and_order_follow_the_reference():
    from open_l2o_b200 import problems
    P, B = 3, 4
    var, const, _ = _capture(problems.confocal_microscopy_3d(batch_size=B, num_points=P, ROI=(5, 6, 7)))
    params = ("I", "x", "y", "z", "sigmaxy", "sigmaz")
    assert [n for n, _, _ in var] == ["%s_var_%d" % (n, i) for i in range(P) for n in params] + ["bg_var"]
    sims = ["I_sim_%d", "x_sim_%d", "y_sim%d", "z_sim_%d", "sigmaxy_sim_%d", "sigmaz_sim_%d"]   # DM/problems.py:871
    assert [n for n, _, _ in const] == [s % i for i in range(P) for s in sims] + ["bg_sim"]
    assert all(s == (B, 1) for _, s, _ in var + const)


def test_confocal_oracle_equals_builder_loss():
    """The product loss (what the autograd path differentiates) and the oracle's dense restatement, same fp32 tensors."""
    from open_l2o_b200 import problems
    for B, P, roi in [(4, 2, (5, 7, 9)), (2, 5, (28, 28, 28))]:
        var, const, loss = _capture(problems.confocal_microscopy_3d(batch_size=B, num_points=P, ROI=roi), seed=3)
        f = co.confocal_f(_rows(var), _rows(const), B, P, roi)
        assert f.dtype == torch.float32
        assert rel_err(f, loss) <= 1e-6, (float(f), float(loss))


def test_confocal_oracle_gradient_matches_central_differences():
    B, P, roi = 2, 2, (4, 5, 6)
    gen = torch.Generator().manual_seed(5)
    x = torch.rand(6 * P + 1, B, generator=gen, dtype=torch.float64) * 1.4 - 0.2   # inside and outside [0, 1]
    sim = torch.rand(6 * P + 1, B, generator=gen, dtype=torch.float64)
    xg = x.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(co.confocal_f(xg, sim, B, P, roi), xg)
    h, fd = 1e-6, torch.zeros_like(x)
    for k in range(x.numel()):
        e = torch.zeros_like(x).view(-1)
        e[k] = h
        e = e.view_as(x)
        fd.view(-1)[k] = (co.confocal_f(x + e, sim, B, P, roi) - co.confocal_f(x - e, sim, B, P, roi)) / (2 * h)
    assert rel_err(g, fd) <= 1e-7


def test_square_cos_oracle_equals_builder_loss():
    from open_l2o_b200 import problems
    var, const, loss = _capture(problems.square_cos(batch_size=16, num_dims=3), seed=1)
    assert [n for n, _, _ in var] == ["x"] and [n for n, _, _ in const] == ["w", "y", "wcos"]
    (_, _, x), = var
    w, y, wcos = (t for _, _, t in const)
    assert rel_err(co.square_cos_f(x, w, y, wcos), loss) <= 1e-6


def test_get_config_entries_and_their_producers():
    from open_l2o_b200 import util
    cw = {"cw": {"net": "CoordinateWiseDeepLSTM", "net_options": {"layers": (20, 20)}, "net_path": None}}
    for name, (n_var, n_const, size) in {"confocal_microscopy_3d": (31, 31, 32), "square_cos": (1, 3, 256)}.items():
        problem, net_config, net_assignments = util.get_config(name)
        assert net_config == cw and net_assignments is None
        var, const, _ = _capture(problem)
        assert (len(var), len(const)) == (n_var, n_const)
        assert sum(t.numel() for _, _, t in var) == (size if name == "square_cos" else 31 * size)
    problem, _, _ = util.get_config("confocal_microscopy_3d")
    assert problem.producer.kind == "confocal_psf" and problem.producer.num_points == 5
    assert problem.producer.roi == (28, 28, 28)
    square, _, _ = util.get_config("square_cos")
    assert getattr(square, "fused", None) is None and getattr(square, "producer", None) is None


def test_confocal_args_follow_the_header_field_order():
    from open_l2o_b200 import _lib
    from tests.test_lib_abi import _struct_fields
    assert [f[0] for f in _lib.ConfocalArgs._fields_] == _struct_fields("l2o_confocal_args")


def test_confocal_grad_checks_arguments_without_gpu():
    from open_l2o_b200 import _lib, engine, problems
    L = _lib.lib()
    fake = ctypes.c_void_p(16)   # never dereferenced: every check below returns before any CUDA call

    def call(batch=2, P=5, roi=(28, 28, 28), x=fake, sim=fake, g=fake):
        a = _lib.ConfocalArgs()
        a.batch, a.num_points = batch, P
        for k in range(3):
            a.roi[k] = roi[k]
        a.x, a.sim, a.g = x, sim, g
        return L.l2o_confocal_grad(ctypes.byref(a), None)

    assert L.l2o_confocal_grad(None, None) == _lib.L2O_E_INVALID
    for kw in (dict(x=None), dict(sim=None), dict(g=None), dict(batch=-1), dict(P=0), dict(roi=(28, 0, 28))):
        assert call(**kw) == _lib.L2O_E_INVALID, kw
    for P, roi in [(5, (64, 64, 64)), (1, (38, 38, 38)), (48, (32, 32, 32)), (1, (1 << 20, 1, 1))]:
        assert not engine.confocal_fits(P, roi)
        assert call(P=P, roi=roi) == _lib.L2O_E_UNSUPPORTED, (P, roi)
        assert getattr(problems.confocal_microscopy_3d(num_points=P, ROI=roi), "fused", None) is None
    assert call(batch=0) == _lib.L2O_OK   # nothing to do, no launch
    assert engine.confocal_fits(47, (32, 32, 32)) and engine.confocal_fits(5, (28, 28, 28))
