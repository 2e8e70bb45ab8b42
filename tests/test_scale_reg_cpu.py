"""CPU: L2O-Scale's regularisers (``scale_reg``) against the fp64 oracle and closed forms, the regularize_time table,
the trainer and driver arguments, and the ``l2o_zoo_hess_form`` argument checks without a device."""
import ctypes as C
import itertools
import os

import pytest
import torch

from open_l2o_b200 import _lib
from open_l2o_b200 import scale_metarun as smr
from open_l2o_b200 import scale_reg as R
from oracle import scale_reg_oracle as O


def _quadratic(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(n, n, generator=g, dtype=torch.float64)
    y = torch.randn(n, generator=g, dtype=torch.float64)
    return W, y, (lambda x: 0.5 * ((W @ x - y) ** 2).sum())


def test_oracle_closed_forms_on_a_quadratic():
    n = 6
    W, y, f = _quadratic(n)
    H = W.T @ W
    x = torch.randn(n, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    # Hutchinson over every sign vector is exactly tr H
    signs = torch.tensor(list(itertools.product([-1.0, 1.0], repeat=n)), dtype=torch.float64)
    assert torch.allclose(O.hutchinson(H, signs), torch.trace(H), rtol=1e-12)
    # Lanczos: sum alpha = trace T = sum of T's eigenvalues
    v0 = O._unit(torch.ones(n, dtype=torch.float64))
    al, be = O.lanczos(H, v0, 4)
    assert torch.allclose(al.sum(), torch.linalg.eigvalsh(O.tridiagonal(al, be)).sum(), rtol=1e-10)
    # power iteration run to convergence gives lambda_max
    # (up to the 1e-6 in the normalisation, which scales the unit vector by 1 / (1 + 1e-6): lambda by about 1 - 2e-6)
    lam = O.power_iteration(H, torch.randn(n, generator=torch.Generator().manual_seed(2), dtype=torch.float64), 500)
    assert abs(float(lam) - float(torch.linalg.eigvalsh(H)[-1])) <= 3e-6 * float(torch.linalg.eigvalsh(H)[-1])
    # jacob: mean g^2
    g = W.T @ (W @ x - y)
    assert torch.allclose(O.regularizer("jacob", f, x), (g * g).mean(), rtol=1e-12)


def _nonquadratic():
    g = torch.Generator().manual_seed(3)
    A = torch.randn(5, 5, generator=g, dtype=torch.float64)
    return lambda x: torch.log1p(((A @ x) ** 2).sum()) + (x ** 4).sum() * 0.1 + torch.sin(x).sum()


@pytest.mark.parametrize("option", R.OPTIONS)
def test_regularizer_generic_path_matches_oracle(option):
    """The product's autograd path on a plain fp64 callable, against the oracle's explicit Hessian; the gradient of
    reg too (the meta-gradient's term), by autograd through the oracle."""
    f = _nonquadratic()
    reg = R.Regularizer(option, hessian_itrs=4, seed=5)
    x = torch.linspace(-0.7, 0.9, 5, dtype=torch.float64).requires_grad_(True)
    objective = lambda ps: f(ps[0])   # noqa: E731
    gen = torch.Generator().manual_seed(9)
    got = reg(objective, x, lambda t: [t], gen)
    (dgot,) = torch.autograd.grad(got, x)
    probes = reg.probes(objective, 5, "cpu", torch.float64) if option in ("hessian", "hessian-esd") else None
    v0 = torch.randn(5, generator=torch.Generator().manual_seed(9)).double() if option == "hessian-ev" else \
        (probes[0] if option == "hessian-esd" else None)
    xr = x.detach().clone().requires_grad_(True)
    with torch.enable_grad():
        g = torch.autograd.grad(f(xr), xr, create_graph=True)[0]
        H = torch.stack([torch.autograd.grad(g[i], xr, create_graph=True)[0] for i in range(5)])
        if option == "jacob":
            want = O.jacob(g)
        elif option == "hessian":
            want = O.hutchinson(H, probes)
        elif option == "hessian-ev":
            want = O.power_iteration(H, v0.double(), 4)
        else:
            want = O.lanczos(H, v0, 4)[0].sum()
    (dwant,) = torch.autograd.grad(want, xr)
    assert abs(float(got) - float(want)) <= 1e-10 * max(1.0, abs(float(want))), (option, float(got), float(want))
    assert torch.allclose(dgot, dwant, rtol=1e-8, atol=1e-10), option
    assert float(O.regularizer(option, f, x.detach(), probes=probes, v0=v0, itrs=4)) == pytest.approx(float(want),
                                                                                                       rel=1e-10)


def test_fixed_probes_are_fixed_per_objective_and_seeded():
    a, b = R.Regularizer("hessian", 10, seed=1), R.Regularizer("hessian", 10, seed=1)
    f1, f2 = (lambda ps: ps[0].sum()), (lambda ps: ps[0].sum())
    p1 = a.probes(f1, 7, "cpu")
    assert p1.shape == (10, 7) and set(p1.unique().tolist()) <= {-1.0, 1.0}
    assert torch.equal(a.probes(f1, 7, "cpu"), p1) and torch.equal(b.probes(f1, 7, "cpu"), p1)
    assert not torch.equal(a.probes(f2, 7, "cpu"), p1)
    e = R.Regularizer("hessian-esd", 10, seed=1).probes(f1, 9, "cpu")
    assert e.shape == (1, 9) and abs(float(e.norm()) - 1.0) < 1e-5


@pytest.mark.parametrize("N", [1, 2, 4, 6, 10, 17])
@pytest.mark.parametrize("scale", [0.0, 0.25, 0.5, 0.9])
def test_regularize_time_table(N, scale):
    b = int(N * scale + 1)
    for i in range(N):
        assert R.reg_switch("posterior", i, N, scale) == (i > b) == O.switch("posterior", i, N, scale)
        assert R.reg_switch("prior", i, N, scale) == (i < b) == O.switch("prior", i, N, scale)
        assert R.reg_switch("none", i, N, scale) is False
        assert R.reg_switch("always", i, N, scale) is True


def test_unknown_option_and_fourth_derivatives_raise_at_construction():
    from open_l2o_b200 import baselines_train as bt
    from open_l2o_b200 import hrnn_train as ht
    with pytest.raises(ValueError):
        R.Regularizer("hessian-trace")
    with pytest.raises(ValueError):
        ht.MetaTrainer([(3,)], reg_option="bogus", device="cpu")
    for option in ("hessian", "hessian-ev", "hessian-esd"):
        with pytest.raises(NotImplementedError, match="reg_optimizee"):
            bt.TrainableAdamTrainer([(3,)], device="cpu", reg_optimizee=True, reg_option=option,
                                    use_second_derivatives=True)
    R.check_options("jacob", True, True)               # third order only: supported
    R.check_options("hessian", True, False)
    R.check_options("hessian", False, True)            # reg_optimizer alone: supported


def test_metarun_regulariser_flags():
    f = smr.parse([])
    assert f.reg_optimizer is False and f.reg_optimizee is False and f.reg_option == "hessian"
    assert f.hessian_itrs == 10 and f.alpha == 5e-4 and f.beta == 1e-4
    assert f.regularize_time == "posterior" and f.reg_scale == 0.5
    base = smr.optimizer_kwargs(f)
    f = smr.parse(["--reg_optimizer", "--reg_optimizee=true", "--reg_option", "hessian-esd", "--hessian_itrs", "4",
                   "--alpha", "0.1", "--beta", "0.2", "--regularize_time", "prior", "--reg_scale", "0.3"])
    assert f.reg_optimizer and f.reg_optimizee and f.reg_option == "hessian-esd" and f.hessian_itrs == 4
    assert (f.alpha, f.beta, f.regularize_time, f.reg_scale) == (0.1, 0.2, "prior", 0.3)
    assert smr.optimizer_kwargs(f) == base             # the optimizer's arguments do not change
    assert smr.parse(["--noreg_optimizer"]).reg_optimizer is False
    assert smr.parse(["--reg_optimizee=false"]).reg_optimizee is False


def test_metarun_hands_the_flags_to_the_trainer(monkeypatch, tmp_path):
    seen = {}

    class Opt(object):
        def meta_trainer(self, var_list, **kw):
            seen.update(kw)

    import open_l2o_b200.trainable_baselines as tb
    monkeypatch.setattr(tb, "register_optimizers", lambda: {"HierarchicalRNN": lambda **kw: Opt()})
    monkeypatch.setattr(smr, "build_problems", lambda entries, device, seed: ([(None, lambda: [torch.zeros(2)])], []))

    def loop(make_trainer, problems, *a, **k):
        make_trainer(((2,),), None)
        return None, []
    f = smr.parse(["--include_quadratic_problems", "--reg_optimizer", "--reg_option", "jacob", "--alpha", "0.5",
                   "--train_dir", str(tmp_path), "--device", "cpu"])
    smr.run(f, out=None, train_optimizer=loop)
    assert seen["reg_optimizer"] is True and seen["reg_optimizee"] is False and seen["reg_option"] == "jacob"
    assert seen["alpha"] == 0.5 and seen["beta"] == 1e-4 and seen["hessian_itrs"] == 10
    assert seen["regularize_time"] == "posterior" and seen["reg_scale"] == 0.5


# ---- C ABI -------------------------------------------------------------------------------------------------------------
def _form(**kw):
    a = _lib.ZooFormArgs()
    b = a.base
    b.family, b.n, b.rows = kw.get("family", _lib.ZOO["QUADRATIC"]), kw.get("n", 4), kw.get("rows", 4)
    b.p0 = kw.get("p0", 2.0)
    fake = 256
    for name in ("x", "v", "A", "y", "c", "f", "out"):
        setattr(b, name, kw.get(name, fake))
    a.k = kw.get("k", 2)
    for name in ("U", "V", "q"):
        setattr(a, name, kw.get(name, fake))
    return a


@pytest.mark.skipif(not os.path.exists(_lib.LIB_PATH), reason="library not built")
def test_hess_form_abi_argument_checks_without_gpu():
    L, Z_ = _lib.lib(), _lib.ZOO
    INV, UNS = _lib.L2O_E_INVALID, _lib.L2O_E_UNSUPPORTED
    assert "l2o_zoo_hess_form" in _lib.EXPORTS
    assert L.l2o_zoo_hess_form(None, None) == INV
    bad = [dict(U=None), dict(V=None), dict(out=None), dict(k=0), dict(k=-3), dict(x=None), dict(family=-1),
           dict(family=21), dict(n=0), dict(rows=5), dict(A=None), dict(y=None), dict(family=Z_["NORM"], p0=0.0),
           dict(family=Z_["RASTRIGIN"], c=None), dict(family=Z_["ROSENBROCK"], n=3),
           dict(family=Z_["OUTWARD_SNAKE"], n=1), dict(family=Z_["DEPENDENCY_CHAIN"], n=1),
           dict(k=0, n=_lib.ZOO_MAX_N + 1, rows=_lib.ZOO_MAX_N + 1)]
    for kw in bad:
        assert L.l2o_zoo_hess_form(C.byref(_form(**kw)), None) == INV, kw
    for kw in (dict(k=_lib.ZOO_MAX_PAIRS + 1), dict(n=_lib.ZOO_MAX_N + 1, rows=_lib.ZOO_MAX_N + 1),
               dict(family=Z_["ISOTROPIC_QUADRATIC"], n=_lib.ZOO_MAX_N + 1)):
        assert L.l2o_zoo_hess_form(C.byref(_form(**kw)), None) == UNS, kw


def test_header_declares_max_pairs():
    hdr = open(os.path.join(_lib.INCLUDE, "l2o_b200.h")).read()
    assert "#define L2O_ZOO_MAX_PAIRS %d" % _lib.ZOO_MAX_PAIRS in hdr
