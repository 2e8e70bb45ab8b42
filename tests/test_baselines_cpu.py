"""CPU: L2O-Scale's baselines (TrainableAdam, LearningRateSchedule, GlobalLearningRate).  The oracle
(oracle/baselines_oracle.py) against the closed forms that pin it, TrainableAdam's literal second moment (NaN at
g = +-1, none at g = 0, a zero beta2_logit meta-gradient), the second-order meta-gradient against central finite
differences, the constructors' checks, the C-ABI's argument validation and the driver name table.  The oracle
meta-gradient here is shared with tests/test_baselines_gpu.py."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import baselines_oracle as B
from open_l2o_b200 import _lib
from tests.test_second_order_cpu import TINY, _assert_fd, _fd_check, _meta, _unrolled_objectives, curved_problem


def tadam_theta(lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, dtype=torch.float64):
    """TrainableAdam's theta from its hyperparameters (TA:64-82), in fp64 then `dtype`."""
    v = [math.log(lr), math.log(b1 / (1 - b1)), math.log(b2 / (1 - b2)), math.log(eps)]
    return torch.tensor(v, dtype=torch.float64).to(dtype)


def baseline_oracle_meta(which, theta, objective, init, T, second, dtype=torch.float64, carry=None, initial_obj=None,
                         need_grad=True):
    """(meta, d meta / d theta, carry) of one unroll through the oracle in `dtype`, for which in ("tadam", "lrs",
    "glr"): from `init` with a fresh state, or from a detached `carry` (truncated BPTT) normalised by `initial_obj`.
    theta: TrainableAdam's [4], the schedule [n_steps], or the global rate [1]."""
    th = theta.to(dtype).clone().requires_grad_(True)
    if carry is None:
        params = [p.to(dtype) for p in init]
        states = [B.tadam_initial_state(p.numel(), dtype) for p in params] if which == "tadam" else 0
    else:
        params = [p.detach() for p in carry[0]]
        states = [{k: v.detach() for k, v in s.items()} for s in carry[1]] if which == "tadam" else carry[1]

    def step(ps, gs, sts):
        if which == "tadam":
            ps, sts, _ = B.tadam_step(th, ps, gs, sts)
            return ps, sts
        ps, itr, _ = B.lrs_step(th, ps, gs, sts)
        return ps, (itr if which == "lrs" else 0)
    objs, params, states = _unrolled_objectives(step, objective, params, states, T, second, carry is None)
    f0 = objs[0].detach() if initial_obj is None else initial_obj
    meta = _meta(objs, f0)
    g = torch.autograd.grad(meta, th)[0] if need_grad else None
    return meta.detach(), g, (params, states, None, f0)


# ---------------------------------------------------------------------------------------------------------------------
# closed forms

def test_glr_step_is_x_minus_lr_g():
    gen = torch.Generator().manual_seed(0)
    x, g = torch.randn(50, generator=gen, dtype=torch.float64), torch.randn(50, generator=gen, dtype=torch.float64)
    for itr in (0, 7):   # the global rate has one entry: every step uses it
        x1, itr1, upd = B.lrs_compute_update(torch.tensor([0.3], dtype=torch.float64), x, g, itr)
        assert torch.equal(x1, x - 0.3 * g) and torch.equal(upd, 0.3 * g) and itr1 == itr + 1


def test_lrs_index_clamps_at_last_entry():
    rates = torch.tensor([0.1, 0.2, 0.3], dtype=torch.float64)
    x, g = torch.ones(4, dtype=torch.float64), torch.full((4,), 2.0, dtype=torch.float64)
    used, itr = [], 0
    for _ in range(6):
        x_new, itr, upd = B.lrs_compute_update(rates, x, g, itr)
        used.append(float(upd[0]) / 2.0)
    assert used == [0.1, 0.2, 0.3, 0.3, 0.3, 0.3] and itr == 6


def test_lrs_default_schedule_does_not_move_x_but_has_a_meta_gradient():
    """initial_rate = 0 (LRS:30): x stays put, and d meta / d rates[0] is still nonzero."""
    objective, init = curved_problem(TINY, seed=1)
    meta, g, (params, _, _, _) = baseline_oracle_meta("lrs", torch.zeros(5, dtype=torch.float64), objective, init, 3, False)
    assert all(torch.equal(p, q) for p, q in zip(params, init))
    # the objectives of x_1 and x_2 see rates[0] and rates[1]; the last step's rate reaches no scored objective
    assert bool((g[:2] != 0).all()) and float(g[2:].abs().max()) == 0.0


@pytest.mark.parametrize("b1", [0.9, 0.999])
def test_tadam_first_step_is_lr_g_over_1e5_plus_eps(b1):
    """Step 1 from the zero state: m^_1 = g and v stays 0, so update = lr g / (sqrt(1e-10) + eps), where eps is
    exp(log_epsilon) + 1e-10 (TA:124)."""
    lr, eps = 1e-3, 1e-8
    th = tadam_theta(lr=lr, b1=b1, eps=eps)
    gen = torch.Generator().manual_seed(1)
    g = torch.randn(40, 1, generator=gen, dtype=torch.float64) * 10.0 ** torch.randint(-6, 4, (40, 1), generator=gen)
    x = torch.randn(40, 1, generator=gen, dtype=torch.float64)
    x1, st, upd = B.tadam_compute_update(th, x, g, B.tadam_initial_state(40))
    want = lr * g / (1e-5 + eps + 1e-10)
    assert torch.allclose(upd, want, rtol=1e-12, atol=0) and torch.allclose(x1, x - want, rtol=1e-12, atol=1e-300)
    assert torch.equal(st["t"], torch.ones(40, 1, dtype=torch.float64)) and float(st["v"].abs().max()) == 0.0


def test_tadam_second_moment_stays_zero_and_update_is_momentum_sgd():
    """v == 0 for every step from the zero state (g never +-1), so update_t = lr m^_t / (1e-5 + eps) with the
    bias-corrected momentum m^_t, about 1e5 lr times a gradient average."""
    lr, b1, eps = 1e-3, 0.8, 1e-8
    th = tadam_theta(lr=lr, b1=b1, eps=eps)
    gen = torch.Generator().manual_seed(2)
    x, st, m = torch.randn(30, 1, generator=gen, dtype=torch.float64), B.tadam_initial_state(30), 0.0
    for t in range(1, 6):
        g = torch.randn(30, 1, generator=gen, dtype=torch.float64) * 0.5
        x, st, upd = B.tadam_compute_update(th, x, g, st)
        m = b1 * m + (1 - b1) * g
        assert float(st["v"].abs().max()) == 0.0
        assert torch.allclose(upd, lr * (m / (1 - b1 ** t)) / (1e-5 + eps + 1e-10), rtol=1e-10, atol=0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_tadam_nan_at_unit_gradient_and_not_at_zero(dtype):
    """g = +-1: pow(g^2, b2) == 1 and v' = 0/0 = NaN, and that coordinate's update and x are NaN from then on.  g = 0
    leaves everything finite, the gradients (first and second order) included."""
    th = tadam_theta(dtype=dtype).requires_grad_(True)
    g = torch.tensor([[1.0], [-1.0], [0.0], [0.5], [1e-30], [1e30]], dtype=dtype, requires_grad=True)
    x = torch.zeros(6, 1, dtype=dtype)
    x1, st, upd = B.tadam_compute_update(th, x, g, B.tadam_initial_state(6, dtype))
    nan = torch.isnan(st["v"]).reshape(-1).tolist()
    assert nan == [True, True, False, False, False, False]
    assert torch.isnan(upd).reshape(-1).tolist() == nan and torch.isnan(x1).reshape(-1).tolist() == nan
    x2, st2, _ = B.tadam_compute_update(th, x1, torch.full((6, 1), 0.25, dtype=dtype), st)
    assert torch.isnan(x2).reshape(-1).tolist() == nan   # NaN stays
    # without the +-1 coordinates (a NaN coordinate's adjoints are NaN, and theta's sum over coordinates with them):
    # finite adjoints through two steps, beta2_logit's exactly 0
    g = g[2:].detach().clone().requires_grad_(True)
    x1, st, _ = B.tadam_compute_update(th, x[2:], g, B.tadam_initial_state(4, dtype))
    x2, st2, _ = B.tadam_compute_update(th, x1, g * 0.5, st)
    d_th, d_g = torch.autograd.grad(x2.sum() + st2["m"].sum() + st2["v"].sum(), (th, g))
    assert bool(torch.isfinite(d_th).all()) and bool(torch.isfinite(d_g).all()) and float(d_th[2]) == 0.0


def test_tadam_beta2_logit_has_zero_meta_gradient():
    """In every reachable state without the NaN, v == 0, so beta2_logit changes nothing: its meta-gradient is exactly
    0, first and second order, while the other three are not."""
    objective, init = curved_problem(TINY, seed=3)
    th = tadam_theta(lr=3e-6, b1=0.7, b2=0.95)
    for second in (False, True):
        _, g, _ = baseline_oracle_meta("tadam", th, objective, init, 4, second)
        assert float(g[2]) == 0.0 and bool((g[[0, 1, 3]] != 0).all()), (second, g)


# ---------------------------------------------------------------------------------------------------------------------
# second-order meta-gradients against central finite differences

@pytest.mark.parametrize("which", ["tadam", "lrs", "glr"])
def test_baseline_oracle_second_order_matches_finite_differences(which):
    """T = 3 on two tiny tensors.  The step sizes are large enough for the optimizee's curvature to matter: an
    effective TrainableAdam rate of lr / (1e-5 + eps) = 0.3, schedule entries 0.1 .. 0.4 (n_steps = 2, so the third step
    reuses the last one), a global rate of 0.3."""
    objective, init = curved_problem(TINY, seed=6)
    if which == "tadam":
        theta = tadam_theta(lr=3e-6, b1=0.8)
    elif which == "lrs":
        theta = torch.tensor([0.1, 0.4], dtype=torch.float64)
    else:
        theta = torch.tensor([0.3], dtype=torch.float64)

    def meta_fn(th, second, need_grad=True):
        return baseline_oracle_meta(which, th, objective, init, 3, second, need_grad=need_grad)
    _assert_fd(_fd_check(meta_fn, theta, 3, seed=2))


# ---------------------------------------------------------------------------------------------------------------------
# Python surface

def test_tadam_constructor_checks():
    from open_l2o_b200.trainable_baselines import TrainableAdam
    for kw in (dict(learning_rate=0.0), dict(learning_rate=-1.0), dict(epsilon=0.0), dict(beta1=0.0), dict(beta1=1.0),
               dict(beta2=0.0), dict(beta2=1.5)):
        with pytest.raises(ValueError):
            TrainableAdam(device="cpu", **kw)
    with pytest.raises(TypeError):   # the reference drivers pass the HRNN cell sizes positionally (SC/metarun.py:371)
        TrainableAdam([10, 20, 20], device="cpu")


def test_rate_constructors_reject_the_drivers_positional_cell_sizes():
    from open_l2o_b200.trainable_baselines import GlobalLearningRate, LearningRateSchedule
    for cls in (GlobalLearningRate, LearningRateSchedule):
        with pytest.raises(TypeError):
            cls([10, 20, 20], device="cpu")


def test_variables_names_and_initial_values():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    from open_l2o_b200.trainable_baselines import GlobalLearningRate, LearningRateSchedule, TrainableAdam
    ta = TrainableAdam(learning_rate=2e-3, beta1=0.8, beta2=0.99, epsilon=1e-7, device="cpu")
    v = ta.get_variables()
    assert list(v) == ["LOL/log_learning_rate", "LOL/beta1_logit", "LOL/beta2_logit", "LOL/log_epsilon"]
    want = np.array([np.log(2e-3), np.log(0.8 / 0.2), np.log(0.99 / 0.01), np.log(1e-7)], dtype=np.float64)
    assert torch.equal(ta.theta, torch.from_numpy(want).float())
    assert torch.equal(tadam_theta(2e-3, 0.8, 0.99, 1e-7, dtype=torch.float32), ta.theta)
    ta.load_variables({"LOL/beta1_logit": 1.5})
    assert float(ta.theta[1]) == 1.5
    lrs = LearningRateSchedule(device="cpu")
    assert list(lrs.get_variables()) == ["LOL/learning_rates"] and lrs.theta.shape == (1000,)
    assert float(lrs.theta.abs().max()) == 0.0
    glr = GlobalLearningRate(device="cpu")
    assert list(glr.get_variables()) == ["LOL/global_learning_rate"]
    assert float(glr.get_variables()["LOL/global_learning_rate"]) == pytest.approx(1e-3)


def test_register_optimizers_names():
    from open_l2o_b200 import coordinatewise_rnn, hierarchical_rnn, trainable_baselines as tb
    opts = tb.register_optimizers()
    assert sorted(opts) == ["CoordinatewiseRNN", "GlobalLearningRate", "HierarchicalRNN", "LearningRateSchedule",
                            "TrainableAdam"]
    assert opts["HierarchicalRNN"] is hierarchical_rnn.HierarchicalRNN
    assert opts["CoordinatewiseRNN"] is coordinatewise_rnn.CoordinatewiseRNN
    assert opts["TrainableAdam"] is tb.TrainableAdam


def test_trainers_default_to_first_order():
    import inspect
    from open_l2o_b200 import baselines_train as bt
    p = inspect.signature(bt._BaselineTrainer.__init__).parameters["use_second_derivatives"]
    assert p.default is False
    for cls in (bt.TrainableAdamTrainer, bt.LearningRateScheduleTrainer, bt.GlobalLearningRateTrainer):
        assert issubclass(cls, bt.MetaTrainerBase)


# ---------------------------------------------------------------------------------------------------------------------
# C-ABI argument validation (host addresses: validation must return before any CUDA call)

def _lib_or_skip():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    return _lib.lib()


def test_tadam_abi_rejects_bad_arguments():
    L = _lib_or_skip()
    assert L.l2o_tadam_theta_count() == 4 and L.l2o_tadam_state_floats() == 3
    n = 4
    sizes = dict(theta=16, g=4 * n, state_old=12 * n, d_state_new=12 * n, d_update=4 * n, d_state_old=12 * n,
                 d_theta=32)
    bufs = {k: (ctypes.c_double * (b // 8 + 4))() for k, b in sizes.items()}
    args = {k: ctypes.addressof(b) for k, b in bufs.items()}
    E = _lib.L2O_E_INVALID
    bwd = lambda **kw: L.l2o_tadam_bwd(ctypes.byref(_lib.TadamBwdArgs(**dict(dict(n=n, **args), **kw))), None)
    for k in args:
        assert bwd(**{k: None}) == E, k                       # null
        assert bwd(**{k: args[k] + 2}) == E, k                # misaligned
    assert bwd(d_theta=args["d_theta"] + 4) == E              # double pointer at a 4-byte offset
    assert bwd(n=0) == E and bwd(n=-3) == E
    own = (ctypes.c_double * 4)()
    assert bwd(d_g=ctypes.addressof(own) + 2) == E
    assert [f[0] for f in _lib.TadamBwdArgs._fields_][-1] == "d_g"
    for k, base in args.items():
        for d_g in (base, base + sizes[k] - 4, base - 4 * (n - 1)):   # first byte, last float, straddling the start
            assert bwd(d_g=d_g) == E, (k, d_g - base)
    st = dict(theta=args["theta"], g=args["g"], state_in=args["state_old"], state_out=args["state_old"])
    step = lambda **kw: L.l2o_tadam_step(ctypes.byref(_lib.TadamStepArgs(**dict(dict(n=n, **st), **kw))), None)
    for k in st:
        assert step(**{k: None}) == E and step(**{k: st[k] + 1}) == E, k
    assert step(n=0) == E and step(x=args["g"] + 2) == E and step(update=args["g"] + 2) == E


def test_lrsgd_abi_rejects_bad_arguments():
    L = _lib_or_skip()
    n, ns = 4, 3
    sizes = dict(rates=4 * ns, g=4 * n, d_update=4 * n, itr=8, d_rates=8 * ns)
    bufs = {k: (ctypes.c_double * (b // 8 + 4))() for k, b in sizes.items()}
    args = {k: ctypes.addressof(b) for k, b in bufs.items()}
    E = _lib.L2O_E_INVALID
    bwd = lambda **kw: L.l2o_lrsgd_bwd(ctypes.byref(_lib.LrsgdBwdArgs(**dict(dict(n=n, n_steps=ns, **args), **kw))), None)
    for k in ("rates", "g", "d_update", "d_rates"):
        assert bwd(**{k: None}) == E, k
    for k in args:
        assert bwd(**{k: args[k] + 2}) == E, k
    assert bwd(d_rates=args["d_rates"] + 4) == E
    assert bwd(n=0) == E and bwd(n_steps=0) == E and bwd(n_steps=-1) == E
    assert [f[0] for f in _lib.LrsgdBwdArgs._fields_][-1] == "d_g"
    for k, base in args.items():
        for d_g in (base, base + sizes[k] - 4, base - 4 * (n - 1)):
            assert bwd(d_g=d_g) == E, (k, d_g - base)
    st = dict(rates=args["rates"], g=args["g"])
    step = lambda **kw: L.l2o_lrsgd_step(ctypes.byref(_lib.LrsgdStepArgs(**dict(dict(n=n, n_steps=ns, **st), **kw))), None)
    for k in st:
        assert step(**{k: None}) == E and step(**{k: st[k] + 2}) == E, k
    assert step(n=0) == E and step(n_steps=0) == E and step(itr=args["itr"] + 2) == E and step(x=args["g"] + 1) == E
