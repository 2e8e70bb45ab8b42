"""Host logic of L2O-Scale's enhanced training recipe without a GPU (SC/metaopt.py:138-176, 354-450, 520-700,
SC/mt_utils.py): the teacher labels, the imitation unroll of ``MetaTrainerBase`` on a torch stepper, the seeded
imitation draws and the curriculum of ``scale_base.train_optimizer``."""
import math
import random

import numpy as np
import pytest
import torch

from open_l2o_b200 import scale_base as sb
from open_l2o_b200.data_generator import teacher_state, teacher_update


def _np_teacher(name, x, grad_fn, steps):
    """TF-1.14 Adam / RMSProp / Nesterov momentum at lr 0.01, hand-rolled in fp64 numpy; returns every iterate."""
    m, v, xs = np.zeros_like(x), np.zeros_like(x), [x.copy()]
    if name == "rmsprop":
        v[:] = 1.0
    for k in range(1, steps + 1):
        g = grad_fn(x)
        if name == "adam":
            m = 0.9 * m + 0.1 * g
            v = 0.999 * v + 0.001 * g * g
            x = x - 0.01 * math.sqrt(1 - 0.999 ** k) / (1 - 0.9 ** k) * m / (np.sqrt(v) + 1e-8)
        elif name == "rmsprop":
            v = 0.9 * v + 0.1 * g * g
            x = x - 0.01 * g / np.sqrt(v + 1e-10)
        else:
            m = 0.9 * m + g
            x = x - 0.01 * (g + 0.9 * m)
        xs.append(x.copy())
    return xs


def _quadratic(seed=0):
    rng = np.random.RandomState(seed)
    a = rng.uniform(0.5, 3.0, size=(3, 4))
    b = rng.randn(3, 4)
    c = rng.randn(5)
    at, bt, ct = (torch.tensor(t, dtype=torch.float32) for t in (a, b, c))

    def objective(ps):
        return (at * (ps[0] - bt) ** 2).sum() + ((ps[1] - ct) ** 2).sum()

    def grad(x):
        return np.concatenate([(2 * a * (x[:12].reshape(3, 4) - b)).reshape(-1), 2 * (x[12:] - c)])
    x0 = rng.randn(17)
    return objective, grad, x0, [(3, 4), 5]


@pytest.mark.parametrize("name", ["adam", "rmsprop", "nag"])
@pytest.mark.parametrize("k", [1, 3])
def test_teacher_labels_sign_and_grouping_against_numpy(name, k):
    """labels[t] = x_prev - x_cur over the t-th group of k teacher steps (the positive step), rows over all partial
    unrolls in run order; grads[t] is the gradient at the group's first point."""
    objective, grad, x0, sizes = _quadratic()
    lens = [2, 3]
    labels, grads = sb.teacher_labels(objective, torch.tensor(x0, dtype=torch.float32), sizes, lens, name, k)
    assert labels.shape == grads.shape == (5, 17) and labels.dtype == torch.float32
    xs = _np_teacher(name, x0.astype(np.float32).astype(np.float64), grad, 5 * k)
    for t in range(5):
        want = xs[t * k] - xs[(t + 1) * k]
        np.testing.assert_allclose(labels[t].double().numpy(), want, rtol=2e-4, atol=2e-6)
        np.testing.assert_allclose(grads[t].double().numpy(), grad(xs[t * k]), rtol=1e-4, atol=1e-5)
    # the teacher moves downhill: x - label lowers the objective on this quadratic
    x1 = torch.tensor(x0, dtype=torch.float32) - labels[0]
    split = lambda x: [x[:12].view(3, 4), x[12:]]
    assert float(objective(split(x1))) < float(objective(split(torch.tensor(x0, dtype=torch.float32))))


def test_teacher_forced_points_are_the_teachers_gradient_points():
    """Teacher forcing x_{t+1} = x_t - labels[t] lands bitwise on the points where grads were recorded."""
    objective, _, x0, sizes = _quadratic(1)
    labels, grads = sb.teacher_labels(objective, torch.tensor(x0, dtype=torch.float32), sizes, [4], "adam", 2)
    x = torch.tensor(x0, dtype=torch.float32)
    for t in range(4):
        xg = x.clone().requires_grad_(True)
        (g,) = torch.autograd.grad(objective([xg[:12].view(3, 4), xg[12:]]), xg)
        assert torch.equal(g, grads[t]), t
        x = x - labels[t]


def test_teacher_update_rejects_an_unknown_name_and_keeps_the_dm_rules():
    x = torch.tensor([1.0, -2.0])
    st = teacher_state(x)
    with pytest.raises(ValueError):
        teacher_update("sgd", x, torch.ones(2), st)
    g = torch.tensor([0.5, -0.25])
    teacher_update("adam", x, g, st)                 # first Adam step: lr * sign(g) up to epsilon
    assert torch.allclose(x, torch.tensor([0.99, -1.99]), atol=1e-6) and st["k"] == 1


class _ToyTrainer(sb.MetaTrainerBase):
    """A MetaTrainerBase with a torch stepper on the CPU: upd = theta0 * g + theta1 * m, m' = 0.5 m + g."""
    what = "toy"

    class State(object):
        def __init__(self, m, x):
            self.m, self.x = m, x

    def __init__(self, shapes, theta):
        self.device = torch.device("cpu")
        self.shapes = [tuple(s) for s in shapes]
        self.sizes = [int(math.prod(s)) for s in self.shapes]
        self.theta = theta.clone().requires_grad_(True)
        self.learning_rate, self.rms_decay, self.rms_epsilon, self.gradient_clip, self.l2_reg = 0.1, 0.9, 1e-10, 1e4, 0.0
        self.use_log_objective, self.use_numerator_epsilon, self.use_second_derivatives = True, False, False
        self.rms = torch.ones_like(self.theta)
        self.global_step = 0

    def initial_state(self, params, theta, _unused=None):
        x = self._x0(params)
        return self.State(torch.zeros_like(x), x)

    def _stepper(self, theta):
        def step(state, g):
            return theta[0] * g + theta[1] * state.m, self.State(0.5 * state.m + g, None)
        return step


def test_imitation_unroll_teacher_forces_and_scores_the_weighted_mse():
    """meta_gradient_mt on a torch stepper: x follows the labels, the meta objective is sum_t (1/T) sum_i
    (upd - label)^2 / 2 / N, replay and re-evaluation agree, and the meta-gradient is that objective's gradient."""
    objective, _, x0, sizes = _quadratic(2)
    shapes = [(3, 4), (5,)]
    params = [torch.tensor(x0[:12], dtype=torch.float32).view(3, 4), torch.tensor(x0[12:], dtype=torch.float32)]
    labels, grads = sb.teacher_labels(objective, torch.tensor(x0, dtype=torch.float32), sizes, [3, 2], "adam", 1)
    theta = torch.tensor([0.02, 0.01])
    tr = _ToyTrainer(shapes, theta)
    meta, g, objs, final = tr.meta_gradient_mt(None, params, labels[:3], grads[:3])
    assert objs == []
    x = torch.cat([p.reshape(-1) for p in params])
    for t in range(3):
        x = x - labels[t]
    assert torch.equal(final.x, x)
    # by hand, fp64
    th = theta.double().requires_grad_(True)
    m, want = torch.zeros(17, dtype=torch.float64), 0.0
    for t in range(3):
        gt = grads[t].double()
        upd = th[0] * gt + th[1] * m
        m = 0.5 * m + gt
        want = want + (1.0 / 3) * 0.5 * ((upd - labels[t].double()) ** 2).sum() / 17
    (gw,) = torch.autograd.grad(want, th)
    want = float(want.detach())
    assert abs(float(meta) - want) <= 1e-6 * abs(want)
    assert torch.allclose(g.double(), gw, rtol=1e-5, atol=0)
    meta_re, g_re, objs_re, final_re = tr.meta_gradient_mt(objective, params, labels[:3], None)
    assert len(objs_re) == 3 and float(meta_re) == float(meta) and torch.equal(g_re, g)
    assert torch.equal(final_re.x, final.x)
    # a run of two partial unrolls: two meta-steps, state carried
    metas, out = tr.train_problem_mt(None, params, labels, grads, [3, 2])
    assert len(metas) == 2 and tr.global_step == 2 and [tuple(o.shape) for o in out] == shapes
    with pytest.raises(ValueError):
        tr.train_problem_mt(None, params, labels, grads, [3, 3])


class _Stub(object):
    """A trainer that records what the driver asks of it; evaluation costs come from a script."""
    device = "cpu"

    def __init__(self, shapes, theta, events, costs):
        self.shapes = [tuple(s) for s in shapes]
        self.theta = torch.zeros(3) if theta is None else theta.clone()
        self.events, self.costs = events, costs

    def _x0(self, params):
        return torch.cat([p.reshape(-1).float() for p in params])

    def train_problem(self, objective, params, num_unrolls, unroll_len):
        self.events.append(("train", num_unrolls, unroll_len))
        self.theta += 1.0
        return [0.0] * num_unrolls, [], params

    def train_problem_mt(self, objective, params, labels, grads, lens):
        self.events.append(("mt", len(lens), tuple(labels.shape)))
        self.theta += 1.0
        return [0.0] * len(lens), params

    def evaluate(self, objective, params, lens):
        self.events.append(("eval", len(lens)))
        return next(self.costs)

    def get_variables(self):
        return {"theta": self.theta.clone()}

    def load_variables(self, values):
        self.events.append(("restore", float(values["theta"][0])))
        self.theta.copy_(values["theta"])


def _problems():
    return [(lambda ps: (ps[0] ** 2).sum(), lambda: [torch.ones(4)])]


def test_seeded_imitation_draws():
    """With if_mt each run is an imitation run when the seeded generator's draw is below mt_ratio (SC/metaopt.py:
    354-360); the teacher labels cover every step of the run."""
    events = []
    sb.train_optimizer(lambda sh, th: _Stub(sh, th, events, iter(())), _problems(), num_problems=1,
                       num_meta_iterations=12, num_unroll_func=lambda: 2, num_partial_unroll_itrs_func=lambda: 3,
                       select_random_problems=False, seed=5, if_mt=True, mt_ratio=0.4, mt_k=2)
    rng = random.Random(5)
    want = ["mt" if rng.random() < 0.4 else "train" for _ in range(12)]
    assert [e[0] for e in events] == want and "mt" in want and "train" in want
    assert all(e == ("mt", 2, (6, 4)) for e in events if e[0] == "mt")
    # off by default: no imitation run and no draw from the generator
    events.clear()
    sb.train_optimizer(lambda sh, th: _Stub(sh, th, events, iter(())), _problems(), 1, 4, lambda: 2, lambda: 3,
                       select_random_problems=False, seed=5, mt_ratio=1.0)
    assert [e[0] for e in events] == ["train"] * 4


def test_curriculum_save_advance_stop_on_scripted_costs(tmp_path):
    """SC/metaopt.py:170-176, 613-690 through train_dm.Curriculum: stage lengths from SCALE_NUM_STEPS, evaluation at
    the next stage's length, "-idx" / "-0" checkpoints on a new best, restore + advance + re-evaluation after
    min_num_eval evaluations with an improvement, stop after min_num_eval without one."""
    events = []
    costs = iter([5.0, 4.0, 4.5,     # save, save, advance (0 -> 1) ...
                  3.9,               # ... the re-evaluation at stage 1
                  4.2, 4.1, 4.0,     # no improvement over 3.9 in three evaluations: stop
                  ])
    save = str(tmp_path / "model.ckpt")
    theta, log = sb.train_optimizer(lambda sh, th: _Stub(sh, th, events, costs), _problems(), num_problems=1,
                                    num_meta_iterations=20, num_unroll_func=lambda: 0,
                                    num_partial_unroll_itrs_func=lambda: 0, select_random_problems=False,
                                    if_cl=True, evaluation_period=1, evaluation_epochs=1, fix_unroll_length=20,
                                    save_path=save)
    assert sb.SCALE_NUM_STEPS == [100, 200, 500, 1000, 1500, 2000, 2500, 3000, 3500, 4000, 4500, 5000]
    assert events == [("train", 5, 20), ("eval", 10),
                      ("train", 5, 20), ("eval", 10),
                      ("train", 5, 20), ("eval", 10), ("restore", 2.0), ("eval", 25),
                      ("train", 10, 20), ("eval", 25),
                      ("train", 10, 20), ("eval", 25),
                      ("train", 10, 20), ("eval", 25)]
    assert len(log) == 6 and float(theta[0]) == 5.0          # six runs, one undone by the restore
    assert float(torch.load(save + "-0")["theta"][0]) == 2.0  # the best: stage 0's second run
    assert sorted(p.name for p in tmp_path.iterdir()) == ["model.ckpt-0"]


def test_evaluation_without_curriculum_saves_the_best_as_zero(tmp_path):
    events = []
    costs = iter([3.0, 2.0, 2.5, 1.0])
    save = str(tmp_path / "m")
    sb.train_optimizer(lambda sh, th: _Stub(sh, th, events, costs), _problems(), 1, 8, lambda: 1, lambda: 20,
                       select_random_problems=False, evaluation_period=2, evaluation_epochs=1, fix_unroll_length=20,
                       fix_num_steps_eval=60, save_path=save)
    assert [e for e in events if e[0] == "eval"] == [("eval", 3)] * 4
    assert float(torch.load(save + "-0")["theta"][0]) == 8.0    # the last (best) evaluation, after eight runs


def test_curriculum_walks_every_stage_and_the_last_evaluates_at_its_own_length():
    """min_num_eval = 1 and costs that improve once and then worsen: every stage trains once, saves, advances and
    re-evaluates.  Evaluation runs at the next stage's length; the last stage, which has none, at its own."""
    events = []
    costs = iter([1.0, 100.0, 50.0] * len(sb.SCALE_NUM_STEPS))
    sb.train_optimizer(lambda sh, th: _Stub(sh, th, events, costs), _problems(), 1, 2 * len(sb.SCALE_NUM_STEPS),
                       lambda: 0, lambda: 0, select_random_problems=False, if_cl=True, evaluation_epochs=1,
                       min_num_eval=1)
    nu = [n // 20 for n in sb.SCALE_NUM_STEPS]
    nxt = lambda s: nu[min(s + 1, len(nu) - 1)]
    want = []
    for s in range(len(nu)):
        want += [("train", nu[s], 20), ("eval", nxt(s)), ("train", nu[s], 20), ("eval", nxt(s)),
                 ("restore", float(s + 1)), ("eval", nxt(s + 1))]
    assert events == want
