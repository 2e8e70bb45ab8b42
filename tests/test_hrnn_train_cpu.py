"""Host-side pieces of the HierarchicalRNN meta-training path that run without a GPU: the theta layout and the small
torch-level cells must agree with the oracle's (SC/optimizer/rnn_cells.py:46-68, trainable_optimizer.py:586-609)."""
import math

import pytest
import torch

from oracle import hrnn_oracle as orc   # checker only


def test_theta_views_match_oracle_layout():
    from open_l2o_b200.hierarchical_rnn import THETA_SPEC
    from open_l2o_b200.scale_base import theta_views
    theta = orc.init_theta(seed=2)
    mine, ref = theta_views(theta, THETA_SPEC), orc.unpack_theta(theta)
    assert list(mine) == list(ref)
    for k in ref:
        assert mine[k].shape == ref[k].shape and torch.equal(mine[k], ref[k]), k
    assert sum(v.numel() for v in mine.values()) == orc.theta_count()


def test_bias_gru_cell_matches_oracle_and_is_differentiable():
    from open_l2o_b200 import hrnn_train as ht
    g = torch.Generator().manual_seed(0)
    ni, nh, rows = 22, 20, 5
    x, h = torch.randn(rows, ni, generator=g, dtype=torch.float64), torch.randn(rows, nh, generator=g, dtype=torch.float64)
    Wg, bg = torch.randn(ni + nh, 2 * nh, generator=g, dtype=torch.float64), torch.randn(2 * nh, generator=g, dtype=torch.float64)
    Wc, bc = torch.randn(ni + nh, nh, generator=g, dtype=torch.float64), torch.randn(nh, generator=g, dtype=torch.float64)
    bias = torch.randn(rows, 3 * nh, generator=g, dtype=torch.float64)
    Wg.requires_grad_(True)
    a = ht._bias_gru(x, h, Wg, bg, Wc, bc, bias)
    b = orc._bias_gru(x, h, Wg, bg, Wc, bc, bias)
    assert torch.allclose(a, b, rtol=0, atol=1e-15)
    (ga,) = torch.autograd.grad(a.sum(), Wg, retain_graph=True)
    (gb,) = torch.autograd.grad(b.sum(), Wg)
    assert torch.allclose(ga, gb, rtol=0, atol=1e-14)


def test_meta_trainer_refuses_to_run_without_cuda():
    from open_l2o_b200 import hrnn_train as ht
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is present")
    with pytest.raises(Exception):
        ht.MetaTrainer([(3, 2), (2,)])


def test_scale_objective_forms():
    from open_l2o_b200 import hrnn_train as ht
    tr = ht.MetaTrainer.__new__(ht.MetaTrainer)     # the formula only: no engine behind it
    objs, f0 = torch.tensor([4.0, 2.0, 1.0], dtype=torch.float64), torch.tensor(4.0, dtype=torch.float64)
    tr.use_log_objective, tr.use_numerator_epsilon = True, False
    want = sum(math.log(v / (4.0 + 1e-6) + 1e-6) for v in (4.0, 2.0, 1.0)) / 3
    assert abs(float(tr.scale_objective(objs.sum(), objs, f0)) - want) < 1e-12
    tr.use_numerator_epsilon = True
    want = sum(math.log((v + 1e-6) / (4.0 + 1e-6)) for v in (4.0, 2.0, 1.0)) / 3
    assert abs(float(tr.scale_objective(objs.sum(), objs, f0)) - want) < 1e-12
    tr.use_log_objective = False
    assert abs(float(tr.scale_objective(objs.sum(), objs, f0)) - 7.0 / (4.0 + 1e-6)) < 1e-12


def test_train_optimizer_sampling_loop_with_a_stub_trainer():
    """metaopt.train_optimizer's loop structure (SC/metaopt.py:117-613) on a stub trainer: problem draws, one trainer per
    optimizee shape, theta handed on between problems, unroll counts from the two callables or the fixed schedule."""
    from open_l2o_b200 import hrnn_train as ht
    calls = []

    class Stub(object):
        device = "cpu"

        def __init__(self, shapes, theta):
            self.shapes = shapes
            self.theta = torch.zeros(4) if theta is None else theta.clone()

        def train_problem(self, objective, params, num_unrolls, unroll_len):
            calls.append((self.shapes, num_unrolls, unroll_len))
            with torch.no_grad():
                self.theta += 1.0
            return [0.0] * num_unrolls, [], params

    problems = [(lambda ps: ps[0].sum(), lambda: [torch.zeros(3, 2)]), (lambda ps: ps[0].sum(), lambda: [torch.zeros(5)])]
    theta, log = ht.train_optimizer(lambda sh, th: Stub(sh, th), problems, num_problems=4, num_meta_iterations=2,
                                    num_unroll_func=lambda: 3, num_partial_unroll_itrs_func=lambda: 7,
                                    select_random_problems=False)
    assert [c[0] for c in calls] == [((3, 2),)] * 2 + [((5,),)] * 2 + [((3, 2),)] * 2 + [((5,),)] * 2
    assert all(c[1:] == (3, 7) for c in calls)
    assert float(theta[0]) == 8.0                      # every run moved the shared theta once, across both trainers
    assert [k for k, _ in log] == [0, 0, 1, 1, 0, 0, 1, 1] and all(len(m) == 3 for _, m in log)
    calls.clear()
    ht.train_optimizer(lambda sh, th: Stub(sh, th), problems[:1], 1, 1, lambda: 0, lambda: 0, fix_unroll=True,
                       fix_unroll_length=20, fix_num_steps=100)
    assert calls == [(((3, 2),), 5, 20)]


def test_train_problem_stopping_rules_on_a_stubbed_unroll():
    """train_problem's control flow without a GPU: carried state, series-wide initial objective, and the two early exits
    of the reference's loop_cond (non-finite objective; objective above obj_train_max_multiplier x initial)."""
    from open_l2o_b200 import hrnn_train as ht
    tr = ht.MetaTrainer.__new__(ht.MetaTrainer)
    tr.device, tr.shapes, tr.sizes = "cpu", [(2,)], [2]
    seen, applied = [], []
    script = iter([[4.0, 3.0], [2.5, 2.0], [30.0, 40.0], [1.0, 1.0]])

    def fake_meta_gradient(objective, params, num_steps, log_learning_rate=None, state=None, initial_obj=None):
        seen.append((state, None if initial_obj is None else float(initial_obj)))
        objs = next(script)
        final = ht.OptimizerState(torch.zeros(21, 2), torch.zeros(1, 20), torch.zeros(1, 20), torch.zeros(1, 4), torch.zeros(2))
        return torch.tensor(-0.1), torch.ones(3), objs, final
    tr.meta_gradient = fake_meta_gradient
    tr.apply_meta_gradient = lambda g: applied.append(1)
    metas, values, out = tr.train_problem(lambda ps: ps[0].sum(), [torch.zeros(2)], num_unrolls=4, unroll_len=2,
                                          obj_train_max_multiplier=5.0)
    assert len(metas) == 2 and values == [4.0, 3.0, 2.5, 2.0] and len(applied) == 2     # third unroll: 30 >= 5 x 4 -> stop
    assert seen[0] == (None, None) and seen[1][0] is not None and seen[1][1] == 4.0 and seen[2][1] == 4.0
    script = iter([[4.0, float("nan")]])
    applied.clear()
    metas, values, _ = tr.train_problem(lambda ps: ps[0].sum(), [torch.zeros(2)], num_unrolls=3, unroll_len=2)
    assert metas == [] and values == [] and applied == []
