"""``python -m open_l2o_b200.scale_metarun``: meta-train one of the five L2O-Scale optimizers on the problem zoo, as
SC/metarun.py does (SC/ = Model_Free_L2O/L2O-Scale/L2O-Scale-Training/), with its flag names and defaults.

The ``--include_*_problems`` flags assemble ``problems_and_data`` in metarun's order (``scale_zoo.problems_and_data``);
each entry is built once, its dataset moved to the device, and handed to ``scale_base.train_optimizer`` as an
``(objective, init_fn)`` pair.  Dataset problems see ``batch_size`` rows per objective evaluation, shuffled epoch by
epoch (``Dataset.batch_indices``) from a generator seeded with ``--seed``; gradient noise and dropout come from a device
generator seeded the same way.  The optimizer comes from ``register_optimizers()`` and its ``meta_trainer``, one trainer
per problem shape, the meta-parameters and the RMSProp accumulator handed on from problem to problem.  The same host
loop serves all five optimizers.  TensorFlow's boolean flags are accepted as ``--flag``, ``--noflag`` and
``--flag=true|false``.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

from . import scale_zoo as zoo

# the metarun flags that reach the optimizer / trainer here, with metarun's defaults (SC/metarun.py:34-235, metaopt.py)
_INT = dict(task=0, worker_tasks=1, num_problems=1, num_meta_iterations=5, num_unroll_scale=40, min_num_unrolls=10,
            num_partial_unroll_itr_scale=20, min_num_itr_partial_unroll=10, cell_size=20, num_cells=2,
            fix_unroll_length=20, fix_num_steps=100, fix_num_steps_eval=100, evaluation_period=1,
            evaluation_epochs=20, save_period=1, mt_k=1, seed=0)
_FLOAT = dict(meta_learning_rate=1e-6, gradient_clip_level=1e4, min_lr=1e-6, max_lr=1e-2, max_log_lr=33.0,
              objective_training_max_multiplier=-1.0, l2_reg=0.0, rms_decay=0.9, rms_epsilon=1e-20, mt_ratio=0.1)
_STR = dict(train_dir="opt/", optimizer="HierarchicalRNN", cell_cls="GRUCell", device="cuda")
_BOOL = dict(zero_init_lr_weights=True, use_relative_lr=True, use_extreme_indicator=False, use_log_means_squared=True,
             use_problem_lr_mean=True, learnable_decay=True, dynamic_output_scale=True, use_log_objective=True,
             use_attention=False, use_second_derivatives=True, use_gradient_shortcut=True, use_lr_shortcut=False,
             use_grad_products=True, use_multiple_scale_decays=False, use_numerator_epsilon=False,
             learnable_inp_decay=True, learnable_rnn_init=True, if_cl=False, fix_unroll=False, if_mt=False)
_INT["num_gradient_scales"] = 4
# the regulariser (SC/optimizer/trainable_optimizer.py:34-41, problems/problem_generator.py:33-36, metaopt.py:63-66)
_REG_BOOL = dict(reg_optimizer=False, reg_optimizee=False)
_REG = dict(reg_option="hessian", hessian_itrs=10, alpha=5e-4, beta=1e-4, regularize_time="posterior", reg_scale=0.5)
_INT["hessian_itrs"] = _REG["hessian_itrs"]
_FLOAT.update(alpha=_REG["alpha"], beta=_REG["beta"], reg_scale=_REG["reg_scale"])
_STR.update(reg_option=_REG["reg_option"], regularize_time=_REG["regularize_time"])
_BOOL.update(_REG_BOOL)
# HierarchicalRNN's constructor flags (SC/metarun.py:373-396)
_HRNN_FLAGS = ("learnable_decay", "dynamic_output_scale", "use_attention", "use_log_objective", "num_gradient_scales",
               "zero_init_lr_weights", "use_log_means_squared", "use_relative_lr", "use_extreme_indicator",
               "max_log_lr", "use_problem_lr_mean", "use_gradient_shortcut", "use_lr_shortcut", "use_grad_products",
               "use_multiple_scale_decays", "learnable_inp_decay", "learnable_rnn_init")
HRNN_CELL_SIZES = [10, 20, 20]


def _bool(s):
    v = str(s).lower()
    if v in ("1", "true", "t", "yes"):
        return True
    if v in ("0", "false", "f", "no"):
        return False
    raise argparse.ArgumentTypeError("not a boolean: %r" % (s,))


def parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    for d, typ in ((_INT, int), (_FLOAT, float), (_STR, str)):
        for name, default in d.items():
            ap.add_argument("--" + name, type=typ, default=default)
    bools = dict(_BOOL)
    bools.update({"include_%s_problems" % name: False for name, _ in zoo.INCLUDE_FLAGS})
    for name, default in bools.items():
        ap.add_argument("--" + name, type=_bool, nargs="?", const=True, default=default)
        ap.add_argument("--no" + name, dest=name, action="store_false")
    return ap


def parse(argv=None):
    return parser().parse_args(argv)


def included(flags):
    return [name for name, _ in zoo.INCLUDE_FLAGS if getattr(flags, "include_%s_problems" % name)]


def sample_numiter(rng: np.random.RandomState, scale, min_steps=50):
    """metaopt.sample_numiter: round(Exp(scale)) + min_steps, clipped to [0, 3 min_steps]."""
    return int(np.clip(np.round(rng.exponential(scale=scale)) + min_steps, 0, 3 * min_steps))


class Batches(object):
    """Index batches of ``batch_size`` rows that cover the dataset epoch by epoch (``Dataset.batch_indices``), drawn
    one at a time."""

    def __init__(self, size, batch_size, rng):
        self.size, self.batch_size, self.rng = int(size), int(batch_size), rng
        self.order = np.arange(self.size)
        self.rng.shuffle(self.order)
        self.pos = 0

    def next(self):
        start, self.pos = self.pos, self.pos + self.batch_size
        if self.pos > self.size:
            self.rng.shuffle(self.order)
            start, self.pos = 0, self.batch_size
        return self.order[start:self.pos]


def build_problems(entries, device, seed=0):
    """``(objective, init_fn)`` pairs for ``scale_base.train_optimizer`` from ``(Spec, dataset, batch_size)`` entries,
    and the built problems."""
    rng = np.random.RandomState(seed)
    noise_gen = torch.Generator(device=device)
    noise_gen.manual_seed(int(seed))
    init_seeds = np.random.RandomState(seed + 1)
    out, built = [], []
    for spec, dataset, batch_size in entries:
        problem = spec.build()
        batch = None
        if dataset is not None:
            data = torch.as_tensor(np.asarray(dataset.data)).to(device)
            labels = torch.as_tensor(np.asarray(dataset.labels)).to(device)
            batches = Batches(len(dataset.data), batch_size, rng)

            def batch(data=data, labels=labels, batches=batches):
                idx = torch.as_tensor(batches.next()).to(device)
                return data.index_select(0, idx), labels.index_select(0, idx)

        def init_fn(problem=problem):
            return problem.init_tensors(int(init_seeds.randint(zoo.MAX_SEED)), device)

        out.append((zoo.training_objective(problem, batch, noise_gen), init_fn))
        built.append(problem)
    return out, built


def optimizer_kwargs(flags):
    """The optimizer's constructor arguments (SC/metarun.py:367-398).  metarun hands ``HRNN_CELL_SIZES`` and the
    HierarchicalRNN flags to every optimizer; TrainableAdam, GlobalLearningRate and LearningRateSchedule take neither
    (the cell sizes land on their first argument, a learning rate, and the reference raises), so they get their
    defaults here.  CoordinatewiseRNN takes the sizes as ``cell_sizes`` and ``--cell_cls`` (LSTMCell: the default
    GRUCell raises in the reference and here)."""
    if flags.optimizer not in ("HierarchicalRNN", "CoordinatewiseRNN"):
        return {}
    kw = {name: getattr(flags, name) for name in _HRNN_FLAGS}
    kw.update(init_lr_range=(flags.min_lr, flags.max_lr), random_seed=flags.seed,
              obj_train_max_multiplier=flags.objective_training_max_multiplier)
    if flags.optimizer == "HierarchicalRNN":
        kw.update(level_sizes=list(HRNN_CELL_SIZES))
    else:
        kw.update(cell_sizes=list(HRNN_CELL_SIZES), cell_cls=flags.cell_cls)
    return kw


def run(flags, out=sys.stdout, train_optimizer=None):
    """Meta-train ``flags.optimizer`` on the included problem sets; returns (theta, log) of ``train_optimizer``."""
    from .scale_base import train_optimizer as default_loop
    from .trainable_baselines import register_optimizers
    loop = train_optimizer or default_loop
    if flags.objective_training_max_multiplier > 0:
        raise NotImplementedError("--objective_training_max_multiplier > 0 is not wired into the sampling loop")
    np.random.seed(flags.seed)   # the problems' constants and unseeded datasets draw from numpy's global generator
    entries = zoo.problems_and_data(included(flags))
    if not entries:
        raise ValueError("no problem set included (pass one or more --include_*_problems flags)")
    problems, _ = build_problems(entries, flags.device, flags.seed)
    opt = register_optimizers()[flags.optimizer](device=flags.device, **optimizer_kwargs(flags))
    trainer_kwargs = dict(learning_rate=flags.meta_learning_rate, gradient_clip=flags.gradient_clip_level,
                          l2_reg=flags.l2_reg, rms_decay=flags.rms_decay, rms_epsilon=flags.rms_epsilon,
                          use_log_objective=flags.use_log_objective, use_numerator_epsilon=flags.use_numerator_epsilon,
                          use_second_derivatives=flags.use_second_derivatives, random_seed=flags.seed)
    trainer_kwargs.update({name: getattr(flags, name) for name in list(_REG_BOOL) + list(_REG)})

    def make_trainer(shapes, theta):
        return opt.meta_trainer([torch.empty(s) for s in shapes], **trainer_kwargs)

    numiter = np.random.RandomState(flags.seed + 2)
    logdir = os.path.join(flags.train_dir, "%s_%s_%d_%d" % (flags.optimizer, flags.cell_cls, flags.cell_size,
                                                             flags.num_cells))
    os.makedirs(logdir, exist_ok=True)
    theta, log = loop(
        make_trainer, problems, flags.num_problems, flags.num_meta_iterations,
        lambda: sample_numiter(numiter, flags.num_unroll_scale, flags.min_num_unrolls),
        lambda: sample_numiter(numiter, flags.num_partial_unroll_itr_scale, flags.min_num_itr_partial_unroll),
        select_random_problems=flags.worker_tasks == 1 or flags.task != 0, fix_unroll=flags.fix_unroll,
        fix_unroll_length=flags.fix_unroll_length, fix_num_steps=flags.fix_num_steps, seed=flags.seed, out=out,
        if_mt=flags.if_mt, mt_ratio=flags.mt_ratio, mt_k=flags.mt_k, if_cl=flags.if_cl,
        evaluation_period=flags.evaluation_period, evaluation_epochs=flags.evaluation_epochs,
        fix_num_steps_eval=flags.fix_num_steps_eval, save_path=os.path.join(logdir, "model"))
    return theta, log


def main(argv=None):
    run(parse(argv))
    return 0


if __name__ == "__main__":
    sys.exit(main())
