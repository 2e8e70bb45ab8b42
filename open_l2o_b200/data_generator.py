"""Imitation-learning data (DM/data_generator.py:35-124): roll a hand-designed optimizer (Adam / RMSProp / Nesterov
momentum, TF-1.14 update rules, lr 0.01: ``teacher_update``, which L2O-Scale's ``scale_base.teacher_labels`` shares) on
the optimizee and record, per unroll, the flattened gradients
``inputs [T, N]`` and the parameter moves ``labels [T, N]`` for every net subset."""
from __future__ import annotations

import numpy as np
import torch

TEACHERS = ("adam", "rmsprop", "nag")


def teacher_state(x: torch.Tensor) -> dict:
    """Fresh slots of a teacher for the coordinates ``x``."""
    return dict(m=torch.zeros_like(x), v=torch.zeros_like(x), k=0)


def teacher_update(name: str, x: torch.Tensor, g: torch.Tensor, st: dict, lr: float = 0.01):
    """One step of a hand-designed teacher with the TF-1.14 update rules, on ``x`` and the slots ``st`` in place.
    The imitation data of L2O-DM (``data_loader.get_data``) and of L2O-Scale (``scale_base.teacher_labels``) both
    come from here."""
    if name == "adam":            # tf.train.AdamOptimizer(0.01)
        st["k"] += 1
        st["m"].mul_(0.9).add_(g, alpha=0.1)
        st["v"].mul_(0.999).addcmul_(g, g, value=0.001)
        lr_t = lr * np.sqrt(1 - 0.999 ** st["k"]) / (1 - 0.9 ** st["k"])
        x.sub_(lr_t * st["m"] / (st["v"].sqrt() + 1e-8))
    elif name == "rmsprop":       # tf.train.RMSPropOptimizer(0.01): decay 0.9, eps 1e-10, ms initialised to 1
        if st["k"] == 0:
            st["v"].fill_(1.0)
        st["k"] += 1
        st["v"].mul_(0.9).addcmul_(g, g, value=0.1)
        x.sub_(lr * g / (st["v"] + 1e-10).sqrt())
    elif name == "nag":           # tf.train.MomentumOptimizer(0.01, 0.9, use_nesterov=True)
        st["m"].mul_(0.9).add_(g)
        x.sub_(lr * (g + 0.9 * st["m"]))
    else:
        raise ValueError("unknown teacher %r (one of %s)" % (name, ", ".join(TEACHERS)))


class data_loader(object):
    def __init__(self, *args):
        """``data_loader(problem, var_x, constants, subsets, scale, optimizers, unroll_len)`` as the reference
        (DM/data_generator.py:35-48; the program is reached through the ``var_x`` handles ``meta_minimize`` returned),
        or the short form ``data_loader(program, optimizers, unroll_len)``."""
        if len(args) == 7:
            _problem, var_x, _constants, _subsets, _scale, optimizers, unroll_len = args
            program = var_x[0]._prog
        elif len(args) == 3:
            program, optimizers, unroll_len = args
        else:
            raise TypeError("data_loader(problem, var_x, constants, subsets, scale, optimizers, unroll_len)")
        self.prog = program
        self.optimizers = optimizers.split(",") if isinstance(optimizers, str) else list(optimizers)
        self.unroll_len = unroll_len
        self.num_subsets = len(program.subsets)

    def _subset_slices(self):
        out = []
        for key in self.prog.net_keys:
            r = [r for r in self.prog.runs if r.key == key][0]
            out.append(slice(r.off, r.off + r.n))
        return out

    def get_data(self, task_i, sess=None, num_unrolls=1, assign_func=None, rd_scale_bound=3.0, if_scale=True, mt_k=1):
        prog = self.prog
        name = self.optimizers[task_i]
        prog.reset_x()                                            # sess.run(self.reset_x): x + constants only
        feed = {}
        if if_scale:
            r_scale = [np.exp(np.random.uniform(-rd_scale_bound, rd_scale_bound, size=v["shape"])).astype(np.float32)
                       for v in prog.variables]
            feed = {p: v for p, v in zip(prog.scale_placeholders, r_scale)}
            prog.assign_x([xv / rs for xv, rs in zip(prog.x_values(), r_scale)])
        prog._apply_scale_feed(feed)
        X = prog.X
        st = teacher_state(X)

        def update(g):
            teacher_update(name, X, g, st)

        sl = self._subset_slices()
        data = {"inputs": [], "labels": []}
        x_prev = X.clone()
        for _ in range(num_unrolls):
            inputs, labels = [], []
            for _s in range(self.unroll_len):
                _, g = prog._value_and_grad(X)
                inputs.append(g.clone())
                update(g)
                for _k in range(mt_k - 1):
                    update(prog._value_and_grad(X)[1])
                labels.append(X - x_prev)
                x_prev = X.clone()
            gi, li = torch.stack(inputs), torch.stack(labels)
            data["inputs"].append([gi[:, s].cpu().numpy() for s in sl])
            data["labels"].append([li[:, s].cpu().numpy() for s in sl])
        return data
