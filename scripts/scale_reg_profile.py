"""Times L2O-Scale meta-training with the regularisers (``--reg_optimizer``) on the GPU.

  * one HierarchicalRNN meta-step (a 20-step unroll, the meta-gradient and the RMSProp meta-step, first order) on
    every problem of ``optimization_test_problems``, ``quadratic_problems`` and ``quadratic_problems_large``, per
    ``reg_option``, with the kernel objective (``training_objective``: Hutchinson on a bare family is one
    ``l2o_zoo_hess_form`` launch; the other options reach the zoo kernels through autograd) against the same
    regulariser on the eager ``torch_objective``;
  * ``l2o_zoo_hess_form`` at n = 2048 (a Quadratic and a Norm, cluster of 8), k = 10, against ten ``l2o_zoo_hvp``
    calls.
Each number is the median over alternated repetitions of CUDA-event times (a meta-step ends in host reads, so its
time is wall time up to a device synchronise).  Writes ``scale_reg_profile_h100.json`` beside this script (or
``--out``), with the GPU's name and power limit read in the same run.

    python scripts/scale_reg_profile.py [--reps 5] [--out path]
"""
import argparse
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from open_l2o_b200 import hrnn_train as ht  # noqa: E402
from open_l2o_b200 import scale_zoo as Z  # noqa: E402
from scripts.measure import alternate, card, emit, event_ms  # noqa: E402

DEV = "cuda"
OPTIONS = ("hessian", "jacob", "hessian-ev", "hessian-esd")


def meta_step(problem, objective, option):
    params = problem.init_tensors(0, DEV)
    tr = ht.MetaTrainer([tuple(p.shape) for p in params], theta=ht._init_theta(0), device=DEV, random_seed=0,
                        reg_optimizer=True, reg_option=option, regularize_time="all")
    llr = torch.full((sum(p.numel() for p in params),), -4.0)

    def run():
        tr.train_step(objective, params, 20, log_learning_rate=llr)
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                  "scale_reg_profile_h100.json"))
    a = ap.parse_args()
    res = {"gpu": card(), "reps": a.reps, "meta_step_ms": {}, "hess_form_ms": {}}
    sets = {"optimization_test": Z.optimization_test_problems(), "quadratic": Z.quadratic_problems(),
            "large_quadratic": Z.quadratic_problems_large()}
    for set_name, entries in sets.items():
        for spec, _, _ in entries:
            problem = spec.build()
            name = "%s/%s%s" % (set_name, spec.callable.__name__, tuple(spec.args))
            for option in OPTIONS:
                t = alternate({"kernel": meta_step(problem, Z.training_objective(problem), option),
                               "torch_eager": meta_step(problem, lambda ps, p=problem: p.torch_objective(ps), option)},
                              a.reps, lambda fn: event_ms(fn, 1, 0), warmup=1)
                t = {k: statistics.median(v) for k, v in t.items()}
                res["meta_step_ms"]["%s/%s" % (name, option)] = t
                print(name, option, t, flush=True)
    for problem in (Z.Quadratic(2048, random_seed=0), Z.Norm(2048, random_seed=0, norm_power=3.)):
        x = problem.init_tensors(0, DEV)[0].reshape(-1).contiguous()
        z = problem.kernel(x)
        P = (torch.randint(0, 2, (10, 2048), generator=torch.Generator().manual_seed(0)).float() * 2 - 1).to(DEV)
        rows = list(P)

        def ten_hvp():
            for p in rows:
                z.hvp(x, p)
        t = alternate({"hess_form_k10": lambda: z.hess_form(x, P), "hvp_x10": ten_hvp}, max(a.reps, 10),
                      lambda fn: event_ms(fn, 20, 0), warmup=2)
        t = {k: statistics.median(v) for k, v in t.items()}
        res["hess_form_ms"][type(problem).__name__ + "(2048)"] = t
        print(type(problem).__name__, t, flush=True)
    emit(res, a.out)


if __name__ == "__main__":
    main()
