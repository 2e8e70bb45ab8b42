"""Times the zoo's analytic objectives on the GPU: the l2o_zoo kernels against the same objectives as torch ops.

For every problem of ``optimization_test_problems`` and ``quadratic_problems``:
  * value-and-gradient (f and df/dx through autograd) and Hessian-vector product (double backward): the kernel path,
    the torch-op restatement eager, and the torch-op restatement captured into a CUDA graph and replayed;
  * one HierarchicalRNN meta-training step (a 20-step unroll, the meta-gradient and the RMSProp meta-step), first and
    second order, with the kernel objective against the eager torch-op objective.  The trainer reads the objective
    values back on the host, so a whole meta-step cannot be graph-captured.
Each number is the median over alternated repetitions (the variants interleaved within each repetition) of CUDA-event
times.  Writes ``scale_zoo_profile_h100.json`` beside this script (or ``--out``), with the GPU's name and power limit.

    python scripts/scale_zoo_profile.py [--reps 15] [--out path]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from open_l2o_b200 import hrnn_train as ht  # noqa: E402
from open_l2o_b200 import scale_zoo as Z  # noqa: E402
from scripts.measure import alternate, card, emit, event_ms, graphed  # noqa: E402

DEV = "cuda"


def objective_calls(problem, x, v, which, hvp):
    obj = getattr(problem, which)
    shape = problem.param_shapes[0]

    def call():
        xg = x.detach().requires_grad_(True)
        f = obj([xg.view(shape)])
        (g,) = torch.autograd.grad(f, xg, create_graph=hvp)
        if hvp:
            (h,) = torch.autograd.grad(g, xg, grad_outputs=v)
            return f, g, h
        return f, g
    return call


def meta_step(problem, which, second, unroll):
    params = problem.init_tensors(11, DEV)
    tr = ht.MetaTrainer([tuple(p.shape) for p in params], theta=ht._init_theta(0), device=DEV,
                        use_second_derivatives=second, learning_rate=0.0)
    obj = getattr(problem, which)
    llr = torch.full((sum(p.numel() for p in params),), -4.0)

    def call():
        _, grad, _, _ = tr.meta_gradient(lambda ps: obj(ps), params, unroll, log_learning_rate=llr)
        tr.apply_meta_gradient(grad)
    return call


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--meta_reps", type=int, default=7)
    ap.add_argument("--unroll", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                  "scale_zoo_profile_h100.json"))
    a = ap.parse_args(argv)
    assert torch.cuda.is_available(), "this profile needs a CUDA device"
    res = {"gpu": card(), "reps": a.reps, "meta_reps": a.meta_reps, "unroll": a.unroll, "sets": {}}
    for set_name, entries in (("optimization_test_problems", Z.optimization_test_problems()),
                              ("quadratic_problems", Z.quadratic_problems())):
        rows = []
        for i, (spec, _, _) in enumerate(entries):
            problem = Z.Spec(spec.callable, spec.args, dict(spec.kwargs, random_seed=i)).build()
            x = problem.init_tensors(i, DEV)[0].reshape(-1).contiguous()
            v = torch.randn_like(x)
            row = {"problem": "%s%s" % (spec.callable.__name__, tuple(spec.args)), "n": x.numel()}
            for hvp in (False, True):
                kern = objective_calls(problem, x, v, "objective", hvp)
                tor = objective_calls(problem, x, v, "torch_objective", hvp)
                t = alternate({"kernel": kern, "torch_eager": tor, "torch_graph": graphed(tor, 3)}, a.reps,
                              lambda fn: event_ms(fn, 20, 0), warmup=3)
                row["hvp_ms" if hvp else "value_grad_ms"] = {k: statistics.median(v) for k, v in t.items()}
            for second in (False, True):
                t = alternate({"kernel": meta_step(problem, "objective", second, a.unroll),
                               "torch_eager": meta_step(problem, "torch_objective", second, a.unroll)},
                              a.meta_reps, lambda fn: event_ms(fn, 1, 0), warmup=3)
                row["meta_step_%s_ms" % ("second" if second else "first")] = {
                    k: statistics.median(v) for k, v in t.items()}
            # the two objectives agree at the timed point
            fk, gk = objective_calls(problem, x, v, "objective", False)()
            ft, gt = objective_calls(problem, x, v, "torch_objective", False)()
            row["max_rel_diff_g"] = float((gk - gt).abs().max() / gt.abs().max().clamp_min(1e-30))
            rows.append(row)
            print(json.dumps(row), flush=True)
        total = {}
        for key in ("value_grad_ms", "hvp_ms", "meta_step_first_ms", "meta_step_second_ms"):
            total[key] = {k: sum(r[key][k] for r in rows) for k in rows[0][key]}
        res["sets"][set_name] = {"problems": rows, "sum_over_problems": total}
        print(json.dumps({set_name: total}), flush=True)
    emit(res, a.out)


if __name__ == "__main__":
    main()
