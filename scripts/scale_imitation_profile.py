"""One imitation meta-step of the HierarchicalRNN against one first-order meta-step, on the BASELINE config #4
optimizee (scale_problems.ConvNet((3, 32, 32), 10, [(3, 3, 32), (5, 5, 32)]), 354,218 coordinates, batch 128), T = 20.

    python scripts/scale_imitation_profile.py --out results/scale_imitation.json [--rounds 5] [--steps 3]

Each meta-step is the meta-gradient of one unroll and the clipped RMSProp step, timed with a host clock between two
device synchronisations; the two kinds alternate over --rounds rounds of --steps meta-steps each.  Also timed: the
Adam teacher's labels for the unroll (teacher_labels, k = 1), and, with CUDA events, the three elementwise passes over
N that an imitation step adds (upd - label, its square-sum, x - label) for all T steps.  Before timing, the replayed
imitation meta-gradient is compared with one that re-evaluates the objective at the teacher-forced points.  The
card's name and power limit are read in the same run."""
import argparse
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from open_l2o_b200 import hrnn_train as ht  # noqa: E402
from open_l2o_b200.scale_base import teacher_labels  # noqa: E402
from open_l2o_b200.scale_problems import ConvNet  # noqa: E402
from scripts.measure import alternate, card, emit, event_ms, wall_ms  # noqa: E402

DEV = "cuda:0"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    T = 20
    prob = ConvNet((3, 32, 32), 10, [(3, 3, 32), (5, 5, 32)])
    params0 = [p.detach() for p in prob.init_tensors(seed=0, device=DEV)]
    gen = torch.Generator().manual_seed(0)
    data = torch.randn(128, 32, 32, 3, generator=gen).to(DEV)
    onehot = torch.nn.functional.one_hot(torch.randint(0, 10, (128,), generator=gen), 10).float().to(DEV)
    obj = lambda ps: prob.objective(ps, data, onehot)   # noqa: E731
    tr = ht.MetaTrainer(prob.param_shapes, device=DEV, random_seed=0)
    N = sum(p.numel() for p in params0)
    llr = (torch.rand(N, generator=gen, dtype=torch.float64) * 3.0 - 6.0).float()
    x0 = torch.cat([p.reshape(-1) for p in params0])
    labels, grads = teacher_labels(obj, x0, prob.param_shapes, [T])

    m_rep, g_rep, _, _ = tr.meta_gradient_mt(None, params0, labels, grads, llr)
    m_eval, g_eval, _, _ = tr.meta_gradient_mt(obj, params0, labels, None, llr)
    agree = {"meta_rel": abs(float(m_rep) - float(m_eval)) / abs(float(m_eval)),
             "grad_rel_maxnorm": float((g_rep - g_eval).abs().max() / g_eval.abs().max())}

    def first_order():
        _, g, _, _ = tr.meta_gradient(obj, params0, T, llr)
        tr.apply_meta_gradient(g)

    def imitation():
        _, g, _, _ = tr.meta_gradient_mt(None, params0, labels, grads, llr)
        tr.apply_meta_gradient(g)

    def teacher():
        teacher_labels(obj, x0, prob.param_shapes, [T])

    upd = torch.randn(N, device=DEV)

    def passes():
        x = x0
        for t in range(T):
            d = upd - labels[t]
            (d * d).sum()
            x = x - labels[t]

    for fn in (first_order, imitation, teacher, passes):   # warm-up of every shape
        fn()
    times = alternate({"first_order_ms": first_order, "imitation_ms": imitation, "teacher_labels_ms": teacher},
                      args.rounds,
                      lambda fn: statistics.median(wall_ms(fn) for _ in range(1 if fn is teacher else args.steps)))
    med = {k: statistics.median(v) for k, v in times.items()}
    med["mt_passes_ms_per_unroll"] = event_ms(passes, 10, 0)
    res = {"card": card(), "shape": {"coordinates": N, "tensors": len(params0), "T": T, "batch": 128},
           "replay_vs_reevaluation": agree, "rounds": times, "median": med,
           "imitation_over_first_order": med["imitation_ms"] / med["first_order_ms"]}
    emit(res, args.out)


if __name__ == "__main__":
    main()
