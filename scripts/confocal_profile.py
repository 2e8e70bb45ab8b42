"""confocal_microscopy_3d at the registry shape (B = 32, P = 5, ROI 28^3, LSTM-20x2, T = 20): the l2o_confocal_grad
producer against torch autograd of the same loss.

    python scripts/confocal_profile.py --out results/confocal.json [--rounds 5] [--launches 100] [--unrolls 5]

(a) f and df/dx of one step: the kernel alone, and the autograd path MetaOptimizer runs with L2O_DISABLE_FUSED=1
    (product loss, autograd.grad, copies into the flat gradient), each timed with CUDA events over --launches calls,
    alternated over --rounds rounds.  Also the max relative difference of the two gradients.
(b) ms per T = 20 training unroll (fx + update + step, synchronised), producer path against L2O_DISABLE_FUSED=1, each
    program past its two eager warm-up unrolls and CUDA-graph capture, --unrolls timed unrolls per round, alternated.
The card's name and power limit are read in the same run."""
import argparse
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from open_l2o_b200 import engine, meta, util  # noqa: E402
from scripts.measure import alternate, card, emit, event_ms, wall_ms  # noqa: E402


def program(fused, T):
    os.environ["L2O_DISABLE_FUSED"] = "0" if fused else "1"
    problem, net_config, net_assignments = util.get_config("confocal_microscopy_3d")
    opt = meta.MetaOptimizer(**net_config)
    ms = opt.meta_minimize(problem, T, learning_rate=0.001, net_assignments=net_assignments)
    prog = opt.program
    assert (prog.producer is not None) == fused
    sess = meta.Session()
    sess.run(ms.reset)
    return prog, sess, ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--unrolls", type=int, default=5)
    args = ap.parse_args()
    T = 20
    pf, sf, mf = program(True, T)
    pa, sa, ma = program(False, T)
    assert torch.equal(pf.X, pa.X)

    # (a) one step's f and df/dx
    p = pf.producer
    B, P, roi = p.sim.shape[1], p.num_points, p.roi
    g = torch.empty_like(pf.X)
    fx = torch.zeros((), dtype=torch.float64, device=pf.X.device)
    kernel = lambda: engine.confocal_grad(pf.X, p.sim, g, B, P, roi, f=fx)   # noqa: E731
    autograd = lambda: pa._value_and_grad(pa.X)   # noqa: E731
    f_k, g_k = pf._value_and_grad(pf.X)
    f_a, g_a = autograd()
    agree = {"f_rel": abs(float(f_k) - float(f_a)) / abs(float(f_a)),
             "g_rel_maxnorm": float((g_k - g_a).abs().max() / g_a.abs().max())}
    step = alternate({"kernel_ms": kernel, "autograd_ms": autograd}, args.rounds,
                     lambda fn: event_ms(fn, args.launches, 1))

    # (b) training unrolls
    def unroll(sess, ms):
        return wall_ms(lambda: sess.run([ms.fx, ms.update, ms.step]))

    for _ in range(3):   # two eager unrolls, then the capture of each program's graph
        unroll(sf, mf)
        unroll(sa, ma)
    train = alternate({"producer_unroll_ms": lambda: unroll(sf, mf), "autograd_unroll_ms": lambda: unroll(sa, ma)},
                      args.rounds, lambda fn: statistics.median(fn() for _ in range(args.unrolls)))

    med = {k: statistics.median(v) for k, v in list(step.items()) + list(train.items())}
    res = {"card": card(), "shape": {"batch": B, "num_points": P, "roi": list(roi), "T": T},
           "launches_per_round": args.launches, "unrolls_per_round": args.unrolls, "gradient_agreement": agree,
           "step": step, "train_unroll": train, "median": med,
           "speedup": {"step": med["autograd_ms"] / med["kernel_ms"],
                       "train_unroll": med["autograd_unroll_ms"] / med["producer_unroll_ms"]}}
    emit(res, args.out)


if __name__ == "__main__":
    main()
