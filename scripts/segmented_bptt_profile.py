"""Segmented BPTT of MetaOptimizer: time, peak memory and meta-gradient agreement of full checkpoints against segments.

    python scripts/segmented_bptt_profile.py --out results/segmented [--reps 5]

Cases (one JSON file, <out>/segmented_bptt.json, and one summary line per case on stdout):
  (a) Rastrigin 1 M x T = 100, fused regime: full vs forced S = 10, alternated unroll by unroll
  (b) the largest Rastrigin N x T = 100 whose full checkpoints exceed the free device memory: the program plans its
      segments itself; N comes from mem_get_info and the planner's byte counts, and the full path's size is computed
      from the shapes, never allocated
  (c) the target-line MLP (LogAndSign k = 5, scale 0.01, 1263 hidden units = 1.0 M coordinates) x T = 20, external
      regime: full vs S = 5
  (d) RNNProp on the 784-100-10 MLP x T = 20: full vs S = 5
Per case: median ms per training unroll (fx + update + step) over --reps unrolls after two warm-up unrolls, the time
the segmented backward spends recomputing checkpoints and in the carried BPTT (CUDA events),
torch.cuda.max_memory_allocated of each program's unrolls, and the max relative dtheta difference of the two programs
when both start an unroll from the same theta.  The card's name and power limit are read in the same run."""
import argparse
import gc
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from open_l2o_b200 import meta, problems, util  # noqa: E402
from scripts.measure import alternate, card, event_ms, wall_ms  # noqa: E402

DM = {"net": "CoordinateWiseDeepLSTM", "net_options": {"layers": (20, 20), "scale": 0.1}}
RNNPROP = {"net": "RNNprop", "net_options": {"layers": (20, 20), "preprocess_name": "fc",
                                             "preprocess_options": {"dim": 20}, "scale": 0.01, "tanh_output": True}}


class Program:
    """One MetaOptimizer training program and its session."""

    def __init__(self, cls, cfg, problem, T, segment):
        kw = dict(cfg) if segment is None else dict(cfg, _bptt_segment=segment)
        self.opt = cls(**kw)
        self.ops = self.opt.meta_minimize(problem, T, learning_rate=0.001)
        self.prog, self.T = self.opt.program, T
        self.sess = meta.Session()
        self.sess.run(self.ops.reset)
        self.it = 0

    def unroll(self):
        ms = wall_ms(lambda: self.sess.run([self.ops.fx, self.ops.update, self.ops.step],
                                           feed_dict={self.opt.step_placeholder: self.it * self.T + 1}))
        self.it += 1
        return ms

    def split(self, reps):
        """Median ms of the segmented backward alone (run eagerly on the last unroll's records, outside any captured
        graph), and of its checkpoint recomputes, from CUDA events."""
        prog, ev = self.prog, []
        rec = prog._recompute

        def timed_recompute(*a):   # events around each recompute inside the one backward
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            rec(*a)
            e1.record()
            ev.append((e0, e1))
        prog._recompute = timed_recompute
        back, recomp = [], []
        for _ in range(reps):
            ev.clear()
            back.append(event_ms(prog._bptt, 1, 0))
            recomp.append(sum(a.elapsed_time(b) for a, b in ev))
        del prog._recompute
        return dict(ms_backward=med(back), ms_recompute=med(recomp),
                    ms_carried_bptt=med([b - r for b, r in zip(back, recomp)]))

    def peak_bytes(self, reps):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        for _ in range(reps):
            self.unroll()
        return torch.cuda.max_memory_allocated()


def release():
    """Free what deleted programs held (a program and its optimizer reference each other) before the next peak."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def med(xs):
    return statistics.median(xs) if xs else None


def compare(name, cls, cfg, make_problem, T, S, reps):
    """Full vs segmented, alternated; both programs start every measured unroll from the full program's theta."""
    full = Program(cls, cfg, make_problem(), T, None)
    seg = Program(cls, cfg, make_problem(), T, S)
    assert not full.prog.segmented and seg.prog.segmented, name
    ddiff = [0.0]

    def full_unroll():
        for k in full.prog.nets:
            seg.prog.nets[k].theta.copy_(full.prog.nets[k].theta)
            for s in ("m", "v"):
                seg.prog.adam[k][s].copy_(full.prog.adam[k][s])
        return full.unroll()

    def seg_unroll():
        ms = seg.unroll()
        for k in full.prog.nets:
            d = full.prog.dtheta[k]
            ddiff.append(float((seg.prog.dtheta[k] - d).abs().max() / d.abs().max()))
        return ms
    t = alternate({"full": full_unroll, "segmented": seg_unroll}, reps + 2, lambda fn: fn())
    t_full, t_seg = t["full"][2:], t["segmented"][2:]   # past two warm-up unrolls
    out = dict(case=name, T=T, S=S, coords=full.prog.N, unrolls=reps, ms_full=med(t_full), ms_segmented=med(t_seg),
               ms_full_all=t_full, ms_segmented_all=t_seg,
               segments=seg.prog.plan.bounds, plan_bytes_full=full.prog.plan.bytes, plan_bytes_segmented=seg.prog.plan.bytes,
               max_rel_dtheta_diff=max(ddiff), **seg.split(reps))
    del full
    release()
    out["peak_bytes_segmented"] = seg.peak_bytes(2)
    del seg
    release()
    full = Program(cls, cfg, make_problem(), T, None)
    out["peak_bytes_full"] = full.peak_bytes(2)
    del full
    release()
    return out


def largest(T, reps):
    """(b): the largest Rastrigin whose full checkpoints do not fit, trained with the segments the planner picks."""
    release()
    free, total = torch.cuda.mem_get_info()
    S = min(range(1, T + 1), key=lambda s: (-(-T // s) + s, s))
    per = sum(meta.plan_segments(T, 80, 1, S=S, boundary_floats=1).bytes.values())
    # what every program allocates per coordinate besides its checkpoints: state, g_rec, x, its working copy, the
    # scale feed, the optimizee's two constants, the forward's working state
    per += 4 * (80 + (T + 1) + 5 + 80)
    N = int(0.8 * free / per) // 1000 * 1000
    full_bytes = sum(meta.plan_segments(T, 80 * N, N, S=T).bytes.values())
    out = dict(case="b_largest_rastrigin", T=T, coords=N, free_bytes_before=free, total_bytes=total,
               full_checkpoint_bytes_computed=full_bytes, full_fits=full_bytes <= free)
    torch.cuda.reset_peak_memory_stats()
    p = Program(meta.MetaOptimizer, {"cw": DM}, problems.rastrigin_separable(num_dims=N), T, None)
    out.update(segments=p.prog.plan.bounds, S=p.prog.plan.S, plan_bytes=p.prog.plan.bytes)
    times = [p.unroll() for _ in range(reps + 2)][2:]
    out.update(ms_segmented=med(times), ms_segmented_all=times, peak_bytes_segmented=torch.cuda.max_memory_allocated(),
               **p.split(reps))
    del p
    release()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cases", default="a,b,c,d")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    res = dict(card=card(), reps=args.reps, cases=[])
    todo = args.cases.split(",")
    runs = {
        "a": lambda: compare("a_rastrigin_1M_T100_fused", meta.MetaOptimizer, {"cw": DM},
                             lambda: problems.rastrigin_separable(num_dims=1_000_000), 100, 10, args.reps),
        "b": lambda: largest(100, args.reps),
        "c": lambda: compare("c_mlp_target_line_T20_external", meta.MetaOptimizer,
                             {"cw": util.get_default_net_config(None)}, lambda: problems.mlp(layers=(1263,)), 20, 5,
                             args.reps),
        "d": lambda: compare("d_rnnprop_mlp_784_100_10_T20", meta.RNNpropMetaOptimizer, {"rp": RNNPROP},
                             lambda: problems.mlp(layers=(100,)), 20, 5, args.reps),
    }
    for c in todo:
        r = runs[c]()
        res["cases"].append(r)
        print(json.dumps({k: v for k, v in r.items() if not k.endswith("_all") and not k.startswith("plan_bytes")}),
              flush=True)
        with open(os.path.join(args.out, "segmented_bptt.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res["card"]))


if __name__ == "__main__":
    main()
