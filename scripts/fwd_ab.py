"""Time the tensor-core forward unroll (l2o_unroll_fwd) alone at the flagship shape: L2O-DM LSTM-20x2 on a separable
Rastrigin problem, 1M coordinates, T = 100.  Two modes, CUDA events around each call:
  - train: checkpoints, g_rec and fx recorded, as the fused meta-training forward runs;
  - infer: fx only, no checkpoints (the forward of evaluate_dm.py).

Compare builds by running it once per library, alternating:
    L2O_LIB=/path/to/libl2o_b200.so python scripts/fwd_ab.py
Prints one JSON line: the library, the card's name and power limit, and the per-call times."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from open_l2o_b200 import _lib  # noqa: E402
from open_l2o_b200.engine import ENGINE_TC, OPT_KINDS, NetHandle  # noqa: E402
from oracle import l2o_oracle as orc  # noqa: E402  (theta initialisation only)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--coords", type=int, default=1_000_000)
    ap.add_argument("--unroll", type=int, default=100)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    n, T, dev = args.coords, args.unroll, "cuda:0"
    gen = torch.Generator().manual_seed(0)
    spec = orc.NetSpec(layers=(20, 20), scale=0.1)
    theta = orc.init_theta(spec, seed=0, out_gain=0.1).to(dev)
    a, b, x0 = (torch.randn(n, generator=gen).to(dev) for _ in range(3))
    h = NetHandle(layers=spec.layers, scale=spec.scale)
    h.set_engine(ENGINE_TC)
    state0 = h.new_state(n, dev)
    ckpt = torch.zeros((T + 1) * h.state_floats * n, device=dev)
    g_rec = torch.empty(T + 1, n, device=dev)
    fx = torch.zeros(T + 1, dtype=torch.float64, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = {"lib": _lib.LIB_PATH, "card": card(), "coords": n, "unroll": T}
    for mode, rec in (("train", dict(ckpt=ckpt, g_rec=g_rec)), ("infer", {})):
        ms = []
        for r in range(args.warmup + args.reps):
            x, state = x0.clone(), state0.clone()
            fx.zero_()
            e0.record()
            h.unroll_fwd(theta, n, T, state, opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=a, opt_b=b, opt_alpha=10.0,
                         opt_fscale=1.0 / n, x=x, fx=fx, **rec)
            e1.record()
            torch.cuda.synchronize()
            if r >= args.warmup:
                ms.append(e0.elapsed_time(e1))
        out[mode] = {"fwd_ms_median": statistics.median(ms), "fwd_ms_min": min(ms), "fwd_ms": ms,
                     "fx_T": float(fx[T]), "x_abs_sum": float(x.double().abs().sum())}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
