"""Time the tensor-core BPTT kernel (l2o_unroll_bwd) alone at the flagship shape: L2O-DM LSTM-20x2 on a separable
Rastrigin problem, 1M coordinates, T = 100, checkpoints from one fused forward unroll.  CUDA events around each call.
`--net rnnprop` times RNNProp's two BPTT passes on the same problem instead.

Compare builds by running it once per library, alternating:
    L2O_LIB=/path/to/libl2o_b200.so python scripts/bptt_ab.py
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
    ap.add_argument("--net", default="dm", choices=["dm", "rnnprop"])
    ap.add_argument("--coords", type=int, default=1_000_000)
    ap.add_argument("--unroll", type=int, default=100)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    n, T, dev = args.coords, args.unroll, "cuda:0"
    gen = torch.Generator().manual_seed(0)
    rnnprop = args.net == "rnnprop"
    if rnnprop:
        spec = orc.NetSpec(layers=(20, 20), preprocess_name="fc", preprocess_options={"dim": 20}, scale=0.01,
                           tanh_output=True, rnnprop=True)
    else:
        spec = orc.NetSpec(layers=(20, 20))
    theta = orc.init_theta(spec, seed=0, out_gain=0.1).to(dev)
    a, b, x0 = (torch.randn(n, generator=gen).to(dev) for _ in range(3))
    h = NetHandle(layers=spec.layers, preprocess_name=spec.preprocess_name, preprocess_options=spec.preprocess_options,
                  scale=spec.scale, tanh_output=spec.tanh_output, n_in=spec.n_in)
    h.set_engine(ENGINE_TC)
    ckpt = torch.zeros((T + 1) * h.state_floats * n, device=dev)
    g_rec = torch.empty(T + 1, n, device=dev)
    in_seq, fwd, bwd = g_rec, {}, {}
    if rnnprop:
        in_seq = torch.empty(T, 2, n, device=dev)
        dseq = torch.empty(T, n, device=dev)
        fwd = dict(m=torch.zeros(n, device=dev), v=torch.zeros(n, device=dev), feat_rec=in_seq, delta_seq=dseq)
        bwd = dict(delta_seq=dseq, scratch=torch.empty(T, n, 20, device=dev))
    h.unroll_fwd(theta, n, T, h.new_state(n, dev), opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=a, opt_b=b,
                 opt_alpha=10.0, opt_fscale=1.0 / n, x=x0.clone(), ckpt=ckpt, g_rec=g_rec, **fwd)
    dtheta = torch.zeros(h.n_theta, dtype=torch.float64, device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for r in range(args.warmup + args.reps):
        dtheta.zero_()
        e0.record()
        h.unroll_bwd(theta, n, T, in_seq, ckpt, dtheta, g_rec=g_rec, **bwd)
        e1.record()
        torch.cuda.synchronize()
        if r >= args.warmup:
            ms.append(e0.elapsed_time(e1))
    print(json.dumps({"lib": _lib.LIB_PATH, "card": card(), "net": args.net, "coords": n, "unroll": T,
                      "bwd_ms_median": statistics.median(ms), "bwd_ms_min": min(ms), "bwd_ms": ms,
                      "dtheta_abs_sum": float(dtheta.abs().sum())}))


if __name__ == "__main__":
    main()
