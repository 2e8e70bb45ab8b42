"""Time one tensor-core unroll kernel alone at the flagship shape: L2O-DM LSTM-20x2 on a separable Rastrigin problem,
1M coordinates, T = 100.  CUDA events around each call.
  --kernel fwd: the forward unroll (l2o_unroll_fwd) in two modes:
      train: checkpoints, g_rec and fx recorded, as the fused meta-training forward runs;
      infer: fx only, no checkpoints (the forward of evaluate_dm.py).
  --kernel bwd: the BPTT (l2o_unroll_bwd) on the checkpoints of one fused forward unroll.  `--net rnnprop` times
      RNNProp's two BPTT passes on the same problem instead.

Compare builds by running it once per library, alternating:
    L2O_LIB=/path/to/libl2o_b200.so python scripts/tc_ab.py --kernel fwd
Prints one JSON line: the library, the card's name and power limit, the per-call times and checksums of the outputs."""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from open_l2o_b200 import _lib  # noqa: E402
from open_l2o_b200.engine import ENGINE_TC, OPT_KINDS, NetHandle  # noqa: E402
from oracle import l2o_oracle as orc  # noqa: E402  (theta initialisation only)
from scripts.measure import card, emit, event_ms  # noqa: E402


def net_spec(kernel, net):
    if net == "rnnprop":
        return orc.NetSpec(layers=(20, 20), preprocess_name="fc", preprocess_options={"dim": 20}, scale=0.01,
                           tanh_output=True, rnnprop=True)
    # The forward has always been timed at the registry's output scale and the BPTT at 1.0; keeping them keeps the
    # checksums comparable with earlier records.
    return orc.NetSpec(layers=(20, 20), scale=0.1 if kernel == "fwd" else 1.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kernel", required=True, choices=["fwd", "bwd"])
    ap.add_argument("--net", default="dm", choices=["dm", "rnnprop"], help="the network of --kernel bwd")
    ap.add_argument("--coords", type=int, default=1_000_000)
    ap.add_argument("--unroll", type=int, default=100)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if args.kernel == "fwd" and args.net != "dm":
        ap.error("--net applies to --kernel bwd only")
    n, T, dev = args.coords, args.unroll, "cuda:0"
    gen = torch.Generator().manual_seed(0)
    spec = net_spec(args.kernel, args.net)
    theta = orc.init_theta(spec, seed=0, out_gain=0.1).to(dev)
    a, b, x0 = (torch.randn(n, generator=gen).to(dev) for _ in range(3))
    problem = dict(opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=a, opt_b=b, opt_alpha=10.0, opt_fscale=1.0 / n)
    h = NetHandle(layers=spec.layers, preprocess_name=spec.preprocess_name, preprocess_options=spec.preprocess_options,
                  scale=spec.scale, tanh_output=spec.tanh_output, n_in=spec.n_in)
    h.set_engine(ENGINE_TC)
    ckpt = torch.zeros((T + 1) * h.state_floats * n, device=dev)
    g_rec = torch.empty(T + 1, n, device=dev)
    out = {"lib": _lib.LIB_PATH, "card": card()}
    if args.kernel == "bwd":
        out["net"] = args.net
    out.update(coords=n, unroll=T)

    if args.kernel == "fwd":
        state0 = h.new_state(n, dev)
        fx = torch.zeros(T + 1, dtype=torch.float64, device=dev)
        for mode, rec in (("train", dict(ckpt=ckpt, g_rec=g_rec)), ("infer", {})):
            ms = []
            for _ in range(args.warmup + args.reps):
                x, state = x0.clone(), state0.clone()
                fx.zero_()
                ms.append(event_ms(lambda: h.unroll_fwd(theta, n, T, state, x=x, fx=fx, **problem, **rec), 1, 0))
            ms = ms[args.warmup:]
            out[mode] = {"fwd_ms_median": statistics.median(ms), "fwd_ms_min": min(ms), "fwd_ms": ms,
                         "fx_T": float(fx[T]), "x_abs_sum": float(x.double().abs().sum())}
    else:
        in_seq, fwd, bwd = g_rec, {}, {}
        if args.net == "rnnprop":
            in_seq = torch.empty(T, 2, n, device=dev)
            dseq = torch.empty(T, n, device=dev)
            fwd = dict(m=torch.zeros(n, device=dev), v=torch.zeros(n, device=dev), feat_rec=in_seq, delta_seq=dseq)
            bwd = dict(delta_seq=dseq, scratch=torch.empty(T, n, 20, device=dev))
        h.unroll_fwd(theta, n, T, h.new_state(n, dev), x=x0.clone(), ckpt=ckpt, g_rec=g_rec, **problem, **fwd)
        dtheta = torch.zeros(h.n_theta, dtype=torch.float64, device=dev)
        ms = []
        for _ in range(args.warmup + args.reps):
            dtheta.zero_()
            ms.append(event_ms(lambda: h.unroll_bwd(theta, n, T, in_seq, ckpt, dtheta, g_rec=g_rec, **bwd), 1, 0))
        ms = ms[args.warmup:]
        out.update(bwd_ms_median=statistics.median(ms), bwd_ms_min=min(ms), bwd_ms=ms,
                   dtheta_abs_sum=float(dtheta.abs().sum()))
    emit(out)


if __name__ == "__main__":
    main()
