"""Time the CoordinatewiseRNN kernels on the GPU with CUDA events and report achieved algorithmic bandwidth.

    python scripts/crnn_profile.py [--reps 50] [--out DIR]

Sizes: the forward step (l2o_crnn_step, in place, x updated) at the BASELINE #4 ConvNet shapes (354,218 coordinates)
and at 32 M coordinates; one meta-training inner step (l2o_crnn_step forward + l2o_crnn_bwd backward, as
crnn_train._Step runs them) at the ConvNet shapes, and a T = 20 unroll of those (objective excluded).

Algorithmic bytes per coordinate: forward 836 (103 planes + g + x read, 103 planes + x written); backward 2,064
(old planes, d_state_new, g, d_update read; d_state_old written).  FLOPs per coordinate of the forward: 2 x 6,040 cell
MACs + 60 readout MACs.  Roofline figures are the H100 SXM data sheet's (3.35 TB/s HBM3, 67 TFLOP/s FP32), not measured.
Prints one JSON line; the card name and power limit come from a read-only nvidia-smi query in the same run.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from scripts.measure import card, emit, event_ms  # noqa: E402

FWD_BYTES, BWD_BYTES = 836, 4 * (103 + 103 + 1 + 1 + 103)
FWD_FLOPS = 2 * (11 * 40 + 31 * 80 + 41 * 80 + 60)
HBM, FP32 = 3.35e12, 67e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("crnn_profile.py measures the GPU kernels and needs a CUDA device")
    from open_l2o_b200 import crnn_train as ct
    from open_l2o_b200.coordinatewise_rnn import CoordinatewiseRNN, metarun_args, step_launch
    from open_l2o_b200.scale_problems import ConvNet
    from tests.helpers import HRNN_CONVNET
    dev = "cuda:0"
    res = dict(card=card(), reps=args.reps)
    n_conv = sum(int(torch.tensor(s).prod()) for s in ConvNet(*HRNN_CONVNET).param_shapes)
    gen = torch.Generator(device=dev).manual_seed(0)
    for tag, n in (("convnet", n_conv), ("32M", 32 * 2 ** 20)):
        opt = CoordinatewiseRNN(random_seed=0, **metarun_args())
        x = torch.randn(n, device=dev, generator=gen)
        g = torch.randn(n, device=dev, generator=gen) * 0.1
        opt.apply_gradients([(g, x)])
        ms = event_ms(lambda: step_launch(opt.theta, g, opt.state, opt.state, x=opt.x), args.reps, 5)
        res["fwd_%s" % tag] = dict(n=n, ms=ms, coord_per_s=n / ms * 1e3, achieved_TBps=n * FWD_BYTES / ms / 1e9,
                                   hbm_share=n * FWD_BYTES / ms * 1e3 / HBM,
                                   fp32_share=n * FWD_FLOPS / ms * 1e3 / FP32)
        del opt, x, g
        torch.cuda.empty_cache()
    # meta-training inner step at the ConvNet shapes: forward + backward of one optimizer step
    n = n_conv
    theta = CoordinatewiseRNN(random_seed=0, **metarun_args()).theta
    tr = ct.MetaTrainer([(n,)], theta=theta, device=dev)
    st = tr.initial_state([torch.randn(n, device=dev, generator=gen)], tr.theta.detach())
    planes = st.planes.detach().contiguous()
    g = torch.randn(n, device=dev, generator=gen) * 0.1
    d_new, d_upd = torch.randn_like(planes) * 1e-3, torch.randn(n, device=dev, generator=gen)
    th = tr.theta.detach()

    def fwd():
        new, upd = torch.empty_like(planes), torch.empty_like(g)
        step_launch(th, g, planes, new, update=upd)

    def bwd():
        ctx = type("Ctx", (), {})()
        ctx.saved_tensors = (th, planes, g)
        ctx.needs_input_grad = (True, True, False)
        ct._Step.backward(ctx, d_new, d_upd)
    f_ms, b_ms = event_ms(fwd, args.reps, 5), event_ms(bwd, args.reps, 5)
    res["train_step_convnet"] = dict(n=n, fwd_ms=f_ms, bwd_ms=b_ms, bwd_achieved_TBps=n * BWD_BYTES / b_ms / 1e9)
    # T = 20 unroll + meta-gradient on a quadratic over the ConvNet coordinate count
    tgt = torch.randn(n, device=dev, generator=gen)
    obj = lambda ps: ((ps[0] - tgt) ** 2).mean()
    p0 = [torch.randn(n, device=dev, generator=gen)]
    ms20 = event_ms(lambda: tr.meta_gradient(obj, p0, 20), max(3, args.reps // 10), 1)
    res["meta_gradient_T20_convnet_ms"] = ms20
    emit(res, args.out and os.path.join(args.out, "crnn_profile.json"))


if __name__ == "__main__":
    main()
