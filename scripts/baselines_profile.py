"""Time L2O-Scale's baseline kernels on the GPU with CUDA events and report achieved algorithmic bandwidth.
(Kernels are timed as CUDA-graph replays of `reps` launches; the meta-gradients as eager calls.)

    python scripts/baselines_profile.py [--reps 50] [--out DIR]

Sizes: the BASELINE #4 ConvNet shapes (354,218 coordinates) and 32 M coordinates.  Per size:
  - l2o_tadam_step in place (x updated), against the same TrainableAdam step written as torch elementwise ops on the
    same GPU, alternated with it in this process; the outputs of both are compared;
  - l2o_tadam_bwd (with d_g), l2o_lrsgd_step in place (x updated), l2o_lrsgd_bwd (with d_g).
And the T = 20 meta-gradient time of each trainer on the ConvNet objective, first and second order.

Algorithmic bytes per coordinate: TrainableAdam step 36 (x g m t v read, x m t v written); its backward 44 (g, 3 old
planes, m and v adjoints, d_update read: 28; 3 plane adjoints and d_g written: 16); schedule step 12 (x g read, x written); its
backward 12 (g, d_update read, d_g written).  The HBM figure is the H100 SXM data sheet's 3.35 TB/s, not a measurement.
Prints one JSON line; the card name and power limit come from a read-only nvidia-smi query in the same run.
"""
import argparse
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from scripts.measure import alternate, card, emit, event_ms, graph_ms  # noqa: E402

TADAM_FWD, TADAM_BWD, LRS_FWD, LRS_BWD = 36, 44, 12, 12
HBM = 3.35e12


def torch_tadam_step(theta, g, st, x):
    """The TrainableAdam step as torch elementwise ops (the scalars as the kernel forms them)."""
    lr, b1, b2 = torch.exp(theta[0]), torch.sigmoid(theta[1]), torch.sigmoid(theta[2])
    eps = torch.exp(theta[3]) + 1e-10
    m, t, v = st[0], st[1], st[2]
    torch.add(t, 1.0, out=t)
    m.mul_(b1).add_((1 - b1) * g)
    v.div_(1 - torch.pow(g * g, b2))
    upd = lr * (m / (1 - torch.pow(b1, t))) / (torch.sqrt(v / (1 - torch.pow(b2, t)) + 1e-10) + eps)
    x.sub_(upd)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("baselines_profile.py measures the GPU kernels and needs a CUDA device")
    from open_l2o_b200 import baselines_train as bt
    from open_l2o_b200.scale_problems import ConvNet
    from open_l2o_b200.engine import _ptr as _p, _stream
    from open_l2o_b200.trainable_baselines import lrsgd_step_launch, tadam_step_launch
    from open_l2o_b200 import _lib
    from tests.helpers import HRNN_CONVNET
    import ctypes as C
    dev = "cuda:0"
    res = dict(card=card(), reps=args.reps)
    net = ConvNet(*HRNN_CONVNET)
    n_conv = sum(int(math.prod(s)) for s in net.param_shapes)
    gen = torch.Generator(device=dev).manual_seed(0)
    theta = torch.tensor([math.log(1e-3), math.log(9.0), math.log(999.0), math.log(1e-8)], device=dev)
    L = _lib.lib()
    for tag, n in (("convnet", n_conv), ("32M", 32 * 2 ** 20)):
        g = torch.randn(n, device=dev, generator=gen) * 0.1
        x0 = torch.randn(n, device=dev, generator=gen)
        # outputs of the kernel and the torch form after three steps from the same state
        xa, sa = x0.clone(), torch.zeros(3, n, device=dev)
        xb, sb = x0.clone(), torch.zeros(3, n, device=dev)
        for _ in range(3):
            tadam_step_launch(theta, g, sa, sa, x=xa)
            torch_tadam_step(theta, g, sb, xb)
        torch.cuda.synchronize()
        rel = lambda a, b: float((a - b).abs().max() / b.abs().max())
        cmp = dict(x=rel(xa, xb), m=rel(sa[0], sb[0]), t=rel(sa[1], sb[1]), v=float((sa[2] - sb[2]).abs().max()))
        kernel_ms = lambda fn: graph_ms(fn, args.reps, 5, 3)   # noqa: E731
        t = alternate({"kernel": lambda: tadam_step_launch(theta, g, sa, sa, x=xa),
                       "torch": lambda: torch_tadam_step(theta, g, sb, xb)}, 5, kernel_ms)
        k_ms, t_ms = statistics.median(t["kernel"]), statistics.median(t["torch"])
        d_new, d_upd = torch.randn(3, n, device=dev, generator=gen), torch.randn(n, device=dev, generator=gen)
        d_old, d_g = torch.empty(3, n, device=dev), torch.empty(n, device=dev)
        d_theta = torch.zeros(4, dtype=torch.float64, device=dev)
        planes = torch.zeros(3, n, device=dev)
        planes[0].normal_(generator=gen)
        ba = _lib.TadamBwdArgs(n=n, theta=_p(theta), g=_p(g), state_old=_p(planes), d_state_new=_p(d_new),
                               d_update=_p(d_upd), d_state_old=_p(d_old), d_theta=d_theta.data_ptr(), d_g=_p(d_g))
        b_ms = kernel_ms(lambda: L.l2o_tadam_bwd(C.byref(ba), _stream()))
        rates, itr = torch.full((1000,), 1e-3, device=dev), torch.zeros(2, dtype=torch.int32, device=dev)
        ls_ms = kernel_ms(lambda: lrsgd_step_launch(rates, g, itr=itr, x=xa))
        d_rates = torch.zeros(1000, dtype=torch.float64, device=dev)
        la = _lib.LrsgdBwdArgs(n=n, rates=_p(rates), n_steps=1000, itr=_p(itr, torch.int32), g=_p(g), d_update=_p(d_upd),
                               d_rates=d_rates.data_ptr(), d_g=_p(d_g))
        lb_ms = kernel_ms(lambda: L.l2o_lrsgd_bwd(C.byref(la), _stream()))
        tb = lambda b, ms: n * b / ms / 1e9
        res[tag] = dict(n=n, tadam_step_ms=k_ms, tadam_step_TBps=tb(TADAM_FWD, k_ms),
                        tadam_step_hbm_share=tb(TADAM_FWD, k_ms) * 1e12 / HBM,
                        torch_tadam_step_ms=t_ms, torch_over_kernel=t_ms / k_ms, kernel_vs_torch_rel=cmp,
                        tadam_bwd_ms=b_ms, tadam_bwd_TBps=tb(TADAM_BWD, b_ms),
                        lrsgd_step_ms=ls_ms, lrsgd_step_TBps=tb(LRS_FWD, ls_ms),
                        lrsgd_bwd_ms=lb_ms, lrsgd_bwd_TBps=tb(LRS_BWD, lb_ms))
        del g, x0, xa, sa, xb, sb, d_new, d_upd, d_old, d_g, planes
        torch.cuda.empty_cache()
    # T = 20 meta-gradient on the ConvNet objective (two images), each trainer, first and second order
    data = torch.rand(2, 32, 32, 3, device=dev, generator=gen)
    labels = torch.eye(10, device=dev)[torch.tensor([3, 7], device=dev)]
    obj = lambda ps: net.objective(ps, data, labels)
    shapes = [tuple(s) for s in net.param_shapes]
    p0 = [torch.randn(s, device=dev, generator=gen) * (math.sqrt(2.0 / math.prod(s[:-1])) if len(s) > 1 else 0.1)
          for s in shapes]
    thetas = dict(TrainableAdam=(bt.TrainableAdamTrainer, theta.cpu()),
                  LearningRateSchedule=(bt.LearningRateScheduleTrainer, torch.full((1000,), 1e-3)),
                  GlobalLearningRate=(bt.GlobalLearningRateTrainer, torch.full((1,), 1e-3)))
    for nm, (cls, th) in thetas.items():
        for second in (False, True):
            tr = cls(shapes, theta=th, device=dev, use_second_derivatives=second)
            torch.cuda.reset_peak_memory_stats()
            ms20 = event_ms(lambda: tr.meta_gradient(obj, p0, 20), max(3, args.reps // 10), 1)
            res["meta_gradient_T20_convnet_%s_%s" % (nm, "second" if second else "first")] = dict(
                ms=ms20, peak_GB=torch.cuda.max_memory_allocated() / 1e9)
    emit(res, args.out and os.path.join(args.out, "baselines_profile.json"))


if __name__ == "__main__":
    main()
