"""Cost of second-order meta-gradients (``use_second_derivatives``) on the GPU.

    python scripts/second_order_profile.py [--reps 50] [--out DIR]

1. Kernel time of l2o_hrnn_coord_bwd and l2o_crnn_bwd without and with the d_g output, at the BASELINE #4 ConvNet
   shapes (354,218 coordinates) and at 32 M coordinates: CUDA events around `reps` back-to-back launches, the two
   variants alternated over `rounds` rounds after a warm-up; min and median over rounds.
2. meta_gradient of a T = 20 unroll on the BASELINE #4 ConvNet optimizee (synthetic batch of 128), first against
   second order, for both trainers: host wall time around work that ends in a device synchronise (alternated, min and
   median over rounds) and torch.cuda.max_memory_allocated of one call.
Prints one JSON line; the card name and power limit come from a read-only nvidia-smi query in the same run.
"""
import argparse
import ctypes as C
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from scripts.measure import alternate, card, emit, event_ms, summary, wall_ms  # noqa: E402


def hrnn_kernel(sizes, reps, rounds, gen):
    from open_l2o_b200 import _lib
    from open_l2o_b200.hrnn_train import _Engine
    from tests.helpers import hrnn_generic_theta
    dev = "cuda:0"
    eng = _Engine(sizes, torch.device(dev))
    N, nt = eng.N, eng.nt
    rnd = lambda *s: torch.randn(*s, device=dev, generator=gen)
    planes = rnd(21, N) * 0.5
    planes[10:12] = torch.rand(2, N, device=dev, generator=gen)
    planes[17:21] = planes[17:21].abs() + 1e-3
    bufs = dict(theta=hrnn_generic_theta(5).to(dev), state_old=planes, g=rnd(N) * 0.1, bias0=rnd(nt, 32) * 0.3,
                zero_flag=torch.zeros(nt, 4, dtype=torch.int32, device=dev), mean_log_lr=planes[12].mean().reshape(1),
                d_state_new=rnd(21, N), d_upd=rnd(N), d_sums=rnd(nt, 24), d_state_old=torch.empty(21, N, device=dev),
                d_theta=torch.zeros(8349, dtype=torch.float64, device=dev),
                d_bias0=torch.zeros(nt, 32, dtype=torch.float64, device=dev),
                d_mean_log_lr=torch.zeros(1, dtype=torch.float64, device=dev))
    d_g = torch.empty(N, device=dev)
    ptrs = {k: v.data_ptr() for k, v in bufs.items()}
    L, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    args = {k: _lib.HrnnBwdArgs(d_g=p, **ptrs) for k, p in (("without_d_g", None), ("with_d_g", d_g.data_ptr()))}
    fns = {k: (lambda a=a: L.l2o_hrnn_coord_bwd(eng._h, C.byref(a), st)) for k, a in args.items()}
    return {k: summary(v) for k, v in alternate(fns, rounds, lambda f: event_ms(f, reps, 0), warmup=3).items()}


def crnn_kernel(n, reps, rounds, gen):
    from open_l2o_b200 import _lib
    from tests.test_crnn_gpu import crnn_generic_theta
    dev = "cuda:0"
    planes = torch.randn(103, n, device=dev, generator=gen) * 0.5
    planes[100] = planes[100].abs() + 1e-3
    planes[101] = torch.rand(n, device=dev, generator=gen)
    planes[102] = planes[102].abs() * 1e-2
    bufs = dict(theta=crnn_generic_theta(5).to(dev), g=torch.randn(n, device=dev, generator=gen) * 0.1,
                state_old=planes, d_state_new=torch.randn(103, n, device=dev, generator=gen),
                d_update=torch.randn(n, device=dev, generator=gen), d_state_old=torch.empty(103, n, device=dev),
                d_theta=torch.zeros(6402, dtype=torch.float64, device=dev))
    d_g = torch.empty(n, device=dev)
    ptrs = {k: v.data_ptr() for k, v in bufs.items()}
    L, st = _lib.lib(), torch.cuda.current_stream().cuda_stream
    args = {k: _lib.CrnnBwdArgs(n=n, d_g=p, **ptrs) for k, p in (("without_d_g", None), ("with_d_g", d_g.data_ptr()))}
    fns = {k: (lambda a=a: L.l2o_crnn_bwd(C.byref(a), st)) for k, a in args.items()}
    return {k: summary(v) for k, v in alternate(fns, rounds, lambda f: event_ms(f, reps, 0), warmup=3).items()}


def meta_gradient_cost(which, rounds, gen, T=20, batch=128):
    from open_l2o_b200 import crnn_train as ct, hrnn_train as ht
    from open_l2o_b200.scale_problems import ConvNet
    from tests.helpers import HRNN_CONVNET, hrnn_generic_theta
    from tests.test_crnn_gpu import crnn_generic_theta
    dev = "cuda:0"
    net = ConvNet(*HRNN_CONVNET)
    data = torch.rand(batch, 32, 32, 3, device=dev, generator=gen)
    labels = torch.nn.functional.one_hot(torch.randint(10, (batch,), device=dev, generator=gen), 10).float()
    obj = lambda ps: net.objective(ps, data, labels)
    shapes = [tuple(s) for s in net.param_shapes]
    p0 = [torch.randn(s, device=dev, generator=gen) * math.sqrt(2.0 / math.prod(s[:-1])) if len(s) > 1
          else torch.full(s, 0.1, device=dev) for s in shapes]
    n = sum(p.numel() for p in p0)
    u = torch.rand(n, generator=torch.Generator().manual_seed(0))
    trainers = {}
    for second in (False, True):
        if which == "hrnn":
            tr = ht.MetaTrainer(shapes, theta=hrnn_generic_theta(5), device=dev, use_second_derivatives=second)
            lr = u * 1.5 - 12.0
        else:
            tr = ct.MetaTrainer(shapes, theta=crnn_generic_theta(7), device=dev, use_second_derivatives=second)
            lr = torch.exp(u * 1.5 - 12.0)
        trainers["second_order" if second else "first_order"] = tr
    res = {k: {} for k in trainers}
    for k, tr in trainers.items():   # warm-up, then one call for the memory high-water mark
        tr.meta_gradient(obj, p0, T, lr)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        _, g, _, _ = tr.meta_gradient(obj, p0, T, lr)
        torch.cuda.synchronize()
        res[k]["max_memory_allocated_GB"] = torch.cuda.max_memory_allocated() / 1e9
        res[k]["peak_over_resident_GB"] = (torch.cuda.max_memory_allocated() - base) / 1e9
        res[k]["grad_finite"] = bool(torch.isfinite(g).all())
        del g
    fns = {k: (lambda tr=tr: tr.meta_gradient(obj, p0, T, lr)) for k, tr in trainers.items()}
    for k, v in alternate(fns, rounds, wall_ms).items():
        res[k].update({"wall_" + m: t for m, t in summary(v).items()}, rounds=len(v))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("second_order_profile.py measures on the GPU and needs a CUDA device")
    from open_l2o_b200.scale_problems import ConvNet
    from tests.helpers import HRNN_CONVNET
    res = dict(card=card(), reps=args.reps, rounds=args.rounds)
    gen = torch.Generator(device="cuda:0").manual_seed(0)
    conv = [int(math.prod(s)) for s in ConvNet(*HRNN_CONVNET).param_shapes]
    big = [8 * 2 ** 20] * 4
    for tag, sizes in (("convnet", conv), ("32M", big)):
        res["hrnn_coord_bwd_%s" % tag] = hrnn_kernel(sizes, args.reps, args.rounds, gen)
        torch.cuda.empty_cache()
        res["crnn_bwd_%s" % tag] = crnn_kernel(sum(sizes), args.reps, args.rounds, gen)
        torch.cuda.empty_cache()
    for which in ("hrnn", "crnn"):
        res["meta_gradient_T20_convnet_%s" % which] = meta_gradient_cost(which, args.rounds, gen)
        torch.cuda.empty_cache()
    emit(res, args.out and os.path.join(args.out, "second_order_profile.json"))


if __name__ == "__main__":
    main()
