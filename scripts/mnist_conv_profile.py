"""The MNIST ConvNet producer (l2o_mnist_conv_grad) on a seeded synthetic MNIST of the real sizes (60,000 + 10,000
images), written to a temporary directory.

    python scripts/mnist_conv_profile.py --out results/mnist_conv.json [--rounds 5] [--calls 50] [--unrolls 3]

(a) f and df/dx of one evaluation at B = 128: the kernel against problems.mnist_conv's torch build (device batch draw,
    gather and scaling, cuDNN convs, batch norm, pooling, fc, cross entropy) and its autograd backward, in fp32 with
    TF32 off.  Both are captured into CUDA graphs of --calls calls and timed over replays, alternated over --rounds
    rounds; the device time per call.  Also the relative difference of f and g on the kernel's batch.
(b) ms per T = 100 training unroll of get_config("mnist_conv") (fx + update + step, synchronised) for the DM net and for
    RNNProp, each on the producer path and with L2O_DISABLE_FUSED=1 (autograd of the torch build), every program past
    its two eager warm-up unrolls and CUDA-graph capture, --unrolls timed unrolls per round, alternated.
The card's name and power limit are read in the same run."""
import argparse
import os
import statistics
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from open_l2o_b200 import engine, meta, meta_rnnprop_train, mnist_data, problems, util  # noqa: E402
from scripts.measure import alternate, card, emit, graph_ms, wall_ms  # noqa: E402
from tests.mnist_fixture import write_mnist  # noqa: E402


def step_variants(data_dir, B):
    """(kernel, torch) callables computing f and df/dx of the ConvNet at a fresh batch, and their agreement."""
    images, labels = mnist_data.device_split(data_dir, "train", "cuda")
    N = images.shape[0]
    sizes = [int(np.prod(s)) for _, s in problems.MNIST_CONV_VARIABLES]
    gen = torch.Generator().manual_seed(1)
    x = (torch.randn(sum(sizes), generator=gen) * 0.05).cuda()
    g_k, g_t = torch.empty_like(x), torch.empty_like(x)
    f_k = torch.zeros((), dtype=torch.float64, device="cuda")
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    idx = torch.zeros(B, dtype=torch.int32, device="cuda")
    ws = torch.empty(engine.mnist_conv_workspace_bytes(B), dtype=torch.uint8, device="cuda")
    offs = np.cumsum([0] + sizes)
    leaves = [x[offs[k]:offs[k + 1]].view(s).detach().requires_grad_(True)
              for k, (_, s) in enumerate(problems.MNIST_CONV_VARIABLES)]
    gts = [g_t[offs[k]:offs[k + 1]].view(s) for k, (_, s) in enumerate(problems.MNIST_CONV_VARIABLES)]

    def kernel():
        engine.mnist_conv_grad(images, labels, x, g_k, B, 0, counter, ws, f=f_k, idx_out=idx)

    def torch_step(batch=None):
        i = torch.randint(0, N, (B,), device="cuda") if batch is None else batch
        pixels = images.index_select(0, i).float() * float(mnist_data.SCALE)
        with torch.enable_grad():
            loss = problems.mnist_conv_forward(leaves, pixels, labels.index_select(0, i))
            grads = torch.autograd.grad(loss, leaves)
        for d, s in zip(gts, grads):
            d.copy_(s)
        return loss.detach()

    kernel()
    f_t = torch_step(idx.long())
    torch.cuda.synchronize()
    agree = {"f_rel": abs(float(f_k) - float(f_t)) / abs(float(f_t)),
             "g_rel_maxnorm": float((g_k - g_t).abs().max() / g_t.abs().max())}
    return kernel, torch_step, agree


def program(data_dir, rnnprop, fused, T):
    os.environ["L2O_DISABLE_FUSED"] = "0" if fused else "1"
    problem, net_config, _ = util.get_config("mnist_conv", net_name="RNNprop" if rnnprop else None, data_dir=data_dir)
    if rnnprop:
        opt = meta_rnnprop_train.MetaOptimizer(0, 0.95, 0.95, **net_config)
        ms = opt.meta_minimize(problem, T, learning_rate=0.001)[0]
    else:
        opt = meta.MetaOptimizer(**net_config)
        ms = opt.meta_minimize(problem, T, learning_rate=0.001)
    assert (opt.program.producer is not None) == fused
    sess = meta.Session()
    sess.run(ms.reset)
    return lambda: sess.run([ms.fx, ms.update, ms.step])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--unrolls", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False      # the torch side in fp32, as the kernel
    torch.backends.cuda.matmul.allow_tf32 = False
    T, B = 100, 128
    with tempfile.TemporaryDirectory() as tmp:
        data_dir = os.path.join(tmp, "MNIST-data")
        write_mnist(data_dir, n_train=60000, n_test=10000, seed=args.seed)

        # (a) one evaluation's f and df/dx
        kernel, torch_step, agreement = step_variants(data_dir, B)
        step = alternate({"kernel_ms": kernel, "torch_graph_ms": torch_step}, args.rounds,
                         lambda fn: graph_ms(fn, args.calls, 10, 3))

        # (b) training unrolls
        runs = {"%s_%s_unroll_ms" % (net, path): program(data_dir, net == "rnnprop", path == "producer", T)
                for net in ("dm", "rnnprop") for path in ("producer", "autograd")}
        for _ in range(3):   # two eager unrolls, then the capture of each program's graph
            for run in runs.values():
                wall_ms(run)
        train = alternate(runs, args.rounds, lambda fn: statistics.median(wall_ms(fn) for _ in range(args.unrolls)))

    med = {k: statistics.median(v) for k, v in list(step.items()) + list(train.items())}
    res = {"card": card(), "shape": {"batch": B, "T": T, "train_images": 55000, "coordinates": 18122},
           "calls_per_graph": args.calls, "unrolls_per_round": args.unrolls, "gradient_agreement": agreement,
           "step": step, "train_unroll": train, "median": med,
           "torch_over_kernel": med["torch_graph_ms"] / med["kernel_ms"],
           "autograd_over_producer": {n: med["%s_autograd_unroll_ms" % n] / med["%s_producer_unroll_ms" % n]
                                      for n in ("dm", "rnnprop")}}
    emit(res, args.out)


if __name__ == "__main__":
    main()
