"""The MNIST MLP producer (l2o_mnist_grad) on a seeded synthetic MNIST of the real sizes (60,000 + 10,000 images),
written to a temporary directory.

    python scripts/mnist_profile.py --out results/mnist.json [--rounds 5] [--calls 100] [--unrolls 3]

(a) f and df/dx at B = 128 for the (20,) and (20, 20) sigmoid MLPs: the kernel against the same computation as fp32
    torch ops (device batch draw, gather and scaling, problems.mlp_value_and_grad's forward, cross entropy and
    hand-written backward).  Both are captured into CUDA graphs of --calls calls and timed over replays, alternated
    over --rounds rounds; the device time per call.  Also the relative difference of f and g on the kernel's batch.
(b) ms per T = 100 training unroll of get_config("mnist") (fx + update + step, synchronised) for the DM net and for
    RNNProp, each on the producer path and with L2O_DISABLE_FUSED=1 (autograd of problems.mnist's torch build), every
    program past its two eager warm-up unrolls and CUDA-graph capture, --unrolls timed unrolls per round, alternated.
The card's name and power limit are read in the same run."""
import argparse
import gzip
import os
import statistics
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from open_l2o_b200 import engine, meta, meta_rnnprop_train, mnist_data, problems, util  # noqa: E402
from scripts.measure import alternate, card, emit, graph_ms, wall_ms  # noqa: E402


def write_mnist(path, n_train, n_test, seed):
    rng = np.random.default_rng(seed)
    os.makedirs(path, exist_ok=True)
    for key, shape, magic in (("train_images", (n_train, 28, 28), 2051), ("train_labels", (n_train,), 2049),
                              ("test_images", (n_test, 28, 28), 2051), ("test_labels", (n_test,), 2049)):
        arr = rng.integers(0, 10 if magic == 2049 else 256, shape, dtype=np.uint8)
        with gzip.open(os.path.join(path, mnist_data.FILES[key] + ".gz"), "wb") as f:
            f.write(np.array([magic] + list(shape), dtype=">u4").tobytes() + arr.tobytes())


def step_variants(data_dir, layers, B):
    """(kernel, torch) callables computing f and df/dx of the sigmoid MLP at a fresh batch, and their agreement."""
    images, labels = mnist_data.device_split(data_dir, "train", "cuda")
    N = images.shape[0]
    sizes, k = [], 784
    for w in tuple(layers) + (10,):
        sizes += [k * w, w]
        k = w
    gen = torch.Generator().manual_seed(1)
    x = (torch.randn(sum(sizes), generator=gen) * 0.01).cuda()
    g_k, g_t = torch.empty_like(x), torch.empty_like(x)
    f_k = torch.zeros((), dtype=torch.float64, device="cuda")
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    idx = torch.zeros(B, dtype=torch.int32, device="cuda")

    def views(flat):
        out, off, k = [], 0, 784
        for w in tuple(layers) + (10,):
            out += [flat[off:off + k * w].view(k, w), flat[off + k * w:off + k * w + w]]
            off, k = off + k * w + w, w
        return out

    xs, gts = views(x), views(g_t)

    def kernel():
        engine.mnist_grad(images, labels, x, g_k, layers, B, "sigmoid", 0, counter, f=f_k, idx_out=idx)

    def torch_step(batch=None):
        i = torch.randint(0, N, (B,), device="cuda") if batch is None else batch
        data = images.index_select(0, i).float() * float(mnist_data.SCALE)
        return problems.mlp_value_and_grad(xs, data, labels.index_select(0, i), "sigmoid", gts)

    kernel()
    f_t = torch_step(idx.long())
    torch.cuda.synchronize()
    agree = {"f_rel": abs(float(f_k) - float(f_t)) / abs(float(f_t)),
             "g_rel_maxnorm": float((g_k - g_t).abs().max() / g_t.abs().max())}
    return kernel, torch_step, agree


def program(data_dir, rnnprop, fused, T):
    os.environ["L2O_DISABLE_FUSED"] = "0" if fused else "1"
    problem, net_config, _ = util.get_config("mnist", net_name="RNNprop" if rnnprop else None, data_dir=data_dir)
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
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--unrolls", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    T, B = 100, 128
    with tempfile.TemporaryDirectory() as tmp:
        data_dir = os.path.join(tmp, "MNIST-data")
        write_mnist(data_dir, 60000, 10000, args.seed)

        # (a) one evaluation's f and df/dx
        step, agreement = {}, {}
        fns = {}
        for layers in ((20,), (20, 20)):
            name = "x".join(str(w) for w in layers)
            kernel, torch_step, agreement[name] = step_variants(data_dir, layers, B)
            fns["kernel_%s_ms" % name] = kernel
            fns["torch_graph_%s_ms" % name] = torch_step
        step = alternate(fns, args.rounds, lambda fn: graph_ms(fn, args.calls, 10, 3))

        # (b) training unrolls
        runs = {"%s_%s_unroll_ms" % (net, path): program(data_dir, net == "rnnprop", path == "producer", T)
                for net in ("dm", "rnnprop") for path in ("producer", "autograd")}
        for _ in range(3):   # two eager unrolls, then the capture of each program's graph
            for run in runs.values():
                wall_ms(run)
        train = alternate(runs, args.rounds, lambda fn: statistics.median(wall_ms(fn) for _ in range(args.unrolls)))

    med = {k: statistics.median(v) for k, v in list(step.items()) + list(train.items())}
    res = {"card": card(), "shape": {"batch": B, "T": T, "train_images": 55000},
           "calls_per_graph": args.calls, "unrolls_per_round": args.unrolls, "gradient_agreement": agreement,
           "step": step, "train_unroll": train, "median": med,
           "torch_over_kernel": {n: med["torch_graph_%s_ms" % n] / med["kernel_%s_ms" % n] for n in ("20", "20x20")},
           "autograd_over_producer": {n: med["%s_autograd_unroll_ms" % n] / med["%s_producer_unroll_ms" % n]
                                      for n in ("dm", "rnnprop")}}
    emit(res, args.out)


if __name__ == "__main__":
    main()
