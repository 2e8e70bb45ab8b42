"""The CIFAR-10 producers (l2o_cifar_conv_grad for cifar_conv, l2o_nas_grad for nas) on a seeded synthetic CIFAR-10 of
the real sizes (50,000 + 10,000 images), written to a temporary directory.  For each network:

    python scripts/cifar_profile.py --out results/cifar.json [--rounds 5] [--calls 50] [--unrolls 3]

(a) f and df/dx of one evaluation at B = 128: the kernel against the problem's torch build (device batch draw,
    gather and pixel lookup, cuDNN convs, batch norm, pooling, fc, cross entropy) and its autograd backward, in fp32
    with TF32 off.  Both are captured into CUDA graphs of --calls calls and timed over replays, alternated over
    --rounds rounds; the device time per call.  Also the relative difference of f and g on the kernel's batch.
(b) ms per T = 100 training unroll of get_config(name) (fx + update + step, synchronised) for the DM net and for
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

from open_l2o_b200 import cifar_data, engine, meta, meta_rnnprop_train, problems, util  # noqa: E402
from scripts.measure import alternate, card, emit, graph_ms, wall_ms  # noqa: E402
from tests.cifar_fixture import write_cifar10  # noqa: E402


NETS = {"cifar_conv": (problems.CIFAR10_VARIABLES, problems.cifar10_forward, engine.cifar_conv_grad,
                       engine.cifar_conv_workspace_bytes),
        "nas": (problems.NAS_VARIABLES, problems.nas_forward, engine.nas_grad, engine.nas_workspace_bytes)}


def step_variants(data_dir, B, name):
    """(kernel, torch) callables computing f and df/dx of the network at a fresh batch, and their agreement."""
    variables, forward, grad, ws_bytes = NETS[name]
    images, labels = cifar_data.device_split(data_dir, "train", "cuda")
    N = images.shape[0]
    sizes = [int(np.prod(s)) for _, s in variables]
    gen = torch.Generator().manual_seed(1)
    x = (torch.randn(sum(sizes), generator=gen) * 0.05).cuda()
    g_k, g_t = torch.empty_like(x), torch.empty_like(x)
    f_k = torch.zeros((), dtype=torch.float64, device="cuda")
    counter = torch.zeros(1, dtype=torch.int64, device="cuda")
    idx = torch.zeros(B, dtype=torch.int32, device="cuda")
    ws = torch.empty(ws_bytes(B), dtype=torch.uint8, device="cuda")
    offs = np.cumsum([0] + sizes)
    leaves = [x[offs[k]:offs[k + 1]].view(s).detach().requires_grad_(True)
              for k, (_, s) in enumerate(variables)]
    values = cifar_data.device_values("cuda")
    gts = [g_t[offs[k]:offs[k + 1]].view(s) for k, (_, s) in enumerate(variables)]

    def kernel():
        grad(images, labels, x, g_k, B, 0, counter, ws, f=f_k, idx_out=idx)

    def torch_step(batch=None):
        i = torch.randint(0, N, (B,), device="cuda") if batch is None else batch
        pixels = values[images.index_select(0, i).long()].reshape(-1, 3, 32, 32).permute(0, 2, 3, 1)
        with torch.enable_grad():
            loss = forward(leaves, pixels, labels.index_select(0, i))
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


def program(data_dir, name, rnnprop, fused, T):
    os.environ["L2O_DISABLE_FUSED"] = "0" if fused else "1"
    problem, net_config, _ = util.get_config(name, net_name="RNNprop" if rnnprop else None, data_dir=data_dir)
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
        data_dir = os.path.join(tmp, "cifar10")
        write_cifar10(data_dir, n_train=50000, n_test=10000, seed=args.seed)

        res = {"card": card(), "calls_per_graph": args.calls, "unrolls_per_round": args.unrolls}
        for name, coords in (("cifar_conv", 13610), ("nas", 7578)):
            # (a) one evaluation's f and df/dx
            kernel, torch_step, agreement = step_variants(data_dir, B, name)
            step = alternate({"kernel_ms": kernel, "torch_graph_ms": torch_step}, args.rounds,
                             lambda fn: graph_ms(fn, args.calls, 10, 3))

            # (b) training unrolls
            runs = {"%s_%s_unroll_ms" % (net, path): program(data_dir, name, net == "rnnprop", path == "producer", T)
                    for net in ("dm", "rnnprop") for path in ("producer", "autograd")}
            for _ in range(3):   # two eager unrolls, then the capture of each program's graph
                for run in runs.values():
                    wall_ms(run)
            train = alternate(runs, args.rounds,
                              lambda fn: statistics.median(wall_ms(fn) for _ in range(args.unrolls)))
            med = {k: statistics.median(v) for k, v in list(step.items()) + list(train.items())}
            res[name] = {"shape": {"batch": B, "T": T, "train_images": 50000, "coordinates": coords},
                         "gradient_agreement": agreement, "step": step, "train_unroll": train, "median": med,
                         "torch_over_kernel": med["torch_graph_ms"] / med["kernel_ms"],
                         "autograd_over_producer": {n: med["%s_autograd_unroll_ms" % n] / med["%s_producer_unroll_ms" % n]
                                                    for n in ("dm", "rnnprop")}}
    emit(res, args.out)


if __name__ == "__main__":
    main()
