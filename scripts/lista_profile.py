"""Time the LISTA-family kernels against the same computation as fp32 torch ops (TF32 off), eager and captured in a
CUDA graph, at the reference's sc configuration (M x N = 256 x 512, K = 16): one training step at B = 128 (forward,
loss, backward and Adam over all 16 layers) and one validation forward at B = 1024.  The versions run alternately in
one process; the kernels' outputs are compared with torch's.  Writes scripts/lista_profile_h100.json (or --out) with
the card's name and power limit read in the same run.

    python scripts/lista_profile.py [--reps 5] [--iters 50]
"""
import argparse
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from open_l2o_b200 import lista, lista_train as lt  # noqa: E402
from open_l2o_b200.engine import adam_step  # noqa: E402
from oracle import lista_oracle as lo  # noqa: E402
from scripts.measure import alternate, card, emit, event_ms, graphed  # noqa: E402
from tests import lfista_lamp_cases as fc  # noqa: E402

M, N, K = 256, 512, 16
B_TRAIN, B_VAL = 128, 1024


def flops(form, B, train, has_dw):
    """GEMM FLOPs from shapes: coupled and LAMP forward 4BMN per layer, backward 4BMN (+2BMN for dW); LISTA forward
    2BMN once (y B1^T) + 2BN^2 per layer with W, backward 2BN^2 (+2BN^2 for dW) per such layer + 2BMN for dB1;
    LFISTA as LISTA with K - 1 Wg and K - 2 Wm products."""
    if form == lista.LFISTA:
        nw = (K - 1) + (K - 2)
        f = 2 * B * M * N + 2 * B * N * N * nw
        return f + 4 * B * N * N * nw + 2 * B * M * N if train else f
    if form in (lista.COUPLED, lista.LAMP):
        f = 4 * B * M * N * K
        return f + (4 + (2 if has_dw else 0)) * B * M * N * K if train else f
    f = 2 * B * M * N + 2 * B * N * N * (K - 1)
    return f + 4 * B * N * N * (K - 1) + 2 * B * M * N if train else f


class TorchVersion:
    """The model's computation as fp32 torch ops with autograd and Keras Adam over the same variables."""

    def __init__(self, m):
        self.m = m
        self.P = {n: v.detach().clone().requires_grad_(True) for n, v in m.variables.items()}
        self.mo = {n: torch.zeros_like(v) for n, v in self.P.items()}
        self.vo = {n: torch.zeros_like(v) for n, v in self.P.items()}
        self.ranks = None if m.ss_rank is None else m.ss_rank.cpu().tolist()

    def forward(self, data, P=None):
        P, m, nm = P or self.P, self.m, self.m.name
        if m.form in (lista.LFISTA, lista.LAMP):
            return fc.model_forward(m, P, data[:, :M], K)
        if m.W_const is not None:
            W = m.W_const[None]
        elif m.share_W:
            W = P[nm + "_W"][None]
        else:
            first = 2 if m.form == lista.LISTA else 1
            W = torch.stack([P[nm + "_W%d" % i] for i in range(first, K + 1)])
        theta = torch.cat([P[nm + "_theta%d" % i] for i in range(1, K + 1)])
        step = torch.cat([P[nm + "_step_size%d" % i] for i in range(1, K + 1)]) if nm + "_step_size1" in P else None
        return lo.forward(m.form, m.A, P.get(nm + "_B"), W, theta, step, data[:, :M], K, m.one_W, self.ranks)[0]

    def train_step(self, data):
        for v in self.P.values():
            v.grad = None
        x = self.forward(data)[-1]
        loss = lo.sc_loss(x, data[:, M:])
        loss.backward()
        with torch.no_grad():
            for n, v in self.P.items():
                if v.grad is not None:
                    lo.keras_adam_step(v, v.grad, self.mo[n], self.vo[n], 1, 1e-4)
        return loss

    def val_pass(self, data):
        with torch.no_grad():
            return self.forward(data)[-1]


def profile(name, reps, iters):
    d = lista.make_data(M, N, (B_TRAIN, B_VAL, 1), seed=0)
    A = d["A"]
    W = lista.alista_weight(A) if name == "alista" else None
    m = lt.build_model(name, A, K, 0.4, False, 1.2, 13.0, W)
    for k in range(K):
        m.create_cell(k)
    if m.form == lista.COUPLED:   # W = A (or the analytic W) over L: a bounded 16-layer recurrence
        for n, v in m.variables.items():
            if "_W" in n:
                v.mul_(1.0 / float(m.scale))
        if m.W_const is not None:
            m.W_const.mul_(1.0 / float(m.scale))
    train = torch.as_tensor(d["train"]).cuda()
    val = torch.as_tensor(d["val"]).cuda()
    tv = TorchVersion(m)

    # outputs: kernel forward and gradients vs the torch version at the same weights
    xk = m.forward(val, K)[-1].clone()
    xt = tv.val_pass(val)
    m.loss_and_grad(train, lista.TASK_SC)
    for v in tv.P.values():
        v.grad = None
    lo.sc_loss(tv.forward(train)[-1], train[:, M:]).backward()
    gerr = max(float((m._grad_span(n, 1).view(v.shape).float() - v.grad).abs().max() / v.grad.abs().max())
               for n, v in tv.P.items() if v.grad is not None and v.grad.abs().max() > 0)
    cmp = {"val_x_K_max_rel_diff": float((xk - xt).abs().max() / xt.abs().max()), "grad_max_rel_diff": gerr}

    tr = lt.KernelTrainer(m, train, val, lista.TASK_SC, 0.0, B_TRAIN, B_VAL, 1)
    tr.begin_stage(1e-4, lt.gradient_scales(K - 1, 1, K))
    start = m.params.clone()

    def k_step():
        m.loss_and_grad(train, lista.TASK_SC, 0.0, tr.gscale)
        adam_step(m.params, m.grads, tr.m, tr.v, 1, lr=1e-4, eps=lt.KERAS_EPS)

    def k_val():
        m.forward(val, K)

    t_step, t_val = (lambda: tv.train_step(train)), (lambda: tv.val_pass(val))
    fns = {"kernel_step": k_step, "kernel_val": k_val, "torch_eager_step": t_step, "torch_eager_val": t_val,
           "torch_graph_step": graphed(t_step, 2), "torch_graph_val": graphed(t_val, 2),
           "kernel_graph_step": graphed(k_step, 2)}
    res = alternate(fns, reps, lambda f: 1e3 * event_ms(f, iters, 1))   # us
    m.params.copy_(start)
    out = {k: statistics.median(v) for k, v in res.items()}
    out["spread"] = {k: [min(v), max(v)] for k, v in res.items()}
    has_dw = name != "alista"
    ft, fv = flops(m.form, B_TRAIN, True, has_dw), flops(m.form, B_VAL, False, has_dw)
    out["flop_train_step"], out["flop_val_pass"] = ft, fv
    out["kernel_step_tflops"] = ft / out["kernel_step"] / 1e6
    out["kernel_val_tflops"] = fv / out["kernel_val"] / 1e6
    out["speedup_vs_torch_graph_step"] = out["torch_graph_step"] / out["kernel_step"]
    out["speedup_vs_torch_graph_val"] = out["torch_graph_val"] / out["kernel_val"]
    out["outputs"] = cmp
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--iters", type=int, default=50)
    p.add_argument("--out", default=os.path.join(ROOT, "scripts", "lista_profile_h100.json"))
    p.add_argument("--models", default="lista,lista_cp,lista_cpss,alista,lfista,lamp")
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lista_profile.py measures on a GPU; none found")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    rec = {"card": card(), "shape": {"M": M, "N": N, "K": K, "B_train": B_TRAIN, "B_val": B_VAL},
           "units": "us per call (median of reps, each the mean of iters calls, CUDA events)", "models": {}}
    for name in a.models.split(","):
        rec["models"][name] = profile(name, a.reps, a.iters)
        r = rec["models"][name]
        print("%-11s step %8.1f us (torch graph %8.1f, eager %8.1f)  val %8.1f us (torch graph %8.1f, eager %8.1f)"
              % (name, r["kernel_step"], r["torch_graph_step"], r["torch_eager_step"], r["kernel_val"],
                 r["torch_graph_val"], r["torch_eager_val"]), r["outputs"], flush=True)
    rec["card_after"] = card()
    emit(rec, a.out)


if __name__ == "__main__":
    main()
