"""Time Twin-L2O on the l2o_minimax_* kernels against the same semantics as batched fp32 torch ops (TF32 off), eager and
captured in one CUDA graph, at the reference's two configurations: the toy seesaw (loss 3, H = 50, dim = 1) and the
matrix game (loss 4, H = 80, dim = 5).  Per configuration it times one training do_fit (B = 128, 100 iterations,
unroll_unit 5: ten segments of forward, backward and two Adam steps) and one 1000-iteration evaluation (B = n_eval =
20).  The versions run alternately in one process from the same starting point; the kernels' outputs are compared with
torch's.  Writes scripts/minimax_profile_h100.json (or --out) with the card's name and power limit read in the same run.

    python scripts/minimax_profile.py [--reps 5] [--iters 5]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from open_l2o_b200 import minimax as mm, minimax_train as tr  # noqa: E402

CONFIGS = {"seesaw": dict(loss=3, hidden=50, dim=1), "matrix_game_dim5": dict(loss=4, hidden=80, dim=5)}
B_TRAIN, B_EVAL, TRAIN_IT, EVAL_IT, UNROLL, META_LR, RESCALE = 128, 20, 100, 1000, 5, 1e-4, 1e-4


class TorchTwin:
    """The same do_fit as batched fp32 torch ops over the R = B dim rows (torch.lstm_cell, autograd, torch Adam)."""

    def __init__(self, twin, loss, data, dim):
        self.loss, self.dim, self.data = loss, dim, data
        self.P = [[v.cuda().requires_grad_(True) for v in twin.state_dict(n).values()] for n in (0, 1)]
        self.opts = [torch.optim.Adam(p, lr=META_LR, capturable=True) for p in self.P]

    def grads(self, u, v):
        if self.loss == 4:
            B, d = self.data.shape[0], self.dim
            gu = torch.bmm(self.data, v.view(B, d, 1)).view(-1)
            gv = torch.bmm(self.data.transpose(1, 2), u.view(B, d, 1)).view(-1)
            return gu, gv
        a, b = self.data[:, 0], self.data[:, 1]
        if self.loss == 3:
            return -b * v * torch.cos(a * math.pi * u) * a * math.pi, -b * torch.sin(a * math.pi * u)
        raise ValueError(self.loss)

    def f(self, u, v):
        if self.loss == 4:
            B, d = self.data.shape[0], self.dim
            return (u.view(B, 1, d) @ self.data @ v.view(B, d, 1)).view(B)
        return -self.data[:, 1] * v * torch.sin(math.pi * u * self.data[:, 0])

    def cell(self, n, x, st):
        wih1, whh1, bih1, bhh1, wih2, whh2, bih2, bhh2, wo, bo = self.P[n]
        h1, c1 = torch.lstm_cell(x, (RESCALE * st[0], RESCALE * st[1]), wih1, whh1, bih1, bhh1)
        h2, c2 = torch.lstm_cell(h1, (RESCALE * st[2], RESCALE * st[3]), wih2, whh2, bih2, bhh2)
        return (h2 @ wo.t() + bo).view(-1), [h1, c1, h2, c2]

    def do_fit(self, u, v, state, optim_it, train):
        lr, wend, B = mm.sche_lr(optim_it), mm.warm_end(optim_it), self.data.shape[0]
        st = [[state[n, k] for k in range(4)] for n in (0, 1)]
        total, lprev = 0.0, 0.0
        for t in range(1, optim_it + 1):
            n = 0 if t % 2 else 1
            gu, gv = self.grads(u.detach(), v.detach())
            x = torch.stack((gu, gv) if n == 0 else (gv, gu), 1)
            delta, st[n] = self.cell(n, x, st[n])
            step = torch.sign(delta) * float(lr[t - 1]) if t < wend else delta
            if n == 0:
                u = u.detach() + step
            else:
                v = v.detach() + step
            if t % (2 * UNROLL) == 0:
                if train:
                    for o in self.opts:
                        o.zero_grad(set_to_none=False)
                    total.backward()
                    for o in self.opts:
                        o.step()
                st = [[s.detach() for s in st[m]] for m in (0, 1)]
                total, lprev = 0.0, 0.0
                u, v = u.detach(), v.detach()
            fl = self.f(u, v)
            lt = fl if n == 0 else -fl
            total = total + (lt + lprev).sum() / B
            lprev = lt
            if n == 0:   # the variable just updated is detached after its reward
                u = u.detach()
            else:
                v = v.detach()
        return u.detach(), v.detach()


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters   # ms


def graphed(fn):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def problems(loss, dim, B, seed):
    if loss == 4:
        return mm.make_matrix_game_data(dim, 0.5, 0.5, 1.0, B, seed)
    rng = np.random.RandomState(seed)
    return np.stack([rng.uniform(0.5, 1.5, B), rng.uniform(0.5, 1.0, B)], 1)


def profile(name, reps, iters):
    c = CONFIGS[name]
    loss, H, dim = c["loss"], c["hidden"], c["dim"]
    twin = mm.TwinOptimizer(H, "cuda", seed=0)
    out = {}
    for mode, B, it in (("train", B_TRAIN, TRAIN_IT), ("eval", B_EVAL, EVAL_IT)):
        train = mode == "train"
        data = mm.problem_tensor(problems(loss, dim, B, 1), loss, dim, "cuda")
        un = mm.Unroll(twin, loss, data, dim, RESCALE)
        un.reset(torch.Generator().manual_seed(2))
        u0, v0, s0, th0 = un.u.clone(), un.v.clone(), un.state.clone(), twin.theta.clone()
        tt = TorchTwin(twin, loss, data, dim)
        opts = tr.make_meta_opts(twin, META_LR) if train else None
        tu, tv = torch.empty_like(u0), torch.empty_like(v0)

        # outputs from the same start, at a meta learning rate of 0 so both versions keep the same weights: final u, v
        # and (training) the last segment's meta-gradient.  (Adam's normalised step would turn fp32 noise in
        # near-zero gradient entries into +-lr, so the weights after real meta-steps are not a useful comparison.)
        for o in (opts or []) + tt.opts:
            o.param_groups[0]["lr"] = 0.0
        un.u.copy_(u0), un.v.copy_(v0), un.state.copy_(s0)
        tr.do_fit(twin, opts, loss, data, dim, UNROLL, it, train, RESCALE, unroll=un)
        with torch.set_grad_enabled(train):
            ru, rv = tt.do_fit(u0.clone(), v0.clone(), s0, it, train)
        cmp = {"u_max_rel_diff": float((un.u - ru).abs().max() / ru.abs().max()),
               "v_max_rel_diff": float((un.v - rv).abs().max() / rv.abs().max())}
        if train:
            tg = torch.stack([torch.cat([p.grad.reshape(-1) for p in ps]) for ps in tt.P]).double()
            cmp["last_segment_meta_grad_max_rel_diff"] = float((twin.grad - tg).abs().max() / tg.abs().max())
        for o in (opts or []) + tt.opts:
            o.param_groups[0]["lr"] = META_LR
        out[mode] = {"batch": B, "iterations": it, "outputs": cmp}

        def k_run():
            un.u.copy_(u0), un.v.copy_(v0), un.state.copy_(s0)
            tr.do_fit(twin, opts, loss, data, dim, UNROLL, it, train, RESCALE, unroll=un)

        def t_run():
            with torch.set_grad_enabled(train):
                a, b = tt.do_fit(u0, v0, s0, it, train)
            tu.copy_(a), tv.copy_(b)

        fns = {"kernel": k_run, "torch_eager": t_run, "torch_graph": graphed(t_run)}
        res = {k: [] for k in fns}
        for _ in range(reps):   # alternate the versions within each repetition
            for k, f in fns.items():
                res[k].append(timed(f, iters))
        twin.theta.copy_(th0)
        twin.refresh()
        r = {k: statistics.median(v) for k, v in res.items()}
        r["spread"] = {k: [min(v), max(v)] for k, v in res.items()}
        r["speedup_vs_torch_graph"] = r["torch_graph"] / r["kernel"]
        r["speedup_vs_torch_eager"] = r["torch_eager"] / r["kernel"]
        out[mode].update(r)
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--iters", type=int, default=5)
    p.add_argument("--out", default=os.path.join(ROOT, "scripts", "minimax_profile_h100.json"))
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("minimax_profile.py measures on a GPU; none found")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    rec = {"card": card(), "units": "ms per do_fit (median of reps, each the mean of iters calls, CUDA events)",
           "setup": {"B_train": B_TRAIN, "train_iterations": TRAIN_IT, "B_eval": B_EVAL, "eval_iterations": EVAL_IT,
                     "unroll_unit": UNROLL, "meta_lr": META_LR, "rescale": RESCALE},
           "configs": {}}
    for name in CONFIGS:
        r = rec["configs"][name] = dict(CONFIGS[name], **profile(name, a.reps, a.iters))
        for mode in ("train", "eval"):
            m = r[mode]
            print("%-17s %-5s kernel %8.3f ms  torch graph %8.3f  eager %8.3f" %
                  (name, mode, m["kernel"], m["torch_graph"], m["torch_eager"]), m["outputs"], flush=True)
    rec["card_after"] = card()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec["card"]))


if __name__ == "__main__":
    main()
