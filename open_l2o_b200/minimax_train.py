"""Twin-L2O meta-training and evaluation (MM = Model_Free_L2O/L2O-Minimax/Twin-L2O.py do_fit :91, fit_optimizer
:470), on the l2o_minimax_* kernels.

    python -m open_l2o_b200.minimax_train --config seesaw_train.json [--eval_interval 5] [--result_dir result]

The JSON keys are the reference's.  Training mode saves epoch<k>min.pth / epoch<k>max.pth every epoch and
bestmin.pth / bestmax.pth at the best evaluation score; test mode loads <load_model>min.pth / max.pth and prints the
score of n_test problems.  Meta-steps are torch.optim.Adam steps, as in the reference.  Evaluation runs all n_eval
problems as one batch (rows are independent).  Plots are not produced.
"""
from __future__ import annotations

import argparse
import json
import os

import numpy as np
import torch

from . import minimax as mm

KEYS_TRAIN = ("seed", "use_second", "meta_lr", "batch_size", "n_train", "train_epochs", "train_optim_iter",
              "eval_optim_iter", "n_eval", "save_train", "hidden_size", "loss", "save_curve", "unroll_unit",
              "rescale", "CL", "mode", "train_data_path", "eval_data_path", "save_name", "load_name")
KEYS_TEST = ("seed", "use_second", "test_optim_iter", "test_epochs", "n_test", "hidden_size", "loss", "unroll_unit",
             "save_curve", "rescale", "CL", "mode", "test_data_path", "save_name", "load_name", "load_model")


def parse_config(params: dict) -> dict:
    """Checks a reference config and fills its defaults (dim = 1)."""
    params = dict(params)
    params["dim"] = params.get("dim", 1)
    need = KEYS_TRAIN if params.get("mode") == "train" else KEYS_TEST
    missing = [k for k in need if k not in params]
    if missing:
        raise KeyError("config lacks %s" % missing)
    if params["use_second"] != 1:
        raise NotImplementedError("use_second = 0 (LSTMCell(1, H)) is not supported")
    return params


def do_fit(twin, meta_opts, loss, data, dim, unroll_unit, optim_it, train, rescale=1e-4, out_mul=1.0,
           cl_ratio=None, gen=None, unroll=None):
    """One do_fit over a batch (data [B][2] or [B][dim][dim] on the device).  Training back-propagates each segment
    of 2 unroll_unit iterations (1 forward and 2 backward launches) and steps both Adams; returns the trajectory
    [optim_it][R][2] and l_t [optim_it][B].  unroll: an Unroll over data already at its starting point (default: a
    fresh one reset with gen)."""
    if cl_ratio is not None and loss == 4:
        raise ValueError("the curriculum (CL) scores problems by their (a, b): losses 1-3 only")
    un = unroll
    if un is None:
        un = mm.Unroll(twin, loss, data, dim, rescale, out_mul)
        un.reset(gen)
    B, seg = un.batch, 2 * unroll_unit
    traj = torch.zeros(optim_it, un.rows, 2, device=twin.device)
    lval = torch.zeros(optim_it, B, device=twin.device)
    t = 1
    while t <= optim_it:
        T = ((t - 1) // seg + 1) * seg   # the next boundary
        if not train or T > optim_it:
            un.forward(t, optim_it + 1, optim_it, traj=traj[t - 1:], lval=lval[t - 1:])
            break
        bufs = un.buffers(T + 1 - t)
        un.forward(t, T + 1, optim_it, traj=traj[t - 1:T], ckpt=bufs["ckpt"], dl=bufs["dl"], lval=lval[t - 1:T])
        weight, chosen = None, B
        if cl_ratio is not None:
            d = data.detach().cpu().numpy()
            # the reference selects before recording the boundary iteration T: its column T - 1 is still 0
            traj_u = traj[:, :, 0].T.cpu().numpy().copy()
            traj_u[:, T - 1:] = 0.0
            keep = mm.get_index(traj_u, d[:, 0], d[:, 1], T, unroll_unit, cl_ratio)
            chosen = len(keep)
            weight = torch.zeros(B, device=twin.device)
            weight[list(keep)] = 1.0
        # sign steps pass zero gradients, and Adam still steps on them (its step count and moments advance); only a
        # curriculum that keeps no problem skips the step, as in the reference
        if chosen > 0:
            coef = mm.reward_coefs(t, T, B).to(twin.device)
            un.backward(t, T, optim_it, bufs["ckpt"], bufs["dl"], coef, weight)
            for n, o in enumerate(meta_opts):
                o.zero_grad()
                o.param_groups[0]["params"][0].grad = twin.grad[n].float()
                o.step()
            twin.refresh()
        t = T + 1
    return traj, lval


def make_meta_opts(twin, lr, eps=1e-8):
    return [torch.optim.Adam([twin.theta[n]], lr=lr, eps=eps) for n in (0, 1)]


def eval_score(loss, data, traj, dim, burn):
    """fit_optimizer's score: mean over problems of sum_{t >= burn} dist_u^2 + dist_v^2 (l1 distances; loss 3's u
    distance is the nearest k / a)."""
    B = data.shape[0]
    au = traj[burn:, :, 0].reshape(-1, B, dim).abs().sum(-1).double().cpu()
    av = traj[burn:, :, 1].reshape(-1, B, dim).abs().sum(-1).double().cpu()
    if loss == 3:
        a = data[:, 0].cpu().numpy()
        au = torch.tensor([[mm.loss3_distance(float(s), float(a[p])) for p, s in enumerate(row)] for row in au.numpy()],
                          dtype=torch.float64)
    return float((au ** 2 + av ** 2).sum(0).mean())


def fit_optimizer(params, result_dir="result", eval_interval=5, device="cuda", log=print):
    torch.manual_seed(params["seed"])
    loss, dim = params["loss"], params["dim"]
    save = os.path.join(result_dir, params["save_name"])
    os.makedirs(save, exist_ok=True)
    twin = mm.TwinOptimizer(params["hidden_size"], device)
    meta_opts = make_meta_opts(twin, params["meta_lr"])
    n_train, n_eval, B = params["n_train"], params["n_eval"], params["batch_size"]
    train = mm.read_toy(params["train_data_path"], n_train)
    evald = mm.read_toy(params["eval_data_path"], n_eval)
    evald = mm.problem_tensor(evald, loss, dim, device)
    np.random.seed(10)
    best = float("inf")
    for epoch in range(params["train_epochs"]):
        np.random.shuffle(train)
        for i in range(n_train // B):
            data = mm.problem_tensor(train[i * B:(i + 1) * B], loss, dim, device)
            ratio = mm.sche_ratio(epoch) if params.get("CL") else None
            _, lval = do_fit(twin, meta_opts, loss, data, dim, params["unroll_unit"], params["train_optim_iter"],
                             True, params["rescale"], cl_ratio=ratio)
            log("epoch %d batch %d mean l_T %.6g" % (epoch, i, float(lval[-1].mean())))
        for n, side in enumerate(("min", "max")):
            torch.save(twin.state_dict(n), os.path.join(save, "epoch%d%s.pth" % (epoch, side)))
        if epoch % eval_interval == 0:
            it = params["eval_optim_iter"]
            traj, _ = do_fit(twin, None, loss, evald, dim, params["unroll_unit"], it, False, params["rescale"])
            score = eval_score(loss, evald, traj, dim, int(0.5 * it))
            log("epoch %d eval score %.6g" % (epoch, score))
            if score < best:
                best = score
                for n, side in enumerate(("min", "max")):
                    torch.save(twin.state_dict(n), os.path.join(save, "best%s.pth" % side))
    return best, twin


def test(params, result_dir="result", device="cuda", log=print):
    loss, dim = params["loss"], params["dim"]
    twin = mm.TwinOptimizer(params["hidden_size"], device)
    load = os.path.join(result_dir, params["load_name"])
    for n, side in enumerate(("min", "max")):
        twin.load_state_dict(n, torch.load(os.path.join(load, params["load_model"] + side + ".pth"),
                                           map_location="cpu"))
    data = mm.read_toy(params["test_data_path"], params["n_test"])
    data = mm.problem_tensor(data, loss, dim, device)
    gen = torch.Generator().manual_seed(70)
    it = params["test_optim_iter"]
    scores = []
    for _ in range(params["test_epochs"]):
        traj, _ = do_fit(twin, None, loss, data, dim, params["unroll_unit"], it, False, params["rescale"], gen=gen)
        scores.append(eval_score(loss, data, traj, dim, int(0.5 * it)))
    log("test score per epoch %s" % scores)
    return scores


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config", required=True, help="a reference JSON config")
    ap.add_argument("--eval_interval", type=int, default=5)
    ap.add_argument("--result_dir", default="result")
    args = ap.parse_args(argv)
    with open(args.config) as f:
        params = parse_config(json.load(f))
    if params["mode"] == "train":
        best, _ = fit_optimizer(params, args.result_dir, args.eval_interval)
        print("best eval score", best)
    else:
        test(params, args.result_dir)


if __name__ == "__main__":
    main()
