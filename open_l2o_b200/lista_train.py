"""Layer-wise training and testing of the LISTA family (MB/train.py:run), on the kernels of ``lista.py``.

    python -m open_l2o_b200.lista_train --model_name lista_cpss --task sc --data_dir D --base_dir E
    python -m open_l2o_b200.lista_train --model_name lista_cpss --task sc --data_dir D --base_dir E \\
        --test --test_files test_data.npy

The schedule's host logic (which variables train in each stage, the 0.3^age gradient multipliers, early stopping,
checkpoints and resume) is kept apart from the step in ``train_layerwise`` so it can run on a stub.
"""
from __future__ import annotations

import argparse
import logging
import os
from typing import Callable, List, Optional

import numpy as np
import torch

from . import lista
from .engine import adam_step

log = logging.getLogger("lista_train")

STAGE_LR = (1.0, 0.2, 0.02)   # base_lr, then base_lr * 0.2 * 0.1^i (MB/train.py:293-323)
PATIENCE = 5                  # EarlyStopping(patience=5, min_delta=0, mode='min') (MB/train.py:298-303)
AGE_DECAY = 0.3               # utils.Adam: g * 0.3^age (MB/utils.py:132)
KERAS_EPS = 1e-7


def gradient_scales(layer_id: int, stage: int, num_layers: int) -> np.ndarray:
    """Multiplier of the gradient of every variable by its creation layer while layer `layer_id` trains.  Stage 0
    trains only the variables created with this layer (utils.Adam(freeze_layer=True)); stages 1 and 2 train all of
    them with 0.3^age.  Variables of later layers are not in the model yet: 0."""
    s = np.zeros(num_layers, np.float32)
    if stage == 0:
        s[layer_id] = 1.0
    else:
        s[:layer_id + 1] = AGE_DECAY ** np.arange(layer_id, -1, -1, dtype=np.float64)
    return s


def fit_stage(train_epoch: Callable[[], None], validate: Callable[[], float], epochs: int,
              patience: int = PATIENCE) -> List[float]:
    """model.fit with EarlyStopping: stop after `patience` epochs in a row without a strictly lower validation
    metric; the weights are not restored.  Returns the validation history."""
    best, wait, hist = np.inf, 0, []
    for _ in range(epochs):
        train_epoch()
        v = float(validate())
        hist.append(v)
        if v < best:
            best, wait = v, 0
        else:
            wait += 1
            if wait >= patience:
                break
    return hist


def last_complete_layer(model_dir: str, num_layers: int) -> int:
    """utils.check_and_load_partial: the number of consecutive layer_<i>/ checkpoints from layer 1."""
    for i in range(num_layers):
        if not os.path.exists(os.path.join(model_dir, "layer_%d" % (i + 1), "model.npz")):
            return i
    return num_layers


def train_layerwise(trainer, num_layers: int, base_lr: float, epochs: int, model_dir: Optional[str] = None):
    """MB/train.py:260-352.  `trainer` provides create_cell(k), begin_stage(lr, gscale), train_epoch(), validate(),
    save(path) and load(path).  Returns the last validation metric."""
    prev = last_complete_layer(model_dir, num_layers) if model_dir else 0
    val = None
    for k in range(num_layers):
        trainer.create_cell(k)
        if k < prev:
            if k == prev - 1:
                trainer.load(os.path.join(model_dir, "layer_%d" % (k + 1), "model.npz"))
                val = trainer.validate()
                log.info("layer %d: restored, val %.6f", k + 1, val)
            continue
        for stage, f in enumerate(STAGE_LR):
            trainer.begin_stage(base_lr * f, gradient_scales(k, stage, num_layers))
            hist = fit_stage(trainer.train_epoch, trainer.validate, epochs)
            val = hist[-1]
            log.info("layer %d stage %d: %d epochs, val %.6f", k + 1, stage, len(hist), val)
        if model_dir:
            path = os.path.join(model_dir, "layer_%d" % (k + 1), "model.npz")
            os.makedirs(os.path.dirname(path), exist_ok=True)
            trainer.save(path)
    return val


def build_model(model_name, A, num_layers, model_lam, share_W, ss_q_per_layer, ss_maxq, alista_W=None,
                device="cuda"):
    if model_name == "lista":
        return lista.Lista(A, num_layers, model_lam, share_W, name="Lista", device=device)
    if model_name == "lista_cp":
        return lista.ListaCp(A, num_layers, model_lam, share_W, name="ListaCp", device=device)
    if model_name == "lista_cpss":
        return lista.ListaCpss(A, num_layers, model_lam, ss_q_per_layer, ss_maxq, share_W, name="ListaCpss",
                               device=device)
    if model_name == "alista":
        return lista.Alista(A, alista_W, num_layers, model_lam, ss_q_per_layer, ss_maxq, name="Alista",
                            device=device)
    if model_name == "lfista":
        return lista.Lfista(A, num_layers, model_lam, share_W, name="Lfista", device=device)
    if model_name == "lamp":
        return lista.Lamp(A, num_layers, model_lam, share_W, name="Lamp", device=device)
    raise NotImplementedError("model %r is not built here (Step-LISTA, TiSTA, GLISTA are out of scope)" % model_name)


class KernelTrainer:
    """The training surface of train_layerwise on the CUDA kernels: per step one forward, loss, backward and Adam."""

    def __init__(self, model, train, val, task, lasso_lam, batch, val_batch, steps_per_epoch, seed=42):
        self.model, self.task, self.lasso_lam = model, task, lasso_lam
        self.train, self.val = train, val
        self.batch, self.val_batch, self.steps = batch, val_batch, steps_per_epoch
        self.rng = np.random.default_rng(seed)
        self.m = torch.zeros_like(model.params)
        self.v = torch.zeros_like(model.params)
        self.gscale = torch.zeros(model.T, dtype=torch.float32, device=model.device)
        self.losses: List[float] = []

    def create_cell(self, k):
        self.model.create_cell(k)

    def begin_stage(self, lr, gscale):
        self.lr, self.t = lr, 0
        self.m.zero_()
        self.v.zero_()
        self.gscale.copy_(torch.as_tensor(gscale))

    def step(self, batch):
        loss = self.model.loss_and_grad(batch, self.task, self.lasso_lam, self.gscale)
        self.t += 1
        adam_step(self.model.params, self.model.grads, self.m, self.v, self.t, lr=self.lr, eps=KERAS_EPS)
        return loss

    def train_epoch(self):
        order = torch.as_tensor(self.rng.permutation(self.train.shape[0]), device=self.train.device)
        tot = None
        for i in range(self.steps):
            idx = order[(i * self.batch) % len(order):][:self.batch]
            loss = self.step(self.train.index_select(0, idx))
            tot = loss.sum() if tot is None else tot + loss.sum()
        self.losses.append(float(tot) / max(1, self.steps))

    def validate(self):
        return evaluate(self.model, self.val, self.task, self.lasso_lam, self.val_batch)[-1]

    def save(self, path):
        np.savez(path, **self.model.state_dict())

    def load(self, path):
        with np.load(path) as d:
            self.model.load_state_dict(d)


def evaluate(model, data, task, lasso_lam, batch):
    """Per-layer metric over `data` (mean over rows): NMSE in dB (EvalNMSE) or the Lasso objective (LassoObjective),
    of each layer's x_k (for LAMP too, whose Keras output interleaves v_k)."""
    M, N, K = model.M, model.N, model.num_cells
    acc, rows = torch.zeros(K, dtype=torch.float64, device=data.device), 0
    for i in range(0, data.shape[0], batch):
        d = data[i:i + batch]
        xs = model.forward(d, K).double()
        y, xt = d[:, :M].double(), d[:, M:].double()
        if task == lista.TASK_SC:
            mse = ((xs - xt) ** 2).mean(dim=2) + 1e-10
            m = 10.0 * torch.log10(mse / ((xt ** 2).mean(dim=1) + 1e-10))
        else:
            e = xs @ model.A.double().T - y
            m = 0.5 * (e ** 2).sum(dim=2) + lasso_lam * xs.abs().sum(dim=2)
        acc += m.sum(dim=1)
        rows += d.shape[0]
    return (acc / rows).tolist()


def final_output(model, data, batch):
    """x_K of every row of `data`, `batch` rows per forward (model.predict's output[:, -N:], MB/train.py:249-252)."""
    out = torch.empty(data.shape[0], model.N, dtype=torch.float32, device=data.device)
    for i in range(0, data.shape[0], batch):
        out[i:i + batch] = model.forward(data[i:i + batch], model.num_cells)[-1]   # forward reuses its buffer
    return out


def run(model_name="lista", task="sc", num_layers=16, model_lam=0.4, lasso_lam=0.005, share_W=False,
        ss_q_per_layer=1.2, ss_maxq=13.0, alista_W_file="W.npy", seed=42, base_lr=0.0005, epochs=100000,
        num_train_images=51200, num_val_images=1024, num_test_images=1024, train_batch_size=128,
        val_batch_size=1024, test_batch_size=1024, test=False, test_files=(), base_dir=".", data_dir=".",
        exp_name="lista_sc", replicate=1, device="cuda"):
    """MB/train.py:run with its flags.  Training returns the last validation metric; test mode evaluates the first
    num_test_images rows of each test file in batches of test_batch_size and returns {file: per-layer metrics}."""
    if task == "cs":
        raise NotImplementedError("the cs task (D, PSNR, im2cols) is not supported")
    if task not in ("sc", "lasso"):
        raise ValueError("invalid task type")
    task_id = lista.TASK_SC if task == "sc" else lista.TASK_LASSO
    model_dir = os.path.join(os.path.abspath(base_dir), "models", exp_name, "replicate_%d" % replicate)
    A = np.load(os.path.join(data_dir, "A.npy"), allow_pickle=True).astype(np.float32)
    W = None
    if model_name.startswith("alista"):
        W = np.load(os.path.join(data_dir, alista_W_file), allow_pickle=True).astype(np.float32)
    model = build_model(model_name, A, num_layers, model_lam, share_W, ss_q_per_layer, ss_maxq, W, device)
    load = lambda f: torch.as_tensor(np.load(os.path.join(data_dir, f), allow_pickle=True).astype(np.float32),
                                     device=device).contiguous()
    if test:
        if last_complete_layer(model_dir, num_layers) != num_layers:
            raise ValueError("Should have a fully trained model!")
        for k in range(num_layers):
            model.create_cell(k)
        with np.load(os.path.join(model_dir, "layer_%d" % num_layers, "model.npz")) as d:
            model.load_state_dict(d)
        res = {}
        for f in test_files:
            data = load(f)[:num_test_images]
            res[f] = evaluate(model, data, task_id, lasso_lam, test_batch_size)
            name = "lasso" if task == "lasso" else "nmse"
            print("%s : %s" % (f, " ".join("%s_layer%d=%.6f" % (name, i, v) for i, v in enumerate(res[f]))))
            if task == "lasso":
                out = final_output(model, data, test_batch_size)
                base = os.path.basename(f)
                base = base[:-4] if base.endswith(".npy") else base
                np.save(os.path.join(model_dir, base + "_final_output.npy"), out.cpu().numpy())
        return res
    train = load("train_data.npy")[:num_train_images]
    val = load("val_data.npy")[:num_val_images]
    trainer = KernelTrainer(model, train, val, task_id, lasso_lam, train_batch_size, val_batch_size,
                            num_train_images // train_batch_size, seed)
    return train_layerwise(trainer, num_layers, base_lr, epochs, model_dir)


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("--model_name", default="lista", choices=["lista", "lista_cp", "lista_cpss", "alista", "lfista",
                                                                   "lamp"])
    p.add_argument("--num_layers", type=int, default=16)
    p.add_argument("--model_lam", type=float, default=0.4)
    p.add_argument("--share_W", action="store_true")
    p.add_argument("--task", default="sc", choices=["sc", "lasso", "cs"])
    p.add_argument("--lasso_lam", type=float, default=0.005)
    p.add_argument("--alista_W_file", default="W.npy")
    p.add_argument("--ss_q_per_layer", type=float, default=1.2)
    p.add_argument("--ss_maxq", type=float, default=13.0)
    p.add_argument("--seed", type=int, default=42)
    p.add_argument("--base_lr", type=float, default=0.0005)
    p.add_argument("--epochs", type=int, default=100000)
    p.add_argument("--num_train_images", type=int, default=51200)
    p.add_argument("--num_val_images", type=int, default=1024)
    p.add_argument("--num_test_images", type=int, default=1024)
    p.add_argument("--train_batch_size", type=int, default=128)
    p.add_argument("--val_batch_size", type=int, default=1024)
    p.add_argument("--test_batch_size", type=int, default=1024)
    p.add_argument("--test_files", action="append", default=[])
    p.add_argument("--test", action="store_true")
    p.add_argument("--base_dir", default=".")
    p.add_argument("--data_dir", default=".")
    p.add_argument("--exp_name", default="lista_sc")
    p.add_argument("--replicate", type=int, default=1)
    a = p.parse_args(argv)
    logging.basicConfig(level=logging.INFO, format="%(message)s")
    return run(**vars(a))


if __name__ == "__main__":
    main()
