"""GPU: the Twin-L2O command line end to end (training with and without the curriculum, evaluation, checkpoints,
test mode) on generated problem files, and Unroll's checks of its problem data."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import minimax_oracle as MO

pytestmark = pytest.mark.gpu


def _toy_file(path, n, seed):
    rng = np.random.RandomState(seed)
    np.savetxt(path, np.stack([rng.uniform(0.5, 1.5, n), rng.uniform(0.5, 1.0, n)], 1))
    return str(path)


def _train_config(tmp_path, name, **kw):
    cfg = {"seed": 0, "use_second": 1, "meta_lr": 0.001, "batch_size": 16, "n_train": 32, "train_epochs": 2,
           "train_optim_iter": 20, "eval_optim_iter": 40, "n_eval": 8, "save_train": 1, "hidden_size": 16, "loss": 3,
           "save_curve": 1, "unroll_unit": 5, "rescale": 0.0001, "CL": 0, "mode": "train", "save_name": name,
           "load_name": ""}
    cfg.update(kw)
    path = tmp_path / (name + ".json")
    path.write_text(json.dumps(cfg))
    return str(path), cfg


def _run(argv, capsys):
    from open_l2o_b200 import minimax_train as tr
    tr.main(argv)
    return capsys.readouterr().out


def _check_checkpoints(out_dir, epochs, hidden):
    names = ["epoch%d%s.pth" % (e, s) for e in range(epochs) for s in ("min", "max")] + ["bestmin.pth", "bestmax.pth"]
    for name in names:
        sd = torch.load(os.path.join(out_dir, name), map_location="cpu")
        net = MO.Net(hidden)
        net.load_state_dict(sd)   # the reference's Optimizer layout: names and shapes
        assert all(torch.isfinite(p).all() for p in net.parameters()), name
    first, last = (torch.load(os.path.join(out_dir, "epoch%dmin.pth" % e)) for e in (0, epochs - 1))
    assert any(not torch.equal(first[k], last[k]) for k in first)   # training moved the weights


@pytest.mark.parametrize("cl", [0, 1])
def test_seesaw_config_trains_evaluates_and_tests(tmp_path, capsys, cl):
    name = "twin_seesaw_CL" if cl else "twin_seesaw"
    train = _toy_file(tmp_path / "train.txt", 32, 1)
    evald = _toy_file(tmp_path / "eval.txt", 8, 2)
    path, cfg = _train_config(tmp_path, name, CL=cl, train_data_path=train, eval_data_path=evald)
    result = str(tmp_path / "result")
    out = _run(["--config", path, "--eval_interval", "1", "--result_dir", result], capsys)
    assert "best eval score" in out and out.count("eval score") == 3
    _check_checkpoints(os.path.join(result, name), 2, 16)

    test_cfg = {"seed": 0, "use_second": 1, "test_optim_iter": 30, "test_epochs": 2, "n_test": 8, "hidden_size": 16,
                "loss": 3, "unroll_unit": 5, "save_curve": 1, "rescale": 0.0001, "CL": 0, "mode": "test",
                "test_data_path": evald, "save_name": name, "load_name": name, "load_model": "best"}
    tpath = tmp_path / "test.json"
    tpath.write_text(json.dumps(test_cfg))
    out = _run(["--config", str(tpath), "--result_dir", result], capsys)
    assert "test score per epoch" in out


def test_matrix_game_config_trains(tmp_path, capsys):
    from open_l2o_b200 import minimax as mm
    train, evald = tmp_path / "dim5_train.txt", tmp_path / "dim5_eval.txt"
    np.savetxt(train, mm.make_matrix_game_data(5, 0.5, 0.5, 1.0, 32, seed=0))
    np.savetxt(evald, mm.make_matrix_game_data(5, 0.5, 0.5, 1.0, 8, seed=1))
    path, _ = _train_config(tmp_path, "twin_matrix_game_dim5", loss=4, dim=5, hidden_size=24, train_epochs=1,
                            train_data_path=str(train), eval_data_path=str(evald))
    result = str(tmp_path / "result")
    _run(["--config", path, "--result_dir", result], capsys)
    for side in ("min", "max"):
        sd = torch.load(os.path.join(result, "twin_matrix_game_dim5", "best%s.pth" % side))
        MO.Net(24).load_state_dict(sd)


def test_curriculum_rejects_matrix_games():
    from open_l2o_b200 import minimax as mm, minimax_train as tr
    twin = mm.TwinOptimizer(8, "cuda", seed=0)
    data = mm.problem_tensor(mm.make_matrix_game_data(5, 0.5, 0.5, 1.0, 4, seed=0), 4, 5, "cuda")
    with pytest.raises(ValueError):
        tr.do_fit(twin, tr.make_meta_opts(twin, 1e-3), 4, data, 5, 5, 20, True, cl_ratio=0.5)


def test_unroll_rejects_data_the_kernels_cannot_read():
    from open_l2o_b200 import minimax as mm
    twin = mm.TwinOptimizer(8, "cuda", seed=0)
    good = torch.rand(6, 2, device="cuda")
    mm.Unroll(twin, 1, good)
    for bad in (good.double(), good.cpu(), torch.rand(2, 6, device="cuda").t(), torch.rand(6, 3, device="cuda"),
                torch.rand(6, 5, 5, device="cuda")):
        with pytest.raises(ValueError):
            mm.Unroll(twin, 1, bad)
    with pytest.raises(ValueError):
        mm.Unroll(twin, 4, torch.rand(6, 5, 4, device="cuda"), dim=5)
    with pytest.raises(ValueError):
        mm.Unroll(twin, 3, good, dim=2)
    mm.Unroll(twin, 4, torch.rand(6, 5, 5, device="cuda"), dim=5)
