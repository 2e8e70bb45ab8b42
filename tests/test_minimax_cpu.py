"""CPU: the Twin-L2O oracle's closed forms, the host logic of open_l2o_b200.minimax and the ABI's argument checks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import minimax_oracle as MO


def _zero_out_nets(H, bias):
    nets = []
    for _ in (0, 1):
        net = MO.Net(H).double()
        with torch.no_grad():
            net.output.weight.zero_()
            net.output.bias.fill_(bias)
        nets.append(net)
    return nets


def _start(B, dim, H, seed=0):
    g = torch.Generator().manual_seed(seed)
    u0 = list(torch.rand(B, dim, generator=g, dtype=torch.float64) - 0.5)
    v0 = list(torch.rand(B, dim, generator=g, dtype=torch.float64) - 0.5)
    st = {n: ([torch.randn(B * dim, H, generator=g, dtype=torch.float64) * 0.01 for _ in range(2)],
              [torch.randn(B * dim, H, generator=g, dtype=torch.float64) * 0.01 for _ in range(2)]) for n in (0, 1)}
    return u0, v0, st


@pytest.mark.parametrize("bias", [0.3, -0.2])
def test_oracle_sign_steps_then_bias_steps(bias):
    optim_it, B = 30, 3
    nets = _zero_out_nets(8, bias)
    u0, v0, st = _start(B, 1, 8)
    data = [torch.tensor([1.0, 0.7], dtype=torch.float64)] * B
    recs, _ = MO.do_fit(nets, 1, data, u0, v0, st, 3, optim_it, 1e-4, train=False)
    lr = MO.sche_lr(optim_it)
    u, v = torch.stack(u0), torch.stack(v0)
    for t in range(1, optim_it + 1):
        step = float(np.sign(bias)) * lr[t - 1] if t < 0.2 * optim_it else bias
        if t % 2:
            u = u + step
        else:
            v = v + step
        assert torch.allclose(recs[t - 1]["u"], u, atol=1e-12) and torch.allclose(recs[t - 1]["v"], v, atol=1e-12)


def test_boundary_update_gets_no_meta_gradient():
    # optim_it 60, unroll 6: sign steps t < 12, boundary at 12.  The boundary's update is the first one that is not a
    # sign step, yet it runs after the first segment's backward and is detached: segment 1's gradient is exactly 0
    # (sign passes zeros), and segment 2's is not
    nets = [MO.Net(6).double() for _ in (0, 1)]
    u0, v0, st = _start(2, 1, 6)
    data = [torch.tensor([1.0, 0.7], dtype=torch.float64)] * 2
    _, segs = MO.do_fit(nets, 2, data, u0, v0, st, 6, 60, 1e-4, train=True)
    assert len(segs) == 5
    assert all(float(g.abs().max()) == 0.0 for n in (0, 1) for g in segs[0][n])
    assert all(float(g.abs().max()) > 0.0 for n in (0, 1) for g in segs[1][n])


@pytest.mark.parametrize("optim_it,n,last_warm", [(100, 20, 19), (1000, 200, 199)])
def test_sche_lr_length_and_indexing(optim_it, n, last_warm):
    from open_l2o_b200 import minimax as mm
    lr = mm.sche_lr(optim_it)
    assert len(lr) == n and lr[0] == 1e-4 and lr[-1] < 1e-1
    assert mm.warm_end(optim_it) == last_warm + 1
    assert MO.is_warm(last_warm, optim_it) and not MO.is_warm(last_warm + 1, optim_it)
    assert lr[last_warm - 1] == MO.sche_lr(optim_it)[last_warm - 1]   # the last sign step's size


def test_loss3_distance_search():
    from open_l2o_b200 import minimax as mm
    assert mm.loss3_distance(0.0, 2.0) == 0.0
    assert abs(mm.loss3_distance(1.2, 2.0) - 0.2) < 1e-12   # nearest k / a is 1.0
    assert abs(mm.loss3_distance(0.3, 2.0) - 0.2) < 1e-12   # 0.5
    assert mm.loss3_distance(0.3, -1.0) == 0.3              # k / a moves away: only k = 0
    for s, a in ((0.77, 1.3), (2.9, 0.6)):
        assert mm.loss3_distance(s, a) == MO.loss3_distance(s, a)
        assert abs(mm.loss3_distance(s, a) - min(abs(s - k / a) for k in range(50))) < 1e-12


def test_get_index_keeps_the_lowest_scores():
    from open_l2o_b200 import minimax as mm
    rng = np.random.RandomState(0)
    B, T = 10, 20
    traj = rng.uniform(-1, 1, (B, T))
    a, b = rng.uniform(0.5, 1.5, B), rng.uniform(0.5, 1.0, B)
    keep = mm.get_index(traj, a, b, 10, 5, 0.5)
    score = [sum((b[i] * np.sin(a[i] * np.pi * x)) ** 2 for x in traj[i, :9]) for i in range(B)]
    assert sorted(keep) == sorted(np.argsort(score)[:5].tolist())
    assert len(mm.get_index(traj, a, b, 10, 5, 0.05)) == B   # int(ratio B) = 0 keeps every problem
    assert mm.sche_ratio(0) == 0.2 and mm.sche_ratio(80) == 1.0 and mm.sche_ratio(81) == 1


def test_matrix_game_data_shapes_and_sparsity():
    from open_l2o_b200 import minimax as mm
    d = mm.make_matrix_game_data(5, 0.5, 0.5, 1.0, 400, seed=1)
    assert d.shape == (400, 25)
    nz = d[d != 0]
    assert nz.min() >= 0.5 and nz.max() < 1.0
    assert abs((d != 0).mean() - 0.5) < 0.03
    assert (mm.make_matrix_game_data(1, 1.0, 0.5, 1.0, 8, seed=2) != 0).all()
    np.testing.assert_array_equal(d, mm.make_matrix_game_data(5, 0.5, 0.5, 1.0, 400, seed=1))


CONFIGS = {
    "toy_train": {"seed": 0, "use_second": 1, "meta_lr": 0.0001, "batch_size": 128, "n_train": 128,
                  "train_epochs": 200, "train_optim_iter": 100, "eval_optim_iter": 1000, "n_eval": 20, "save_train": 1,
                  "hidden_size": 50, "loss": 3, "save_curve": 1, "unroll_unit": 5, "rescale": 0.0001, "CL": 1,
                  "mode": "train", "train_data_path": "t.txt", "eval_data_path": "e.txt", "save_name": "twin_seesaw_CL",
                  "load_name": ""},
    "toy_test": {"seed": 0, "use_second": 1, "test_optim_iter": 2000, "test_epochs": 5, "n_test": 100,
                 "hidden_size": 50, "loss": 3, "unroll_unit": 5, "save_curve": 1, "rescale": 0.0001, "CL": 0,
                 "mode": "test", "test_data_path": "t.txt", "save_name": "twin_seesaw", "load_name": "twin_seesaw",
                 "load_model": "best"},
    "matrix_train": {"seed": 0, "use_second": 1, "save_curve": 1, "save_train": 1, "meta_lr": 0.0001,
                     "batch_size": 128, "n_train": 128, "train_epochs": 300, "train_optim_iter": 100,
                     "eval_optim_iter": 1000, "n_eval": 20, "hidden_size": 80, "loss": 4, "unroll_unit": 5,
                     "rescale": 0.0001, "CL": 0, "mode": "train", "train_data_path": "t.txt",
                     "eval_data_path": "e.txt", "save_name": "twin_matrix_game_dim5", "load_name": "", "dim": 5},
    "matrix_test": {"seed": 0, "use_second": 1, "test_optim_iter": 2000, "test_epochs": 5, "n_test": 100,
                    "hidden_size": 80, "loss": 4, "unroll_unit": 5, "save_curve": 1, "rescale": 0.0001, "CL": 0,
                    "mode": "test", "test_data_path": "t.txt", "save_name": "m", "load_name": "m",
                    "load_model": "best", "dim": 5},
}


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_config_parsing(name):
    from open_l2o_b200 import minimax_train as tr
    p = tr.parse_config(CONFIGS[name])
    assert p["dim"] == CONFIGS[name].get("dim", 1)
    bad = dict(CONFIGS[name])
    del bad["hidden_size"]
    with pytest.raises(KeyError):
        tr.parse_config(bad)


def test_state_dict_names_and_shapes():
    from open_l2o_b200 import minimax as mm
    for H in (50, 80):
        ref = MO.Net(H)
        spec = mm.param_spec(H)
        assert [(k, tuple(v.shape)) for k, v in ref.state_dict().items()] == [(k, tuple(s)) for k, s in spec]
        assert sum(int(np.prod(s)) for _, s in spec) == 12 * H * H + 25 * H + 1


def _lib_or_skip():
    from open_l2o_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built (run __graft_entry__.build())")
    return _lib, _lib.lib()


def test_abi_argument_errors():
    _lib, L = _lib_or_skip()
    for H in (50, 80, 128):
        assert L.l2o_minimax_theta_count(H) == 12 * H * H + 25 * H + 1
    buf = (C.c_float * 64)()
    p = C.cast(buf, C.c_void_p)

    def args(**kw):
        a = _lib.MinimaxArgs()
        a.loss, a.batch, a.dim, a.hidden, a.t0, a.t1, a.warm_end = 1, 4, 1, 50, 1, 3, 1
        a.out_mul, a.rescale = 1.0, 1e-4
        a.image, a.data, a.u, a.v, a.state = p, p, p, p, p
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    nb = C.c_size_t()
    ok = args()
    assert L.l2o_minimax_workspace_bytes(C.byref(ok), C.byref(nb)) == _lib.L2O_OK
    assert nb.value == 8 * 2 * 4 * (8 * 50 + 1 + 4 * 50 + 5)
    invalid = [dict(loss=0), dict(loss=5), dict(batch=0), dict(dim=0), dict(hidden=0), dict(t0=0), dict(t1=1),
               dict(warm_end=0), dict(image=None), dict(data=None), dict(u=None), dict(state=None),
               dict(warm_end=2), dict(u=C.c_void_p(p.value + 2))]
    for kw in invalid:
        a = args(**kw)
        assert L.l2o_minimax_workspace_bytes(C.byref(a), C.byref(nb)) == _lib.L2O_E_INVALID, kw
        assert L.l2o_minimax_fwd(C.byref(a), None) == _lib.L2O_E_INVALID, kw
    for kw in (dict(hidden=129), dict(loss=4, dim=33), dict(loss=3, dim=2)):
        a = args(**kw)
        assert L.l2o_minimax_fwd(C.byref(a), None) == _lib.L2O_E_UNSUPPORTED, kw
    a = args(loss=4, dim=32, hidden=128)
    assert L.l2o_minimax_workspace_bytes(C.byref(a), C.byref(nb)) == _lib.L2O_OK
    g = _lib.MinimaxGrads()
    assert L.l2o_minimax_bwd(C.byref(ok), None, None) == _lib.L2O_E_INVALID
    assert L.l2o_minimax_bwd(C.byref(ok), C.byref(g), None) == _lib.L2O_E_INVALID   # no theta, ckpt, dl, coef
    assert L.l2o_minimax_image(None, p, 50, None) == _lib.L2O_E_INVALID
    assert L.l2o_minimax_image(p, p, 129, None) == _lib.L2O_E_UNSUPPORTED
