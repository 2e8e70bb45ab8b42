"""CPU: the CoordinatewiseRNN oracle (oracle/crnn_oracle.py) and the package's CPU-side pieces (argument checks, theta
layout, the ctypes ABI of the new entry points)."""
import ctypes
import json
import math
import os
import re

import pytest
import torch

from oracle import crnn_oracle as CR
from open_l2o_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(HERE), "include", "l2o_b200.h")


def test_cell_reproduces_the_hand_vectors():
    for case in json.load(open(os.path.join(HERE, "golden", "lstm_cell_hand.json"))):
        t = lambda k: torch.tensor(case[k], dtype=torch.float64)
        h, c = CR.lstm_cell(t("x"), t("h"), t("c"), t("w"), t("b"))
        assert torch.allclose(h, t("h_next"), atol=1e-14, rtol=0), case["name"]
        assert torch.allclose(c, t("c_next"), atol=1e-14, rtol=0), case["name"]


def _problem(seed, shapes=((7, 3), (5,)), dtype=torch.float64):
    gen = torch.Generator().manual_seed(seed)
    theta = CR.init_theta(seed, dtype=dtype)
    P = CR.unpack_theta(theta)
    params = [torch.randn(s, generator=gen, dtype=dtype) for s in shapes]
    states = [CR.initial_state(P, p.numel(), gen, dtype=dtype) for p in params]
    grads = [torch.randn(s, generator=gen, dtype=dtype) * 3 for s in shapes]
    return theta, params, states, grads


def test_first_step_scales_by_asinh_and_keeps_ms_at_one():
    theta, params, states, grads = _problem(0)
    P = CR.unpack_theta(theta)
    for g, st in zip(grads, states):
        s, ms = CR.rms_scaling(g, st["decay"], st["rms"])
        assert torch.allclose(ms, torch.ones_like(ms), atol=0, rtol=0)   # decay = rms = 1: ms' = ms = 1
        assert torch.allclose(s.reshape(-1), torch.asinh(g.reshape(-1) / math.sqrt(1 + 1e-16)), atol=1e-13)
    _, new, _ = CR.step(theta, params, grads, states)
    for st in new:
        assert torch.equal(st["rms"], torch.ones_like(st["rms"]))


def test_learning_rate_change_is_bounded():
    theta, params, states, grads = _problem(1)
    P = CR.unpack_theta(theta)
    P["learning_rate_weights"].copy_(torch.randn(20, 1, dtype=torch.float64) * 2)    # init makes the ratio exactly 1
    for _ in range(3):
        old = [s["learning_rate"] for s in states]
        params, states, _ = CR.step(theta, params, grads, states)
        for o, s in zip(old, states):
            r = s["learning_rate"] / o
            assert float(r.min()) > 0 and float(r.max()) < 2
            assert float((r - 1).abs().max()) > 1e-3


def test_rnn_slot_packs_c_before_h():
    theta, params, states, grads = _problem(2)
    P = CR.unpack_theta(theta)
    _, new, _ = CR.step(theta, params, grads, states)
    g, st = grads[0], states[0]
    s, _ = CR.rms_scaling(g, st["decay"], st["rms"])
    h1, c1 = CR.lstm_cell(s, st["rnn"][:, 10:20], st["rnn"][:, 0:10], P["cell_0/kernel"], P["cell_0/bias"])
    assert torch.equal(new[0]["rnn"][:, 0:10], c1) and torch.equal(new[0]["rnn"][:, 10:20], h1)
    assert not torch.allclose(c1, h1)


def test_all_zero_ms_predicate_is_literal():
    theta, params, states, grads = _problem(3)
    st = dict(states[0])
    st["rms"] = torch.zeros_like(st["rms"])
    st["decay"] = torch.full_like(st["decay"], 0.5)
    _, ms = CR.rms_scaling(grads[0], st["decay"], st["rms"])
    assert torch.allclose(ms.reshape(-1), grads[0].reshape(-1) ** 2 + 1e-12)   # decay forced to 0
    st["rms"][0] = 1.0                                                           # not ALL zero: decay 0.5 applies
    _, ms = CR.rms_scaling(grads[0], st["decay"], st["rms"])
    assert torch.allclose(ms[1:].reshape(-1), 0.5 * (grads[0].reshape(-1)[1:] ** 2 + 1e-12))


def test_fp32_oracle_agrees_with_fp64():
    th64, p64, s64, g64 = _problem(4)
    th32 = th64.float()
    p32 = [p.float() for p in p64]
    s32 = [{k: v.float() for k, v in s.items()} for s in s64]
    g32 = [g.float() for g in g64]
    for _ in range(4):
        p64, s64, _ = CR.step(th64, p64, g64, s64)
        p32, s32, _ = CR.step(th32, p32, g32, s32)
    for a, b in zip(p32, p64):
        assert float((a.double() - b).abs().max() / b.abs().max()) < 1e-5
    for a, b in zip(s32, s64):
        for k in a:
            assert float((a[k].double() - b[k]).abs().max() / b[k].abs().max()) < 1e-5, k


def test_theta_layout_matches_the_spec():
    from open_l2o_b200 import coordinatewise_rnn as cw
    assert CR.theta_count() == 6402
    assert sum(math.prod(s) for _, s in cw.THETA_SPEC) == 6402
    assert [s for _, s in cw.THETA_SPEC] == [s for _, s in CR.theta_spec()]
    short = [n.split("/")[-1] for n, _ in cw.THETA_SPEC]
    assert short[:6] == ["update_weights", "decay_weights", "decay_bias", "learning_rate_weights",
                         "learning_rate_bias", "init_vector"]
    assert cw.theta_spec("BasicLSTMCell")[-1][0] == "LOL/multi_rnn_cell/cell_2/basic_lstm_cell/bias"
    th = cw._init_theta(0, zero_init_lr_weights=True)
    o = dict(zip([n for n, _ in cw.THETA_SPEC], torch.split(th, [math.prod(s) for _, s in cw.THETA_SPEC])))
    assert float(o["LOL/decay_bias"]) == pytest.approx(2.2)
    assert float(o["LOL/learning_rate_weights"].abs().max()) == 0.0
    lim = math.sqrt(6 / (11 + 40))
    k0 = o["LOL/multi_rnn_cell/cell_0/lstm_cell/kernel"]
    assert float(k0.abs().max()) <= lim and float(k0.abs().max()) > 0.8 * lim


def test_constructor_checks():
    from open_l2o_b200.coordinatewise_rnn import CoordinatewiseRNN, metarun_args
    with pytest.raises(TypeError, match="CR:99"):
        CoordinatewiseRNN([10, 20, 20], "GRUCell")
    with pytest.raises(ValueError):
        CoordinatewiseRNN([10, 20, 20], "LSTMCell", init_lr_range=(1.0,))
    with pytest.raises(ValueError):
        CoordinatewiseRNN([10, 20, 20], "LSTMCell", init_lr_range=(1.0, 0.5))
    with pytest.raises(NotImplementedError, match="cell_sizes"):
        CoordinatewiseRNN([20, 20], "LSTMCell")
    with pytest.raises(NotImplementedError, match="learnable_decay"):
        CoordinatewiseRNN([10, 20, 20], "LSTMCell", learnable_decay=False)
    with pytest.raises(NotImplementedError, match="dynamic_output_scale"):
        CoordinatewiseRNN([10, 20, 20], "LSTMCell", dynamic_output_scale=False)
    with pytest.raises(NotImplementedError):
        CoordinatewiseRNN([10, 20, 20], "LSTMBlockCell")
    args = metarun_args()
    assert args["cell_cls"] == "LSTMCell" and args["cell_sizes"] == [10, 20, 20]
    assert args["init_lr_range"] == (1e-6, 1e-2) and args["zero_init_lr_weights"] is True


def _struct_fields(name):
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    m = re.search(r"typedef struct\s*\{([^}]*)\}\s*%s\s*;" % name, src)
    assert m, name
    return [re.findall(r"[A-Za-z_][A-Za-z_0-9]*", d.strip())[-1] for d in m.group(1).split(";") if d.strip()]


def test_crnn_ctypes_structs_follow_the_header():
    for cname, cls in [("l2o_crnn_step_args", _lib.CrnnStepArgs), ("l2o_crnn_bwd_args", _lib.CrnnBwdArgs)]:
        assert [f[0] for f in cls._fields_] == _struct_fields(cname), cname


def test_crnn_entry_points_validate_without_gpu():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    assert L.l2o_crnn_theta_count() == 6402 and L.l2o_crnn_state_floats() == 103
    E = _lib.L2O_E_INVALID
    buf = (ctypes.c_double * 8)()
    base = ctypes.addressof(buf)                 # host addresses: validation must reject before any CUDA call
    good = dict(n=4, theta=base, g=base, state_in=base, state_out=base, x=None, update=None)
    assert L.l2o_crnn_step(None, None) == E
    for k in ("theta", "g", "state_in", "state_out"):
        a = _lib.CrnnStepArgs(**dict(good, **{k: None}))
        assert L.l2o_crnn_step(ctypes.byref(a), None) == E, k
    for n in (0, -3):
        assert L.l2o_crnn_step(ctypes.byref(_lib.CrnnStepArgs(**dict(good, n=n))), None) == E
    for k in ("theta", "g", "state_in", "state_out", "x", "update"):
        a = _lib.CrnnStepArgs(**dict(good, **{k: base + 2}))
        assert L.l2o_crnn_step(ctypes.byref(a), None) == E, k
    bgood = dict(n=4, theta=base, g=base, state_old=base, d_state_new=base, d_update=base, d_state_old=base,
                 d_theta=base)
    assert L.l2o_crnn_bwd(None, None) == E
    for k in bgood:
        if k == "n":
            continue
        assert L.l2o_crnn_bwd(ctypes.byref(_lib.CrnnBwdArgs(**dict(bgood, **{k: None}))), None) == E, k
        assert L.l2o_crnn_bwd(ctypes.byref(_lib.CrnnBwdArgs(**dict(bgood, **{k: base + 2}))), None) == E, k
    assert L.l2o_crnn_bwd(ctypes.byref(_lib.CrnnBwdArgs(**dict(bgood, d_theta=base + 4))), None) == E
    assert L.l2o_crnn_bwd(ctypes.byref(_lib.CrnnBwdArgs(**dict(bgood, n=0))), None) == E
