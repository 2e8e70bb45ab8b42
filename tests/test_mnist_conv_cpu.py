"""CPU tests of problems.mnist_conv and the registry entry mnist_conv (DM/problems.py:291-347, DM/util.py:164-169), and
of the l2o_mnist_conv_grad ABI without a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from open_l2o_b200 import _lib, mnist_data, problems, util
from open_l2o_b200.variables import variable_getter
from tests.mnist_fixture import write_mnist

NAMES = ["conv_layer1/weights1", "conv_layer1/biases1", "conv_layer2/weights1", "conv_layer2/biases1", "fc_weights",
         "fc_bias"]
SHAPES = [(3, 3, 1, 16), (16,), (5, 5, 16, 32), (32,), (512, 10), (10,)]


def _run(build, params=None):
    """Run build() with CPU tensors for its variables; returns ({name: tensor}, loss, the indices drawn)."""
    made = {}

    def getter(name, shape, dtype, initializer, trainable):
        assert trainable, name   # the data are not variables
        if name not in made:
            made[name] = params[name] if params is not None else initializer(shape, torch.Generator().manual_seed(
                len(made)))
        return made[name]

    drawn = []
    real = torch.randint

    def spy(*a, **k):
        out = real(*a, **k)
        drawn.append(out.clone())
        return out

    with variable_getter(getter):
        torch.randint = spy
        try:
            loss = build()
        finally:
            torch.randint = real
    return made, loss, drawn[-1]


def test_registry_producer_matches_the_reference(tmp_path):
    write_mnist(str(tmp_path))
    problem, net_config, assignments = util.get_config("mnist_conv", data_dir=str(tmp_path))
    assert assignments is None and net_config == {"cw": util.get_default_net_config(None)}
    p = problem.producer
    assert p.kind == "mnist_conv" and p.batch_norm is True and p.batch_size == 128
    assert p.mode == "train" and p.data_dir == str(tmp_path)
    assert util.get_config("mnist_conv", path="/some/net", data_dir=str(tmp_path))[0].producer.mode == "test"
    assert util.get_config("mnist_conv", path="/some/net", mode="validation",
                           data_dir=str(tmp_path))[0].producer.mode == "validation"
    rp = util.get_config("mnist_conv", net_name="RNNprop", data_dir=str(tmp_path))[1]
    assert list(rp) == ["rp"] and rp["rp"]["net"] == "RNNprop"
    made, loss, idx = _run(problem)
    assert list(made) == NAMES and [tuple(v.shape) for v in made.values()] == SHAPES
    assert sum(v.numel() for v in made.values()) == 18122 == _lib.MNIST_CONV_COORDS
    for name, v in made.items():   # weights N(0, 0.01), biases zero (DM/problems.py:312-318,330-337)
        if v.dim() == 1:
            assert torch.count_nonzero(v) == 0, name
        else:
            assert abs(float(v.std()) - 0.01) < 0.2 * 0.01 and abs(float(v.mean())) < 0.005, name
    assert idx.shape == (128,) and int(idx.max()) < 1000
    assert loss.shape == () and np.isfinite(float(loss))


def test_missing_directory_fails_before_anything_runs(tmp_path):
    with pytest.raises(FileNotFoundError, match=re.escape(str(tmp_path / "nowhere"))):
        util.get_config("mnist_conv", data_dir=str(tmp_path / "nowhere"))


def numpy_forward(params, pixels, labels):
    """DM/problems.py:302-345 in float64 NumPy with explicit loops over the VALID windows (HWIO weights, NHWC)."""
    w1, b1, w2, b2, wf, bf = [np.asarray(p, dtype=np.float64) for p in params]
    B = pixels.shape[0]
    h = pixels.astype(np.float64).reshape(B, 28, 28, 1)

    def conv(x, w, b):
        k = w.shape[0]
        H = x.shape[1] - k + 1
        out = np.zeros((B, H, H, w.shape[3]))
        for i in range(H):
            for j in range(H):
                win = x[:, i:i + k, j:j + k, :]                          # [B, k, k, C_in]
                out[:, i, j, :] = np.tensordot(win, w, axes=([1, 2, 3], [0, 1, 2]))
        return out + b

    def bn_relu_pool(z):
        mu = z.mean(axis=(0, 1, 2))
        var = ((z - mu) ** 2).mean(axis=(0, 1, 2))                       # biased
        a = np.maximum((z - mu) / np.sqrt(var + 1e-3), 0.0)
        P = z.shape[1] // 2                                              # VALID: 9 -> 4 drops row / column 8
        out = np.zeros((B, P, P, z.shape[3]))
        for i in range(P):
            for j in range(P):
                out[:, i, j, :] = a[:, 2 * i:2 * i + 2, 2 * j:2 * j + 2, :].max(axis=(1, 2))
        return out

    h = bn_relu_pool(conv(h, w1, b1))
    h = bn_relu_pool(conv(h, w2, b2))
    assert h.shape == (B, 4, 4, 32)
    logits = np.maximum(h.reshape(B, -1) @ wf + bf, 0.0)                 # NHWC flatten, then the logits' ReLU
    m = logits.max(axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(logits - m).sum(axis=1))
    return float(np.mean(lse - logits[np.arange(B), labels]))


def test_torch_build_equals_a_numpy_forward_of_the_spec(tmp_path):
    write_mnist(str(tmp_path), seed=4)
    build = problems.mnist_conv(batch_size=16, data_dir=str(tmp_path))
    gen = torch.Generator().manual_seed(11)
    params = {n: torch.randn(s, generator=gen, dtype=torch.float64) * (0.3 if len(s) > 1 else 0.5)
              for n, s in zip(NAMES, SHAPES)}
    torch.manual_seed(1)
    _, loss, idx = _run(build, params)
    d = mnist_data.load_mnist(str(tmp_path))["train"]
    ref = numpy_forward([params[n].numpy() for n in NAMES], d.pixels()[idx.numpy()], d.labels[idx.numpy()])
    assert abs(float(loss) - ref) <= 1e-10 * abs(ref), (float(loss), ref)


def test_without_batch_norm_builds_and_its_producer_keeps_the_flag(tmp_path):
    write_mnist(str(tmp_path))
    build = problems.mnist_conv(batch_norm=False, data_dir=str(tmp_path))
    assert build.producer.batch_norm is False
    made, loss, _ = _run(build)
    assert list(made) == NAMES and np.isfinite(float(loss))


def test_mnist_conv_args_follow_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(_lib.INCLUDE, "l2o_b200.h")).read(), flags=re.S)
    m = re.search(r"typedef struct\s*\{([^}]*)\}\s*l2o_mnist_conv_args\s*;", src)
    assert int(re.search(r"#define L2O_MNIST_CONV_LAYOUT (\d+)", src).group(1)) == _lib.MNIST_CONV_LAYOUT
    want = [re.findall(r"[A-Za-z_][A-Za-z_0-9]*", d.strip())[-1] for d in m.group(1).split(";") if d.strip()]
    assert [f[0] for f in _lib.MnistConvArgs._fields_] == want
    assert int(re.search(r"#define L2O_MNIST_CONV_COORDS (\d+)", src).group(1)) == _lib.MNIST_CONV_COORDS
    assert int(re.search(r"#define L2O_MNIST_CONV_MAX_BATCH (\d+)", src).group(1)) == _lib.MNIST_CONV_MAX_BATCH


def test_mnist_conv_grad_validates_without_gpu():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    assert L.l2o_mnist_conv_workspace_bytes(0) == _lib.L2O_E_INVALID
    assert L.l2o_mnist_conv_workspace_bytes(1025) == _lib.L2O_E_INVALID
    sizes = [L.l2o_mnist_conv_workspace_bytes(b) for b in (1, 128, 1024)]
    assert 0 < sizes[0] < sizes[1] < sizes[2] and all(s % 16 == 0 for s in sizes)
    assert L.l2o_mnist_conv_grad(None, None) == _lib.L2O_E_INVALID
    buf = ctypes.create_string_buffer(64)
    base = (ctypes.addressof(buf) + 15) & ~15   # 16-byte aligned

    def args(**kw):
        a = _lib.MnistConvArgs()
        a.batch, a.num_examples = 128, 100
        a.counter = a.images = a.labels = a.x = a.g = a.workspace = base
        a.workspace_bytes = L.l2o_mnist_conv_workspace_bytes(128)
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    for bad in (dict(batch=0), dict(batch=1025), dict(num_examples=0), dict(counter=None), dict(images=None),
                dict(labels=None), dict(x=None), dict(g=None), dict(workspace=None),
                dict(workspace_bytes=L.l2o_mnist_conv_workspace_bytes(128) - 1),
                dict(batch=129), dict(workspace=base + 8), dict(x=base + 4), dict(scale=base + 4), dict(g=base + 2),
                dict(counter=base + 4), dict(f=base + 4), dict(idx_out=base + 2)):
        assert L.l2o_mnist_conv_grad(ctypes.byref(args(**bad)), None) == _lib.L2O_E_INVALID, bad
    off = (ctypes.c_int64 * _lib.MNIST_CONV_LAYOUT)()
    for b in (0, 1025):
        assert L.l2o_mnist_conv_workspace_layout(b, off) == _lib.L2O_E_INVALID
    assert L.l2o_mnist_conv_workspace_layout(128, None) == _lib.L2O_E_INVALID
    from open_l2o_b200.engine import mnist_conv_workspace_layout
    for b in (1, 200, 1024):   # z1, z2, the 96 batch-norm constants and dlogits lie inside the workspace, 16-aligned
        lay = mnist_conv_workspace_layout(b)
        ends = dict(z1=b * 10816 * 4, z2=b * 2592 * 4, bn=96 * 4, dl=b * 16 * 4)
        assert all(lay[k] % 16 == 0 and lay[k] + ends[k] <= L.l2o_mnist_conv_workspace_bytes(b) for k in ends), lay
        spans = sorted((lay[k], lay[k] + ends[k]) for k in ends)
        assert all(e <= s for (_, e), (s, _) in zip(spans, spans[1:])), spans
    from open_l2o_b200.engine import mnist_conv_fits
    assert mnist_conv_fits(1) and mnist_conv_fits(1024) and not mnist_conv_fits(0) and not mnist_conv_fits(1025)
