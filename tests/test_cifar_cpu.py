"""CPU tests of the CIFAR-10 reader (cifar_data), problems.cifar10 and problems.nas and their registry entries
cifar_conv and nas (DM/problems.py:369-458,540-634, DM/util.py:170-175,185-190), their producers' ``accepts``, and the
l2o_cifar_conv_grad and l2o_nas_grad ABIs without a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from open_l2o_b200 import _lib, cifar_data, meta, problems, util
from open_l2o_b200.variables import variable_getter
from tests.cifar_fixture import records, write_cifar10
from tests.mnist_fixture import write_mnist

NAMES = ["conv_layer1/weights1", "conv_layer1/biases1", "conv_layer2/weights1", "conv_layer2/biases1", "fc_weights",
         "fc_bias"]
SHAPES = [(3, 3, 3, 16), (16,), (5, 5, 16, 32), (32,), (32, 10), (10,)]


@pytest.fixture(scope="module")
def data_dir(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("cifar") / "cifar10")
    write_cifar10(d, n_train=1000, n_test=300, seed=3)
    return d


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


# ---- the reader ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("archive", [False, True], ids=["folder", "tarball"])
def test_reader_returns_the_records_of_both_layouts(tmp_path, archive):
    d = str(tmp_path / "cifar10")
    tr_img, tr_lab, te_img, te_lab = write_cifar10(d, n_train=57, n_test=11, seed=1, archive=archive)
    assert os.path.isdir(os.path.join(d, cifar_data.FOLDER)) != archive
    train, test = cifar_data.load_cifar10(d, "train"), cifar_data.load_cifar10(d, "test")
    assert train.images.dtype == np.uint8 and train.images.shape == (57, 3, 32, 32)
    assert np.array_equal(train.images, tr_img) and np.array_equal(train.labels, tr_lab)
    assert np.array_equal(test.images, te_img) and np.array_equal(test.labels, te_lab)
    assert test.num_examples == 11


def test_reader_prefers_the_folder_over_the_tarball(tmp_path):
    d = str(tmp_path)
    write_cifar10(d, n_train=10, n_test=5, seed=1, archive=True)
    folder = write_cifar10(d, n_train=20, n_test=5, seed=2)
    assert np.array_equal(cifar_data.load_cifar10(d, "train").images, folder[0])


def test_pixels_divide_by_255_in_float32_and_read_nhwc(tmp_path):
    img = np.arange(3 * 32 * 32, dtype=np.int64).reshape(1, 3, 32, 32) % 256   # every byte value, many times
    os.makedirs(tmp_path / cifar_data.FOLDER)
    for name in cifar_data.FILES["train"] + cifar_data.FILES["test"]:
        (tmp_path / cifar_data.FOLDER / name).write_bytes(records(img, [7]))
    split = cifar_data.load_cifar10(str(tmp_path), "test")
    px = split.pixels()
    assert px.dtype == np.float32 and px.shape == (1, 32, 32, 3)
    want = img.transpose(0, 2, 3, 1).astype(np.float32) / np.float32(255)
    assert np.array_equal(px, want)
    v = np.arange(256, dtype=np.float32)
    assert np.array_equal(cifar_data.VALUES, v / np.float32(255))
    # the quotient, not the product with 1/255 that MNIST uses: the two differ for some byte values
    assert not np.array_equal(cifar_data.VALUES, v * np.float32(1.0 / 255.0))
    for p in range(256):   # each the correctly rounded quotient: no other fp32 is closer to p / 255
        q = float(cifar_data.VALUES[p])
        for nb in (np.nextafter(np.float32(q), np.float32(2)), np.nextafter(np.float32(q), np.float32(-1))):
            assert abs(q - p / 255) <= abs(float(nb) - p / 255), p


def test_missing_data_names_the_directory_and_the_files(tmp_path):
    where = str(tmp_path / "nowhere")
    with pytest.raises(FileNotFoundError, match=re.escape(where)) as e:
        cifar_data.load_cifar10(where, "train")
    assert "data_batch_1.bin" in str(e.value) and "test_batch.bin" in str(e.value)
    assert cifar_data.ARCHIVE in str(e.value)
    with pytest.raises(FileNotFoundError, match=re.escape(where)):
        util.get_config("cifar_conv", data_dir=where)


def test_bad_record_sizes_and_labels_are_errors_naming_the_file(tmp_path):
    d = tmp_path / "short"
    write_cifar10(str(d), n_train=10, n_test=4)
    bad = d / cifar_data.FOLDER / "test_batch.bin"
    bad.write_bytes(bad.read_bytes()[:-1])
    with pytest.raises(ValueError, match="test_batch.bin"):
        cifar_data.load_cifar10(str(d), "test")
    bad.write_bytes(b"")
    with pytest.raises(ValueError, match="test_batch.bin"):
        cifar_data.load_cifar10(str(d), "test")
    d = tmp_path / "label"
    write_cifar10(str(d), n_train=10, n_test=4)
    bad = d / cifar_data.FOLDER / "data_batch_3.bin"
    raw = bytearray(bad.read_bytes())
    raw[cifar_data.RECORD_BYTES] = 10   # the second record's label
    bad.write_bytes(bytes(raw))
    with pytest.raises(ValueError, match="data_batch_3.bin"):
        cifar_data.load_cifar10(str(d), "train")


def test_only_train_and_test_are_splits(data_dir):
    for mode in ("validation", "eval", ""):
        with pytest.raises(ValueError, match="Mode"):
            cifar_data.load_cifar10(data_dir, mode)
        with pytest.raises(ValueError, match="Mode"):
            problems.cifar10(mode=mode, data_dir=data_dir)


# ---- the registry and the problem ---------------------------------------------------------------------------------

def test_registry_entry_matches_the_reference(data_dir):
    problem, net_config, assignments = util.get_config("cifar_conv", data_dir=data_dir)
    assert assignments is None and net_config == {"cw": util.get_default_net_config(None)}
    p = problem.producer
    assert p.kind == "cifar_conv" and p.batch_norm is True and p.batch_size == 128
    assert p.mode == "train" and p.data_dir == data_dir
    assert util.get_config("cifar_conv", path="/some/net", data_dir=data_dir)[0].producer.mode == "test"
    assert util.get_config("cifar_conv", mode="test", data_dir=data_dir)[0].producer.mode == "test"
    rp = util.get_config("cifar_conv", net_name="RNNprop", data_dir=data_dir)[1]
    assert list(rp) == ["rp"] and rp["rp"]["net"] == "RNNprop"
    made, loss, idx = _run(problem)
    assert list(made) == NAMES and [tuple(v.shape) for v in made.values()] == SHAPES
    assert sum(v.numel() for v in made.values()) == 13610 == _lib.CIFAR_CONV_COORDS
    for name, v in made.items():   # weights N(0, 0.01), biases zero (DM/problems.py:421-427,439-446)
        if v.dim() == 1:
            assert torch.count_nonzero(v) == 0, name
        else:
            assert abs(float(v.std()) - 0.01) < 0.25 * 0.01 and abs(float(v.mean())) < 0.005, name
    assert idx.shape == (128,) and int(idx.max()) < 1000
    assert loss.shape == () and np.isfinite(float(loss))


def test_data_dir_defaults_per_problem(tmp_path, monkeypatch):
    """"cifar10" for cifar_conv and "MNIST-data" for the MNIST problems, relative to the working directory."""
    write_cifar10(str(tmp_path / "cifar10"), n_train=20, n_test=5)
    write_mnist(str(tmp_path / "MNIST-data"), n_train=5100, n_test=10)
    monkeypatch.chdir(tmp_path)
    assert util.get_config("cifar_conv")[0].producer.data_dir == "cifar10"
    for name in ("mnist", "mnist_conv"):
        assert util.get_config(name)[0].producer.data_dir == "MNIST-data"


def numpy_forward(params, pixels, labels):
    """DM/problems.py:410-456 in float64 NumPy with explicit loops over the stride-2 VALID windows (HWIO weights,
    NHWC pixels)."""
    w1, b1, w2, b2, wf, bf = [np.asarray(p, dtype=np.float64) for p in params]
    B = pixels.shape[0]
    h = pixels.astype(np.float64)

    def conv(x, w, b):
        k = w.shape[0]
        H = (x.shape[1] - k) // 2 + 1                                     # VALID, stride 2
        out = np.zeros((B, H, H, w.shape[3]))
        for i in range(H):
            for j in range(H):
                win = x[:, 2 * i:2 * i + k, 2 * j:2 * j + k, :]          # [B, k, k, C_in]
                out[:, i, j, :] = np.tensordot(win, w, axes=([1, 2, 3], [0, 1, 2]))
        return out + b

    def bn_relu_pool(z):
        mu = z.mean(axis=(0, 1, 2))
        var = ((z - mu) ** 2).mean(axis=(0, 1, 2))                       # biased
        a = np.maximum((z - mu) / np.sqrt(var + 1e-3), 0.0)
        P = z.shape[1] // 2                                              # VALID: 15 -> 7 drops row / column 14
        out = np.zeros((B, P, P, z.shape[3]))
        for i in range(P):
            for j in range(P):
                out[:, i, j, :] = a[:, 2 * i:2 * i + 2, 2 * j:2 * j + 2, :].max(axis=(1, 2))
        return out

    z1 = conv(h, w1, b1)
    assert z1.shape == (B, 15, 15, 16)
    h = bn_relu_pool(z1)
    assert h.shape == (B, 7, 7, 16)
    z2 = conv(h, w2, b2)
    assert z2.shape == (B, 2, 2, 32)
    h = bn_relu_pool(z2)
    assert h.shape == (B, 1, 1, 32)
    logits = np.maximum(h.reshape(B, -1) @ wf + bf, 0.0)                 # flatten, then the logits' ReLU
    m = logits.max(axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(logits - m).sum(axis=1))
    return float(np.mean(lse - logits[np.arange(B), labels]))


def test_torch_build_equals_a_numpy_forward_of_the_spec(data_dir):
    build = problems.cifar10(batch_size=16, data_dir=data_dir)
    gen = torch.Generator().manual_seed(11)
    params = {n: torch.randn(s, generator=gen, dtype=torch.float64) * (0.3 if len(s) > 1 else 0.5)
              for n, s in zip(NAMES, SHAPES)}
    torch.manual_seed(1)
    _, loss, idx = _run(build, params)
    d = cifar_data.load_cifar10(data_dir, "train")
    ref = numpy_forward([params[n].numpy() for n in NAMES], d.pixels()[idx.numpy()], d.labels[idx.numpy()])
    assert abs(float(loss) - ref) <= 1e-10 * abs(ref), (float(loss), ref)


def test_without_batch_norm_builds_and_its_producer_keeps_the_flag(data_dir):
    build = problems.cifar10(batch_norm=False, data_dir=data_dir)
    assert build.producer.batch_norm is False
    made, loss, _ = _run(build)
    assert list(made) == NAMES and np.isfinite(float(loss))


# ---- the producer's accepts ---------------------------------------------------------------------------------------

def _layout(build, reverse=False):
    variables, constants = meta._get_variables(build, torch.Generator().manual_seed(0), "cpu")
    order = list(range(len(variables)))[::-1 if reverse else 1]
    slices, _, _ = meta.plan_arena(variables, [order], ["cw"], {"cw": None})
    return variables, slices, constants


def test_producer_takes_batch_norm_and_the_kernels_batches_in_creation_order(data_dir):
    build = problems.cifar10(batch_size=4, data_dir=data_dir)
    p = build.producer
    assert p.kind == "cifar_conv"
    layout = _layout(build)
    assert p.accepts(*layout)
    assert not p.accepts(*_layout(build, reverse=True))
    variables, slices, constants = layout
    for j in range(len(variables)):
        renamed = [dict(v, name=v["name"] + "_other") if i == j else v for i, v in enumerate(variables)]
        assert not p.accepts(renamed, slices, constants), j
    assert not problems.cifar10(batch_norm=False, batch_size=4, data_dir=data_dir).producer.accepts(*layout)
    for batch, fits in [(1, True), (1024, True), (1025, False)]:
        assert problems.cifar10(batch_size=batch, data_dir=data_dir).producer.accepts(*layout) == fits, batch
    # the MNIST ConvNet's variables share the names but not the shapes
    mnist_like = [dict(v, shape=[512, 10]) if v["name"] == "fc_weights" else v for v in variables]
    assert not p.accepts(mnist_like, slices, constants)


# ---- the ABI ------------------------------------------------------------------------------------------------------

def test_cifar_conv_args_follow_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(_lib.INCLUDE, "l2o_b200.h")).read(), flags=re.S)
    m = re.search(r"typedef struct\s*\{([^}]*)\}\s*l2o_cifar_conv_args\s*;", src)
    want = [re.findall(r"[A-Za-z_][A-Za-z_0-9]*", d.strip())[-1] for d in m.group(1).split(";") if d.strip()]
    assert [f[0] for f in _lib.CifarConvArgs._fields_] == want
    assert [f[0] for f in _lib.CifarConvArgs._fields_] == [f[0] for f in _lib.MnistConvArgs._fields_]
    assert int(re.search(r"#define L2O_CIFAR_CONV_LAYOUT (\d+)", src).group(1)) == _lib.CIFAR_CONV_LAYOUT
    assert int(re.search(r"#define L2O_CIFAR_CONV_COORDS (\d+)", src).group(1)) == _lib.CIFAR_CONV_COORDS
    assert int(re.search(r"#define L2O_CIFAR_CONV_MAX_BATCH (\d+)", src).group(1)) == _lib.CIFAR_CONV_MAX_BATCH


def test_cifar_conv_grad_validates_without_gpu():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    assert L.l2o_cifar_conv_workspace_bytes(0) == _lib.L2O_E_INVALID
    assert L.l2o_cifar_conv_workspace_bytes(1025) == _lib.L2O_E_INVALID
    sizes = [L.l2o_cifar_conv_workspace_bytes(b) for b in (1, 128, 1024)]
    assert 0 < sizes[0] < sizes[1] < sizes[2] and all(s % 16 == 0 for s in sizes)
    assert L.l2o_cifar_conv_grad(None, None) == _lib.L2O_E_INVALID
    buf = ctypes.create_string_buffer(64)
    base = (ctypes.addressof(buf) + 15) & ~15   # 16-byte aligned

    def args(**kw):
        a = _lib.CifarConvArgs()
        a.batch, a.num_examples = 128, 100
        a.counter = a.images = a.labels = a.x = a.g = a.workspace = base
        a.workspace_bytes = L.l2o_cifar_conv_workspace_bytes(128)
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    for bad in (dict(batch=0), dict(batch=1025), dict(num_examples=0), dict(counter=None), dict(images=None),
                dict(labels=None), dict(x=None), dict(g=None), dict(workspace=None),
                dict(workspace_bytes=L.l2o_cifar_conv_workspace_bytes(128) - 1),
                dict(batch=129), dict(workspace=base + 8), dict(x=base + 4), dict(scale=base + 4), dict(g=base + 2),
                dict(counter=base + 4), dict(f=base + 4), dict(idx_out=base + 2)):
        assert L.l2o_cifar_conv_grad(ctypes.byref(args(**bad)), None) == _lib.L2O_E_INVALID, bad
    off = (ctypes.c_int64 * _lib.CIFAR_CONV_LAYOUT)()
    for b in (0, 1025):
        assert L.l2o_cifar_conv_workspace_layout(b, off) == _lib.L2O_E_INVALID
    assert L.l2o_cifar_conv_workspace_layout(128, None) == _lib.L2O_E_INVALID
    from open_l2o_b200.engine import cifar_conv_fits, cifar_conv_workspace_layout
    for b in (1, 200, 1024):   # z1, z2, the 96 batch-norm constants and dlogits lie inside the workspace, 16-aligned
        lay = cifar_conv_workspace_layout(b)
        ends = dict(z1=b * 3600 * 4, z2=b * 128 * 4, bn=96 * 4, dl=b * 16 * 4)
        assert all(lay[k] % 16 == 0 and lay[k] + ends[k] <= L.l2o_cifar_conv_workspace_bytes(b) for k in ends), lay
        spans = sorted((lay[k], lay[k] + ends[k]) for k in ends)
        assert all(e <= s for (_, e), (s, _) in zip(spans, spans[1:])), spans
    assert cifar_conv_fits(1) and cifar_conv_fits(1024) and not cifar_conv_fits(0) and not cifar_conv_fits(1025)


# ---- nas (DM/problems.py:540-634, DM/util.py:185-190) ---------------------------------------------------------------

NAS_NAMES = [s + v for s in ("node0", "node0_onto_node2", "node1", "node1_onto_node3") for v in ("/weights1", "/biases1")]
NAS_NAMES += ["fc_weights", "fc_bias"]
NAS_SHAPES = [(3, 3, 3, 16), (16,)] + [(3, 3, 16, 16), (16,)] * 3 + [(16, 10), (10,)]


def test_nas_registry_entry_matches_the_reference(data_dir):
    problem, net_config, assignments = util.get_config("nas", data_dir=data_dir)
    assert assignments is None and net_config == {"cw": util.get_default_net_config(None)}
    p = problem.producer
    assert p.kind == "nas" and p.batch_norm is True and p.batch_size == 128
    assert p.mode == "train" and p.data_dir == data_dir
    assert util.get_config("nas", path="/some/net", data_dir=data_dir)[0].producer.mode == "test"
    rp = util.get_config("nas", net_name="RNNprop", data_dir=data_dir)[1]
    assert list(rp) == ["rp"] and rp["rp"]["net"] == "RNNprop"
    made, loss, idx = _run(problem)
    assert list(made) == NAS_NAMES and [tuple(v.shape) for v in made.values()] == NAS_SHAPES
    assert sum(v.numel() for v in made.values()) == 7578 == _lib.NAS_COORDS
    for name, v in made.items():   # weights N(0, 0.01), biases zero (DM/problems.py:588-594,617-624)
        if v.dim() == 1:
            assert torch.count_nonzero(v) == 0, name
        else:
            assert abs(float(v.std()) - 0.01) < 0.25 * 0.01 and abs(float(v.mean())) < 0.005, name
    assert idx.shape == (128,) and int(idx.max()) < 1000 and np.isfinite(float(loss))


def test_nas_data_dir_defaults_to_cifar10(tmp_path, monkeypatch):
    write_cifar10(str(tmp_path / "cifar10"), n_train=20, n_test=5)
    monkeypatch.chdir(tmp_path)
    assert util.get_config("nas")[0].producer.data_dir == "cifar10"
    with pytest.raises(ValueError, match="Mode"):
        util.get_config("nas", mode="validation")


def nas_numpy_forward(params, pixels, labels):
    """DM/problems.py:584-632 in float64 NumPy with explicit loops: SAME 3x3 convs over a zero-padded input, and TF's
    SAME average pool, which divides each window's sum by its in-image cells."""
    w0, b0, wa, ba, w1, b1, wb, bb, wf, bf = [np.asarray(p, dtype=np.float64) for p in params]
    B = pixels.shape[0]

    def conv(x, w, b):
        xp = np.pad(x, ((0, 0), (1, 1), (1, 1), (0, 0)))
        out = np.zeros((B, 32, 32, w.shape[3]))
        for i in range(32):
            for j in range(32):
                out[:, i, j, :] = np.tensordot(xp[:, i:i + 3, j:j + 3, :], w, axes=([1, 2, 3], [0, 1, 2]))
        z = out + b
        mu = z.mean(axis=(0, 1, 2))
        var = ((z - mu) ** 2).mean(axis=(0, 1, 2))
        return np.maximum((z - mu) / np.sqrt(var + 1e-3), 0.0)

    def avgpool(x):
        out = np.zeros_like(x)
        for i in range(32):
            for j in range(32):
                rows, cols = range(max(i - 1, 0), min(i + 2, 32)), range(max(j - 1, 0), min(j + 2, 32))
                cells = [x[:, r, c, :] for r in rows for c in cols]
                out[:, i, j, :] = sum(cells) / len(cells)
        return out

    node0 = conv(pixels.astype(np.float64), w0, b0)
    n0o2 = conv(node0, wa, ba)
    node1 = conv(node0, w1, b1)
    n1o3 = conv(node1, wb, bb)
    node3 = avgpool(node1) + n0o2 + n1o3 + node0
    logits = np.maximum(node3.reshape(B, -1, 16).mean(axis=1) @ wf + bf, 0.0)
    m = logits.max(axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(logits - m).sum(axis=1))
    return float(np.mean(lse - logits[np.arange(B), labels]))


def test_nas_average_pool_divides_by_the_in_image_cells():
    """The torch op nas_forward uses for tf.nn.avg_pool SAME: 4 cells at a corner, 6 on an edge, 9 inside."""
    F = torch.nn.functional
    x = torch.ones(1, 1, 32, 32, dtype=torch.float64)
    x[0, 0, 0, 0] = 5.0
    y = F.avg_pool2d(x, 3, 1, padding=1, count_include_pad=False)
    assert float(y[0, 0, 0, 0]) == (5 + 3) / 4 and float(y[0, 0, 0, 1]) == (5 + 5) / 6 and float(y[0, 0, 5, 5]) == 1


def test_nas_torch_build_equals_a_numpy_forward_of_the_spec(data_dir):
    build = problems.nas(batch_size=4, data_dir=data_dir)
    gen = torch.Generator().manual_seed(12)
    params = {n: torch.randn(s, generator=gen, dtype=torch.float64) * (0.3 if len(s) > 1 else 0.5)
              for n, s in zip(NAS_NAMES, NAS_SHAPES)}
    params["fc_weights"] = params["fc_weights"] * 10   # the mean over positions shrinks the features: keep logits O(1)
    torch.manual_seed(2)
    _, loss, idx = _run(build, params)
    d = cifar_data.load_cifar10(data_dir, "train")
    ref = nas_numpy_forward([params[n].numpy() for n in NAS_NAMES], d.pixels()[idx.numpy()], d.labels[idx.numpy()])
    assert abs(float(loss) - ref) <= 1e-10 * abs(ref), (float(loss), ref)


def test_nas_producer_takes_batch_norm_and_the_kernels_batches_in_creation_order(data_dir):
    build = problems.nas(batch_size=4, data_dir=data_dir)
    p = build.producer
    layout = _layout(build)
    assert p.accepts(*layout)
    assert not p.accepts(*_layout(build, reverse=True))
    variables, slices, constants = layout
    for j in range(len(variables)):
        renamed = [dict(v, name=v["name"] + "_other") if i == j else v for i, v in enumerate(variables)]
        assert not p.accepts(renamed, slices, constants), j
    assert not problems.nas(batch_norm=False, batch_size=4, data_dir=data_dir).producer.accepts(*layout)
    for batch, fits in [(1, True), (1024, True), (1025, False)]:
        assert problems.nas(batch_size=batch, data_dir=data_dir).producer.accepts(*layout) == fits, batch
    assert not problems.cifar10(batch_size=4, data_dir=data_dir).producer.accepts(*layout)


def test_nas_args_follow_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(_lib.INCLUDE, "l2o_b200.h")).read(), flags=re.S)
    m = re.search(r"typedef struct\s*\{([^}]*)\}\s*l2o_nas_args\s*;", src)
    want = [re.findall(r"[A-Za-z_][A-Za-z_0-9]*", d.strip())[-1] for d in m.group(1).split(";") if d.strip()]
    assert [f[0] for f in _lib.NasArgs._fields_] == want
    assert int(re.search(r"#define L2O_NAS_LAYOUT (\d+)", src).group(1)) == _lib.NAS_LAYOUT
    assert int(re.search(r"#define L2O_NAS_COORDS (\d+)", src).group(1)) == _lib.NAS_COORDS
    assert int(re.search(r"#define L2O_NAS_MAX_BATCH (\d+)", src).group(1)) == _lib.NAS_MAX_BATCH


def test_nas_grad_validates_without_gpu():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    assert L.l2o_nas_workspace_bytes(0) == _lib.L2O_E_INVALID
    assert L.l2o_nas_workspace_bytes(1025) == _lib.L2O_E_INVALID
    sizes = [L.l2o_nas_workspace_bytes(b) for b in (1, 128, 1024)]
    assert 0 < sizes[0] < sizes[1] < sizes[2] and all(s % 16 == 0 for s in sizes)
    assert L.l2o_nas_grad(None, None) == _lib.L2O_E_INVALID
    buf = ctypes.create_string_buffer(64)
    base = (ctypes.addressof(buf) + 15) & ~15

    def args(**kw):
        a = _lib.NasArgs()
        a.batch, a.num_examples = 128, 100
        a.counter = a.images = a.labels = a.x = a.g = a.workspace = base
        a.workspace_bytes = L.l2o_nas_workspace_bytes(128)
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    for bad in (dict(batch=0), dict(batch=1025), dict(num_examples=0), dict(counter=None), dict(images=None),
                dict(labels=None), dict(x=None), dict(g=None), dict(workspace=None),
                dict(workspace_bytes=L.l2o_nas_workspace_bytes(128) - 1),
                dict(batch=129), dict(workspace=base + 8), dict(x=base + 4), dict(scale=base + 4), dict(g=base + 2),
                dict(counter=base + 4), dict(f=base + 4), dict(idx_out=base + 2)):
        assert L.l2o_nas_grad(ctypes.byref(args(**bad)), None) == _lib.L2O_E_INVALID, bad
    off = (ctypes.c_int64 * _lib.NAS_LAYOUT)()
    for b in (0, 1025):
        assert L.l2o_nas_workspace_layout(b, off) == _lib.L2O_E_INVALID
    assert L.l2o_nas_workspace_layout(128, None) == _lib.L2O_E_INVALID
    from open_l2o_b200.engine import nas_fits, nas_workspace_layout
    for b in (1, 200, 1024):
        lay = nas_workspace_layout(b)
        ends = dict(z0=b * 16384 * 4, za=b * 16384 * 4, z1=b * 16384 * 4, zb=b * 16384 * 4, bn=128 * 4, dl=b * 16 * 4)
        assert all(lay[k] % 16 == 0 and lay[k] + ends[k] <= L.l2o_nas_workspace_bytes(b) for k in ends), lay
        spans = sorted((lay[k], lay[k] + ends[k]) for k in ends)
        assert all(e <= s for (_, e), (s, _) in zip(spans, spans[1:])), spans
    assert nas_fits(1) and nas_fits(1024) and not nas_fits(0) and not nas_fits(1025)
