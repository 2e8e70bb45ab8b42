"""CPU tests of the MNIST reader (mnist_data), problems.mnist and the registry entries mnist / mnist_relu /
mnist_deeper (DM/problems.py:254-288, DM/util.py:145-163), and of the l2o_mnist_grad ABI without a GPU."""
import ctypes
import gzip
import os
import re

import numpy as np
import pytest
import torch

from open_l2o_b200 import _lib, mnist_data, problems, util
from open_l2o_b200.variables import variable_getter
from tests.mnist_fixture import idx_bytes, write_mnist


@pytest.mark.parametrize("gz", [True, False])
def test_reader_round_trips_and_splits_like_read_data_sets(tmp_path, gz):
    tri, trl, tei, tel = write_mnist(str(tmp_path), gz=gz)
    d = mnist_data.load_mnist(str(tmp_path))
    assert d["validation"].num_examples == 5000 and d["train"].num_examples == 1000 and d["test"].num_examples == 1000
    np.testing.assert_array_equal(d["validation"].images, tri[:5000].reshape(5000, 784))
    np.testing.assert_array_equal(d["train"].images, tri[5000:].reshape(1000, 784))
    np.testing.assert_array_equal(d["test"].images, tei.reshape(1000, 784))
    np.testing.assert_array_equal(d["validation"].labels, trl[:5000])
    np.testing.assert_array_equal(d["train"].labels, trl[5000:])
    np.testing.assert_array_equal(d["test"].labels, tel)
    assert d["train"].images.dtype == np.uint8 and d["train"].labels.dtype == np.uint8
    # read_data_sets: images.astype(float32) * (1.0 / 255.0)
    want = tri[5000:].reshape(1000, 784).astype(np.float32) * (1.0 / 255.0)
    assert want.dtype == np.float32
    np.testing.assert_array_equal(d["train"].pixels(), want)
    assert d["train"].pixels()[0].view(np.uint32).tolist() == want[0].view(np.uint32).tolist()
    assert mnist_data.load_mnist(str(tmp_path)) is d   # read once per directory


def _rewrite(path, stem, raw):
    os.remove(os.path.join(path, stem + ".gz"))
    with gzip.open(os.path.join(path, stem + ".gz"), "wb") as f:
        f.write(raw)


def test_reader_errors_name_the_directory(tmp_path):
    empty = tmp_path / "empty"
    empty.mkdir()
    with pytest.raises(FileNotFoundError, match=re.escape(str(empty))) as e:
        mnist_data.load_mnist(str(empty))
    assert "train-images-idx3-ubyte" in str(e.value) and "t10k-labels-idx1-ubyte" in str(e.value)

    bad = str(tmp_path / "magic")
    write_mnist(bad, n_train=5000, n_test=10)
    _rewrite(bad, mnist_data.FILES["train_images"], idx_bytes(np.zeros((5000, 28, 28)), 2049))
    with pytest.raises(ValueError, match=re.escape(bad) + ".*magic"):
        mnist_data.load_mnist(bad)

    bad = str(tmp_path / "count")
    write_mnist(bad, n_train=5000, n_test=10)
    _rewrite(bad, mnist_data.FILES["test_labels"], idx_bytes(np.zeros(9), 2049))
    with pytest.raises(ValueError, match=re.escape(bad) + ".*10 images but 9 labels"):
        mnist_data.load_mnist(bad)

    bad = str(tmp_path / "small")
    write_mnist(bad, n_train=4999, n_test=10)
    with pytest.raises(ValueError, match=re.escape(bad) + ".*between 0 and 4999"):
        mnist_data.load_mnist(bad)


def _capture(build):
    """Run a problem's build() with CPU tensors for its variables; returns ({name: shape}, loss)."""
    shapes = {}

    def getter(name, shape, dtype, initializer, trainable):
        assert trainable, name   # the data are not variables
        shapes[name] = tuple(shape)
        return initializer(shape, torch.Generator().manual_seed(len(shapes)))

    with variable_getter(getter):
        loss = build()
    return shapes, loss


@pytest.mark.parametrize("name,layers,act", [("mnist", (20,), "sigmoid"), ("mnist_relu", (20,), "relu"),
                                             ("mnist_deeper", (20, 20), "sigmoid")])
def test_registry_producer_matches_the_reference(tmp_path, name, layers, act):
    write_mnist(str(tmp_path))
    problem, net_config, assignments = util.get_config(name, data_dir=str(tmp_path))
    assert assignments is None and net_config == {"cw": util.get_default_net_config(None)}
    p = problem.producer
    assert p.kind == "mnist_mlp" and p.layers == layers and p.activation == act
    assert p.mode == "train" and p.batch_size == 128
    assert util.get_config(name, path="/some/net", data_dir=str(tmp_path))[0].producer.mode == "test"
    assert util.get_config(name, path="/some/net", mode="validation", data_dir=str(tmp_path))[0].producer.mode \
        == "validation"
    rp = util.get_config(name, net_name="RNNprop", data_dir=str(tmp_path))[1]
    assert list(rp) == ["rp"] and rp["rp"]["net"] == "RNNprop"
    shapes, loss = _capture(problem)
    want, k = {}, 784
    for i, w in enumerate(layers + (10,)):
        want["mlp/linear_%d/w" % i], want["mlp/linear_%d/b" % i] = (k, w), (w,)
        k = w
    assert shapes == want and list(shapes) == list(want)
    assert loss.shape == () and np.isfinite(float(loss))


def test_missing_directory_fails_before_anything_runs(tmp_path):
    with pytest.raises(FileNotFoundError, match="nowhere"):
        util.get_config("mnist", data_dir=str(tmp_path / "nowhere"))


def test_build_draws_a_fresh_batch_at_every_evaluation(tmp_path):
    write_mnist(str(tmp_path), seed=3)
    build = problems.mnist((20,), data_dir=str(tmp_path))
    drawn = []
    real = torch.randint

    def spy(*a, **k):
        out = real(*a, **k)
        drawn.append(out.clone())
        return out

    torch.manual_seed(0)
    params = {}

    def getter(name, shape, dtype, initializer, trainable):
        if name not in params:
            params[name] = initializer(shape, torch.Generator().manual_seed(len(params)))
        return params[name]

    with variable_getter(getter):
        torch.randint = spy
        try:
            losses = [float(build()) for _ in range(3)]
        finally:
            torch.randint = real
    assert len(drawn) == 3 and all(d.shape == (128,) and int(d.min()) >= 0 and int(d.max()) < 1000 for d in drawn)
    assert not torch.equal(drawn[0], drawn[1]) and not torch.equal(drawn[1], drawn[2])
    assert len(set(losses)) == 3
    # the loss is the reference's on the batch drawn
    d = mnist_data.load_mnist(str(tmp_path))["train"]
    x = torch.from_numpy(d.pixels()[drawn[2].numpy()])
    h = torch.sigmoid(x @ params["mlp/linear_0/w"] + params["mlp/linear_0/b"])
    ref = torch.nn.functional.cross_entropy(h @ params["mlp/linear_1/w"] + params["mlp/linear_1/b"],
                                            torch.from_numpy(d.labels[drawn[2].numpy()]).long())
    assert losses[2] == float(ref)


def test_mnist_args_follow_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(_lib.INCLUDE, "l2o_b200.h")).read(), flags=re.S)
    m = re.search(r"typedef struct\s*\{([^}]*)\}\s*l2o_mnist_args\s*;", src)
    want = [re.findall(r"[A-Za-z_][A-Za-z_0-9]*", d.strip())[-1] for d in m.group(1).split(";") if d.strip()]
    assert [f[0] for f in _lib.MnistArgs._fields_] == want
    for name in ("INPUT", "CLASSES", "MAX_HIDDEN", "MAX_WIDTH", "MAX_BATCH", "SIGMOID", "RELU"):
        assert int(re.search(r"#define L2O_MNIST_%s (\d+)" % name, src).group(1)) == getattr(_lib, "MNIST_" + name)


def test_mnist_grad_validates_without_gpu():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    assert L.l2o_mnist_grad(None, None) == _lib.L2O_E_INVALID
    buf = ctypes.create_string_buffer(8)
    ok = dict(batch=128, num_examples=100, n_layers=2, activation=0)

    def args(**kw):
        a = _lib.MnistArgs()
        for k, v in dict(ok, **kw).items():
            setattr(a, k, v)
        a.hidden[0] = 20
        a.counter = a.images = a.labels = a.x = a.g = ctypes.addressof(buf)
        return a

    for bad in (dict(batch=0), dict(batch=1025), dict(num_examples=0), dict(n_layers=1), dict(n_layers=6),
                dict(activation=2), dict(h0=0), dict(h0=65)):
        h0 = bad.pop("h0", 20)
        a = args(**bad)
        a.hidden[0] = h0
        assert L.l2o_mnist_grad(ctypes.byref(a), None) == _lib.L2O_E_INVALID, bad
    a = args()
    a.g = None
    assert L.l2o_mnist_grad(ctypes.byref(a), None) == _lib.L2O_E_INVALID
    from open_l2o_b200.engine import mnist_fits
    assert mnist_fits((20,), 128) and mnist_fits((64,) * 4, 1024)
    assert not mnist_fits((), 128) and not mnist_fits((64,) * 5, 128) and not mnist_fits((65,), 128)
    assert not mnist_fits((20,), 1025)
