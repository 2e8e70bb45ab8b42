"""MNIST from a local directory, split as the reference's loader splits it (``mnist_dataset.load_mnist()``, i.e. TF's
``read_data_sets("MNIST-data")`` with ``validation_size=5000``).  Nothing here downloads: a missing file is a
``FileNotFoundError`` naming the directory and the files expected there.

Pixels and labels stay ``uint8``.  The value a network sees is ``float32(p) * float32(1 / 255)``, what
``read_data_sets``' ``images.astype(float32) * (1.0 / 255.0)`` gives; ``pixels()`` returns exactly that, and the
l2o_mnist_grad kernel forms the same product in-kernel."""
from __future__ import annotations

import gzip
import os
from dataclasses import dataclass

import numpy as np

FILES = {
    "train_images": "train-images-idx3-ubyte",
    "train_labels": "train-labels-idx1-ubyte",
    "test_images": "t10k-images-idx3-ubyte",
    "test_labels": "t10k-labels-idx1-ubyte",
}
VALIDATION_SIZE = 5000
IMAGE_MAGIC, LABEL_MAGIC = 2051, 2049
SCALE = np.float32(1.0 / 255.0)


@dataclass(frozen=True)
class Split:
    images: np.ndarray   # [N, 784] uint8
    labels: np.ndarray   # [N] uint8

    @property
    def num_examples(self) -> int:
        return int(self.images.shape[0])

    def pixels(self) -> np.ndarray:
        """The float32 images the reference's loader returns."""
        return self.images.astype(np.float32) * SCALE


def _find(data_dir, stem):
    """``stem.gz`` (the reference's download layout) or ``stem`` (torchvision's MNIST/raw layout)."""
    for name in (stem + ".gz", stem):
        path = os.path.join(data_dir, name)
        if os.path.isfile(path):
            return path
    return None


def _read(path, magic, ndim):
    opener = gzip.open if path.endswith(".gz") else open
    with opener(path, "rb") as f:
        raw = f.read()
    head = 4 * (1 + ndim)
    if len(raw) < head:
        raise ValueError("{}: truncated IDX header".format(path))
    fields = np.frombuffer(raw[:head], dtype=">u4")
    if int(fields[0]) != magic:
        raise ValueError("{}: invalid magic number {} (expected {})".format(path, int(fields[0]), magic))
    dims = [int(d) for d in fields[1:]]
    count = int(np.prod(dims))
    if len(raw) - head != count:
        raise ValueError("{}: {} bytes of data, the header's dimensions {} need {}".format(path, len(raw) - head, dims,
                                                                                          count))
    return np.frombuffer(raw, dtype=np.uint8, offset=head).reshape(dims)


def _pair(data_dir, kind):
    img_path, lab_path = _find(data_dir, FILES[kind + "_images"]), _find(data_dir, FILES[kind + "_labels"])
    images = _read(img_path, IMAGE_MAGIC, 3)
    labels = _read(lab_path, LABEL_MAGIC, 1)
    if images.shape[0] != labels.shape[0]:
        raise ValueError("{}: {} images but {} labels".format(data_dir, images.shape[0], labels.shape[0]))
    if images.shape[1:] != (28, 28):
        raise ValueError("{}: images are {}, expected 28 x 28".format(img_path, images.shape[1:]))
    if labels.size and int(labels.max()) > 9:
        raise ValueError("{}: label {} is not a digit".format(lab_path, int(labels.max())))
    return images.reshape(images.shape[0], 784), labels


_cache = {}


def load_mnist(data_dir="MNIST-data"):
    """{"train", "validation", "test"} -> Split, read once per directory and process."""
    key = os.path.abspath(data_dir)
    if key in _cache:
        return _cache[key]
    missing = [stem for stem in FILES.values() if _find(data_dir, stem) is None]
    if missing:
        raise FileNotFoundError("MNIST not found in {!r}: expected {} (each .gz or uncompressed); this project never "
                                "downloads them".format(data_dir, ", ".join(missing)))
    train_images, train_labels = _pair(data_dir, "train")
    test_images, test_labels = _pair(data_dir, "test")
    if not 0 <= VALIDATION_SIZE <= len(train_images):
        raise ValueError("{}: validation size should be between 0 and {}. Received: {}.".format(
            data_dir, len(train_images), VALIDATION_SIZE))
    out = {
        "validation": Split(train_images[:VALIDATION_SIZE], train_labels[:VALIDATION_SIZE]),
        "train": Split(train_images[VALIDATION_SIZE:], train_labels[VALIDATION_SIZE:]),
        "test": Split(test_images, test_labels),
    }
    _cache[key] = out
    return out


_device_cache = {}


def device_split(data_dir, mode, device):
    """(images [N, 784], labels [N]) of one split as uint8 torch tensors on ``device``, uploaded once per process.
    They are not optimizee variables: resetting an optimizee never touches them."""
    import torch
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    key = (os.path.abspath(data_dir), mode, str(device))
    if key not in _device_cache:
        split = load_mnist(data_dir)[mode]
        _device_cache[key] = (torch.from_numpy(np.array(split.images)).to(device),
                              torch.from_numpy(np.array(split.labels)).to(device))
    return _device_cache[key]
