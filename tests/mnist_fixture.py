"""A seeded synthetic MNIST in IDX format, written into a test's temporary directory (no test needs the real files)."""
import gzip
import os

import numpy as np

from open_l2o_b200.mnist_data import FILES


def idx_bytes(arr, magic):
    arr = np.ascontiguousarray(arr, dtype=np.uint8)
    return np.array([magic] + list(arr.shape), dtype=">u4").tobytes() + arr.tobytes()


def write_mnist(path, n_train=6000, n_test=1000, seed=0, gz=True):
    """Writes the four files into ``path``; returns (train_images, train_labels, test_images, test_labels)."""
    rng = np.random.default_rng(seed)
    data = (rng.integers(0, 256, (n_train, 28, 28), dtype=np.uint8), rng.integers(0, 10, n_train, dtype=np.uint8),
            rng.integers(0, 256, (n_test, 28, 28), dtype=np.uint8), rng.integers(0, 10, n_test, dtype=np.uint8))
    os.makedirs(path, exist_ok=True)
    for key, arr, magic in zip(("train_images", "train_labels", "test_images", "test_labels"), data,
                               (2051, 2049, 2051, 2049)):
        raw = idx_bytes(arr, magic)
        if gz:
            with gzip.open(os.path.join(path, FILES[key] + ".gz"), "wb") as f:
                f.write(raw)
        else:
            with open(os.path.join(path, FILES[key]), "wb") as f:
                f.write(raw)
    return data
