"""CIFAR-10 from a local directory in the reference's binary layout (DM/problems.py:352-366,379-384): the ``train``
split is ``cifar-10-batches-bin/data_batch_{1..5}.bin`` and the ``test`` split ``cifar-10-batches-bin/test_batch.bin``.
Without that directory the same members are read from ``cifar-10-binary.tar.gz`` (the file the reference downloads),
without extracting it.  Nothing here downloads: if neither is present, a ``FileNotFoundError`` names the directory and
the files expected there.  The reference has no validation split, so ``train`` and ``test`` are the only modes.

A record is 3073 bytes: the label, then the R, G and B planes, each 32 x 32 row-major.  Pixels and labels stay
``uint8`` in the file's plane order, [N][3][32][32].  The value a network sees is ``float32(p) / float32(255)``, the
reference's ``tf.math.divide(image, 255)`` on the float32 image (a correctly rounded division, not the product with
1/255 MNIST uses); ``pixels()`` returns exactly that, NHWC, and l2o_cifar_conv_grad forms the same quotient
in-kernel."""
from __future__ import annotations

import os
import tarfile
from dataclasses import dataclass

import numpy as np

FOLDER = "cifar-10-batches-bin"
ARCHIVE = "cifar-10-binary.tar.gz"
FILES = {
    "train": ["data_batch_{}.bin".format(i) for i in range(1, 6)],
    "test": ["test_batch.bin"],
}
RECORD_BYTES = 1 + 3 * 32 * 32
VALUES = np.arange(256, dtype=np.float32) / np.float32(255)   # the value of each pixel byte, fp32(p) / fp32(255)


@dataclass(frozen=True)
class Split:
    images: np.ndarray   # [N, 3, 32, 32] uint8, the record's plane order
    labels: np.ndarray   # [N] uint8

    @property
    def num_examples(self) -> int:
        return int(self.images.shape[0])

    def pixels(self) -> np.ndarray:
        """The float32 NHWC images [N, 32, 32, 3] the reference's reader yields."""
        return VALUES[self.images.transpose(0, 2, 3, 1)]


def _records(raw, name):
    if len(raw) == 0 or len(raw) % RECORD_BYTES:
        raise ValueError("{}: {} bytes is not a positive multiple of the {}-byte record".format(name, len(raw),
                                                                                                RECORD_BYTES))
    rec = np.frombuffer(raw, dtype=np.uint8).reshape(-1, RECORD_BYTES)
    labels = rec[:, 0]
    if int(labels.max()) > 9:
        raise ValueError("{}: label {} is not a CIFAR-10 class".format(name, int(labels.max())))
    return rec[:, 1:].reshape(-1, 3, 32, 32), labels


def _read_members(data_dir, names):
    """The raw bytes of each ``names`` member: from the extracted folder if it exists, else from the archive."""
    folder = os.path.join(data_dir, FOLDER)
    archive = os.path.join(data_dir, ARCHIVE)
    if os.path.isdir(folder):
        out = []
        for n in names:
            path = os.path.join(folder, n)
            if not os.path.isfile(path):
                raise FileNotFoundError("CIFAR-10 file {!r} not found; this project never downloads it".format(path))
            with open(path, "rb") as f:
                out.append((path, f.read()))
        return out
    if os.path.isfile(archive):
        with tarfile.open(archive, "r:gz") as tar:
            members = {m.name: m for m in tar.getmembers() if m.isfile()}
            out = []
            for n in names:
                key = FOLDER + "/" + n
                if key not in members:
                    raise FileNotFoundError("{!r} has no member {!r}".format(archive, key))
                out.append((archive + ":" + key, tar.extractfile(members[key]).read()))
            return out
    expected = ", ".join(FOLDER + "/" + n for n in FILES["train"] + FILES["test"])
    raise FileNotFoundError("CIFAR-10 not found in {!r}: expected {} or {}; this project never downloads them".format(
        data_dir, expected, ARCHIVE))


_cache = {}


def load_cifar10(data_dir="cifar10", mode="train"):
    """Split ``mode`` ("train" or "test") of the CIFAR-10 copy in ``data_dir``, read once per directory and process."""
    if mode not in FILES:
        raise ValueError("Mode {} not recognised: CIFAR-10 has the splits {}".format(mode, sorted(FILES)))
    key = (os.path.abspath(data_dir), mode)
    if key not in _cache:
        parts = [_records(raw, name) for name, raw in _read_members(data_dir, FILES[mode])]
        _cache[key] = Split(np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]))
    return _cache[key]


_device_cache = {}
_values_cache = {}


def device_split(data_dir, mode, device):
    """(images [N, 3072], labels [N]) of one split as uint8 torch tensors on ``device``, uploaded once per process.
    They are not optimizee variables: resetting an optimizee never touches them."""
    import torch
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    key = (os.path.abspath(data_dir), mode, str(device))
    if key not in _device_cache:
        split = load_cifar10(data_dir, mode)
        _device_cache[key] = (torch.from_numpy(split.images.reshape(split.num_examples, -1).copy()).to(device),
                              torch.from_numpy(np.array(split.labels)).to(device))
    return _device_cache[key]


def device_values(device):
    """VALUES as a float32 torch tensor on ``device``, uploaded once per process: the pixel value of each byte."""
    import torch
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    if str(device) not in _values_cache:
        _values_cache[str(device)] = torch.from_numpy(VALUES.copy()).to(device)
    return _values_cache[str(device)]
