"""A seeded synthetic CIFAR-10 in the binary record layout, written into a test's temporary directory (no test needs the
real files): ``cifar-10-batches-bin/`` extracted, or the ``cifar-10-binary.tar.gz`` archive holding the same members."""
import io
import os
import tarfile

import numpy as np

from open_l2o_b200.cifar_data import ARCHIVE, FILES, FOLDER


def records(images, labels):
    """The bytes of the records: per example, the label then the [3][32][32] planes."""
    images = np.ascontiguousarray(images, dtype=np.uint8).reshape(len(labels), -1)
    return np.concatenate([np.asarray(labels, dtype=np.uint8)[:, None], images], axis=1).tobytes()


def write_cifar10(path, n_train=2000, n_test=500, seed=0, archive=False):
    """Writes the five training batches (n_train examples split over them) and the test batch into ``path``, as the
    extracted folder or, with ``archive``, as the gzipped tarball only.  Returns (train_images, train_labels,
    test_images, test_labels), images [N][3][32][32] uint8."""
    rng = np.random.default_rng(seed)
    data = (rng.integers(0, 256, (n_train, 3, 32, 32), dtype=np.uint8), rng.integers(0, 10, n_train, dtype=np.uint8),
            rng.integers(0, 256, (n_test, 3, 32, 32), dtype=np.uint8), rng.integers(0, 10, n_test, dtype=np.uint8))
    cuts = np.linspace(0, n_train, 6).astype(int)
    members = [(name, records(data[0][lo:hi], data[1][lo:hi]))
               for name, lo, hi in zip(FILES["train"], cuts[:-1], cuts[1:])]
    members.append((FILES["test"][0], records(data[2], data[3])))
    os.makedirs(path, exist_ok=True)
    if archive:
        with tarfile.open(os.path.join(path, ARCHIVE), "w:gz") as tar:
            for name, raw in members:
                info = tarfile.TarInfo(FOLDER + "/" + name)
                info.size = len(raw)
                tar.addfile(info, io.BytesIO(raw))
    else:
        os.makedirs(os.path.join(path, FOLDER), exist_ok=True)
        for name, raw in members:
            with open(os.path.join(path, FOLDER, name), "wb") as f:
                f.write(raw)
    return data
