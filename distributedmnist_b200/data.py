"""MNIST data pipeline: IDX decode, normalisation, in-memory DataSet, synthetic data.

Behavioural parity with the reference (src/mnist_data.py):

* images are decoded to fp32 ``(x - 127.5) / 255`` in [-0.5, 0.5], NHWC
  ``[N, 28, 28, 1]`` (mnist_data.py:132-145); labels are int64 (:147-154);
* ``DataSet`` shuffles at construction and at every epoch wrap and serves
  contiguous slices (:81-84, :102-130);
* the "validation" split IS the 10k test set (:200-201);
* every replica sees the full training set -- ``worker_id`` / ``n_workers`` are
  accepted and do not shard (:162-163, :212-213);
* ``fake_data`` yields constant all-ones images with label 0 (:104-112).

Differences, on purpose: the shuffle seed is explicit (the reference seeds numpy
with ``int(time.time())``, :55) and derived per replica so replicas draw
independent streams reproducibly; nothing is ever downloaded (no network) --
when the IDX files are absent a *learnable* synthetic MNIST-shaped set is
generated so time-to-accuracy curves remain meaningful.
"""
from __future__ import annotations

import gzip
import os
import struct
from collections import namedtuple
from typing import Optional, Tuple

import numpy as np

IMAGE_SIZE = 28
NUM_CHANNELS = 1
PIXEL_DEPTH = 255
NUM_LABELS = 10

TRAIN_IMAGES = "train-images-idx3-ubyte.gz"
TRAIN_LABELS = "train-labels-idx1-ubyte.gz"
TEST_IMAGES = "t10k-images-idx3-ubyte.gz"
TEST_LABELS = "t10k-labels-idx1-ubyte.gz"

Datasets = namedtuple("Datasets", ["train", "validation", "test"])


def _open_maybe_gz(path: str):
    with open(path, "rb") as f:
        magic = f.read(2)
    return gzip.open(path, "rb") if magic == b"\x1f\x8b" else open(path, "rb")


def normalize_images(u8: np.ndarray) -> np.ndarray:
    """uint8 [0,255] -> fp32 [-0.5, 0.5] (reference mnist_data.py:141)."""
    return (u8.astype(np.float32) - (PIXEL_DEPTH / 2.0)) / PIXEL_DEPTH


def extract_data(filename: str, num_images: Optional[int] = None) -> np.ndarray:
    """IDX3 image file -> fp32 NHWC ``[N, 28, 28, 1]`` in [-0.5, 0.5]."""
    with _open_maybe_gz(filename) as bs:
        magic, n, rows, cols = struct.unpack(">IIII", bs.read(16))
        if magic != 2051:
            raise ValueError("%s: bad IDX3 magic %d" % (filename, magic))
        if num_images is not None:
            n = min(n, num_images)
        buf = bs.read(rows * cols * n)
    data = np.frombuffer(buf, dtype=np.uint8)
    if data.size != rows * cols * n:
        raise ValueError("%s: truncated (%d of %d bytes)" % (filename, data.size, rows * cols * n))
    return normalize_images(data).reshape(n, rows, cols, 1)


def extract_labels(filename: str, num_images: Optional[int] = None) -> np.ndarray:
    """IDX1 label file -> int64 ``[N]``."""
    with _open_maybe_gz(filename) as bs:
        magic, n = struct.unpack(">II", bs.read(8))
        if magic != 2049:
            raise ValueError("%s: bad IDX1 magic %d" % (filename, magic))
        if num_images is not None:
            n = min(n, num_images)
        buf = bs.read(n)
    return np.frombuffer(buf, dtype=np.uint8).astype(np.int64)


def write_idx_images(path: str, u8_images: np.ndarray) -> None:
    """Write a uint8 ``[N, R, C]`` array as a gzipped IDX3 file (tests, tooling)."""
    n, r, c = u8_images.shape
    with gzip.open(path, "wb") as f:
        f.write(struct.pack(">IIII", 2051, n, r, c))
        f.write(np.ascontiguousarray(u8_images, dtype=np.uint8).tobytes())


def write_idx_labels(path: str, labels: np.ndarray) -> None:
    with gzip.open(path, "wb") as f:
        f.write(struct.pack(">II", 2049, labels.shape[0]))
        f.write(np.ascontiguousarray(labels, dtype=np.uint8).tobytes())


class DataSet:
    """In-memory shuffled dataset with ``next_batch`` (reference mnist_data.py:41-130)."""

    def __init__(self, images, labels, fake_data: bool = False, one_hot: bool = False,
                 reshape: bool = False, seed: Optional[int] = None):
        self._rng = np.random.RandomState(seed if seed is not None else 0)
        self.one_hot = one_hot
        self.fake_data = fake_data
        if fake_data:
            self._num_examples = 10000
            images = np.ones((0, IMAGE_SIZE, IMAGE_SIZE, 1), np.float32)
            labels = np.zeros((0,), np.int64)
        else:
            images = np.asarray(images)
            labels = np.asarray(labels)
            assert images.shape[0] == labels.shape[0], (
                "images.shape: %s labels.shape: %s" % (images.shape, labels.shape))
            self._num_examples = images.shape[0]
            if reshape:
                assert images.shape[3] == 1
                images = images.reshape(images.shape[0], images.shape[1] * images.shape[2])
        self._images = images
        self._labels = labels
        self._epochs_completed = 0
        self._index_in_epoch = 0
        self._perm = np.arange(self._num_examples)
        if not fake_data:
            # the initial shuffle re-orders the arrays themselves (one copy at start-up; `images` / `labels` then expose a
            # per-replica order, as in the reference); the per-epoch reshuffles only draw a new permutation
            perm = self._rng.permutation(self._num_examples)
            self._images = self._images[perm]
            self._labels = self._labels[perm]

    def _shuffle(self) -> None:
        # A fresh permutation per epoch, applied when a batch is drawn (row gather of `batch_size` examples) instead of
        # re-ordering the whole arrays: at ~0.15 ms per 256-image step an epoch of 60 000 images lasts ~35 ms, and copying
        # 188 MB per epoch would be a large share of that.
        self._perm = self._rng.permutation(self._num_examples)

    @property
    def images(self):
        return self._images

    @property
    def labels(self):
        return self._labels

    @property
    def num_examples(self) -> int:
        return self._num_examples

    @property
    def epochs_completed(self) -> int:
        return self._epochs_completed

    def next_batch(self, batch_size: int, fake_data: bool = False) -> Tuple[np.ndarray, np.ndarray]:
        if fake_data or self.fake_data:
            imgs = np.ones((batch_size, IMAGE_SIZE, IMAGE_SIZE, 1), np.float32)
            if self.one_hot:
                lab = np.zeros((batch_size, NUM_LABELS), np.int64)
                lab[:, 0] = 1
            else:
                lab = np.zeros((batch_size,), np.int64)
            return imgs, lab
        assert batch_size <= self._num_examples
        start = self._index_in_epoch
        self._index_in_epoch += batch_size
        if self._index_in_epoch > self._num_examples:
            self._epochs_completed += 1
            self._shuffle()
            start = 0
            self._index_in_epoch = batch_size
        end = self._index_in_epoch
        idx = self._perm[start:end]
        return self._images[idx], self._labels[idx]

    def next_batch_indices(self, batch_size: int) -> np.ndarray:
        """The row indices ``next_batch`` would use (same epoch / reshuffle bookkeeping), for input pipelines that gather
        straight into their own (page-locked) buffers."""
        assert not self.fake_data and batch_size <= self._num_examples
        start = self._index_in_epoch
        self._index_in_epoch += batch_size
        if self._index_in_epoch > self._num_examples:
            self._epochs_completed += 1
            self._shuffle()
            start = 0
            self._index_in_epoch = batch_size
        return self._perm[start:self._index_in_epoch]


# ----------------------------------------------------------------------------
# Synthetic MNIST-shaped data
# ----------------------------------------------------------------------------

def _class_prototypes(rng: np.random.RandomState) -> np.ndarray:
    """Ten smooth 28x28 'glyph' prototypes in [0,1]: a few random strokes blurred."""
    protos = np.zeros((NUM_LABELS, IMAGE_SIZE, IMAGE_SIZE), np.float32)
    yy, xx = np.mgrid[0:IMAGE_SIZE, 0:IMAGE_SIZE].astype(np.float32)
    for c in range(NUM_LABELS):
        img = np.zeros((IMAGE_SIZE, IMAGE_SIZE), np.float32)
        for _ in range(3 + c % 3):
            x0, y0, x1, y1 = rng.uniform(5, 23, size=4)
            for t in np.linspace(0.0, 1.0, 24):
                cx, cy = x0 + t * (x1 - x0), y0 + t * (y1 - y0)
                img += np.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / (2 * 1.3 ** 2))
        protos[c] = np.clip(img / max(img.max(), 1e-6) * 1.4, 0.0, 1.0)
    return protos


def make_synthetic_mnist(num_train: int = 60000, num_test: int = 10000, seed: int = 1234,
                         noise: float = 0.25) -> Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """Learnable synthetic set with MNIST's shapes/dtypes/value range.

    Each example = class prototype, randomly shifted by up to +-2 px, scaled in
    intensity, plus Gaussian pixel noise; quantised to uint8 then normalised
    exactly like real MNIST so the downstream path is identical.
    """
    rng = np.random.RandomState(seed)
    protos = _class_prototypes(rng)

    def gen(n: int) -> Tuple[np.ndarray, np.ndarray]:
        labels = rng.randint(0, NUM_LABELS, size=n).astype(np.int64)
        shifts = rng.randint(-2, 3, size=(n, 2))
        gain = rng.uniform(0.7, 1.0, size=n).astype(np.float32)
        out = np.empty((n, IMAGE_SIZE, IMAGE_SIZE), np.uint8)
        chunk = 4096
        for s in range(0, n, chunk):
            e = min(n, s + chunk)
            base = protos[labels[s:e]] * gain[s:e, None, None]
            for j in range(e - s):
                base[j] = np.roll(base[j], (int(shifts[s + j, 0]), int(shifts[s + j, 1])), axis=(0, 1))
            base = base + rng.normal(0.0, noise, size=base.shape).astype(np.float32)
            out[s:e] = (np.clip(base, 0.0, 1.0) * 255.0).astype(np.uint8)
        return normalize_images(out).reshape(n, IMAGE_SIZE, IMAGE_SIZE, 1), labels

    tr_x, tr_y = gen(num_train)
    te_x, te_y = gen(num_test)
    return tr_x, tr_y, te_x, te_y


def _find_idx(train_dir: str, name: str) -> Optional[str]:
    for cand in (name, name[:-3]):  # .gz or already gunzipped
        p = os.path.join(train_dir, cand)
        if os.path.exists(p):
            return p
    return None


def read_data_sets(train_dir: str, fake_data: bool = False, one_hot: bool = False, reshape: bool = False,
                   worker_id: int = -1, n_workers: int = -1, seed: int = 66478,
                   synthetic: bool = True, synthetic_sizes: Tuple[int, int] = (60000, 10000)) -> Datasets:
    """Reference ``read_data_sets`` (mnist_data.py:156-210) without the download."""
    # Independent, reproducible stream per replica (reference: time-seeded, :55).
    wid = max(worker_id, 0)
    train_seed = (seed * 1000003 + 7919 * wid + 1) % (2 ** 31 - 1)
    if fake_data:
        mk = lambda: DataSet([], [], fake_data=True, one_hot=one_hot)
        return Datasets(train=mk(), validation=mk(), test=mk())
    paths = [_find_idx(train_dir, n) for n in (TRAIN_IMAGES, TRAIN_LABELS, TEST_IMAGES, TEST_LABELS)]
    if all(p is not None for p in paths):
        train_images = extract_data(paths[0], 60000)
        train_labels = extract_labels(paths[1], 60000)
        test_images = extract_data(paths[2], 10000)
        test_labels = extract_labels(paths[3], 10000)
    elif synthetic:
        # Loud, because accuracy / time-to-accuracy numbers of a run on this data are NOT MNIST numbers (the generated
        # classes are far easier); the only other sign would be the missing "Extracting ..." lines.
        import logging
        logging.getLogger("dmnist").warning(
            "*** MNIST IDX files not found under %r: training on SYNTHETIC MNIST-shaped data (--synthetic_data=true). "
            "Precision / loss / time-to-accuracy of this run are not MNIST results. ***" % train_dir)
        train_images, train_labels, test_images, test_labels = make_synthetic_mnist(
            synthetic_sizes[0], synthetic_sizes[1], seed=seed)
    else:
        raise FileNotFoundError(
            "MNIST IDX files not found under %r and --synthetic_data=false (no network: nothing is downloaded)"
            % train_dir)
    train = DataSet(train_images, train_labels, reshape=reshape, seed=train_seed)
    # "validation" is the test set, as in the reference (mnist_data.py:200-201).
    validation = DataSet(test_images, test_labels, reshape=reshape, seed=seed + 17)
    return Datasets(train=train, validation=validation, test=None)


def load_mnist(train_dir: str = "MNIST-data", worker_id: int = -1, n_workers: int = -1, **kw) -> Datasets:
    return read_data_sets(train_dir, worker_id=worker_id, n_workers=n_workers, **kw)
