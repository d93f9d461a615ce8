"""--device_data on the host side (no GPU needed): the flag combinations that are refused, and the index feed that replaces
the batch packer -- its index sequence, what gathering with it yields, and when it rewrites its page-locked buffers."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.train import _IndexFeed, check_device_data_flags, train


@pytest.fixture
def clean_flags():
    FLAGS.reset()
    saved = {k: os.environ.pop(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") if k in os.environ}
    yield FLAGS
    FLAGS.reset()
    os.environ.update(saved)


def _train_cpu(tmp_path, *extra):
    FLAGS.parse(["--train_dir=%s" % (tmp_path / "train"), "--batch_size=32", "--max_steps=3", "--model=mlp2",
                 "--mlp_hidden=32", "--device_data=true"] + list(extra))
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64), fake_data=FLAGS.fake_data)
    return train(ctx, ds.train, ds.validation, FLAGS)


def test_device_data_with_fake_data_is_refused(tmp_path, clean_flags):
    with pytest.raises(ValueError, match="--device_data cannot be combined with --fake_data"):
        _train_cpu(tmp_path, "--fake_data=true")
    assert not (tmp_path / "train").exists()                 # refused before anything was set up


def test_device_data_on_the_torch_engine_is_refused(tmp_path, clean_flags):
    with pytest.raises(ValueError, match="--device_data needs the sm_90a engine"):
        _train_cpu(tmp_path)
    assert not (tmp_path / "train").exists()


@pytest.mark.parametrize("backend", ["nccl", "gloo"])
def test_device_data_on_a_non_fused_backend_is_refused(backend):
    flags = SimpleNamespace(device_data=True, fake_data=False, backend=backend)
    ds = SimpleNamespace(fake_data=False)
    with pytest.raises(ValueError, match=r"--device_data needs the sm_90a engine .*--backend=%s" % backend):
        check_device_data_flags(flags, SimpleNamespace(on_gpu=True), ds)
    for ok in ("auto", "fused"):                              # the sm_90a engine's backends pass
        check_device_data_flags(SimpleNamespace(device_data=True, fake_data=False, backend=ok), SimpleNamespace(on_gpu=True), ds)
    check_device_data_flags(SimpleNamespace(device_data=False, fake_data=True, backend=backend), SimpleNamespace(on_gpu=False), ds)


def _twins(n, seed, count):
    imgs, labels, _, _ = mnist_data.make_synthetic_mnist(n, 10, seed=seed)
    return [mnist_data.DataSet(imgs, labels, seed=seed + 1) for _ in range(count)]


@pytest.fixture
def no_pinning(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self, *a, **k: self)      # no CUDA on the CPU tier


def test_index_feed_yields_the_datasets_index_sequence_and_gathers_next_batch(no_pinning):
    N, B = 1000, 96                                           # B does not divide N: every epoch drops a remainder
    a, b, c = _twins(N, 9, 3)
    feed = _IndexFeed(a, B)
    table_x = np.asarray(a.images, np.float32).reshape(N, 784)
    table_y = np.asarray(a.labels, np.int64)
    for _ in range(35):                                       # 35 x 96 = 3360 rows: three epoch wraps
        idx = feed.next()
        assert idx.dtype == torch.int32 and idx.shape == (B,)
        ref = b.next_batch_indices(B)
        np.testing.assert_array_equal(idx.numpy(), ref)
        x, y = c.next_batch(B)
        assert table_x[idx.numpy()].tobytes() == np.asarray(x, np.float32).reshape(B, 784).tobytes()
        assert table_y[idx.numpy()].tobytes() == np.asarray(y, np.int64).tobytes()
    assert a.epochs_completed == b.epochs_completed == 3


class _RecordingEngine:
    """Stands in for the engine: records each buffer it is handed and checks that none it may still be reading changed."""

    def __init__(self):
        self.handed = []                                      # (step, buffer, contents when handed over)

    def step_indices(self, buf):
        for step, b, snap in self.handed[-2:]:                # the DMAs of the last two steps may not have run yet
            assert torch.equal(b, snap), "buffer of step %d rewritten after %d more launches" % (step, len(self.handed) - step)
        self.handed.append((len(self.handed), buf, buf.clone()))


def test_index_feed_rewrites_a_buffer_only_after_two_more_steps_were_launched(no_pinning):
    (ds,) = _twins(500, 4, 1)
    feed = _IndexFeed(ds, 64)
    eng = _RecordingEngine()
    for _ in range(40):
        eng.step_indices(feed.next())
    last = {}
    for step, buf, _snap in eng.handed:
        key = buf.data_ptr()
        if key in last:
            assert step - last[key] >= 3, "a buffer was handed out again %d steps later" % (step - last[key])
        last[key] = step
    assert len(last) == len(feed.ring) >= 3
