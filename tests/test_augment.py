"""Random affine augmentation on the CPU (``--augment_max_shift`` / ``_rotation`` / ``_scale``): the flags and their
refusals, the numpy emulation of the draws, the float64 warp, the torch engine's augmented step, and a gloo mlp2
``train()`` run whose training batches are augmented while its evaluations are not."""
import math
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from distributedmnist_b200 import augment as AU
from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.engine import TorchEngine
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.models.lenet import dropout_keep_mask
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.train import train


@pytest.fixture
def clean_flags():
    FLAGS.reset()
    saved = {k: os.environ.pop(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") if k in os.environ}
    yield FLAGS
    FLAGS.reset()
    os.environ.update(saved)


def _flags(**kw):
    d = dict(augment_max_shift=0.0, augment_max_rotation=0.0, augment_max_scale=0.0)
    d.update(kw)
    return SimpleNamespace(**d)


def _images(n, seed=0):
    return np.random.default_rng(seed).uniform(-0.5, 0.5, (n, 28, 28))


# ---- flags -------------------------------------------------------------------------------------------------------------
def test_flags_default_off_and_parse(clean_flags):
    assert AU.from_flags(FLAGS) is None
    FLAGS.parse(["--augment_max_shift=2", "--augment_max_rotation", "15", "--augment_max_scale=0.1"])
    assert AU.from_flags(FLAGS) == AU.Ranges(2.0, 15.0, 0.1)
    FLAGS.reset()
    FLAGS.parse(["--augment_max_rotation=180"])
    assert AU.from_flags(FLAGS) == AU.Ranges(0.0, 180.0, 0.0)
    assert AU.from_flags(_flags(augment_max_shift=8.0, augment_max_scale=0.999)) == AU.Ranges(8.0, 0.0, 0.999)


@pytest.mark.parametrize("kw", [dict(augment_max_shift=-1.0), dict(augment_max_shift=8.5), dict(augment_max_rotation=-0.1),
                                dict(augment_max_rotation=181.0), dict(augment_max_scale=1.0), dict(augment_max_scale=-0.2),
                                dict(augment_max_shift=float("nan")), dict(augment_max_rotation=float("inf")),
                                dict(augment_max_scale=float("nan"))])
def test_out_of_range_or_non_finite_values_are_refused(kw):
    name = "--" + next(iter(kw))
    with pytest.raises(ValueError, match=name):
        AU.check_flags(_flags(**kw))
    with pytest.raises(ValueError, match=name):
        TorchEngine("mlp2", 4, torch.device("cpu"), lambda n: torch.zeros(n), mlp_hidden=64).arm_augment(
            kw.get("augment_max_shift", 0.0), kw.get("augment_max_rotation", 0.0), kw.get("augment_max_scale", 0.0))


def test_train_refuses_before_any_work(tmp_path, clean_flags):
    FLAGS.parse(["--train_dir=%s" % tmp_path, "--augment_max_shift=9", "--model=mlp2", "--mlp_hidden=32"])
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(64, 32))
    with pytest.raises(ValueError, match="--augment_max_shift"):
        train(ctx, ds.train, ds.validation, FLAGS)
    assert not os.listdir(tmp_path)


# ---- the draws ---------------------------------------------------------------------------------------------------------
def test_hash_is_the_dropout_hash():
    """hash_mix is csrc/common.cuh's (the one models/lenet.py emulates for the dropout mask)."""
    mix = 0x1234ABCD
    h = AU.hash_mix(mix, np.arange(64 * 32, dtype=np.uint64))
    want = dropout_keep_mask(mix, 64, 32, 0.5).numpy().reshape(-1)
    assert np.array_equal((h >> np.uint64(8)) < (1 << 23), want)


def test_draws_lie_in_the_unit_interval_and_differ_everywhere():
    mix = AU.seed_mix(66478, 0)
    u = AU.uniforms(mix, 5, 512)
    assert u.shape == (512, 4) and u.min() >= 0.0 and u.max() < 1.0
    assert np.array_equal(u * 2 ** 24, np.floor(u * 2 ** 24))                   # multiples of 2^-24: exact in fp32
    assert np.array_equal(u.astype(np.float32).astype(np.float64), u)
    assert 0.45 < u.mean() < 0.55 and u.min() < 0.01 and u.max() > 0.99
    assert len(np.unique(u)) > 0.99 * u.size                                    # rows and k differ
    assert not np.array_equal(u[:, 0], u[:, 1]) and not np.array_equal(u[:, 2], u[:, 3])
    others = [AU.uniforms(AU.seed_mix(66478, 1), 5, 512),                        # replica
              AU.uniforms(mix, 6, 512),                                         # iteration
              AU.uniforms(AU.seed_mix(66479, 0), 5, 512)]                        # seed
    for v in others:
        assert np.mean(v == u) < 0.01
    assert AU.seed_mix(66478, 0) != AU.seed_mix(66478, 1)
    from distributedmnist_b200.models.lenet import dropout_seed_mix
    assert AU.seed_mix(66478, 0) != dropout_seed_mix(66478, 0, 0)


def test_draws_do_not_depend_on_the_batch_size():
    mix = AU.seed_mix(7, 3)
    big = AU.uniforms(mix, 2 ** 32 - 1, 8192)
    for rows in (1, 96, 256):
        assert np.array_equal(AU.uniforms(mix, 2 ** 32 - 1, rows), big[:rows])
    assert np.array_equal(AU.uniforms(mix, 2 ** 32 + 4, 4), AU.uniforms(mix, 4, 4))   # the iteration is a u32


def test_rank_mix_steps_to_the_next_rank():
    for seed, rank in ((66478, 0), (7, 3), (2 ** 31 + 5, 6)):
        assert (AU.seed_mix(seed, rank) + AU.RANK_MIX) & 0xFFFFFFFF == AU.seed_mix(seed, rank + 1)


def test_restart_start_iteration():
    """Past the iterations that went into the restored step: g with K <= N, K g with K > N (count-triggered runs only),
    g for interval / cdf runs; a u32."""
    assert AU.start_iteration(0, True, 4, 1) == 0
    assert AU.start_iteration(13, True, 1, 1) == 13
    assert AU.start_iteration(13, True, 6, 8) == 13                   # K < N: one iteration per global step
    assert AU.start_iteration(13, True, 8, 8) == 13
    assert AU.start_iteration(13, True, 4, 1) == 52
    assert AU.start_iteration(13, True, 16, 8) == 208
    assert AU.start_iteration(13, False, 16, 8) == 13                 # interval: not a function of the global step
    assert AU.start_iteration(2 ** 31, True, 4, 1) == 0


# ---- the warp ----------------------------------------------------------------------------------------------------------
def test_zero_ranges_are_the_identity():
    img = _images(16).astype(np.float32)
    out = AU.augment_batch(img, AU.seed_mix(1, 0), 3, AU.Ranges(0.0, 0.0, 0.0))
    assert out.dtype == np.float32 and np.array_equal(out, img)
    flat = img.reshape(16, 784)
    assert np.array_equal(AU.augment_batch(flat, 5, 0, AU.Ranges(0.0, 0.0, 0.0)), flat)


@pytest.mark.parametrize("tx,ty", [(3, -2), (-8, 8), (1, 0), (0, 5), (30, 0)])
def test_integer_shift_fills_with_the_background(tx, ty):
    img = _images(4, 1)
    out = AU.warp(img, 1.0, 0.0, tx, ty)
    want = np.full_like(img, AU.BACKGROUND)
    # out[y, x] = img[y - ty, x - tx]
    ys, xs = slice(max(ty, 0), 28 + min(ty, 0)), slice(max(tx, 0), 28 + min(tx, 0))
    yd, xd = slice(max(-ty, 0), 28 + min(-ty, 0)), slice(max(-tx, 0), 28 + min(-tx, 0))
    if abs(tx) < 28 and abs(ty) < 28:
        want[:, ys, xs] = img[:, yd, xd]
    assert np.array_equal(out, want)


def test_quarter_turns_are_rot90():
    img = _images(3, 2)
    # theta = +90 degrees samples src[27 - x][y]: np.rot90 clockwise; -90 degrees counter-clockwise
    for theta, k in ((math.pi / 2, -1), (-math.pi / 2, 1)):
        out = AU.warp(img, *AU.affine(theta, 1.0, 0.0, 0.0))
        want = np.rot90(img, k, axes=(1, 2))
        assert np.max(np.abs(out - want)) <= 1e-12
    out = AU.warp(img, *AU.affine(math.pi, 1.0, 0.0, 0.0))
    assert np.max(np.abs(out - img[:, ::-1, ::-1])) <= 1e-12


def test_zoom_and_half_pixel_shift_interpolate():
    img = _images(2, 3)
    half = AU.warp(img, 1.0, 0.0, 0.5, 0.0)          # samples x - 0.5: the mean of two neighbours
    assert np.allclose(half[:, :, 1:], 0.5 * (img[:, :, 1:] + img[:, :, :-1]), atol=1e-15)
    assert np.allclose(half[:, :, 0], 0.5 * (img[:, :, 0] + AU.BACKGROUND), atol=1e-15)
    big = AU.warp(img, *AU.affine(0.0, 1e6, 0.0, 0.0))   # zoom in a million times: the centre's 2x2 blend everywhere
    c = img[:, 13:15, 13:15].mean(axis=(1, 2))
    assert np.allclose(big, c[:, None, None], atol=1e-5)
    tiny = AU.warp(img, *AU.affine(0.0, 1e-3, 0.0, 0.0))  # zoom out: everything but the centre is background
    assert np.all(tiny[:, :13, :] == AU.BACKGROUND)


def test_augmented_batch_matches_its_coefficients():
    img = _images(32, 4).astype(np.float32)
    r = AU.Ranges(2.0, 30.0, 0.2)
    mix = AU.seed_mix(66478, 2)
    out = AU.augment_batch(img, mix, 17, r)
    a, b, tx, ty = AU.coefficients(AU.uniforms(mix, 17, 32), r)
    assert np.array_equal(out, AU.warp(img, a, b, tx, ty).astype(np.float32))
    theta = np.arctan2(b, a)
    s = 1.0 / np.hypot(a, b)
    assert np.all(np.abs(theta) <= math.radians(30.0) + 1e-12) and np.all(np.abs(s - 1.0) <= 0.2 + 1e-12)
    assert np.all(np.abs(tx) <= 2.0) and np.all(np.abs(ty) <= 2.0)
    assert out.min() >= -0.5 - 1e-7 and out.max() <= 0.5 + 1e-7
    assert not np.array_equal(out, img)


# ---- the torch engine --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["lenet", "mlp2"])
def test_torch_engine_trains_on_the_augmented_batch(model):
    B = 8
    g = torch.Generator().manual_seed(5)
    shape = (B, 28, 28, 1) if model == "lenet" else (B, 784)
    x, y = torch.rand(*shape, generator=g) - 0.5, torch.randint(0, 10, (B,), generator=g)
    r = AU.Ranges(3.0, 20.0, 0.1)

    def engine():
        return TorchEngine(model, B, torch.device("cpu"), lambda n: torch.zeros(n), seed=9, rank=1, mlp_hidden=64)

    eng = engine()
    eng.arm_augment(*r, start_iteration=41)
    eng.load_batch(x, y)
    eng.forward_backward(0)
    got = eng.augmented_batch()
    want = AU.augment_batch(x.numpy(), AU.seed_mix(9, 1), 41, r)
    assert got.shape == x.shape and np.array_equal(got.numpy(), want)
    assert eng.augment_iteration() == 42
    ref = engine()                                  # fed the augmented images, no augmentation: the same gradient
    ref.load_batch(torch.from_numpy(want), y)
    ref.forward_backward(0)
    assert torch.equal(ref.grads, eng.grads)
    eng.forward_backward(0)                         # the next iteration draws anew
    assert not torch.equal(eng.augmented_batch(), got)
    assert eng.evaluate(x, y) == ref.evaluate(x, y)                 # evaluation is never augmented
    eng.arm_augment(0.0, 0.0, 0.0)
    assert eng.augmented_batch() is None


# ---- train() -----------------------------------------------------------------------------------------------------------
def _train(train_dir, *extra, steps=8):
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=32", "--max_steps=%d" % steps, "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000", "--initial_learning_rate=0.05",
                 "--backend=gloo"] + list(extra))
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    return train(ctx, ds.train, ds.validation, FLAGS), ds


def test_gloo_mlp2_run_augments_training_only(tmp_path, clean_flags, caplog, capsys, monkeypatch):
    from distributedmnist_b200.checkpoint import Saver
    from distributedmnist_b200.evaluator import evaluate
    seen, evals = [], []
    fb, ev = TorchEngine.forward_backward, TorchEngine.evaluate

    def record_step(self, step):
        fb(self, step)
        seen.append((self._images.clone(), self.augmented_batch().clone(), self.augment_iteration()))

    def record_eval(self, images, labels, *a, **kw):
        evals.append(np.array(images, copy=True))
        return ev(self, images, labels, *a, **kw)

    monkeypatch.setattr(TorchEngine, "forward_backward", record_step)
    monkeypatch.setattr(TorchEngine, "evaluate", record_eval)
    d = tmp_path / "aug"
    res, ds = _train(str(d), "--augment_max_shift=2", "--augment_max_rotation=15", "--augment_max_scale=0.1",
                     "--eval_every_steps=4")
    assert len(seen) == res["final_step"] >= 8
    assert any("Random affine augmentation of the training images: shift up to 2 px, rotation up to 15 degrees"
               in r.getMessage() for r in caplog.records)
    mix = AU.seed_mix(FLAGS.seed, 0)
    r = AU.Ranges(2.0, 15.0, 0.1)
    for i, (plain, aug, it) in enumerate(seen):
        assert it == i + 1
        assert not torch.equal(plain, aug)
        assert np.array_equal(aug.numpy(), AU.augment_batch(plain.numpy(), mix, i, r))
    # the in-training evaluations score the validation images as they are
    assert evals and all(np.array_equal(e, ds.validation.images) for e in evals)
    # the evaluator scores the checkpoint on unaugmented images, although the flags are still set
    evals.clear()
    FLAGS.parse(["--checkpoint_dir=%s" % d, "--eval_dir=%s" % (tmp_path / "eval"), "--run_once=true"])
    capsys.readouterr()
    assert evaluate(ds.validation, FLAGS, device=torch.device("cpu")) == str(res["final_step"])
    m = re.search(r"Num examples: 64  Precision @ 1: ([0-9.]+) Loss: ([0-9.]+) Time: ", capsys.readouterr().out)
    assert m and evals and np.array_equal(evals[0], ds.validation.images)
    state, _step = Saver.restore(Saver.latest(str(d)))
    eng = TorchEngine("mlp2", 32, torch.device("cpu"), lambda n: torch.zeros(n), mlp_hidden=32)
    eng.params.copy_(eng.spec.from_state_dict(state))
    loss, acc = ev(eng, ds.validation.images, ds.validation.labels)
    assert float(m.group(2)) == pytest.approx(loss, abs=2e-6) and float(m.group(1)) == pytest.approx(acc, abs=2e-6)
