"""Elastic distortion on the CPU (``--augment_elastic_alpha`` / ``_sigma``): the flags and their refusals, the draws and
their key, the field against scipy's Gaussian filter, the warp with a field, the torch engine's augmented step, a gloo
mlp2 ``train()`` run whose training batches are distorted while its evaluations are not, and the trajectory harness's
augment stage on emulated elastic steps seeded right and wrong."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.ndimage
import torch

from distributedmnist_b200 import augment as AU
from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.engine import TorchEngine
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.ops import trajectory as T
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.train import train

EL = AU.Elastic(34.0, 4.0)
AFFINE = AU.Ranges(2.0, 15.0, 0.1)


@pytest.fixture
def clean_flags():
    FLAGS.reset()
    saved = {k: os.environ.pop(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") if k in os.environ}
    yield FLAGS
    FLAGS.reset()
    os.environ.update(saved)


def _flags(**kw):
    d = dict(augment_max_shift=0.0, augment_max_rotation=0.0, augment_max_scale=0.0, augment_elastic_alpha=0.0,
             augment_elastic_sigma=4.0)
    d.update(kw)
    return SimpleNamespace(**d)


def _images(n, seed=0):
    return np.random.default_rng(seed).uniform(-0.5, 0.5, (n, 28, 28))


def _engine(model="mlp2", B=4, rank=0):
    return TorchEngine(model, B, torch.device("cpu"), lambda n: torch.zeros(n), seed=9, rank=rank, mlp_hidden=64)


# ---- flags -------------------------------------------------------------------------------------------------------------
def test_flags_default_off_and_parse(clean_flags):
    assert AU.elastic_from_flags(FLAGS) is None
    FLAGS.parse(["--augment_elastic_alpha=34"])
    assert AU.elastic_from_flags(FLAGS) == AU.Elastic(34.0, 4.0) and AU.from_flags(FLAGS) is None
    FLAGS.reset()
    FLAGS.parse(["--augment_elastic_alpha", "8", "--augment_elastic_sigma=0.5", "--augment_max_shift=2"])
    assert AU.elastic_from_flags(FLAGS) == AU.Elastic(8.0, 0.5) and AU.from_flags(FLAGS) == AU.Ranges(2.0, 0.0, 0.0)
    assert AU.elastic_from_flags(_flags(augment_elastic_alpha=64.0, augment_elastic_sigma=8.0)) == AU.Elastic(64.0, 8.0)
    AU.check_flags(_flags())


@pytest.mark.parametrize("kw,name", [
    (dict(augment_elastic_alpha=-1.0), "--augment_elastic_alpha"),
    (dict(augment_elastic_alpha=64.5), "--augment_elastic_alpha"),
    (dict(augment_elastic_alpha=float("nan")), "--augment_elastic_alpha"),
    (dict(augment_elastic_alpha=float("inf")), "--augment_elastic_alpha"),
    (dict(augment_elastic_alpha=1.0, augment_elastic_sigma=0.4), "--augment_elastic_sigma"),
    (dict(augment_elastic_alpha=1.0, augment_elastic_sigma=8.5), "--augment_elastic_sigma"),
    (dict(augment_elastic_alpha=1.0, augment_elastic_sigma=float("nan")), "--augment_elastic_sigma"),
    (dict(augment_elastic_sigma=3.0), "--augment_elastic_sigma needs --augment_elastic_alpha"),
])
def test_out_of_range_non_finite_or_orphan_values_are_refused(kw, name):
    with pytest.raises(ValueError, match=name):
        AU.check_flags(_flags(**kw))
    if "augment_elastic_alpha" in kw:              # the engine refuses the same values (alpha 0 there is simply off)
        with pytest.raises(ValueError, match=name):
            _engine().arm_augment(0.0, 0.0, 0.0, elastic=AU.Elastic(kw.get("augment_elastic_alpha", 0.0),
                                                                    kw.get("augment_elastic_sigma", 4.0)))


@pytest.mark.parametrize("flag", ["--augment_elastic_alpha=65", "--augment_elastic_sigma=2"])
def test_train_refuses_before_any_work(tmp_path, clean_flags, flag):
    FLAGS.parse(["--train_dir=%s" % tmp_path, flag, "--model=mlp2", "--mlp_hidden=32"])
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(64, 32))
    with pytest.raises(ValueError, match=flag.split("=")[0]):
        train(ctx, ds.train, ds.validation, FLAGS)
    assert not os.listdir(tmp_path)


# ---- the draws and the field -------------------------------------------------------------------------------------------
def test_elastic_keys_differ_from_every_affine_key():
    """E_r = seed_mix(s, r) + ELASTIC_MIX equals some affine key seed_mix(s, r') = seed_mix(s, r) + (r' - r) RANK_MIX
    only if ELASTIC_MIX = k RANK_MIX (mod 2^32) with k = r' - r; for up to 1024 replicas |k| < 1024."""
    k = np.arange(-1023, 1024, dtype=np.int64)
    assert not np.any((k * AU.RANK_MIX) % 2 ** 32 == AU.ELASTIC_MIX)
    keys = {AU.seed_mix(7, r) for r in range(1024)}
    assert not keys & {(AU.seed_mix(7, r) + AU.ELASTIC_MIX) & 0xFFFFFFFF for r in range(1024)}


def test_draws_follow_the_documented_hash():
    mix, it, rows = AU.seed_mix(3, 2), 2 ** 32 - 1, 5
    v = AU.elastic_uniforms(mix, it, rows)
    key = int(AU.hash_mix((mix + AU.ELASTIC_MIX) & 0xFFFFFFFF, it))
    for b, d, p in ((0, 0, 0), (1, 1, 783), (4, 0, 29), (3, 1, 400)):
        h = int(AU.hash_mix(key, 1568 * b + 784 * d + p))
        assert v[b, d, p] == 2.0 * ((h >> 8) * 2.0 ** -24) - 1.0
    assert np.array_equal(v.astype(np.float32).astype(np.float64), v) and v.min() >= -1.0 and v.max() < 1.0
    assert np.array_equal(AU.elastic_uniforms(mix, it, 2), v[:2])       # a row's draws do not depend on the batch size
    with pytest.raises(ValueError, match="at most 2739137 rows"):
        AU.elastic_uniforms(mix, it, AU.MAX_ELASTIC_BATCH + 1)
    assert 1568 * AU.MAX_ELASTIC_BATCH <= 2 ** 32 < 1568 * (AU.MAX_ELASTIC_BATCH + 1)


@pytest.mark.parametrize("sigma", [0.5, 1.3, 4.0, 8.0])
def test_field_is_alpha_times_scipy_gaussian_filter(sigma):
    mix, it, rows = AU.seed_mix(11, 1), 77, 6
    el = AU.Elastic(34.0, sigma)
    f = AU.elastic_field(mix, it, rows, el)
    v = AU.elastic_uniforms(mix, it, rows).reshape(rows, 2, 28, 28)
    want = np.stack([[el.alpha * scipy.ndimage.gaussian_filter(v[b, d], sigma, mode="constant", cval=0.0, truncate=4.0)
                      for d in range(2)] for b in range(rows)])
    assert f.shape == (rows, 2, 28, 28) and np.abs(f - want).max() <= 1e-12
    w = AU.gaussian_weights(sigma)
    assert len(w) == int(4 * sigma + 0.5) + 1 <= 33
    assert abs(w[0] + 2 * w[1:].sum() - 1.0) <= 1e-15 and np.all(np.diff(w) < 0)


# ---- the warp ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ex,ey", [(0, 0), (1, 0), (0, -2), (3, 5), (-27, 1), (30, 0)])
def test_integer_constant_field_is_an_integer_shift(ex, ey):
    img = _images(3, 1)
    f = np.zeros((3, 2, 28, 28))
    f[:, 0], f[:, 1] = ex, ey
    got = AU.warp(img, 1.0, 0.0, 0.0, 0.0, field=f)
    want = np.full_like(img, AU.BACKGROUND)            # output (x, y) reads source (x + ex, y + ey)
    ys, xs = slice(max(0, -ey), min(28, 28 - ey)), slice(max(0, -ex), min(28, 28 - ex))
    ys_src, xs_src = slice(max(0, ey), min(28, 28 + ey)), slice(max(0, ex), min(28, 28 + ex))
    if abs(ex) < 28 and abs(ey) < 28:                  # else every output pixel is background
        want[:, ys, xs] = img[:, ys_src, xs_src]
    assert np.array_equal(got, want)


def test_warp_without_field_is_unchanged_and_field_composes_before_the_affine_map():
    img = _images(4, 2)
    a, b, tx, ty = (np.array(v) for v in ([0.9, 1.1, 1.0, 0.7], [0.2, -0.1, 0.0, 0.3], [1.5, 0.0, -2.0, 0.25],
                                          [0.0, 1.0, 3.0, -0.5]))
    assert np.array_equal(AU.warp(img, a, b, tx, ty, field=None), AU.warp(img, a, b, tx, ty))
    assert np.array_equal(AU.warp(img, a, b, tx, ty, field=np.zeros((4, 2, 784))), AU.warp(img, a, b, tx, ty))
    # a constant field (ex, ey) under the affine map is the affine map with the shift tx - ex, ty - ey
    f = np.zeros((4, 2, 28, 28))
    f[:, 0], f[:, 1] = 0.75, -1.25
    assert np.allclose(AU.warp(img, a, b, tx, ty, field=f), AU.warp(img, a, b, tx - 0.75, ty + 1.25), atol=1e-12)


def test_augment_batch_without_elastic_is_unchanged():
    img = _images(8, 3).astype(np.float32)
    mix = AU.seed_mix(5, 0)
    assert np.array_equal(AU.augment_batch(img, mix, 9, AFFINE, None), AU.augment_batch(img, mix, 9, AFFINE))
    out = AU.augment_batch(img, mix, 9, AFFINE, EL)
    c = AU.coefficients(AU.uniforms(mix, 9, 8), AFFINE)
    want = AU.warp(img, *c, field=AU.elastic_field(mix, 9, 8, EL)).astype(np.float32)
    assert out.dtype == np.float32 and np.array_equal(out, want)
    assert not np.array_equal(out, AU.augment_batch(img, mix, 9, AFFINE))


# ---- the torch engine and train() --------------------------------------------------------------------------------------
@pytest.mark.parametrize("model,ranges", [("lenet", AFFINE), ("mlp2", AU.Ranges(0.0, 0.0, 0.0))])
def test_torch_engine_trains_on_the_distorted_batch(model, ranges):
    B = 8
    g = torch.Generator().manual_seed(5)
    shape = (B, 28, 28, 1) if model == "lenet" else (B, 784)
    x, y = torch.rand(*shape, generator=g) - 0.5, torch.randint(0, 10, (B,), generator=g)
    eng = _engine(model, B, rank=1)
    eng.arm_augment(*ranges, start_iteration=41, elastic=EL)
    eng.load_batch(x, y)
    eng.forward_backward(0)
    got = eng.augmented_batch()
    want = AU.augment_batch(x.numpy(), AU.seed_mix(9, 1), 41, ranges, EL)
    assert got.shape == x.shape and np.array_equal(got.numpy(), want)
    assert eng.augment_iteration() == 42
    ref = _engine(model, B, rank=1)
    ref.load_batch(torch.from_numpy(want), y)
    ref.forward_backward(0)
    assert torch.equal(ref.grads, eng.grads)
    assert eng.evaluate(x, y) == ref.evaluate(x, y)                 # evaluation is never distorted
    eng.arm_augment(0.0, 0.0, 0.0, elastic=AU.Elastic(0.0, 4.0))     # alpha 0: off
    assert eng.augmented_batch() is None


def test_gloo_mlp2_run_distorts_training_only(tmp_path, clean_flags, caplog, monkeypatch):
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
    FLAGS.parse(["--train_dir=%s" % (tmp_path / "el"), "--batch_size=32", "--max_steps=6", "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000",
                 "--initial_learning_rate=0.05", "--backend=gloo", "--augment_elastic_alpha=34",
                 "--augment_elastic_sigma=3", "--eval_every_steps=3"])
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    res = train(ctx, ds.train, ds.validation, FLAGS)
    assert len(seen) == res["final_step"] >= 6
    assert any("elastic distortion alpha 34 px, sigma 3 px, draws from iteration 0;" in r.getMessage()
               for r in caplog.records)
    mix, el = AU.seed_mix(FLAGS.seed, 0), AU.Elastic(34.0, 3.0)
    for i, (plain, aug, it) in enumerate(seen):
        assert it == i + 1
        assert np.array_equal(aug.numpy(), AU.augment_batch(plain.numpy(), mix, i, AU.Ranges(0.0, 0.0, 0.0), el))
        assert not torch.equal(plain, aug)
    assert evals and all(np.array_equal(e, ds.validation.images) for e in evals)


# ---- the trajectory harness's augment stage ----------------------------------------------------------------------------
def _counter(it):
    return torch.from_numpy(np.array([it & 0xFFFFFFFF, 0], dtype=np.uint32).view(np.int32))


def _fault_images(x, mix, it, ranges, el, fault):
    """The buffer an elastic step with ``fault`` would write, in fp32 like the kernel."""
    n = x.shape[0]
    if fault == "next_iteration":
        it += 1
    c = AU.coefficients(AU.uniforms(mix, it, n), ranges)
    f = AU.elastic_field(mix, it, n, el)
    if fault == "swapped_components":
        f = f[:, ::-1]
    if fault == "no_field":
        f = None
    return AU.warp(x, *c, field=f).astype(np.float32).reshape(n, 784)


def _stage(ranges, fault=None, steps=3, B=16, start=2 ** 32 - 2):
    mix = AU.seed_mix(5, 0)
    gen = torch.Generator().manual_seed(4)
    batches = [(torch.rand(B, 28, 28, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen))
               for _ in range(steps)]
    init = dict(aug_counter=_counter(start))
    records = [dict(aug_images=torch.from_numpy(_fault_images(x.numpy(), mix, start + t, ranges, EL, fault)),
                    aug_counter=_counter(start + t + 1)) for t, (x, _y) in enumerate(batches)]
    upd = dict(aug=(ranges, mix), aug_start=start, elastic=EL)
    return T.augment_stage_results("lenet", init, records, batches, upd)


@pytest.mark.parametrize("ranges", [AFFINE, AU.Ranges(0.0, 0.0, 0.0)], ids=["affine", "elastic_only"])
def test_emulated_elastic_steps_pass_with_every_premise(ranges):
    res = _stage(ranges)
    assert not T.failures(res), T.failures(res)
    worst = T.worst_by_stage("lenet", res)
    for p in ("iteration_minus_1", "iteration_plus_1", "next_rank", "swapped_components", "no_field", "sigma_1.25"):
        assert "augment.premise.%s_detectable" % p in worst, sorted(worst)
    assert "augment[err/bound]" in worst and all(0 <= v <= 1 for v in worst.values()), worst


@pytest.mark.parametrize("fault", ["next_iteration", "swapped_components", "no_field"])
def test_seeded_elastic_fault_fails_at_the_augment_stage(fault):
    bad = T.failures(_stage(AFFINE, fault))
    assert bad and all(".augment[err/bound]" in n for n, _, _ in bad), bad[:10]
