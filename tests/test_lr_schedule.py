"""Learning-rate warmup and cosine decay on the CPU: the schedule against TF's ``cosine_decay`` and the closed forms of
torch's ``LinearLR`` / ``CosineAnnealingLR``, its exact identities, the refusals of ``check_lr_schedule_flags``, the torch
engine applying the scheduled rate, and ``FusedBackend`` refusing a host-evaluated rate once a block has one armed."""
import logging
import math
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.backends import LocalBackend
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.schedule import LearningRateSchedule, cosine_decay, exponential_decay
from distributedmnist_b200.train import check_lr_schedule_flags, train

SCRAPERS = [r".*step ([0-9]*),.*", r"Num examples: ([0-9]*)  Precision @ 1: ([\.0-9]*) Loss: ([\.0-9]*) Time: ([\.0-9]*)",
            r".* step=([0-9]*)", r".*ELAPSED TIMES (.*)", r".*ITERATION TIMES (.*)"]       # tools/benchmark.py
EPS = 2.0 ** -52


# ---- independent references ---------------------------------------------------------------------------------------
def tf_cosine_decay(lr0, step, decay_steps, alpha):
    """``tf.compat.v1.train.cosine_decay``, written out as TF computes it."""
    global_step = min(step, decay_steps)
    completed_fraction = global_step / decay_steps
    cosine_decayed = 0.5 * (1.0 + math.cos(math.pi * completed_fraction))
    decayed = (1 - alpha) * cosine_decayed + alpha
    return lr0 * decayed


def torch_linear_lr(lr0, step, total_iters, start_factor):
    """Closed form of ``torch.optim.lr_scheduler.LinearLR(start_factor, end_factor=1.0, total_iters)``."""
    return lr0 * (start_factor + (1.0 - start_factor) * min(total_iters, step) / total_iters)


def torch_cosine_annealing(lr0, step, t_max, eta_min):
    """Closed form of ``torch.optim.lr_scheduler.CosineAnnealingLR(T_max, eta_min)`` (no clamp: valid for s <= T_max)."""
    return eta_min + (lr0 - eta_min) * (1.0 + math.cos(math.pi * step / t_max)) / 2


SHAPES = [(0.1, 3, 1.0 / 3, 10, 0.0), (0.05, 100, 0.25, 1000, 0.0), (0.4, 500, 0.125, 20000, 0.01),
          (1.6, 1, 0.0, 7, 0.5), (0.02, 0, 1.0 / 3, 333, 0.1), (0.3, 64, 0.5, 0, 0.0), (0.25, 2, 0.1, 4, 0.0)]


def _probe_steps(w, t):
    top = 3 * max(t, w, 1)
    s = set(range(0, min(top, 2000) + 1)) | {int(x) for x in np.linspace(0, top, 500)}
    s |= {x for x in (w - 1, w, w + 1, t - 1, t, t + 1, 2 * t, 3 * t) if x >= 0}
    return sorted(s)


@pytest.mark.parametrize("lr0,w,f0,t,alpha", SHAPES)
def test_schedule_matches_tf_and_torch_closed_forms(lr0, w, f0, t, alpha):
    """Within a few double ulps of lr0 at every probed step, s = 0, W - 1, W, T - 1 and T included: against torch's
    LinearLR x CosineAnnealingLR up to T (torch's cosine does not clamp), and against TF's clamped form up to 3T."""
    sched = LearningRateSchedule(lr0, 10 ** 6, 0.999, warmup_steps=w, warmup_start=f0, cosine_steps=t, cosine_alpha=alpha)
    tol = 8 * EPS * lr0
    for s in _probe_steps(w, t):
        got = sched(s)
        warm = torch_linear_lr(1.0, s, w, f0) if w else 1.0
        if t:
            assert abs(got - tf_cosine_decay(lr0, s, t, alpha) * warm) <= tol, (s, got)
            if s <= t:
                assert abs(got - torch_cosine_annealing(lr0, s, t, alpha * lr0) * warm) <= tol, (s, got)
        else:
            assert abs(got - lr0 * warm) <= tol, (s, got)
        if w and s < w:
            assert abs(got - (tf_cosine_decay(lr0, s, t, alpha) if t else lr0) * warm) <= tol
            assert got < (tf_cosine_decay(lr0, s, t, alpha) if t else lr0)


@pytest.mark.parametrize("t", [1, 2, 7, 100, 12345, 2 ** 31])
def test_sin_squared_form_is_the_half_cosine(t):
    """The cancellation-free form equals (1 + cos) / 2 to within 1e-15 where the cosine is not near its end."""
    for s in sorted({0, 1, t // 4, t // 3, t // 2} | {int(x) for x in np.linspace(0, t // 2, 200)}):
        c = 0.5 * (1.0 + math.cos(math.pi * s / t))
        assert abs(cosine_decay(s, t, 0.0) - c) <= 1e-15 * c, (t, s)


@pytest.mark.parametrize("decay_steps,rate", [(1, 0.999), (7, 0.95), (100, 0.5), (3, 1.0)])
def test_no_warmup_and_no_cosine_is_the_old_schedule_bit_for_bit(decay_steps, rate):
    for cuts, factor in (((), 1.0), ((5, 9, 9, 40), 0.1), ((0, 3), 0.5)):
        sched = LearningRateSchedule(0.05, decay_steps, rate, factor=factor, cuts=cuts)
        assert not sched.shaped
        for s in list(range(120)) + [999, 10 ** 6 + 3]:
            lr = exponential_decay(0.05, s, decay_steps, rate)
            c = sum(1 for x in cuts if x <= s)
            want = lr * factor ** c if c else lr
            assert sched(s) == want and sched(s) == 0.05 * rate ** float(s // decay_steps) * (factor ** c if c else 1.0)


@pytest.mark.parametrize("alpha", [0.0, 0.01, 0.1, 0.5, 0.999])
def test_cosine_ends_exactly_at_alpha(alpha):
    """From step T on the rate is exactly lr0 * alpha (times the cuts): alpha = 0 stops the weights."""
    for w, t in ((0, 10), (3, 10), (9, 10), (0, 1), (50, 1000)):
        sched = LearningRateSchedule(0.3, 1, 0.9, warmup_steps=w, warmup_start=0.2, cosine_steps=t, cosine_alpha=alpha)
        for s in (t, t + 1, 2 * t, 10 ** 9):
            assert sched(s) == 0.3 * alpha
        assert sched(t - 1) > 0.3 * alpha
        sched.factor, sched.cuts = 0.5, [t]
        assert sched(t) == 0.3 * alpha * 0.5
    assert LearningRateSchedule(0.3, 1, 0.9, cosine_steps=5)(5) == 0.0


def test_warmup_is_exact_at_its_ends_and_multiplies_the_staircase():
    sched = LearningRateSchedule(0.2, 4, 0.5, warmup_steps=8, warmup_start=0.25)
    assert sched(0) == 0.2 * 0.25
    for s in range(8):
        assert sched(s) == 0.2 * 0.5 ** float(s // 4) * (0.25 + (0.75 * s) / 8)
    assert sched(8) == 0.2 * 0.5 ** 2.0
    # the cosine counts from step 0: the warmup multiplies its first steps
    c = LearningRateSchedule(0.2, 4, 0.5, warmup_steps=8, warmup_start=0.25, cosine_steps=16)
    for s in range(8):
        assert c(s) == 0.2 * cosine_decay(s, 16, 0.0) * (0.25 + (0.75 * s) / 8)
    assert c(8) == 0.2 * cosine_decay(8, 16, 0.0)


def test_from_flags_reads_the_four_flags():
    FLAGS.reset()
    try:
        FLAGS.parse(["--lr_warmup_steps=5", "--lr_warmup_start_factor=0.1", "--lr_cosine_decay_steps=50",
                     "--lr_cosine_alpha=0.02"])
        sched = LearningRateSchedule.from_flags(FLAGS, 60000, 1)
        assert (sched.warmup_steps, sched.warmup_start, sched.cosine_steps, sched.cosine_alpha) == (5, 0.1, 50, 0.02)
        assert sched.describe() == dict(warmup_steps=5, warmup_start_factor=0.1, cosine_decay_steps=50,
                                        cosine_alpha=0.02)
        FLAGS.reset()
        sched = LearningRateSchedule.from_flags(FLAGS, 60000, 1)
        assert (sched.warmup_steps, sched.warmup_start, sched.cosine_steps, sched.cosine_alpha) == (0, 1.0 / 3, 0, 0.0)
        assert not sched.shaped
    finally:
        FLAGS.reset()


# ---- refusals -------------------------------------------------------------------------------------------------------
def _flags(*args):
    FLAGS.reset()
    FLAGS.parse(list(args))
    return FLAGS


@pytest.mark.parametrize("args,msg", [
    (["--lr_warmup_steps=-1"], r"--lr_warmup_steps must lie in \[0, 2\^32 - 1\)"),
    (["--lr_warmup_steps=4294967295"], r"--lr_warmup_steps must lie"),
    (["--lr_cosine_decay_steps=-5"], r"--lr_cosine_decay_steps must lie"),
    (["--lr_cosine_decay_steps=4294967295"], r"--lr_cosine_decay_steps must lie"),
    (["--lr_warmup_steps=3", "--lr_warmup_start_factor=1.0"], r"--lr_warmup_start_factor must lie in \[0, 1\)"),
    (["--lr_warmup_steps=3", "--lr_warmup_start_factor=-0.1"], r"--lr_warmup_start_factor must lie"),
    (["--lr_warmup_steps=3", "--lr_warmup_start_factor=nan"], r"--lr_warmup_start_factor must lie"),
    (["--lr_warmup_steps=3", "--lr_warmup_start_factor=inf"], r"--lr_warmup_start_factor must lie"),
    (["--lr_cosine_decay_steps=9", "--lr_cosine_alpha=1"], r"--lr_cosine_alpha must lie in \[0, 1\)"),
    (["--lr_cosine_decay_steps=9", "--lr_cosine_alpha=-0.5"], r"--lr_cosine_alpha must lie"),
    (["--lr_cosine_decay_steps=9", "--lr_cosine_alpha=nan"], r"--lr_cosine_alpha must lie"),
    (["--lr_warmup_start_factor=0.5"], r"--lr_warmup_start_factor needs --lr_warmup_steps >= 1"),
    (["--lr_cosine_alpha=0.1"], r"--lr_cosine_alpha needs --lr_cosine_decay_steps >= 1"),
    (["--lr_cosine_decay_steps=9", "--learning_rate_decay_factor=0.9"],
     r"--lr_cosine_decay_steps replaces the staircase decay, so --learning_rate_decay_factor would do nothing"),
    (["--lr_cosine_decay_steps=9", "--num_epochs_per_decay=2"],
     r"so --num_epochs_per_decay would do nothing"),
    (["--lr_cosine_decay_steps=9", "--learning_rate_decay_factor=0.999", "--num_epochs_per_decay=2"],
     r"so --learning_rate_decay_factor and --num_epochs_per_decay would do nothing"),
])
def test_refusals_name_their_reason(args, msg):
    try:
        with pytest.raises(ValueError, match=msg):
            check_lr_schedule_flags(_flags(*args))
    finally:
        FLAGS.reset()


@pytest.mark.parametrize("args", [
    [], ["--lr_warmup_steps=1"], ["--lr_warmup_steps=4294967294", "--lr_warmup_start_factor=0"],
    ["--lr_cosine_decay_steps=1"], ["--lr_cosine_decay_steps=4294967294", "--lr_cosine_alpha=0.999"],
    ["--lr_warmup_steps=10", "--lr_warmup_start_factor=0.01", "--lr_cosine_decay_steps=100", "--lr_cosine_alpha=0.05"],
    ["--learning_rate_decay_factor=0.9", "--num_epochs_per_decay=1", "--lr_warmup_steps=10"],
    ["--lr_plateau_patience=1", "--eval_every_steps=5", "--lr_cosine_decay_steps=10"],
])
def test_accepted_combinations(args):
    try:
        check_lr_schedule_flags(_flags(*args))
    finally:
        FLAGS.reset()


def test_refused_before_any_work(tmp_path, monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    with pytest.raises(ValueError, match="--lr_cosine_alpha needs"):
        _train(str(tmp_path / "d"), "--lr_cosine_alpha=0.5")
    assert not os.path.exists(str(tmp_path / "d"))


# ---- the torch engine -----------------------------------------------------------------------------------------------
def _train(train_dir, *extra, steps=6):
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=32", "--max_steps=%d" % steps, "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000", "--initial_learning_rate=0.05",
                 "--backend=gloo", "--dropout_keep_prob=1.0"] + list(extra))
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    return train(ctx, ds.train, ds.validation, FLAGS)


def test_torch_engine_applies_the_warmup(tmp_path, monkeypatch, caplog):
    """One replica on the CPU with W = 3: the rate of each of the first steps, estimated from the parameter delta and the
    gradient, is the scheduled one, not the staircase's."""
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    seen = []
    real = LocalBackend.sync_step

    def spy(self, params, grads, lr, local_step, k, delay_s=0.0):
        w0 = params.detach().double().clone()
        info = real(self, params, grads, lr, local_step, k, delay_s)
        seen.append((local_step, w0, grads.detach().double().clone(), params.detach().double().clone()))
        return info

    monkeypatch.setattr(LocalBackend, "sync_step", spy)
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(str(tmp_path / "warm"), "--lr_warmup_steps=3", "--lr_warmup_start_factor=0.2", steps=5)
    FLAGS.reset()
    sched = res["optimizer"].lr_schedule
    plain = LearningRateSchedule(0.05, sched.decay_steps, sched.decay_rate)
    assert res["lr_schedule"] == dict(warmup_steps=3, warmup_start_factor=0.2, cosine_decay_steps=0, cosine_alpha=0.0)
    assert [s for s, *_ in seen] == list(range(len(seen))) and len(seen) >= 5
    for s, w0, g, w1 in seen:
        rate = -float(((w1 - w0) * g).sum() / (g * g).sum())
        assert rate == pytest.approx(sched(s), rel=1e-4), s
        if s < 3:
            assert sched(s) == plain(s) * (0.2 + (0.8 * s) / 3)
            assert rate != pytest.approx(plain(s), rel=1e-3)
        else:
            assert sched(s) == plain(s)
    msgs = [m.getMessage() for m in caplog.records]
    line = [m for m in msgs if m.startswith("Learning rate schedule: ")]
    assert line == ["Learning rate schedule: 0.05 decayed by 0.999 every %d global steps, linear warmup from 0.2 of it "
                    "over global steps 0 to 2; the update of global step #0 is made at %g" % (sched.decay_steps, 0.01)]
    assert not any(re.match(p, line[0]) for p in SCRAPERS)


def test_torch_engine_results_carry_the_schedule_when_off(tmp_path, monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    res = _train(str(tmp_path / "off"), steps=2)
    FLAGS.reset()
    assert res["lr_schedule"] == dict(warmup_steps=0, warmup_start_factor=1.0 / 3, cosine_decay_steps=0,
                                      cosine_alpha=0.0)


# ---- no double application ------------------------------------------------------------------------------------------
def test_fused_backend_refuses_a_host_rate_once_a_schedule_is_armed():
    """set_lr_schedule hands its words to the entry point; with a schedule armed, sync_step and interval_tick (which pass
    a rate the host evaluated) raise before they launch anything."""
    from distributedmnist_b200.parallel.fused import FusedBackend
    calls = []
    be = FusedBackend.__new__(FusedBackend)
    be.lib = SimpleNamespace(dm_sync_set_lr_schedule=lambda *a: calls.append(a))
    be.ctrl = SimpleNamespace(local_ptr=0x1000)
    be.set_lr_schedule(3, 0.25, 0, 0.0)
    assert calls == [(0x1000, 3, 0.25, 0, 0.0)] and be.lr_schedule_armed
    with pytest.raises(RuntimeError, match="sync_step passes a learning rate the host evaluated"):
        be.sync_step(None, None, 0.1, 0, 1)
    with pytest.raises(RuntimeError, match="interval_tick passes a learning rate the host evaluated"):
        be.interval_tick(None, None, 1, 0.1, 0)
    be.set_lr_schedule(0, 1.0 / 3, 7, 0.5)
    assert be.lr_schedule_armed
    be.set_lr_schedule(0, 1.0 / 3, 0, 0.0)
    assert not be.lr_schedule_armed and len(calls) == 3
