"""``--eval_snapshot`` on the CPU: the snapshot protocol's element-level model (both writer orders, and the hazards its two
checks exist for), the flag combinations, the pass trigger of the snapshot modes and the multi-run accuracy plot."""
import os
import random
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.protocol import ProtocolHazard, SnapshotModel, explore_schedules
from distributedmnist_b200.train import check_eval_flags, eval_due

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the snapshot protocol (csrc/eval_snapshot.cu) -------------------------------------------------------------------
@pytest.mark.parametrize("interval", [False, True], ids=["global_step_before_pushes", "global_step_after_pushes"])
@pytest.mark.parametrize("numel", [2, 3])
def test_every_schedule_accepts_only_one_step(interval, numel):
    """n = 2 writers, k = 1, 2 steps: under EVERY interleaving an accepted snapshot holds one version, the one it reports."""
    def make():
        m = SnapshotModel(n=2, steps=2, numel=numel, interval=interval)
        make.models.append(m)
        return m
    make.models = []
    runs = explore_schedules(make, max_runs=400000)
    assert runs > 1000
    steps = {tuple(m.accepted) for m in make.models}
    assert {(0,), (1,), (2,)} <= steps           # the initial weights and both committed steps are each scored somewhere


@pytest.mark.parametrize("interval", [False, True])
def test_random_schedules_with_retries(interval):
    """3 steps, 3 elements, 4 attempts: sampled schedules; accepted snapshots are consistent, and retries accept more."""
    rng = random.Random(7)
    accepted = 0
    for _ in range(3000):
        m = SnapshotModel(n=2, steps=3, numel=3, interval=interval, attempts=4)
        m.run(lambda runnable: rng.choice(runnable))
        accepted += len(m.accepted)
    assert accepted > 2000


@pytest.mark.parametrize("interval", [False, True])
def test_ring_laps_fail_the_attempt_and_stay_consistent(interval):
    """A ring of 2 slots with 4 steps: a reader can find its candidate's slot reused; such attempts fail, others stay exact."""
    rng = random.Random(11)
    for _ in range(3000):
        m = SnapshotModel(n=2, steps=4, numel=2, interval=interval, ring=2, attempts=3)
        m.run(lambda runnable: rng.choice(runnable))


@pytest.mark.parametrize("interval", [False, True])
@pytest.mark.parametrize("removed", ["validate", "wait_done"])
def test_model_detects_the_hazards_without_its_checks(interval, removed):
    with pytest.raises(ProtocolHazard, match="holds element"):
        explore_schedules(lambda: SnapshotModel(n=2, steps=2, numel=2, interval=interval, **{removed: False}))


# ---- flags -------------------------------------------------------------------------------------------------------------
def _flags(**kw):
    base = dict(eval_every_steps=10, backend="auto", model="lenet", interval_method=False, worker_times_cdf_method=False,
                eval_snapshot=True)
    base.update(kw)
    return SimpleNamespace(**base)


GPU = SimpleNamespace(on_gpu=True, world_size=8)


@pytest.mark.parametrize("k", range(1, 9))
def test_snapshot_flag_accepts_every_k_and_interval_for_lenet(k):
    check_eval_flags(_flags(), GPU, k, dataset_test=object())                 # one flag set for a whole K sweep
    check_eval_flags(_flags(interval_method=True), GPU, k, dataset_test=object())
    check_eval_flags(_flags(worker_times_cdf_method=True), GPU, k, dataset_test=object())


@pytest.mark.parametrize("model", ["mlp2", "mlp3"])
def test_snapshot_flag_keeps_refusing_mlp(model):
    for interval in (False, True):
        with pytest.raises(ValueError, match="implemented for lenet"):
            check_eval_flags(_flags(model=model, interval_method=interval), GPU, 1, dataset_test=object())


def test_without_snapshot_flag_the_refusals_point_to_it():
    for kw, k, msg in [(dict(interval_method=True), 8, "interval commits push weights"), (dict(), 7, "K < N")]:
        with pytest.raises(ValueError, match=msg) as e:
            check_eval_flags(_flags(eval_snapshot=False, **kw), GPU, k, dataset_test=object())
        assert "--eval_snapshot=true" in str(e.value)
    with pytest.raises(ValueError, match="needs the validation set"):
        check_eval_flags(_flags(), GPU, 1, dataset_test=None)


def test_flag_is_registered_and_off_by_default():
    FLAGS.reset()
    try:
        assert FLAGS.eval_snapshot is False
        FLAGS.parse(["--eval_snapshot=true"])
        assert FLAGS.eval_snapshot is True
    finally:
        FLAGS.reset()


# ---- trigger -----------------------------------------------------------------------------------------------------------
def _triggers(steps, every, restored=0):
    mark, out = restored, []
    for s in steps:
        if eval_due(s, mark, every):
            mark = s
            out.append(s)
    return out


def test_trigger_follows_crossed_multiples_when_steps_jump():
    assert _triggers(range(1, 31), 10) == [10, 20, 30]
    # K < N: a late chief fast-forwards, consumed steps jump by more than E -- one pass per crossing, not per multiple
    assert _triggers([3, 9, 14, 15, 37, 38, 40, 41, 59, 61], 10) == [14, 37, 40, 59, 61]
    # interval mode: the same step is consumed several times in a row
    assert _triggers([0, 0, 5, 5, 10, 10, 10, 11, 20], 5) == [5, 10, 20]
    assert _triggers([101, 105, 112], 10, restored=100) == [112]          # counted from the restored step
    assert not eval_due(7, 0, 0)


# ---- plot --------------------------------------------------------------------------------------------------------------
def test_plot_draws_one_curve_per_configuration(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import benchmark as bm
    dirs = []
    for k in (1, 4, 8):
        d = tmp_path / ("k%d" % k)
        d.mkdir()
        rows = np.array([(10 * k, 1000.0, 0.002, 10000, 8000 + k, 0.4), (20 * k, 1000.3, 0.002, 10000, 9000 + k, 0.3),
                         (30 * k, 1000.9, 0.002, 10000, 9500 + k, 0.2)])
        np.save(str(d / "worker0_eval.npy"), rows)
        dirs.append(str(d))
    out = bm.plot_device_time_precision(dirs, str(tmp_path), labels=["K=1", "K=4", "K=8"])
    assert out.endswith("device_time_precision.png") and os.path.getsize(out) > 0
    with open(out, "rb") as f:
        assert f.read(8) == b"\x89PNG\r\n\x1a\n"
    with pytest.raises(ValueError, match="labels"):
        bm.plot_device_time_precision(dirs, str(tmp_path), labels=["K=1"])
    assert bm.plot_device_time_precision(dirs[0], str(tmp_path)) == out         # the one-directory call
