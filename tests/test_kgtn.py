"""K > N gradients per update (mode A, "replicas compute multiple batches per update"), on the CPU: the count-triggered
protocol model explored schedule by schedule, the host optimizer on the local and gloo backends, the training driver and
the evaluation flags."""
import json
import os
from types import SimpleNamespace

import pytest
import torch

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
from distributedmnist_b200.parallel.backends import LocalBackend
from distributedmnist_b200.parallel.context import ReplicaContext, init_context
from distributedmnist_b200.parallel.launcher import run_replicas
from distributedmnist_b200.parallel.protocol import CountTriggerModel, ProtocolHazard, explore_schedules
from distributedmnist_b200.schedule import LearningRateSchedule
from distributedmnist_b200.train import check_eval_flags, train

HERE = os.path.dirname(os.path.abspath(__file__))


# ---- protocol model ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("iters", [(3, 3), (4, 3), (3, 4)])
def test_count_trigger_every_schedule_is_sound(iters):
    """2 replicas, K = 3: every interleaving commits >= K gradients of the committed step, never reads an accumulator
    mid-add, ends with replicas equal to the serial replay, and leaves no step with K gradients uncommitted."""
    totals = set()

    def make():
        m = CountTriggerModel(2, 3, iters)
        made.append(m)
        return m
    made = []
    runs = explore_schedules(make, max_runs=100000)
    assert runs > 1000
    for m in made:
        totals.update(c[4] for c in m.commits)
        assert len(m.commits) >= sum(iters) // 4          # at most 3 of the other replica's gradients can be lost per step
    assert min(totals) == 3 and max(totals) == 4          # 4: a close raced the K-th one and was still counted


@pytest.mark.parametrize("removed, msg", [("fence", "without a commit"), ("busy_wait", "while it was adding")])
def test_count_trigger_model_fails_without_the_fence_or_the_busy_wait(removed, msg):
    with pytest.raises(ProtocolHazard, match=msg):
        explore_schedules(lambda: CountTriggerModel(2, 3, 3, **{removed: False}))


def test_count_trigger_single_replica_commits_every_k():
    m = CountTriggerModel(1, 4, 8)
    assert explore_schedules(lambda: m) == 1
    assert [c[4] for c in m.commits] == [4, 4] and m.accepted == [8] and m.dropped == [0]


# ---- host optimizer ---------------------------------------------------------------------------------------------------
def test_local_backend_update_is_the_mean_of_k_batch_gradients():
    be = LocalBackend(ReplicaContext(0, 1, 0, torch.device("cpu"), "none"))
    opt = SyncReplicasOptimizer(be, LearningRateSchedule(0.1, 1000, 1.0), 4, 1)
    gen = torch.Generator().manual_seed(3)
    w = torch.randn(100, generator=gen, dtype=torch.float64)
    params = w.clone()
    for step in range(3):
        gs = [torch.randn(100, generator=gen, dtype=torch.float64) for _ in range(4)]
        for i, g in enumerate(gs):
            info = opt.apply_gradients(params, g.clone())
            assert info.applied == (i == 3)
        w = w - 0.1 * torch.stack(gs).sum(0) / 4
        assert torch.allclose(params, w, rtol=0, atol=1e-12)
        assert info.global_step == step + 1 and info.count == 4
    assert opt.accepted_steps == 12 and opt.dropped_steps == 0 and opt.global_step == 3


def test_optimizer_refuses_k_below_one():
    be = LocalBackend(ReplicaContext(0, 1, 0, torch.device("cpu"), "none"))
    with pytest.raises(ValueError, match=">= 1"):
        SyncReplicasOptimizer(be, LearningRateSchedule(0.1, 1000, 1.0), 0, 1)


def test_gloo_two_replicas_k3(tmp_path):
    out = str(tmp_path / "out")
    argv = [os.path.join(HERE, "_kgtn_gloo_worker.py"), str(tmp_path / "res_RANK.json"), "--model=mlp2", "--mlp_hidden=32",
            "--batch_size=16", "--backend=gloo", "--initial_learning_rate=0.05", "--save_interval_secs=1000",
            "--train_dir=%s" % (tmp_path / "train"), "--max_steps=20", "--num_replicas_to_aggregate=3"]
    codes = run_replicas(argv, 2, timeout=180, out_dir=out)
    logs = [open(os.path.join(out, f)).read() for f in sorted(os.listdir(out))]
    assert codes == [0, 0], "\n".join(l[-2000:] for l in logs)
    a, b = [json.load(open(tmp_path / ("res_%d.json" % r))) for r in range(2)]
    assert [c[3] for c in a["commits"]] == [c[3] for c in b["commits"]]     # bit-identical after every update
    assert a["final_fp"] == b["final_fp"] and a["final_step"] == b["final_step"] == 21
    assert [c[0] for c in a["commits"]] == list(range(1, 22))
    for ca, cb in zip(a["commits"], b["commits"]):
        assert ca[1] == cb[1] >= 3 and ca[2] + cb[2] == ca[1] and ca[2] >= 1 and cb[2] >= 1
    assert a["accepted"] + b["accepted"] == sum(c[1] for c in a["commits"])
    assert a["accepted"] == a["calls"] and a["dropped"] == b["dropped"] == 0
    assert sum(a["losses"][-10:]) < sum(a["losses"][:10])


# ---- training driver and flags ------------------------------------------------------------------------------------------
@pytest.fixture
def clean_flags():
    FLAGS.reset()
    saved = {k: os.environ.pop(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") if k in os.environ}
    yield FLAGS
    FLAGS.reset()
    os.environ.update(saved)


def test_train_one_replica_k4(tmp_path, clean_flags):
    FLAGS.parse(["--train_dir=%s" % (tmp_path / "train"), "--batch_size=32", "--max_steps=10", "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000", "--initial_learning_rate=0.05",
                 "--num_replicas_to_aggregate=4"])
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    res = train(ctx, ds.train, ds.validation, FLAGS)
    assert res["final_step"] == 11 and res["accepted"] == 44 and res["dropped"] == 0
    assert len(res["steps"]) == 43                      # 4 local iterations per global step; the 44th ends the loop
    assert res["steps"][:5] == [0, 0, 0, 1, 1]
    assert res["optimizer"].lr_schedule.decay_steps == \
        LearningRateSchedule.from_flags(FLAGS, ds.train.num_examples, 4).decay_steps


def test_restarted_k4_run_draws_past_the_iterations_it_restored(tmp_path, clean_flags, caplog, monkeypatch):
    """Random affine augmentation with K = 4 on one replica: a run restored at global step g used the draws of iterations
    0 .. 4g - 1 (4 per step), so the restarted run draws from 4g on and no iteration's draws are used twice."""
    from distributedmnist_b200.engine import TorchEngine
    seen = []
    fb = TorchEngine.forward_backward

    def record_step(self, step):
        fb(self, step)
        seen[-1].append(self.augment_iteration() - 1)          # the iteration whose draws this step used

    monkeypatch.setattr(TorchEngine, "forward_backward", record_step)
    finals = []
    for steps in (12, 20):
        seen.append([])
        caplog.clear()
        FLAGS.reset()
        FLAGS.parse(["--train_dir=%s" % (tmp_path / "train"), "--batch_size=32", "--max_steps=%d" % steps, "--model=mlp2",
                     "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000",
                     "--initial_learning_rate=0.05", "--num_replicas_to_aggregate=4", "--augment_max_shift=2",
                     "--augment_max_rotation=15", "--augment_max_scale=0.1"])
        ctx = init_context(FLAGS, want_gpu=False)
        ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                                   synthetic_sizes=(256, 64))
        res = train(ctx, ds.train, ds.validation, FLAGS)
        finals.append(res["final_step"])
        assert res["accepted"] == len(seen[-1])
        start = 4 * finals[0] if steps == 20 else 0
        assert any("draws from iteration %d;" % start in r.getMessage() for r in caplog.records), \
            [r.getMessage() for r in caplog.records if "draws from" in r.getMessage()]
    first, second = seen
    assert finals == [13, 21] and first == list(range(52)) and second == list(range(52, 84))
    assert not set(first) & set(second)


GPU = SimpleNamespace(on_gpu=True, world_size=2)


def _flags(**kw):
    base = dict(eval_every_steps=10, backend="auto", model="lenet", interval_method=False, worker_times_cdf_method=False,
                eval_snapshot=False)
    base.update(kw)
    return SimpleNamespace(**base)


@pytest.mark.parametrize("k", [3, 16, 50])
def test_live_eval_pass_is_refused_for_k_above_n_and_the_snapshot_is_accepted(k):
    with pytest.raises(ValueError, match="K > N") as e:
        check_eval_flags(_flags(), GPU, k, dataset_test=object())
    assert "--eval_snapshot=true" in str(e.value)
    check_eval_flags(_flags(eval_snapshot=True), GPU, k, dataset_test=object())
