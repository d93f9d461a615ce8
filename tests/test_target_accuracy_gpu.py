"""``--target_accuracy`` on the GPU: lenet runs through ``train()`` that stop at S = g + STOP_MARGIN and end exactly as a run
with ``--max_steps=S`` (pipelined and non-pipelined loop), the device threshold at ``need - 1`` / ``need``, snapshot passes
(a dropped pass never stops the run; K > N and interval end at min(max_steps, S)), the synchronise count per step, and the
multi-replica runs."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_OF_N, INTERVAL = 0, 1
VAL = 1000


@pytest.fixture
def flags(monkeypatch):
    from distributedmnist_b200.flags import FLAGS
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    FLAGS.reset()
    yield FLAGS
    FLAGS.reset()


def _train(d, *extra, steps=300):
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import train
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % d, "--batch_size=128", "--max_steps=%d" % steps, "--eval_every_steps=10",
                 "--initial_learning_rate=0.05", "--log_every=1000", "--save_results_period=1000000",
                 "--save_interval_secs=1000"] + list(extra))
    ctx = init_context(FLAGS)
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True, synthetic_sizes=(8192, VAL))
    return train(ctx, ds.train, ds.validation, FLAGS)


def _rows(d):
    return np.load(os.path.join(str(d), "worker0_eval.npy"))


def _ckpt(d, step):
    with open(os.path.join(str(d), "model.ckpt-%d.data-00000-of-00001" % step), "rb") as f:
        return f.read()


def _reachable(rows, upto):
    """(g, correct): the first row with the best count among the rows of steps <= upto; every earlier row is below it."""
    early = rows[rows[:, 0] <= upto]
    best = int(early[:, 4].max())
    g = int(early[early[:, 4] == best][0, 0])
    return g, best


@pytest.mark.parametrize("pipelined", [True, False], ids=["pipelined", "non_pipelined"])
def test_lenet_stops_at_g_plus_margin_like_max_steps(tmp_path, flags, pipelined):
    from distributedmnist_b200.train import STOP_MARGIN
    # --device_data: the index feed draws batches on the training thread, so every run trains on the same batch sequence
    loop = ["--pipeline_steps=%s" % ("true" if pipelined else "false"), "--device_data=true"]
    _train(tmp_path / "ref", *loop)
    g, best = _reachable(_rows(tmp_path / "ref"), 250)
    s = g + STOP_MARGIN
    res = _train(tmp_path / "armed", *loop, "--target_accuracy=%r" % (best / VAL))
    cut = _train(tmp_path / "cut", *loop, steps=s)
    assert res["time_to_accuracy"]["global_step"] == g, res["time_to_accuracy"]
    assert res["final_step"] == cut["final_step"] == s + 1
    assert _ckpt(tmp_path / "armed", s + 1) == _ckpt(tmp_path / "cut", s + 1)
    a, c = _rows(tmp_path / "armed"), _rows(tmp_path / "cut")
    np.testing.assert_array_equal(a[:, [0, 3, 4, 5]], c[:, [0, 3, 4, 5]])
    assert (a[a[:, 0] < g, 4] < best).all() and int(a[a[:, 0] == g, 4][0]) == best
    rep = res["time_to_accuracy"]
    with open(str(tmp_path / "armed" / "worker0_time_to_accuracy.json")) as f:
        assert json.load(f) == rep
    assert rep["reached"] and rep["global_step"] == g and rep["correct"] == best and rep["need"] == best
    assert rep["clock"] == "device %globaltimer" and 0 < rep["train_time_s"] < rep["wall_time_s"]
    print("\n%s: g=%d S=%d correct=%d train_time=%.4f s wall=%.4f s" % ("pipelined" if pipelined else "non-pipelined", g, s,
                                                                        best, rep["train_time_s"], rep["wall_time_s"]))


def _engine(B=256, seed=5):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaLeNetEngine(B, be, seed=seed, use_graph=True)
    eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 4, 0.7), 1, 1))
    return eng, be


def _valset(n, seed):
    from distributedmnist_b200.ops.selfcheck import mnist_like
    g = torch.Generator().manual_seed(seed)
    return mnist_like(g, n), torch.randint(0, 10, (n,), generator=g)


def _stop_word(eng):
    torch.cuda.synchronize()
    return int(eng._stop.view(torch.int32, 0, 1).cpu()[0])


def test_device_threshold_is_need_not_need_minus_one():
    eng, _be = _engine()
    eng.arm_eval(*_valset(2500, 6))
    correct = int(eng.run_eval()[4])
    assert 0 < correct < 2500
    eng.arm_stop()
    eng.arm_target(correct + 1, 2)                       # one row short: no stop
    eng.enqueue_eval()
    assert _stop_word(eng) == 0
    eng.arm_target(correct, 2)                           # exactly need: S = epoch (0) + 2
    eng.enqueue_eval()
    assert _stop_word(eng) == 2
    eng.arm_target(1, 5)                                 # a stop is set once
    eng.enqueue_eval()
    assert _stop_word(eng) == 2
    # every step's last kernel copies the stop word to the host
    g = torch.Generator().manual_seed(3)
    buf = eng.pack_batch(torch.rand(256, 784, generator=g) - 0.5, torch.randint(0, 10, (256,), generator=g))
    ev, _l, _s = eng.step_packed(buf)
    ev.synchronize()
    assert eng.stop_step() == 2


def _emulate(eng, g, mode, phases=7):
    from distributedmnist_b200.ops.lib import stream_ptr
    eng.lib.dm_snap_test_emulate(eng.backend.ctrl.local_ptr, eng.params, eng.params.numel(), g, mode, 1, phases, stream_ptr())


@pytest.mark.parametrize("mode", [K_OF_N, INTERVAL], ids=["k_of_n", "interval"])
def test_dropped_snapshot_pass_never_stops_and_the_snapshot_step_does(mode):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaLeNetEngine(256, be, seed=5, use_graph=True)
    eng._interval = mode == INTERVAL
    eng.arm_eval(*_valset(2500, 6), snapshot=True)
    eng.arm_stop()
    eng.arm_target(1, 2)
    _emulate(eng, 1, mode, phases=1 | 2)                 # committed and pushed, done never released: every attempt fails
    eng.enqueue_eval()
    torch.cuda.synchronize()
    assert [st for _r, st in eng.eval_records_with_status()] == [-1]
    assert _stop_word(eng) == 0
    _emulate(eng, 1, mode, phases=4)                     # done arrives: the next pass scores the snapshot of step 1
    eng.enqueue_eval()
    torch.cuda.synchronize()
    (rec, status), = eng.eval_records_with_status()
    assert status > 0 and rec[0] == 1 and rec[4] >= 1
    assert _stop_word(eng) == 1 + 2                      # the snapshot's step, not the chief's epoch (0)


@pytest.mark.parametrize("extra", [["--num_replicas_to_aggregate=4"], ["--interval_method=true", "--interval_ms=2"]],
                         ids=["k4_of_1", "interval"])
def test_snapshot_runs_end_at_min_max_steps_and_s(tmp_path, flags, extra):
    from distributedmnist_b200.train import STOP_MARGIN
    args = ["--eval_snapshot=true", "--pipeline_steps=true"] + extra
    _train(tmp_path / "ref", *args, steps=200)
    rows = _rows(tmp_path / "ref")
    _g, best = _reachable(rows, 120)
    need = max(1, best - 30)                             # timing decides which steps a snapshot pass scores: leave room
    res = _train(tmp_path / "armed", *args, "--target_accuracy=%r" % (need / VAL), steps=200)
    rep = res["time_to_accuracy"]
    assert rep["reached"], (rep, _rows(tmp_path / "armed"))
    a = _rows(tmp_path / "armed")
    first = int(np.argmax(a[:, 4] >= need))
    assert (a[:first, 4] < need).all() and int(a[first, 0]) == rep["global_step"]
    s = min(200, rep["global_step"] + STOP_MARGIN)
    assert max(res["steps"]) <= s < res["final_step"], (res["steps"][-5:], res["final_step"], s)
    print("\n%s: reached at snapshot step %d, S = %d, final step %d" % (extra[0], rep["global_step"], s, res["final_step"]))


def test_armed_run_adds_no_synchronisation_per_step(tmp_path, flags, monkeypatch):
    """An armed run whose target is never reached makes as many synchronise calls per step as an unarmed one: the
    difference between a 100-step and a 200-step run is the same with and without the target."""
    from distributedmnist_b200.train import _AsyncCheckpointer
    calls = {"sync": 0, "at_final_save": None}

    def counted(fn):
        def wrapper(*a, **k):
            calls["sync"] += 1
            return fn(*a, **k)
        return wrapper
    monkeypatch.setattr(torch.cuda, "synchronize", counted(torch.cuda.synchronize))
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", counted(torch.cuda.Stream.synchronize))
    monkeypatch.setattr(torch.cuda.Event, "synchronize", counted(torch.cuda.Event.synchronize))
    real_save = _AsyncCheckpointer.save

    def save(self, *a, **k):
        calls["at_final_save"] = calls["sync"]
        return real_save(self, *a, **k)
    monkeypatch.setattr(_AsyncCheckpointer, "save", save)
    counts = {}
    for tag, extra in (("armed", ["--target_accuracy=1.0"]), ("off", [])):
        for steps in (100, 200):
            calls.update(sync=0, at_final_save=None)
            res = _train(tmp_path / ("%s_%d" % (tag, steps)), *extra, steps=steps)
            assert res["final_step"] == steps + 1
            counts[(tag, steps)] = calls["at_final_save"]
    per_armed = counts[("armed", 200)] - counts[("armed", 100)]
    per_off = counts[("off", 200)] - counts[("off", 100)]
    assert per_armed == per_off, counts


def _replica_runs(tmp_path, name, extra, steps, n=2):
    from distributedmnist_b200.parallel.launcher import run_replicas
    worker = os.path.join(ROOT, "tests", "_snapshot_eval_worker.py")
    d = tmp_path / name
    codes = run_replicas([worker, str(d / "rank_RANK"), "--train_dir=%s" % (d / "train_dir"), "--batch_size=128",
                          "--max_steps=%d" % steps, "--initial_learning_rate=0.05", "--save_interval_secs=1000",
                          "--log_every=50", "--eval_every_steps=10"] + extra, n, timeout=600, out_dir=str(d / "out"))
    logs = "\n".join(open(os.path.join(d, "out", f)).read()[-1500:] for f in sorted(os.listdir(d / "out")))
    assert codes == [0] * n, (name, logs)
    ranks = []
    for r in range(n):
        with open(str(d / ("rank_%d.json" % r))) as f:
            ranks.append((np.load(str(d / ("rank_%d.npy" % r))), json.load(f)))
    return ranks, d / "train_dir"


@pytest.mark.multigpu
def test_two_replicas_k_equals_n_stop_at_the_same_step(tmp_path):
    from distributedmnist_b200.train import STOP_MARGIN
    _ranks, ref_dir = _replica_runs(tmp_path, "ref", [], 300)
    g, best = _reachable(_rows(ref_dir), 250)
    ranks, train_dir = _replica_runs(tmp_path, "armed", ["--target_accuracy=%r" % (best / 10000)], 300)
    with open(str(train_dir / "worker0_time_to_accuracy.json")) as f:
        rep = json.load(f)
    assert rep["global_step"] == g
    assert [m["final_step"] for _p, m in ranks] == [g + STOP_MARGIN + 1] * 2
    assert np.array_equal(ranks[0][0].view(np.uint32), ranks[1][0].view(np.uint32))


@pytest.mark.multigpu
def test_two_replicas_k1_of_2_with_straggler_end_cleanly(tmp_path):
    ranks, train_dir = _replica_runs(tmp_path, "k1", ["--num_replicas_to_aggregate=1", "--inject_straggler=1:1.0:1000",
                                                      "--eval_snapshot=true", "--target_accuracy=0.2"], 300)
    with open(str(train_dir / "worker0_time_to_accuracy.json")) as f:
        rep = json.load(f)
    if rep["reached"]:
        s = rep["global_step"] + 2
        assert all(m["final_step"] > min(300, s) for _p, m in ranks)
