"""Snapshot passes on the GPU (``CudaLeNetEngine.arm_eval(snapshot=True)``, csrc/eval_snapshot.cu): an exact copy of quiescent
weights, deterministic interleavings with an emulated peer on one stream, a concurrent paced writer, and interval mode end to
end on one replica."""
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_OF_N, INTERVAL = 0, 1


def _engine(B=256, seed=5, use_graph=True):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    return CudaLeNetEngine(B, be, seed=seed, use_graph=use_graph), be


def _valset(n, seed):
    from distributedmnist_b200.ops.selfcheck import mnist_like
    g = torch.Generator().manual_seed(seed)
    return mnist_like(g, n), torch.randint(0, 10, (n,), generator=g)


def _fields(rec):
    gs, _t0, _t1, n, correct, loss = rec
    return gs, n, correct, float(loss)


def _bits(t):
    return t.view(torch.int32)


def _f(g, n):
    """The emulated peer's push of step g: g + (i mod 1024) / 1024, exact in fp32."""
    i = torch.arange(n, device="cuda", dtype=torch.int64)
    return (torch.bitwise_and(i, 1023).to(torch.float32) / 1024.0) + float(g)


def _emulate(eng, g, mode, phases=7):
    from distributedmnist_b200.ops.lib import stream_ptr
    eng.lib.dm_snap_test_emulate(eng.backend.ctrl.local_ptr, eng.params, eng.params.numel(), g, mode, 1, phases, stream_ptr())


def _attempt(eng, a, part):
    """One part of snapshot attempt `a` of a 4-attempt pass, launched eagerly."""
    from distributedmnist_b200.ops.lib import stream_ptr
    lib, ctrl, st = eng.lib, eng.backend.ctrl.local_ptr, eng._snap_state
    if part == "select":
        lib.dm_snap_select(ctrl, st, a, int(eng._interval), eng.SNAP_WATCHDOG_MS, stream_ptr())
    elif part == "copy":
        lib.dm_snap_copy(st, eng.params, eng._snap, eng._snap16, eng.params.numel(), *eng._snap_bf_ranges, stream_ptr())
    else:
        lib.dm_snap_validate(ctrl, st, a, eng.SNAP_ATTEMPTS, stream_ptr())


def _armed(mode, use_graph=False, n=2500):
    eng, be = _engine(use_graph=use_graph)
    eng._interval = mode == INTERVAL           # which commit-word layout select reads (attach_optimizer sets it in training)
    eng.arm_eval(*_valset(n, 6), snapshot=True)
    return eng, be


def test_quiescent_snapshot_is_exact_and_scores_like_the_live_pass():
    from distributedmnist_b200.ops.lib import stream_ptr
    eng, _ = _engine(use_graph=True)
    x, y = _valset(2500, 6)
    eng.arm_eval(x, y, snapshot=True)
    eng.enqueue_eval()
    torch.cuda.synchronize()
    recs = eng.eval_records_with_status()
    assert len(recs) == 1 and recs[0][1] == 1                       # accepted on the first attempt
    snap, step = eng.eval_snapshot()
    assert step == 0 and torch.equal(_bits(snap), _bits(eng.params))
    ref16 = torch.empty_like(eng._snap16)
    eng.lib.dm_f32_to_bf16(snap, ref16, snap.numel(), stream_ptr())
    rg = eng._snap_bf_ranges
    for b, e in zip(rg[0::2], rg[1::2]):
        assert torch.equal(eng._snap16[b:e].view(torch.int16), ref16[b:e].view(torch.int16))
    snap_rec = recs[0][0]
    eng.arm_eval(x, y)                                               # the live pass over the same weights
    eng.enqueue_eval()
    torch.cuda.synchronize()
    live = eng.eval_records()
    assert len(live) == 1
    assert _fields(snap_rec) == _fields(live[0]) == _fields(eng.run_eval())


@pytest.mark.parametrize("mode", [K_OF_N, INTERVAL], ids=["k_of_n", "interval"])
def test_interleavings_on_one_stream(mode):
    eng, be = _armed(mode)
    n = eng.params.numel()
    p, pb = eng._ev_views
    _emulate(eng, 1, mode)
    # a commit (with its pushes and done) between copy and validate: that attempt is rejected, the next scores g + 1
    _attempt(eng, 0, "select")
    _attempt(eng, 0, "copy")
    _emulate(eng, 2, mode)
    _attempt(eng, 0, "validate")
    for part in ("select", "copy", "validate"):
        _attempt(eng, 1, part)
    for a in (2, 3):                                                 # attempts after an accepted one do nothing
        for part in ("select", "copy", "validate"):
            _attempt(eng, a, part)
    eng._launch_eval(publish=True, p=p, pb=pb)
    torch.cuda.synchronize()
    (rec, status), = eng.eval_records_with_status()
    assert status == 2 and rec[0] == 2
    snap, step = eng.eval_snapshot()
    assert step == 2 and torch.equal(_bits(snap), _bits(_f(2, n)))
    st = eng.eval_snapshot_stats()
    assert st["attempts"] == 2 and st["rejected"] == 1 and st["accepted_passes"] == 1

    # a commit whose writer never releases done: every attempt ends in the watchdog, the record is dropped, no hang
    _emulate(eng, 3, mode, phases=1 | 2)
    t0 = time.time()
    eng.enqueue_eval()
    torch.cuda.synchronize()
    assert time.time() - t0 < 5.0
    assert eng.eval_records() == [] and eng.eval_dropped == 1
    assert eng.eval_snapshot() is None
    st = eng.eval_snapshot_stats()
    assert st["timeouts"] == 4 and st["failed_passes"] == 1
    _emulate(eng, 3, mode, phases=4)                                 # ... once done arrives, step 3 is scored
    eng.enqueue_eval()
    torch.cuda.synchronize()
    (rec,) = eng.eval_records()
    snap, step = eng.eval_snapshot()
    assert rec[0] == step == 3 and torch.equal(_bits(snap), _bits(_f(3, n)))

    # more than a ring lap (64 commits) since the last pass: the newest step is found
    for g in range(4, 4 + 70):
        _emulate(eng, g, mode)
    eng.enqueue_eval()
    torch.cuda.synchronize()
    (rec,) = eng.eval_records()
    snap, step = eng.eval_snapshot()
    assert rec[0] == step == 73 and torch.equal(_bits(snap), _bits(_f(73, n)))
    be.check_error()


@pytest.mark.parametrize("mode", [K_OF_N, INTERVAL], ids=["k_of_n", "interval"])
def test_restore_with_an_empty_ring_scores_the_restored_step(mode):
    eng, be = _engine(use_graph=True)
    eng._interval = mode == INTERVAL
    be.set_global_step(57)
    eng.params.copy_(_f(57, eng.params.numel()) * 0.01)
    eng.params_updated()
    eng.arm_eval(*_valset(2500, 6), snapshot=True)
    eng.enqueue_eval()
    torch.cuda.synchronize()
    (rec, status), = eng.eval_records_with_status()
    snap, step = eng.eval_snapshot()
    assert status == 1 and rec[0] == step == 57 and torch.equal(_bits(snap), _bits(eng.params))


@pytest.mark.parametrize("mode", [K_OF_N, INTERVAL], ids=["k_of_n", "interval"])
def test_concurrent_paced_writer(mode):
    """One writer CTA on a second stream commits rounds into the arena while snapshot passes run on the training stream.
    Every accepted snapshot equals f(g, .) of the step it reports; acceptance and retry counts are printed."""
    from distributedmnist_b200.ops.lib import stream_ptr
    eng, be = _armed(mode, use_graph=True)
    n = eng.params.numel()
    _emulate(eng, 1, mode)
    torch.cuda.synchronize()
    g = 1
    side = torch.cuda.Stream()
    report, before = {}, {}
    for pace_us, rounds in ((0.0, 600), (400.0, 150)):
        flag = torch.zeros(4, dtype=torch.int32).pin_memory()
        eng.lib.dm_snap_test_writer(be.ctrl.local_ptr, eng.params, n, g, rounds, pace_us, mode, flag, stream_ptr(side))
        t0 = time.time()
        while int(flag[0]) == 0:                                     # the writer is resident before any snapshot launches
            assert time.time() - t0 < 30.0, "writer CTA never started"
            time.sleep(1e-4)
        passes = accepted = 0
        steps = []
        while int(flag[0]) != 2 and passes < 400:
            eng.enqueue_eval()
            torch.cuda.current_stream().synchronize()
            passes += 1
            for rec, status in eng.eval_records_with_status():
                if status > 0:
                    snap, step = eng.eval_snapshot()
                    assert rec[0] == step
                    assert torch.equal(_bits(snap), _bits(_f(step, n))), "snapshot of step %d is not f(%d, .)" % (step, step)
                    accepted += 1
                    steps.append(step)
        side.synchronize()
        assert steps == sorted(steps)
        g += rounds
        st = eng.eval_snapshot_stats()
        report["pace_%gus" % pace_us] = dict(passes=passes, accepted=accepted, **{k: v - before.get(k, 0) for k, v in st.items()})
        before = st
    print("\nconcurrent snapshot (%s): %s" % ("interval" if mode else "k_of_n", report))
    be.check_error()


def test_interval_end_to_end_on_one_replica(tmp_path):
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.checkpoint import Saver
    from distributedmnist_b200.flags import FLAGS
    train_dir, eval_dir = str(tmp_path / "train_dir"), str(tmp_path / "eval_dir")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="0")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    tr = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_distributed_train.py"), "--job_name=worker",
                         "--task_id=0", "--worker_hosts=localhost:1234", "--batch_size=128", "--max_steps=30",
                         "--interval_method=true", "--interval_ms=5", "--eval_every_steps=2", "--eval_snapshot=true",
                         "--initial_learning_rate=0.05", "--train_dir=" + train_dir, "--log_every=50"],
                        env=env, capture_output=True, text=True, timeout=600)
    log = tr.stdout + tr.stderr
    assert tr.returncode == 0, log[-3000:]
    assert sorted(f for f in os.listdir(train_dir) if f.endswith("_eval.npy")) == ["worker0_eval.npy"]
    rows = np.load(os.path.join(train_dir, "worker0_eval.npy"))
    assert len(rows) >= 2, rows
    assert (np.diff(rows[:, 0]) >= 0).all(), rows[:, 0]
    assert (rows[:, 3] == 10000).all()
    # the last row: the final pass, after the last step (no other writer at N = 1) -> the final weights
    FLAGS.reset()
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=FLAGS.synthetic_data, fake_data=FLAGS.fake_data)
    state, _ = Saver.restore(Saver.latest(train_dir))
    eng, _be = _engine(use_graph=False)
    eng.params.copy_(eng.spec.from_state_dict(state).to(eng.params.device))
    eng.params_updated()
    eng.arm_eval(ds.validation.images, ds.validation.labels)
    ref = eng.run_eval()
    assert int(rows[-1, 4]) == ref[4] and rows[-1, 5] == ref[5] / ref[3], (rows[-1], ref)
    ev = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_eval.py"), "--run_once=true",
                         "--checkpoint_dir=" + train_dir, "--eval_dir=" + eval_dir], env=env, capture_output=True,
                        text=True, timeout=600)
    out = ev.stdout + ev.stderr
    assert ev.returncode == 0, out[-3000:]
    m = re.search(r"Num examples: 10000  Precision @ 1: ([0-9.]+) Loss: ([0-9.]+) Time", out)
    assert m, out[-2000:]
    assert int(rows[-1, 4]) == round(float(m.group(1)) * 10000)
    assert abs(rows[-1, 5] - float(m.group(2))) <= 2.0 ** -10 * float(m.group(2)) + 1e-6


def test_keep_holds_the_last_accepted_snapshot_across_a_failed_pass(monkeypatch):
    eng, _ = _engine(use_graph=True)
    monkeypatch.setattr(eng, "SNAP_KEEP", True)
    eng.arm_eval(*_valset(2500, 6), snapshot=True)
    n = eng.params.numel()
    assert eng.eval_snapshot() is None                               # nothing accepted yet
    _emulate(eng, 1, K_OF_N)
    eng.enqueue_eval()
    _emulate(eng, 2, K_OF_N, phases=1 | 2)                           # committed and pushed, done never released
    eng.enqueue_eval()
    torch.cuda.synchronize()
    assert [st for _r, st in eng.eval_records_with_status()] == [1, -1]
    snap, step = eng.eval_snapshot()
    assert step == 1 and torch.equal(_bits(snap), _bits(_f(1, n)))


def _two_gpu_runs(tmp_path, name, extra, max_steps, n=2):
    """Chief pass on and off for one configuration on n replicas (tests/_snapshot_eval_worker.py)."""
    import json

    from distributedmnist_b200.parallel.launcher import run_replicas
    worker = os.path.join(ROOT, "tests", "_snapshot_eval_worker.py")
    out = {}
    for tag, ev in (("on", ["--eval_every_steps=20", "--eval_snapshot=true"]), ("off", [])):
        d = tmp_path / ("%s_%s" % (name, tag))
        codes = run_replicas([worker, str(d / "rank_RANK"), "--train_dir=%s" % (d / "train_dir"), "--batch_size=128",
                              "--max_steps=%d" % max_steps, "--initial_learning_rate=0.05", "--save_interval_secs=1000",
                              "--log_every=50"] + extra + ev, n, timeout=600, out_dir=str(d / "out"))
        logs = "\n".join(open(os.path.join(d, "out", f)).read()[-1500:] for f in sorted(os.listdir(d / "out")))
        assert codes == [0] * n, (name, tag, logs)
        ranks = []
        for r in range(n):
            with open(str(d / ("rank_%d.json" % r))) as f:
                ranks.append((np.load(str(d / ("rank_%d.npy" % r))), json.load(f)))
        out[tag] = (ranks, sorted(f for f in os.listdir(d / "train_dir") if f.endswith("_eval.npy")), d / "train_dir")
    return out


def _check_two_gpu_runs(name, out):
    for tag, (ranks, eval_files, _d) in out.items():
        for r in range(1, len(ranks)):
            assert np.array_equal(ranks[0][0].view(np.uint32), ranks[r][0].view(np.uint32)), "%s/%s: replicas differ" % (name, tag)
        assert all(m["evals"] == [] for _p, m in ranks[1:])           # only the chief evaluates
        assert eval_files == (["worker0_eval.npy"] if tag == "on" else []), (name, tag, eval_files)
    ranks, _files, train_dir = out["on"]
    rows = np.load(str(train_dir / "worker0_eval.npy"))
    assert len(rows) >= 1 and (np.diff(rows[:, 0]) >= 0).all() and (rows[:, 3] == 10000).all(), rows
    chief = ranks[0][1]
    # the newest row comes from the newest accepted pass, whose snapshot the chief kept
    assert chief["kept_step"] == int(rows[-1, 0]), (chief["kept_step"], rows[-1])
    gs, _t0, _t1, n_ex, correct, loss_sum = chief["standalone"]
    assert n_ex == 10000 and int(rows[-1, 4]) == correct and rows[-1, 5] == loss_sum / n_ex, (rows[-1], chief["standalone"])
    print("\n%s: chief dropped steps with eval on %d, off %d; snapshot passes dropped %d; %s"
          % (name, chief["dropped_steps"], out["off"][0][0][1]["dropped_steps"], chief["eval_dropped"],
             chief["snapshot_stats"]))


@pytest.mark.multigpu
def test_two_replicas_k1_of_2_with_straggler(tmp_path):
    """K = 1 of 2, rank 1 delayed 1 ms per step on the device: the chief scores snapshots while the real K-of-N kernels
    push into its arena."""
    name = "k1_of_2_straggler"
    _check_two_gpu_runs(name, _two_gpu_runs(tmp_path, name, ["--num_replicas_to_aggregate=1",
                                                              "--inject_straggler=1:1.0:1000"], 200))


@pytest.mark.multigpu
def test_two_replicas_interval(tmp_path):
    """Interval mode at N = 2: either replica commits a tick and pushes into the chief's arena at any time."""
    name = "interval_n2"
    _check_two_gpu_runs(name, _two_gpu_runs(tmp_path, name, ["--interval_method=true", "--interval_ms=5"], 60))
