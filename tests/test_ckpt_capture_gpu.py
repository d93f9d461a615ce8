"""Checkpoint captures on the GPU (``_CudaEngine.arm_checkpoint`` / ``enqueue_checkpoint``): the live capture after every
launched step against a second engine, validated snapshots next to an emulated peer (csrc/eval_snapshot.cu's test writer),
a capture right after a restore, ``train()`` end to end with a checkpoint every step, and no host synchronisation per
checkpoint."""
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


def _engine(model="lenet", B=256, seed=5, optimizer=True):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine, CudaMlpEngine
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaLeNetEngine(B, be, seed=seed, use_graph=True) if model == "lenet" else \
        CudaMlpEngine(model, B, be, seed=seed, use_graph=True)
    if optimizer:
        eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 4, 0.7), 1, 1))
    return eng, be


def _packed(eng, n, seed):
    g = torch.Generator().manual_seed(seed)
    B = eng.batch_size
    return [eng.pack_batch(torch.rand(B, 784, generator=g) - 0.5, torch.randint(0, 10, (B,), generator=g)) for _ in range(n)]


def _bits(t):
    return t.view(torch.int32)


def _f(g, n):
    """The emulated peer's push of step g: g + (i mod 1024) / 1024, exact in fp32 (host tensor)."""
    return (torch.bitwise_and(torch.arange(n, dtype=torch.int64), 1023).to(torch.float32) / 1024.0) + float(g)


def _emulate(eng, g, mode, phases=7):
    from distributedmnist_b200.ops.lib import stream_ptr
    eng.lib.dm_snap_test_emulate(eng.backend.ctrl.local_ptr, eng.params, eng.params.numel(), g, mode, 1, phases, stream_ptr())


def test_lenet_live_capture_after_every_step_is_bit_exact():
    """K = N: a capture after every launched step, each waited for only after the next step has been launched, equals the
    arena a second engine with the same seed and batches holds after the same number of steps."""
    steps = 12
    ref, _ = _engine()
    expect = []
    for buf in _packed(ref, steps, 7):
        ev, _l, _s = ref.step_packed(buf)
        ev.synchronize()
        torch.cuda.synchronize()
        expect.append(ref.params.cpu())
    ref._leave_native_runner()
    del ref

    eng, be = _engine()
    eng.arm_checkpoint(snapshot=False)
    bufs = _packed(eng, steps, 7)
    got = []
    for i in range(steps):
        eng.step_packed(bufs[i])
        if i > 0:
            seq, b, step = eng.checkpoint_wait()              # the capture after step i - 1, step i still in flight
            got.append((step, eng.ckpt_host[b].clone()))
        eng.enqueue_checkpoint(i & 1)
    seq, b, step = eng.checkpoint_wait()
    got.append((step, eng.ckpt_host[b].clone()))
    torch.cuda.synchronize()
    be.check_error()
    eng._leave_native_runner()
    assert seq == steps
    for i, (step, arena) in enumerate(got):
        assert step == i + 1, (i, step)                        # restored (0) + launched
        assert torch.equal(_bits(arena), _bits(expect[i])), "capture after step %d differs from the reference" % (i + 1)


def test_mlp2_live_capture_equals_the_arena_after_a_synchronise():
    eng, be = _engine("mlp2")
    eng.arm_checkpoint(snapshot=False)
    for i, buf in enumerate(_packed(eng, 8, 9)):
        eng.step_packed(buf)
        eng.enqueue_checkpoint(i & 1)
        seq, b, step = eng.checkpoint_wait()
        torch.cuda.synchronize()
        assert seq == i + 1 and step == i + 1
        assert torch.equal(_bits(eng.ckpt_host[b]), _bits(eng.params.cpu()))
    be.check_error()
    eng._leave_native_runner()


@pytest.mark.parametrize("mode", [K_OF_N, INTERVAL], ids=["k_of_n", "interval"])
def test_snapshot_capture_next_to_a_concurrent_paced_writer(mode):
    """One writer CTA on a second stream commits rounds into the arena while captures run on the current stream.  Every
    accepted capture equals f(g, .) of the step its record names, accepted steps never decrease; counts are printed."""
    from distributedmnist_b200.ops.lib import stream_ptr
    eng, be = _engine(optimizer=False)
    eng._interval = mode == INTERVAL              # which commit-word layout select reads (attach_optimizer sets it in training)
    eng.arm_checkpoint(snapshot=True)
    n = eng.params.numel()
    _emulate(eng, 1, mode)
    torch.cuda.synchronize()
    g = 1
    side = torch.cuda.Stream()
    report = {}
    for pace_us, rounds in ((0.0, 600), (400.0, 150)):
        flag = torch.zeros(4, dtype=torch.int32).pin_memory()
        eng.lib.dm_snap_test_writer(be.ctrl.local_ptr, eng.params, n, g, rounds, pace_us, mode, flag, stream_ptr(side))
        t0 = time.time()
        while int(flag[0]) == 0:
            assert time.time() - t0 < 30.0, "writer CTA never started"
            time.sleep(1e-4)
        captures, steps = 0, []
        while int(flag[0]) != 2 and captures < 400:
            eng.enqueue_checkpoint(captures & 1)
            _seq, b, step = eng.checkpoint_wait()
            captures += 1
            if step >= 0:
                assert torch.equal(_bits(eng.ckpt_host[b]), _bits(_f(step, n))), "capture of step %d is not f(%d, .)" % (step, step)
                steps.append(step)
        side.synchronize()
        assert steps == sorted(steps)
        if pace_us > 0:
            assert steps, "no capture was accepted next to a writer that pauses %g us between commits" % pace_us
        g += rounds
        report["pace_%gus" % pace_us] = dict(captures=captures, accepted=len(steps), rejected=captures - len(steps))
    print("\nconcurrent checkpoint capture (%s): %s %s" % ("interval" if mode else "k_of_n", report, eng.checkpoint_stats()))
    be.check_error()


@pytest.mark.parametrize("mode", [K_OF_N, INTERVAL], ids=["k_of_n", "interval"])
def test_failed_captures_write_no_file_and_are_retried_at_the_next_step(tmp_path, mode):
    """A back-to-back writer: most captures fail.  The checkpointer writes no file for them and enqueues the retry at its
    next call; every file it writes holds f(g, .) of its step."""
    from distributedmnist_b200.checkpoint import Saver, get_checkpoint_state
    from distributedmnist_b200.ops.lib import stream_ptr
    from distributedmnist_b200.train import _AsyncCheckpointer
    eng, be = _engine(optimizer=False)
    eng._interval = mode == INTERVAL
    eng.arm_checkpoint(snapshot=True)
    n = eng.params.numel()
    _emulate(eng, 1, mode)
    torch.cuda.synchronize()

    class _Flat:
        def to_state_dict(self, flat):
            return {"arena": flat.clone()}
    train_dir = str(tmp_path / "train")
    ck = _AsyncCheckpointer(train_dir, _Flat(), 1000.0, engine=eng, timeout_s=5.0)
    enqueued = []
    real = eng.enqueue_checkpoint
    eng.enqueue_checkpoint = lambda buf: enqueued.append(buf) or real(buf)
    saved = []
    real_save = ck.saver.save
    ck.saver.save = lambda d, state, step: saved.append(step) or real_save(d, state, step)
    flag = torch.zeros(4, dtype=torch.int32).pin_memory()
    side = torch.cuda.Stream()
    eng.lib.dm_snap_test_writer(be.ctrl.local_ptr, eng.params, n, 1, 3000, 0.0, mode, flag, stream_ptr(side))
    t0 = time.time()
    while int(flag[0]) == 0:
        assert time.time() - t0 < 30.0, "writer CTA never started"
        time.sleep(1e-4)
    ck._next = 0.0                                      # due now; afterwards only retries enqueue (interval 1000 s)
    while not saved:                                    # (once the writer has finished, a capture is accepted)
        ck.maybe_save(None, 0)
        assert time.time() - t0 < 60.0
    ck._queue.join()
    ck.close()
    side.synchronize()
    print("\nback-to-back writer (%s): %d captures, %d failed, %d written" % ("interval" if mode else "k_of_n",
                                                                               len(enqueued), ck.failed, len(saved)))
    assert ck.failed >= 1 and len(saved) == 1 and len(enqueued) == ck.failed + 1
    st = get_checkpoint_state(train_dir)
    assert st.all_model_checkpoint_paths == ["model.ckpt-%d" % saved[0]]
    state, step = Saver.restore(Saver.latest(train_dir))
    assert step == saved[0] and torch.equal(_bits(state["arena"]), _bits(_f(step, n)))
    be.check_error()


@pytest.mark.parametrize("snapshot", [False, True], ids=["live", "snapshot"])
@pytest.mark.parametrize("mode", [K_OF_N, INTERVAL], ids=["k_of_n", "interval"])
def test_capture_after_a_restore_reports_the_restored_step(mode, snapshot):
    eng, be = _engine(optimizer=False)
    eng._interval = mode == INTERVAL
    be.set_global_step(57)
    eng.params.copy_(_f(57, eng.params.numel()).cuda() * 0.01)
    eng.params_updated()
    eng.arm_checkpoint(snapshot=snapshot)
    eng.enqueue_checkpoint(0)
    _seq, b, step = eng.checkpoint_wait()
    assert step == 57 and torch.equal(_bits(eng.ckpt_host[b]), _bits(eng.params.cpu()))


def _env():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="0")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    return env


@pytest.mark.parametrize("model,extra", [("lenet", ["--num_replicas_to_aggregate=3"]),
                                         ("mlp2", ["--num_replicas_to_aggregate=3"]),
                                         ("lenet", ["--interval_method=true", "--interval_ms=2"])],
                         ids=["k3_lenet", "k3_mlp2", "interval_lenet"])
def test_train_checkpoints_every_step_end_to_end(tmp_path, model, extra):
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.checkpoint import Saver, get_checkpoint_state, resolve_checkpoint_path, step_from_path
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.models import get_model
    train_dir, eval_dir = str(tmp_path / "train_dir"), str(tmp_path / "eval_dir")
    live = str(tmp_path / "live.npy")
    tr = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "_ckpt_worker.py"), live, "--batch_size=128",
                         "--max_steps=40", "--model=%s" % model, "--initial_learning_rate=0.05", "--save_interval_secs=0.001",
                         "--train_dir=" + train_dir, "--log_every=50"] + extra,
                        env=_env(), capture_output=True, text=True, timeout=600)
    log = tr.stdout + tr.stderr
    assert tr.returncode == 0, log[-3000:]
    st = get_checkpoint_state(train_dir)
    paths = st.all_model_checkpoint_paths
    assert len(paths) >= 2 and paths[-1] == st.model_checkpoint_path, paths
    steps = [step_from_path(p) for p in paths]
    assert steps == sorted(set(steps)), steps
    assert resolve_checkpoint_path(train_dir, st) == Saver.latest(train_dir)
    for p in paths:
        _state, step = Saver.restore(os.path.join(train_dir, p))
        assert step == step_from_path(p)
    spec = get_model(model)[0]
    final, step = Saver.restore(Saver.latest(train_dir))
    flat = spec.from_state_dict(final)
    arena = torch.from_numpy(np.load(live))[:spec.arena_numel]
    mask = spec.valid_mask()
    assert torch.equal(_bits(flat[mask]), _bits(arena[mask])), "the final checkpoint is not the arena after the run"
    print("\n%s %s: kept checkpoints at steps %s" % (model, " ".join(extra), steps))
    if model != "lenet":
        return
    FLAGS.reset()
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=FLAGS.synthetic_data, fake_data=FLAGS.fake_data)
    eng, _be = _engine(optimizer=False)
    eng.params.copy_(flat.to(eng.params.device))
    eng.params_updated()
    eng.arm_eval(ds.validation.images, ds.validation.labels)
    ref = eng.run_eval()
    ev = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_eval.py"), "--run_once=true",
                         "--checkpoint_dir=" + train_dir, "--eval_dir=" + eval_dir], env=_env(), capture_output=True,
                        text=True, timeout=600)
    out = ev.stdout + ev.stderr
    assert ev.returncode == 0, out[-3000:]
    m = re.search(r"Num examples: (\d+)  Precision @ 1: ([0-9.]+) Loss", out)
    assert m and int(m.group(1)) == ref[3], out[-2000:]
    assert ref[4] == round(float(m.group(2)) * ref[3]), (ref, m.group(0))


def test_checkpoints_add_no_host_synchronisation(tmp_path, monkeypatch):
    """``train()`` in this process, K = N lenet: a run that checkpoints after every consumed step makes exactly as many
    synchronise calls inside the training loop as one that never checkpoints.  Calls are counted until the final save is
    entered: that save waits for a capture still in flight, which depends on how fast the saver thread freed the arenas."""
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.checkpoint import get_checkpoint_state
    from distributedmnist_b200.engine_cuda import _CudaEngine
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import _AsyncCheckpointer, train
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    calls = {"sync": 0, "captures": 0, "at_final_save": None}

    def counted(fn, key):
        def wrapper(*a, **k):
            calls[key] += 1
            return fn(*a, **k)
        return wrapper
    monkeypatch.setattr(torch.cuda, "synchronize", counted(torch.cuda.synchronize, "sync"))
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", counted(torch.cuda.Stream.synchronize, "sync"))
    monkeypatch.setattr(torch.cuda.Event, "synchronize", counted(torch.cuda.Event.synchronize, "sync"))
    monkeypatch.setattr(_CudaEngine, "enqueue_checkpoint", counted(_CudaEngine.enqueue_checkpoint, "captures"))
    real_save = _AsyncCheckpointer.save

    def save(self, *a, **k):
        calls["at_final_save"] = (calls["sync"], calls["captures"])
        return real_save(self, *a, **k)
    monkeypatch.setattr(_AsyncCheckpointer, "save", save)
    counts = {}
    try:
        for name, secs in (("every_step", "0"), ("never", "1e9"), ("every_step_again", "0")):
            FLAGS.reset()
            d = tmp_path / name
            FLAGS.parse(["--train_dir=%s" % d, "--batch_size=128", "--max_steps=200", "--save_interval_secs=%s" % secs,
                         "--initial_learning_rate=0.05", "--log_every=1000", "--save_results_period=1000000"])
            ctx = init_context(FLAGS)
            ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True, synthetic_sizes=(4096, 256))
            calls.update(sync=0, captures=0, at_final_save=None)
            res = train(ctx, ds.train, ds.validation, FLAGS)
            assert calls["at_final_save"] is not None
            counts[name] = calls["at_final_save"]
            assert res["final_step"] == 201
            kept = get_checkpoint_state(str(d)).all_model_checkpoint_paths
            assert kept[-1] == "model.ckpt-201"
            if secs == "1e9":
                assert kept == ["model.ckpt-201"] and counts[name][1] == 0
            else:
                # at most one capture in flight and two host arenas: how many are taken depends on the disk, not on the loop
                assert len(kept) >= 2 and counts[name][1] >= 2, (kept, counts[name])
    finally:
        FLAGS.reset()
    print("\n(synchronise calls, captures) before the final save: %s" % counts)
    assert counts["every_step"][0] == counts["never"][0] == counts["every_step_again"][0], counts
