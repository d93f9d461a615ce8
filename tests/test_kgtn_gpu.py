"""K > N gradients per update on the GPU (csrc/fused_interval.cu with the count trigger): the engines' graph-replayed steps
bit for bit against the exact emulation of ops/aggrefs.py, the device accounting, the training driver with snapshot
evaluation, and several replicas with a delayed one."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from distributedmnist_b200.ops import aggrefs as A
from distributedmnist_b200.schedule import LearningRateSchedule

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _backend():
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    return FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))


def _engine_commits(make_engine, k, commits=3):
    """``commits`` x ``k`` graph-replayed iterations on one replica: after every k-th the fp32 arena must be
    sgd(w, interval_accumulate(the k gradients), fp32(lr(step) / k)) bit for bit."""
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    be = _backend()
    eng = make_engine(be)
    sched = LearningRateSchedule(0.05, 2, 0.999)
    eng.attach_optimizer(SyncReplicasOptimizer(be, sched, k, 1))
    assert eng._kgtn_k == k and not eng._bucketed
    be.set_global_step(3001)
    be.kgtn_arm()
    gen = torch.Generator().manual_seed(9)
    B = eng.batch_size
    shape = (B, 28, 28) if isinstance(eng, CudaLeNetEngine) else (B, 784)
    for c in range(commits):
        torch.cuda.synchronize()
        step = be.device_epoch if c == 0 else step + 1
        gs = []
        for i in range(k):
            eng.load_batch(torch.rand(*shape, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen))
            eng.train_step()
            torch.cuda.synchronize()
            if i == 0:
                w = A.f32(eng.params)          # the first iteration adopted the previous commit
            gs.append(A.f32(eng.grads))
        want = A.sgd(w, A.interval_accumulate(gs), A.step_scale(sched, step, k))
        got = A.bits(eng.params)
        bad = np.flatnonzero(got != A.bits(want))
        assert bad.size == 0, "commit %d: %d of %d weights differ, first at %d" % (c, bad.size, got.size, bad[0])
    be.check_error()
    st = be.read_status()
    assert st["accepted_steps"] == k * commits and st["dropped_steps"] == 0, st
    eng.train_step()                           # adopts the last commit
    torch.cuda.synchronize()
    st = be.read_status()
    assert st["epoch"] == 3001 + commits and st["last_count"] == k, st
    assert eng.launches_per_step > 0
    return eng


def test_lenet_k4_one_replica_is_bit_exact():
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    eng = _engine_commits(lambda be: CudaLeNetEngine(128, be, seed=3, rank=0, use_graph=True), 4)
    kt = eng.time_kernels(3)                   # bench.py --kernel-times: the K > N kernels, not the fused sync kernel
    assert "kgtn_end" in kt and "kgtn_begin" in kt and "fused_sync_sgd" not in kt and kt["kgtn_end"] > 0


def test_mlp2_k2_one_replica_is_bit_exact():
    from distributedmnist_b200.engine_cuda import CudaMlpEngine
    _engine_commits(lambda be: CudaMlpEngine("mlp2", 128, be, hidden=1024, seed=3, use_graph=True), 2)


def test_drop_connect_with_k_above_n_is_refused():
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    be = _backend()
    eng = CudaLeNetEngine(32, be, use_graph=False)
    with pytest.raises(ValueError, match="drop_connect"):
        eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.01, 10, 1.0), 3, 1,
                                                   drop_connect_probability=0.5))


def test_native_runner_steps_commit_every_k():
    """step_packed (input DMA + graph launch in one native call), as the training loop and bench.py drive it."""
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    be = _backend()
    eng = CudaLeNetEngine(256, be, seed=1, use_graph=True)
    eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.01, 10, 1.0), 4, 1))
    gen = torch.Generator().manual_seed(2)
    bufs = [eng.pack_batch(torch.rand(256, 28, 28, generator=gen) - 0.5, torch.randint(0, 10, (256,), generator=gen))
            for _ in range(4)]
    for i in range(41):
        ev = eng.step_packed(bufs[i % 4])
    ev[0].synchronize()
    assert eng._runner is not None
    st = be.read_status()
    assert st["epoch"] == 10 and st["accepted_steps"] == 40 and st["dropped_steps"] == 0 and st["error"] == 0, st


def test_train_k3_one_replica_snapshot_eval_matches_the_evaluator(tmp_path):
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.checkpoint import Saver
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.flags import FLAGS
    train_dir, eval_dir = str(tmp_path / "train_dir"), str(tmp_path / "eval_dir")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="0")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    tr = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_distributed_train.py"), "--job_name=worker",
                         "--task_id=0", "--worker_hosts=localhost:1234", "--batch_size=128", "--max_steps=20",
                         "--num_replicas_to_aggregate=3", "--eval_every_steps=4", "--eval_snapshot=true",
                         "--initial_learning_rate=0.05", "--train_dir=" + train_dir, "--log_every=50"],
                        env=env, capture_output=True, text=True, timeout=600)
    log = tr.stdout + tr.stderr
    assert tr.returncode == 0, log[-3000:]
    rows = np.load(os.path.join(train_dir, "worker0_eval.npy"))
    assert len(rows) >= 3 and (np.diff(rows[:, 0]) >= 0).all() and (rows[:, 3] == 10000).all(), rows
    FLAGS.reset()
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=FLAGS.synthetic_data, fake_data=FLAGS.fake_data)
    state, step = Saver.restore(Saver.latest(train_dir))
    assert step == 21 and int(rows[-1, 0]) == 21, (step, rows[-1])
    eng = CudaLeNetEngine(256, _backend(), seed=5, use_graph=False)
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


# ---- several replicas (tests/_kgtn_worker.py) -------------------------------------------------------------------------
def _run_worker(tmp_path, n, k, iters, delay_us, nvls):
    from distributedmnist_b200.parallel.launcher import run_replicas
    os.environ["DMNIST_NVLS"] = "1" if nvls else "0"       # inherited by the helper processes
    try:
        codes = run_replicas([os.path.join(HERE, "_kgtn_worker.py"), str(tmp_path / "res_RANK.json"), str(k), str(iters),
                              str(delay_us)], n, timeout=300, out_dir=str(tmp_path / "out"))
    finally:
        os.environ.pop("DMNIST_NVLS")
    logs = "\n".join(open(os.path.join(tmp_path, "out", f)).read()[-1500:] for f in sorted(os.listdir(tmp_path / "out")))
    assert codes == [0] * n, logs
    return [json.load(open(tmp_path / ("res_%d.json" % r))) for r in range(n)]


@pytest.mark.multigpu
@pytest.mark.parametrize("nvls", [True, False])
def test_multi_replica_k_above_n_with_a_delayed_replica(tmp_path, nvls):
    n = min(torch.cuda.device_count(), 8)
    k = 2 * n + 1
    res = _run_worker(tmp_path, n, k, 400, 1000.0, nvls)
    steps = {r["steps"] for r in res}
    assert len(steps) == 1 and res[0]["steps"] >= 10, [r["steps"] for r in res]
    steps = res[0]["steps"]
    assert len({r["fp"] for r in res}) == 1                                # replicas bit-identical once quiescent
    assert all(r["err"] < 1e-5 * max(1.0, r["pmax"]) for r in res), [r["err"] for r in res]
    assert sum(r["ticks_committed"] for r in res) == steps                 # exactly one committer per step
    totals = {}
    for r in res:
        for epoch, _late, _mask, count in r["rows"]:
            if epoch > 0:
                totals[epoch] = count                                      # divisor of the step that produced `epoch`
    assert totals and all(c >= k for c in totals.values()), totals
    accepted = sum(r["accepted"] for r in res)
    assert accepted >= k * steps
    if len(totals) == steps:
        assert accepted == sum(totals.values())
    # every accumulated or dropped iteration is accounted for exactly once
    assert sum(r["accepted"] + r["dropped"] + r["pending"] for r in res) == sum(r["iters"] for r in res)
    slow, fast = res[n - 1], res[0]
    assert slow["accepted"] < fast["accepted"]                             # the delayed replica contributes fewer
    assert fast["wall_s"] < 2.0 * slow["wall_s"] + 1.0                      # ... and nobody waits for it
    if nvls and n >= 2:
        assert all(r["nvls"] for r in res) or not any(r["nvls"] for r in res)
