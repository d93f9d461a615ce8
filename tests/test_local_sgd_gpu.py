"""Local SGD (``--local_sgd_steps``, csrc/fused_local.cu) on H100s.

1. The local update on one replica, bit for bit against ``ops/aggrefs.py`` over the whole LeNet arena after every step,
   with the shadow equal to RNE(weights), under the staircase, warmup and cosine schedules; the averaging steps (the
   identity with one replica) and the statistics.
2. The averaging arithmetic over N = 2, 3, 4 and 8 arenas in one process: ls_average_kernel alone, once per shard owner,
   bit for bit against ``aggrefs.local_average``.  No barrier runs: nothing here waits on another replica.
3. Engine steps on one replica, graph-replayed back to back, stage by stage (ops/trajectory.py, mode "local"), for LeNet
   and mlp3.
4. ``train()`` on one replica with the in-training evaluation, a target, the device-resident training set and
   augmentation; the polling evaluator reproduces the last pass's count on the final checkpoint, and a restart continues
   the global step and averages at the next multiple of H.
5. Several GPUs (tests/_local_sgd_worker.py, skipped below 2 GPUs): replicas bit-identical after every averaging step and
   not between them, the average against the recorded copies with and without NVLS, a target run that ends on the same
   step everywhere, and a lognormal straggler run that reports its barrier wait."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch

from distributedmnist_b200.ops import aggrefs as A

pytestmark = pytest.mark.gpu

STEP0 = 3001
HERE = os.path.dirname(os.path.abspath(__file__))


def _lib():
    from distributedmnist_b200.ops.lib import load
    return load()


def _table(ptrs):
    return (ctypes.c_void_p * 8)(*([int(p) for p in ptrs] + [int(ptrs[0])] * (8 - len(ptrs))))


def _assert_exact(what, params, shadow, want):
    torch.cuda.synchronize()
    got, exp = A.bits(params), A.bits(want)
    bad = np.flatnonzero(got != exp)
    assert bad.size == 0, "%s: %d of %d weights differ, first at %d: got %r, want %r" % (
        what, bad.size, got.size, bad[0], got.view(np.float32)[bad[0]], exp.view(np.float32)[bad[0]])
    sh = shadow.view(torch.int16).cpu().numpy().view(np.uint16)
    bad = np.flatnonzero(sh != A.bf16_bits(want))
    assert bad.size == 0, "%s: %d of %d shadow elements differ from RNE(weights), first at %d" % (
        what, bad.size, sh.size, bad[0])


# ---- 1. the local update, one replica -------------------------------------------------------------------------------------
@pytest.mark.parametrize("sched", ["staircase", "warmup", "cosine"])
def test_local_step_one_replica_bit_for_bit(sched):
    from distributedmnist_b200.models import get_model
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    try:
        spec, _ = get_model("lenet")
        n = spec.arena_numel
        params = be.allocate(n)
        params.copy_(spec.init_flat(7).cuda())
        be.attach_shadow(params)
        stats = torch.zeros(int(_lib().dm_local_stats_bytes()), dtype=torch.uint8, device="cuda")
        if sched == "staircase":
            s = LearningRateSchedule(0.05, STEP0 + 2, 0.5)
        elif sched == "warmup":
            s = LearningRateSchedule(0.05, 1, 1.0, warmup_steps=STEP0 + 3, warmup_start=0.25)
        else:
            s = LearningRateSchedule(0.05, 1, 1.0, warmup_steps=STEP0 + 2, warmup_start=0.1, cosine_steps=STEP0 + 4,
                                     cosine_alpha=0.05)
        be.set_lr_schedule(s.warmup_steps, s.warmup_start, s.cosine_steps, getattr(s, "cosine_alpha", 0.0))
        be.set_global_step(STEP0)
        H = 3
        gen = torch.Generator(device="cuda").manual_seed(3)
        w = A.f32(params)
        rounds = 0
        for j in range(7):
            g = torch.randn(n, generator=gen, device="cuda") * 0.5
            be.enqueue_local_step(params, g, H, s.initial_learning_rate, s.decay_rate, s.decay_steps)
            be.enqueue_local_average(params, stats, H)
            w = A.sgd(w, A.f32(g), A.step_scale(s, STEP0 + j, 1))
            if (STEP0 + j + 1) % H == 0:
                w = A.local_average([w])
                rounds += 1
            _assert_exact("%s step %d" % (sched, j), params, be.shadow, w)
            info = be.mirror_info(j + 1)
            assert info.global_step == STEP0 + j + 1 and info.accepted and info.count == 1
        assert be.device_epoch == STEP0 + 7
        st = be.local_stats(stats)
        assert st["rounds"] == rounds == 2 and st["wait_max_ns"] <= st["wait_total_ns"]
        be.enqueue_local_average(params, stats, 1, close=False)        # the end-of-run average closes no step
        _assert_exact("%s final" % sched, params, be.shadow, w)
        assert be.device_epoch == STEP0 + 7 and be.local_stats(stats)["rounds"] == 3
        be.check_error()
    finally:
        be.close()


# ---- 2. the averaging arithmetic over N arenas on one GPU -------------------------------------------------------------------
@pytest.mark.parametrize("nranks", [2, 3, 4, 8])
@pytest.mark.parametrize("ctas", [0, 5])
def test_average_peer_path_bit_for_bit(nranks, ctas):
    from distributedmnist_b200.models import get_model
    lib = _lib()
    spec, _ = get_model("lenet")
    n = spec.arena_numel
    gen = torch.Generator(device="cuda").manual_seed(nranks)
    ws = [torch.randn(n, generator=gen, device="cuda") * (q + 1) for q in range(nranks)]
    ws[0][:8] = 0.0
    ws[1][8:16] = -ws[0][8:16]                      # sums that cancel exactly
    before = [A.f32(w) for w in ws]
    ctrl = torch.zeros(int(lib.dm_sync_ctrl_bytes()), dtype=torch.uint8, device="cuda")
    sp = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    tab = _table([w.data_ptr() for w in ws])
    lib.dm_local_average_shard(ctrl, tab, 0, nranks, n, 2, ctas, sp, None)    # epoch 0: an averaging step of H = 2
    for q in range(1, nranks):
        lib.dm_local_average_shard(ctrl, tab, q, nranks, n, 2, ctas, sp, None)
    torch.cuda.synchronize()
    want = A.bits(A.local_average(before))
    for q in range(nranks):
        bad = int((A.bits(ws[q]) != want).sum())
        assert bad == 0, "arena %d: %d of %d elements differ" % (q, bad, n)
    # an epoch word that is not a multiple of H: the kernel leaves every arena alone
    ctrl[int(lib.dm_sync_ctrl_offset(b"epoch"))] = 1
    again = [w.clone() for w in ws]
    for w in ws:
        w.add_(1.0)
    for q in range(nranks):
        lib.dm_local_average_shard(ctrl, tab, q, nranks, n, 2, ctas, sp, None)
    torch.cuda.synchronize()
    assert all(torch.equal(w, a + 1.0) for w, a in zip(ws, again))


# ---- 3. engine steps, one replica -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("model,B", [("lenet", 256), ("mlp3", 512)])
def test_engine_steps_stage_by_stage(model, B):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine, CudaMlpEngine
    from distributedmnist_b200.ops import trajectory as T
    from distributedmnist_b200.ops.trajectory import StepRecorder
    from distributedmnist_b200.parallel.aggregators import LocalSGDOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    if model == "lenet":
        eng = CudaLeNetEngine(B, be, seed=3, rank=0, keep_prob=0.5, use_graph=True)
    else:
        eng = CudaMlpEngine(model, B, be, hidden=4096, seed=3, use_graph=True)
    sched = LearningRateSchedule(0.05, 1, 0.999)
    eng.attach_optimizer(LocalSGDOptimizer(be, sched, 1, period=2))
    assert eng._local == 2 and not eng._bucketed and not eng._interval and not eng._async
    be.set_global_step(STEP0)
    rec = StepRecorder(eng)
    gen = torch.Generator().manual_seed(9)
    shape = (B, 28, 28) if model == "lenet" else (B, 784)
    batches = [(torch.rand(*shape, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen)) for _ in range(6)]
    for x, y in batches:
        eng.load_batch(x.numpy(), y.numpy())
        eng.train_step()
        rec.record()
    torch.cuda.synchronize()
    be.check_error()
    assert be.device_epoch == STEP0 + 6
    upd = T.update_of(eng, sched, STEP0)
    assert upd["mode"] == "local" and upd["period"] == 2
    if model == "lenet":
        res = T.lenet_trajectory_results(model, eng.spec, rec.init, rec.records, batches, upd, eng.seed, eng.rank,
                                         eng.keep_prob, 0.0)
    else:
        res = T.mlp_trajectory_results(model, eng.spec, rec.init, rec.records, batches, upd)
    print("\nTRAJECTORY local.%s %s" % (model, json.dumps(T.worst_by_stage(model, res), sort_keys=True)))
    bad = T.failures(res)
    assert not bad, "%d of %d checks failed, first: %s" % (len(bad), len(res), bad[:20])
    w = eng.params.clone()
    assert eng.local_finish() == STEP0 + 6
    assert torch.equal(eng.params, w)                   # one replica: the final average is the identity
    assert eng.local_stats()["rounds"] == 4             # global steps 3002, 3004, 3006, and the final average after 3007


# ---- 4. train(), one replica ----------------------------------------------------------------------------------------------
def _train(d, *extra, steps=120):
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import train
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % d, "--batch_size=128", "--max_steps=%d" % steps, "--eval_every_steps=20",
                 "--local_sgd_steps=5", "--save_interval_secs=1000", "--log_every=20"] + list(extra))
    ctx = init_context(FLAGS)
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True, synthetic_sizes=(8192, 2048))
    try:
        return train(ctx, ds.train, ds.validation, FLAGS)
    finally:
        FLAGS.reset()


@pytest.fixture
def one_replica(monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)


def test_train_with_evaluation_target_device_data_and_augmentation(tmp_path, one_replica, capsys):
    from distributedmnist_b200.checkpoint import Saver
    from distributedmnist_b200.flags import FLAGS
    d = str(tmp_path / "run")
    res = _train(d, "--target_accuracy=0.5", "--device_data", "--augment_max_shift=1.5", "--augment_max_rotation=8")
    tta = res["time_to_accuracy"]
    T = res["final_step"]
    evals = res["evals"]
    steps = [int(r[0]) for r in evals]
    if tta["reached"]:
        g = tta["global_step"]
        assert g % 20 == 0 and T == g + 2 * 5 + 1        # S = g + 2H, and the run ends as --max_steps = S does
    else:
        assert T == 121
    assert steps[-1] == T and all(s % 20 == 0 for s in steps[:-1])
    rep = res["local_sgd"]
    assert rep["period"] == 5 and rep["rounds"] == T // 5 + 1 and rep["wait_total_s"] >= 0.0
    with open(os.path.join(d, "worker0_local_sgd.json")) as f:
        assert json.load(f) == rep
    state, step = Saver.restore(Saver.latest(d))
    assert step == T
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200 import evaluator
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True, synthetic_sizes=(8192, 2048))
    capsys.readouterr()
    FLAGS.reset()
    FLAGS.parse(["--checkpoint_dir=%s" % d, "--eval_dir=%s" % str(tmp_path / "eval"), "--run_once=true"])
    try:
        assert int(evaluator.evaluate(ds.validation, FLAGS, torch.device("cuda", 0), max_evals=1)) == T
    finally:
        FLAGS.reset()
    m = re.search(r"Num examples: 2048  Precision @ 1: ([0-9.]+) Loss", capsys.readouterr().out)
    assert m and round(float(m.group(1)) * 2048) == int(evals[-1][4])


def test_train_restart_continues_the_global_step(tmp_path, one_replica):
    from distributedmnist_b200.checkpoint import Saver
    d = str(tmp_path / "run")
    first = _train(d, steps=41)
    T1 = first["final_step"]
    assert T1 == 42 and Saver.restore(Saver.latest(d))[1] == 42
    second = _train(d, steps=90)
    assert second["steps"][0] == T1 + 1 and second["final_step"] == 91
    # averaging steps 45, 50, ..., 90, and the final average after 91: the first round is at the next multiple of H
    assert second["local_sgd"]["rounds"] == 10 + 1
    assert Saver.restore(Saver.latest(d))[1] == 91


# ---- 5. several GPUs (tests/_local_sgd_worker.py) ---------------------------------------------------------------------------
def _multi(tmp_path, n, nvls, *args):
    from distributedmnist_b200.parallel.launcher import run_replicas
    os.environ["DMNIST_NVLS"] = "1" if nvls else "0"       # inherited by the helper processes
    try:
        codes = run_replicas([os.path.join(HERE, "_local_sgd_worker.py"), str(tmp_path / "train"),
                              str(tmp_path / "res_RANK.npz")] + list(args), n, timeout=600, out_dir=str(tmp_path / "out"))
    finally:
        os.environ.pop("DMNIST_NVLS")
    logs = "\n".join(open(os.path.join(tmp_path, "out", f)).read()[-1500:] for f in sorted(os.listdir(tmp_path / "out")))
    assert codes == [0] * n, logs
    return [dict(np.load(str(tmp_path / ("res_%d.npz" % r)))) for r in range(n)]


@pytest.mark.multigpu
@pytest.mark.parametrize("nvls", [False, True], ids=["p2p", "nvls"])
def test_multi_gpu_replicas_agree_after_every_average(tmp_path, nvls):
    n = min(torch.cuda.device_count(), 8)
    if nvls and n < 4:
        pytest.skip("the NVLS case needs 4 GPUs")
    H = 4
    res = _multi(tmp_path, n, nvls, "--max_steps=21", "--local_sgd_steps=%d" % H)
    steps = res[0]["steps"].tolist()
    assert steps == list(range(1, 23)) and all(r["steps"].tolist() == steps for r in res)
    for t, s in enumerate(steps):
        same = len({A.bits(r["after"][t]).tobytes() for r in res}) == 1
        assert same == (s % H == 0), (s, same)
    # each average against the copies every replica held after the step before it (the step's update applied)
    for t, s in enumerate(steps):
        if s % H or t == 0:
            continue
        want = A.local_average([r["before"][t] for r in res])
        got = res[0]["after"][t].astype(np.float64)
        if nvls:                  # the switch picks the summation order: within n roundings of the sum
            top = sum(np.abs(r["before"][t]).astype(np.float64) for r in res)
            assert np.all(np.abs(got - want) <= n * np.spacing(top.astype(np.float32)))
        else:
            assert A.bits(res[0]["after"][t]).tolist() == A.bits(want).tolist()
    assert len({A.bits(r["final"]).tobytes() for r in res}) == 1 and all(int(r["final_step"]) == 22 for r in res)
    assert all(bool(r["nvls"]) == nvls for r in res)


@pytest.mark.multigpu
def test_multi_gpu_target_run_ends_on_the_same_step(tmp_path):
    n = min(torch.cuda.device_count(), 8)
    H = 4
    res = _multi(tmp_path, n, False, "--max_steps=400", "--local_sgd_steps=%d" % H, "--eval_every_steps=8",
                 "--target_accuracy=0.2")
    ends = {int(r["final_step"]) for r in res}
    assert len(ends) == 1
    tta = json.load(open(tmp_path / "train" / "worker0_time_to_accuracy.json"))
    assert tta["reached"], tta
    assert ends == {tta["global_step"] + 2 * H + 1}
    assert len({A.bits(r["final"]).tobytes() for r in res}) == 1


@pytest.mark.multigpu
def test_multi_gpu_lognormal_stragglers_report_their_wait(tmp_path):
    n = min(torch.cuda.device_count(), 8)
    res = _multi(tmp_path, n, False, "--max_steps=200", "--local_sgd_steps=16", "--inject_straggler=*:lognormal:100:1.0")
    assert {int(r["final_step"]) for r in res} == {201}
    for r in res:
        rep = json.loads(str(r["report"]))
        assert rep["rounds"] == 201 // 16 + 1 and rep["wait_total_s"] > 0.0 and rep["wait_max_s"] > 0.0
    assert len({A.bits(r["final"]).tobytes() for r in res}) == 1
