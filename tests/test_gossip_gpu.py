"""Gossip SGD (``--gossip_method``, csrc/fused_gossip.cu) on H100s.

1. Engine steps on one replica, graph-replayed back to back, stage by stage (ops/trajectory.py, mode "gossip"), for
   LeNet at B = 256 and mlp3 at B = 512.  For LeNet every recorded buffer is also bit for bit that of a
   ``--local_sgd_steps=1`` engine fed the same batches.
2. N = 2 to 8 replicas on one GPU (tests/_gossip_replicas_worker.py), one stream each, with the last replica slowed by a
   device sleep: every replica's arena after every iteration bit for bit against ``aggrefs.gossip_mix`` of the
   emulated half steps; for N <= 3 equal to the local-SGD kernels with H = 1; G2 from the %globaltimer stamps, with the
   bound reached by the replica opposite the slow one; the fast replicas waited; no error word; after the closing
   dm_local_average every arena is ``aggrefs.local_average`` of the mixed arenas.
3. ``train()`` on one replica with the in-training evaluation, a target, the device-resident training set and
   augmentation: the report, the JSON file, the log line, the final checkpoint reproducing the final pass's count, and a
   restart that continues the global step.
4. Several GPUs (tests/_gossip_worker.py, skipped below 2 GPUs): lognormal stragglers, and a target run; every replica
   ends on the same step with identical final weights."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from distributedmnist_b200.ops import aggrefs as A

pytestmark = pytest.mark.gpu

STEP0 = 3001
HERE = os.path.dirname(os.path.abspath(__file__))


# ---- 1. engine steps, one replica -----------------------------------------------------------------------------------------
def _engine(model, B, opt_cls, **kw):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine, CudaMlpEngine
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    if model == "lenet":
        eng = CudaLeNetEngine(B, be, seed=3, rank=0, keep_prob=0.5, use_graph=True)
    else:
        eng = CudaMlpEngine(model, B, be, hidden=4096, seed=3, use_graph=True)
    sched = LearningRateSchedule(0.05, 1, 0.999)
    eng.attach_optimizer(opt_cls(be, sched, 1, **kw))
    be.set_global_step(STEP0)
    return be, eng, sched


def _run(eng, batches):
    from distributedmnist_b200.ops.trajectory import StepRecorder
    rec = StepRecorder(eng)
    for x, y in batches:
        eng.load_batch(x.numpy(), y.numpy())
        eng.train_step()
        rec.record()
    torch.cuda.synchronize()
    eng.backend.check_error()
    return rec


@pytest.mark.parametrize("model,B", [("lenet", 256), ("mlp3", 512)])
def test_engine_steps_stage_by_stage(model, B):
    from distributedmnist_b200.ops import trajectory as T
    from distributedmnist_b200.parallel.aggregators import GossipSGDOptimizer, LocalSGDOptimizer
    be, eng, sched = _engine(model, B, GossipSGDOptimizer)
    assert eng._gossip and not eng._local and not eng._bucketed and not eng._interval and not eng._async
    gen = torch.Generator().manual_seed(9)
    shape = (B, 28, 28) if model == "lenet" else (B, 784)
    batches = [(torch.rand(*shape, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen)) for _ in range(6)]
    rec = _run(eng, batches)
    assert be.device_epoch == STEP0 + 6
    upd = T.update_of(eng, sched, STEP0)
    assert upd["mode"] == "gossip"
    if model == "lenet":
        res = T.lenet_trajectory_results(model, eng.spec, rec.init, rec.records, batches, upd, eng.seed, eng.rank,
                                         eng.keep_prob, 0.0)
    else:
        res = T.mlp_trajectory_results(model, eng.spec, rec.init, rec.records, batches, upd)
    print("\nTRAJECTORY gossip.%s %s" % (model, json.dumps(T.worst_by_stage(model, res), sort_keys=True)))
    bad = T.failures(res)
    assert not bad, "%d of %d checks failed, first: %s" % (len(bad), len(res), bad[:20])
    st = eng.gossip_stats()
    assert st["iterations"] == 6 and st["waits"] == 0 and st["wait_max_ns"] <= st["wait_total_ns"]
    w = eng.params.clone()
    assert eng.gossip_finish() == STEP0 + 6
    assert torch.equal(eng.params, w)                   # one replica: the closing average is the identity
    if model != "lenet":
        return
    # the MLP kernels add their bias gradients with atomics in no fixed order, so only LeNet is compared bit for bit
    be2, eng2, _ = _engine(model, B, LocalSGDOptimizer, period=1)
    rec2 = _run(eng2, batches)
    assert eng.launches_per_step == eng2.launches_per_step - 2      # local SGD's five kernels -> gossip's three
    for t, (a, b) in enumerate(zip(rec.records, rec2.records)):
        assert a.keys() == b.keys()
        for k in a:
            xs, ys = (a[k], b[k]) if isinstance(a[k], list) else ([a[k]], [b[k]])
            for x, y in zip(xs, ys):
                assert torch.equal(x.view(torch.uint8), y.view(torch.uint8)), "step %d: %s differs" % (t, k)
    be.close()
    be2.close()


# ---- 2. N replicas on one GPU ---------------------------------------------------------------------------------------------
def test_replicas_on_one_gpu(tmp_path):
    out = str(tmp_path / "gossip.npz")
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    r = subprocess.run([sys.executable, os.path.join(HERE, "_gossip_replicas_worker.py"), out], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
    d = dict(np.load(out))
    sys.path.insert(0, HERE)
    import _gossip_replicas_worker as W
    from distributedmnist_b200.schedule import LearningRateSchedule
    scale = A.step_scale(LearningRateSchedule(W.LR, 1, 1.0), 0, 1)
    assert scale == np.float32(W.LR)
    for n in range(2, 9):
        p = "n%d_" % n
        assert d[p + "errors"].tolist() == [0] * (2 * n), "n=%d: error words %s" % (n, d[p + "errors"])
        assert d[p + "epochs"].tolist() == [W.ITERS] * n
        # every iteration of every replica bit for bit against the emulation
        w = [d["w0"]] * n
        for s in range(W.ITERS):
            hs = [A.sgd(w[q], d["grads"][q][s], scale) for q in range(n)]
            w = [A.gossip_mix(hs, q) for q in range(n)]
            for q in range(n):
                bad = int((A.bits(d[p + "rec"][q][s]) != A.bits(w[q])).sum())
                assert bad == 0, "n=%d replica %d iteration %d: %d of %d weights differ" % (n, q, s, bad, w[q].size)
        if n >= 4:
            assert len({A.bits(x).tobytes() for x in d[p + "mixed"]}) == n     # a sparse ring: the replicas differ
        else:
            # every replica mixes every half step: bit for bit the local-SGD kernels with H = 1
            assert np.array_equal(A.bits(d[p + "rec"]), A.bits(d[p + "local"]))
        # the closing average of every arena, and the shadow
        avg = A.local_average(list(d[p + "mixed"]))
        for q in range(n):
            assert np.array_equal(A.bits(d[p + "final"][q]), A.bits(avg)), "n=%d: arena %d after the average" % (n, q)
            assert np.array_equal(d[p + "shadow"][q], A.bf16_bits(avg))
        # G2: at every moment two replicas at ring distance k have passed barrier counts at most k apart (the pass
        # stamps), and have begun iterations at most k apart (the apply stamps)
        ta, tp = d[p + "t_arrive"].astype(np.int64), d[p + "t_pass"].astype(np.int64)
        dist = lambda a, b: min(abs(a - b), n - abs(a - b))     # noqa: E731
        for i in range(n):
            for j in range(n):
                k = dist(i, j)
                for s in range(k, W.ITERS):
                    assert tp[i][s - k] <= tp[j][s], "n=%d: %d passed barrier %d before %d passed %d" % (n, j, s, i, s - k)
                    assert ta[i][s - k] <= ta[j][s], "n=%d: %d began iteration %d before %d began %d" % (n, j, s, i, s - k)
        # the bound is reached: while the slow replica computes, the one opposite begins floor(N / 2) iterations more
        z, D = n - 1, n // 2
        o = (z + D) % n
        assert any(ta[o][s + D - 1] < ta[z][s] for s in range(W.ITERS - D + 1)), "n=%d: lead %d never reached" % (n, D)
        stats = json.loads(str(d[p + "stats"]))
        assert [st["iterations"] for st in stats] == [W.ITERS] * n
        assert all(stats[q]["waits"] > 0 for q in range(n) if q != z), stats
        assert all(st["wait_max_ns"] <= st["wait_total_ns"] for st in stats)


# ---- 3. train(), one replica ----------------------------------------------------------------------------------------------
def _train(d, *extra, steps=120):
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import train
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % d, "--batch_size=128", "--max_steps=%d" % steps, "--eval_every_steps=20",
                 "--gossip_method", "--save_interval_secs=1000", "--log_every=20"] + list(extra))
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
        assert g % 20 == 0 and T == g + 2 + 1            # S = g + max(2, floor(1 / 2)), and the run ends as S does
    else:
        assert T == 121
    assert steps[-1] == T and all(s % 20 == 0 for s in steps[:-1])
    rep = res["gossip"]
    assert rep["replicas"] == 1 and rep["neighbourhood"] == 1 and rep["iterations"] == T and rep["waits"] == 0
    with open(os.path.join(d, "worker0_gossip.json")) as f:
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
    assert second["gossip"]["iterations"] == 91 - 42
    assert Saver.restore(Saver.latest(d))[1] == 91


# ---- 4. several GPUs (tests/_gossip_worker.py) ------------------------------------------------------------------------------
def _multi(tmp_path, n, *args, nvls=False):
    from distributedmnist_b200.parallel.launcher import run_replicas
    os.environ["DMNIST_NVLS"] = "1" if nvls else "0"     # the closing average; the mix uses the peer path either way
    try:
        codes = run_replicas([os.path.join(HERE, "_gossip_worker.py"), str(tmp_path / "train"),
                              str(tmp_path / "res_RANK.npz")] + list(args), n, timeout=600, out_dir=str(tmp_path / "out"))
    finally:
        os.environ.pop("DMNIST_NVLS")
    logs = "\n".join(open(os.path.join(tmp_path, "out", f)).read()[-1500:] for f in sorted(os.listdir(tmp_path / "out")))
    assert codes == [0] * n, logs
    return [dict(np.load(str(tmp_path / ("res_%d.npz" % r)))) for r in range(n)]


@pytest.mark.multigpu
@pytest.mark.parametrize("nvls", [False, True], ids=["p2p", "nvls"])
def test_multi_gpu_lognormal_stragglers_end_together(tmp_path, nvls):
    n = min(torch.cuda.device_count(), 8)
    if nvls and n < 4:
        pytest.skip("the NVLS case needs 4 GPUs")
    res = _multi(tmp_path, n, "--max_steps=200", "--inject_straggler=*:lognormal:100:1.0", nvls=nvls)
    assert {int(r["final_step"]) for r in res} == {201}
    for r in res:
        rep = json.loads(str(r["report"]))
        assert rep["replicas"] == n and rep["iterations"] == 201 and rep["wait_total_s"] > 0.0
    assert len({A.bits(r["final"]).tobytes() for r in res}) == 1


@pytest.mark.multigpu
def test_multi_gpu_target_run_ends_on_the_same_step(tmp_path):
    n = min(torch.cuda.device_count(), 8)
    res = _multi(tmp_path, n, "--max_steps=400", "--eval_every_steps=8", "--target_accuracy=0.2")
    ends = {int(r["final_step"]) for r in res}
    assert len(ends) == 1
    tta = json.load(open(tmp_path / "train" / "worker0_time_to_accuracy.json"))
    assert tta["reached"], tta
    assert ends == {tta["global_step"] + max(2, n // 2) + 1}
    assert len({A.bits(r["final"]).tobytes() for r in res}) == 1
