"""Stale synchronous parallel (``--ssp_staleness`` with ``--async_method``, csrc/fused_async.cu) on one H100.

1. Engine steps on one replica, graph-replayed back to back, for LeNet (B = 256) and mlp3 with s = 0 and s = 3: stage by
   stage against float64 and the update bit for bit (ops/trajectory.py, mode "async"), and for LeNet every recorded
   buffer bit for bit equal to the same steps of a plain asynchronous engine.  One replica never waits.
2. N = 2, 4 and 8 replicas on one GPU (tests/_ssp_replicas_worker.py, one stream each), integer updates that count
   themselves, one slow replica, s in {0, 1, 4}: B1 and B2 at every pull, B3 for every update, the tickets a
   permutation, the final master copies exact, the bound reached exactly, and the fast replicas waiting.  A small
   watchdog turns a protocol bug into the error word instead of a long stall.
3. Retirement: a replica that stops half way retires, and the others finish with no error word.
4. ``train()`` on one replica with ``--ssp_staleness=0``: evaluation, a target and the device-resident training set; the
   report, its JSON file, and the final checkpoint reproducing the final pass's count.
5. Several GPUs (tests/_ssp_worker.py, skipped below 2 GPUs, the NVLS case below 4): ``train()`` with a straggler and
   s = 2 -- the clock lead and the staleness within their bounds, every replica's update count within s + 3 of every
   other's, and every copy of the weights identical."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
STEP0 = 3001
RETIRED = 0xFFFFFFFF


# ---- 1. engine steps, one replica -----------------------------------------------------------------------------------
def _engine(model, B, s):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine, CudaMlpEngine
    from distributedmnist_b200.ops.trajectory import StepRecorder
    from distributedmnist_b200.parallel.aggregators import AsyncSGDOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    if model == "lenet":
        eng = CudaLeNetEngine(B, be, seed=3, rank=0, keep_prob=0.5, use_graph=True)
    else:
        eng = CudaMlpEngine(model, B, be, hidden=4096, seed=3, use_graph=True)
    sched = LearningRateSchedule(0.05, 1, 0.999)
    eng.attach_optimizer(AsyncSGDOptimizer(be, sched, 1, ssp_staleness=s))
    assert eng._async and eng._ssp == s
    be.set_global_step(STEP0)
    return eng, be, sched, StepRecorder(eng)


@pytest.mark.parametrize("s", [0, 3])
@pytest.mark.parametrize("model,B", [("lenet", 256), ("mlp3", 512)])
def test_engine_steps_match_plain_async(model, B, s):
    from distributedmnist_b200.ops import trajectory as T
    gen = torch.Generator().manual_seed(9)
    shape = (B, 28, 28) if model == "lenet" else (B, 784)
    batches = [(torch.rand(*shape, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen)) for _ in range(6)]
    runs = {}
    for bound in (-1, s):
        eng, be, sched, rec = _engine(model, B, bound)
        for x, y in batches:
            eng.load_batch(x.numpy(), y.numpy())
            eng.train_step()
            rec.record()
        torch.cuda.synchronize()
        be.check_error()
        runs[bound] = (eng, be, sched, rec)
    eng, be, sched, rec = runs[s]
    plain = runs[-1][0]
    assert eng.launches_per_step == plain.launches_per_step + 2       # the wait and the clock publication
    upd = T.update_of(eng, sched, STEP0)
    assert upd["mode"] == "async"
    if model == "lenet":
        res = T.lenet_trajectory_results(model, eng.spec, rec.init, rec.records, batches, upd, eng.seed, eng.rank,
                                         eng.keep_prob, 0.0)
    else:
        res = T.mlp_trajectory_results(model, eng.spec, rec.init, rec.records, batches, upd)
    print("\nTRAJECTORY ssp%d.%s %s" % (s, model, json.dumps(T.worst_by_stage(model, res), sort_keys=True)))
    bad = T.failures(res)
    assert not bad, "%d of %d checks failed, first: %s" % (len(bad), len(res), bad[:20])
    # every recorded buffer of every step, bit for bit -- for LeNet, whose step is bit-reproducible; the MLP kernels add
    # their bias gradients with atomics in no fixed order, so there the trajectory check above is the comparison
    for a, b in zip(runs[-1][3].records, rec.records) if model == "lenet" else ():
        for k in a:
            ta, tb = a[k], b[k]
            for u, v in (zip(ta, tb) if isinstance(ta, list) else [(ta, tb)]):
                if isinstance(u, torch.Tensor):
                    assert torch.equal(u.contiguous().view(torch.uint8), v.contiguous().view(torch.uint8)), k
                else:
                    assert u == v, k
    st = eng.ssp_stats()
    assert st["clock"] == 6 and st["waits"] == 0 and st["lead_max"] == 0 and st["wait_total_ns"] == 0
    assert st["pairs"].tolist() == [[c, RETIRED] for c in range(6)]       # no peer
    assert eng.async_finish() == plain.async_finish() == STEP0 + 6
    if model == "lenet":
        assert torch.equal(eng.params.view(torch.int32), plain.params.view(torch.int32))


# ---- 2. and 3. N replicas on one GPU ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def replica_cases(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("ssp") / "cases.json")
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    r = subprocess.run([sys.executable, os.path.join(HERE, "_ssp_replicas_worker.py"), out], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
    with open(out) as f:
        return json.load(f)


def _case(cases, n, s, iters):
    return next(c for c in cases if c["n"] == n and c["s"] == s and c["iters"] == iters)


def _check_bounds(c):
    """B1, B2 and B3 at every pull and update, the permutation of the tickets and the exact final copies; returns each
    replica's bound statistics."""
    n, s, iters = c["n"], c["s"], c["iters"]
    assert c["errors"] == [0] * n
    tickets = []
    for q in range(n):
        pulled = np.array(c["pulled"][q])                       # [iteration, replica]: updates held by the pull
        ssp = c["ssp"][q]
        assert ssp["clock"] == iters[q] and ssp["lead_max"] <= s
        pairs = np.array(ssp["pairs"], dtype=np.int64)
        assert pairs[:, 0].tolist() == list(range(iters[q]))
        for j in range(iters[q]):
            assert pulled[j, q] == j, (q, j)                    # B1: all of my own updates
            lo = int(pairs[j, 1])
            for p in range(n):
                if p != q:                                      # B1: c - s of a running peer, all of a retired one
                    assert pulled[j, p] >= min(j - s, iters[p]), (q, j, p, pulled[j].tolist())
            if lo != RETIRED:
                assert j - lo <= s, (q, j, lo)                  # B2
        a = c["async"][q]
        assert a["updates"] == iters[q]
        rs = np.array(a["pairs"], dtype=np.int64)
        assert ((rs[:, 1] - rs[:, 0]) <= (n - 1) * (2 * s + 1)).all(), rs.tolist()      # B3
        tickets += rs[:, 1].tolist()
    assert sorted(tickets) == list(range(sum(iters)))
    for q in range(n):
        assert c["master"][q] == [float(u) for u in iters]      # every update in every copy, exactly
        assert c["boards"][q] == [RETIRED] * n                  # every replica retired
    return c["ssp"]


@pytest.mark.parametrize("s", [0, 1, 4])
@pytest.mark.parametrize("n", [2, 4, 8])
def test_replicas_on_one_gpu_keep_the_bound(replica_cases, n, s):
    ssp = _check_bounds(_case(replica_cases, n, s, [24] * n))
    fast = ssp[:n - 1]
    assert any(b["lead_max"] == s for b in fast), [b["lead_max"] for b in ssp]      # the wait is not over-conservative
    assert all(b["waits"] > 0 and b["wait_total_ns"] > 0 for b in fast), [b["waits"] for b in ssp]


@pytest.mark.parametrize("s,iters", [(0, [12, 24, 24, 24]), (1, [24, 24, 24, 12])])
def test_a_retired_replica_blocks_nobody(replica_cases, s, iters):
    _check_bounds(_case(replica_cases, 4, s, iters))


# ---- 4. train(), one replica --------------------------------------------------------------------------------------------
@pytest.fixture
def one_replica(monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)


def test_train_with_evaluation_target_and_device_data(tmp_path, one_replica, capsys):
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200 import evaluator
    from distributedmnist_b200.checkpoint import Saver
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import train
    d = str(tmp_path / "run")
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % d, "--batch_size=128", "--max_steps=120", "--eval_every_steps=20", "--async_method",
                 "--ssp_staleness=0", "--save_interval_secs=1000", "--log_every=20", "--target_accuracy=0.999",
                 "--device_data"])
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True, synthetic_sizes=(8192, 2048))
    try:
        res = train(init_context(FLAGS), ds.train, ds.validation, FLAGS)
    finally:
        FLAGS.reset()
    T = res["final_step"]
    assert 121 <= T <= 122 or res["time_to_accuracy"]["reached"]
    rep = res["ssp"]
    assert rep == dict(s=0, waits=0, wait_total_ns=0, wait_max_ns=0, lead_max=0, updates=T)
    assert res["staleness"]["updates"] == T and res["staleness"]["max"] == 0
    with open(os.path.join(d, "worker0_ssp.json")) as f:
        assert json.load(f) == rep
    evals = res["evals"]
    assert [int(r[0]) for r in evals][:6] == [20, 40, 60, 80, 100, 120] and int(evals[-1][0]) == T
    state, step = Saver.restore(Saver.latest(d))
    assert step == T
    capsys.readouterr()
    FLAGS.parse(["--checkpoint_dir=%s" % d, "--eval_dir=%s" % str(tmp_path / "eval"), "--run_once=true"])
    try:
        assert int(evaluator.evaluate(ds.validation, FLAGS, torch.device("cuda", 0), max_evals=1)) == T
    finally:
        FLAGS.reset()
    m = re.search(r"Num examples: 2048  Precision @ 1: ([0-9.]+) Loss", capsys.readouterr().out)
    assert m and round(float(m.group(1)) * 2048) == int(evals[-1][4])


# ---- 5. several GPUs (tests/_ssp_worker.py) ---------------------------------------------------------------------------
@pytest.mark.multigpu
@pytest.mark.parametrize("nvls", [False, True], ids=["p2p", "nvls"])
def test_multi_gpu_train_with_a_straggler(tmp_path, nvls):
    from distributedmnist_b200.parallel.launcher import run_replicas
    n = min(torch.cuda.device_count(), 8)
    if n < 2:
        pytest.skip("needs 2 GPUs")
    if nvls and n < 4:
        pytest.skip("the NVLS case needs 4 GPUs")
    s = 2
    os.environ["DMNIST_NVLS"] = "1" if nvls else "0"       # inherited by the helper processes
    try:
        codes = run_replicas([os.path.join(HERE, "_ssp_worker.py"), str(tmp_path / "train"), str(tmp_path / "res_RANK.json"),
                              "400", "%d:1.0:2000" % (n - 1), str(s)], n, timeout=600, out_dir=str(tmp_path / "out"))
    finally:
        os.environ.pop("DMNIST_NVLS")
    logs = "\n".join(open(os.path.join(tmp_path, "out", f)).read()[-1500:] for f in sorted(os.listdir(tmp_path / "out")))
    assert codes == [0] * n, logs
    res = [json.load(open(tmp_path / ("res_%d.json" % r))) for r in range(n)]
    T = res[0]["final_step"]
    assert all(r["final_step"] == T for r in res)
    assert len({r["params"] for r in res}) == 1 and len({r["master"] for r in res}) == 1
    assert res[0]["params"] == res[0]["master"]
    assert sum(r["updates"] for r in res) == T
    assert all(r["nvls"] == nvls for r in res)
    assert all(r["lead_max"] <= s for r in res), [r["lead_max"] for r in res]
    assert all(r["max_tau"] <= (n - 1) * (2 * s + 1) for r in res), [r["max_tau"] for r in res]
    u = [r["updates"] for r in res]
    assert max(u) - min(u) <= s + 3, u                  # DESIGN.md §4: the bound plus the end-of-run slack
    assert all(r["waits"] > 0 for r in res[:n - 1]), [r["waits"] for r in res]
