"""Asynchronous SGD (``--async_method``, csrc/fused_async.cu) on one H100.

1. The kernels on one replica, bit for bit against ``ops/aggrefs.py`` over the whole LeNet arena after every apply: the
   master copy, the pulled working arena and its bf16 shadow, the tickets, and the rate under the staircase, warmup and
   cosine schedules.
2. N = 2, 4 and 8 replicas on one GPU in one process: N control blocks, master copies and working arenas as plain device
   allocations, the peer path, begin / end sequences interleaved on N concurrent streams.  This is safe only because no
   async kernel waits on a word another replica writes.
3. Engine steps on one replica, graph-replayed back to back, stage by stage against float64 and the update bit for bit
   (ops/trajectory.py, mode "async"), for LeNet and mlp3.
4. ``train()`` on one replica with the in-training evaluation, a target, the device-resident training set and
   augmentation, and a restart from a mid-run checkpoint; the standalone evaluator reproduces the last pass's count on the
   final checkpoint.
5. The NVLS branch of the apply on one GPU: the master copy behind a one-device multicast object, every update reduced
   through the multicast address and pulled back through the unicast one on the same stream, bit for bit.
6. Several GPUs (tests/_async_worker.py, skipped below 2 GPUs, the NVLS case below 4): ``train()`` on every replica with a
   straggler -- every master copy and working arena identical after the end barrier, the replicas' updates summing to
   the final step, the straggler applying fewer updates while the others keep their pace."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

STEP0 = 3001


def _lib():
    from distributedmnist_b200.ops.lib import load
    return load()


def _table(ptrs):
    return (ctypes.c_void_p * 8)(*([int(p) for p in ptrs] + [int(ptrs[0])] * (8 - len(ptrs))))


# ---- 1. kernels, one replica -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sched", ["staircase", "warmup", "cosine"])
def test_kernels_one_replica_bit_for_bit(sched):
    from distributedmnist_b200.models import get_model
    from distributedmnist_b200.ops import aggrefs as A
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    spec, _ = get_model("lenet")
    n = spec.arena_numel
    params = be.allocate(n)
    params.copy_(spec.init_flat(7).cuda())
    master = be.allocate(n)
    be.attach_shadow(params)
    stats = torch.zeros(int(_lib().dm_async_stats_bytes()), dtype=torch.uint8, device="cuda")
    if sched == "staircase":
        s = LearningRateSchedule(0.05, STEP0 + 2, 0.5)     # halves from the third step on
    elif sched == "warmup":
        s = LearningRateSchedule(0.05, 1, 1.0, warmup_steps=STEP0 + 3, warmup_start=0.25)
    else:
        s = LearningRateSchedule(0.05, 1, 1.0, warmup_steps=STEP0 + 2, warmup_start=0.1, cosine_steps=STEP0 + 4,
                                 cosine_alpha=0.05)
    be.set_lr_schedule(s.warmup_steps, s.warmup_start, s.cosine_steps, getattr(s, "cosine_alpha", 0.0))
    be.set_global_step(STEP0)
    be.async_arm(master, params, stats)
    gen = torch.Generator(device="cuda").manual_seed(3)
    w = A.f32(master)
    for j in range(6):
        be.enqueue_async_begin(master, params)
        torch.cuda.synchronize()
        assert A.bits(params).tolist() == A.bits(w).tolist()
        assert (be.shadow.view(torch.int16).cpu().numpy().view("<u2") == A.bf16_bits(w)).all()
        assert be.device_epoch == STEP0 + j
        g = torch.randn(n, generator=gen, device="cuda") * 0.5
        be.enqueue_async_end(master, g, stats, s.initial_learning_rate, s.decay_rate, s.decay_steps)
        torch.cuda.synchronize()
        scale = A.step_scale(s, STEP0 + j, 1)
        w = A.async_apply(w, [A.async_update(A.f32(g), scale)])
        got = A.bits(master)
        assert (got != A.bits(w)).sum() == 0, (j, int((got != A.bits(w)).sum()))
        info = be.mirror_info(j + 1)
        assert info.global_step == STEP0 + j + 1 and info.accepted and info.count == 1
    st = be.async_stats(stats)
    assert st["updates"] == 6 and st["hist"][0] == 6 and st["tau_sum"] == 0 and st["tau_max"] == 0
    assert st["pairs"].tolist() == [[STEP0 + j, STEP0 + j] for j in range(6)]
    be.check_error()
    be.close()


# ---- 5. the NVLS branch on one GPU ----------------------------------------------------------------------------------------
def _one_device_multicast(nbytes):
    """(unicast pointer, multicast pointer) of a VMM allocation bound to a multicast object of this one device; skips when
    the device or the fabric offers no multicast."""
    lib = _lib()
    if int(lib.dm_vmm_multicast_supported(0)) != 1:
        pytest.skip("the device has no multicast (NVLS) support")
    size = int(lib.dm_vmm_round_size(nbytes, 0, 1))
    assert size >= nbytes
    h, fd, p = ctypes.c_ulonglong(), ctypes.c_int(-1), ctypes.c_void_p()
    assert lib.dm_vmm_create(size, 0, ctypes.byref(h), ctypes.byref(fd), ctypes.byref(p)) == 0
    lib.dm_close_fd(fd.value)
    mch, mcfd = ctypes.c_ulonglong(), ctypes.c_int(-1)
    if lib.dm_mc_create(size, 1, ctypes.byref(mch), ctypes.byref(mcfd)) != 0:
        pytest.skip("no multicast object over one device on this fabric")
    lib.dm_close_fd(mcfd.value)
    assert lib.dm_mc_add_device(mch, 0) == 0
    assert lib.dm_mc_bind(mch, h, size) == 0
    mp = ctypes.c_void_p()
    assert lib.dm_vmm_map(mch, size, 0, ctypes.byref(mp)) == 0
    return int(p.value), int(mp.value)


def test_nvls_apply_is_visible_to_the_next_pull():
    """Back-to-back iterations on one stream, nothing synchronised in between: each pull reads through the unicast address
    the update the previous apply reduced through the multicast address."""
    from distributedmnist_b200.ops import aggrefs as A
    lib = _lib()
    numel, U = 1 << 20, 12
    uni, mc = _one_device_multicast(numel * 4)
    gen = torch.Generator(device="cuda").manual_seed(11)
    lib.dm_memset_async(uni, 0, numel * 4, None)     # the master copy starts at zero
    ctrl = torch.zeros(int(lib.dm_sync_ctrl_bytes()), dtype=torch.uint8, device="cuda")
    stats = torch.zeros(int(lib.dm_async_stats_bytes()), dtype=torch.uint8, device="cuda")
    params = torch.zeros(numel, device="cuda")
    grads = [torch.randn(numel, generator=gen, device="cuda") for _ in range(U)]
    pulled = []
    ct, mt = _table([ctrl.data_ptr()]), _table([uni])
    sp = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for j in range(U):
        lib.dm_async_begin(ct, 0, ctypes.c_void_p(uni), params, None, numel, 0, sp)
        pulled.append(params.clone())
        lib.dm_async_end(ct, mt, grads[j], stats, 0, 1, numel, 0.01, 1.0, 1, 0, sp, ctypes.c_void_p(mc))
    lib.dm_async_begin(ct, 0, ctypes.c_void_p(uni), params, None, numel, 0, sp)
    pulled.append(params.clone())
    torch.cuda.synchronize()
    w = np.zeros(numel, np.float32)
    scale = A.step_scale(lambda s: 0.01, 0, 1)
    for j in range(U + 1):
        assert (A.bits(pulled[j]) != A.bits(w)).sum() == 0, j
        if j < U:
            w = A.async_apply(w, [A.async_update(A.f32(grads[j]), scale)])


# ---- 2. N replicas on one GPU ---------------------------------------------------------------------------------------------
class _Replicas:
    """N replicas' control blocks, master copies, working arenas and staleness buffers in plain device memory of one GPU."""

    def __init__(self, nranks, numel, init):
        lib = _lib()
        self.lib, self.n, self.numel = lib, nranks, numel
        self.ctrl = [torch.zeros(int(lib.dm_sync_ctrl_bytes()), dtype=torch.uint8, device="cuda") for _ in range(nranks)]
        self.master = [init.clone() for _ in range(nranks)]
        self.params = [torch.zeros_like(init) for _ in range(nranks)]
        self.stats = [torch.zeros(int(lib.dm_async_stats_bytes()), dtype=torch.uint8, device="cuda") for _ in range(nranks)]
        self.streams = [torch.cuda.Stream() for _ in range(nranks)]
        self.ct = _table([c.data_ptr() for c in self.ctrl])
        self.mt = _table([m.data_ptr() for m in self.master])

    def begin(self, q):
        self.lib.dm_async_begin(self.ct, q, self.master[q], self.params[q], None, self.numel, 16,
                                ctypes.c_void_p(self.streams[q].cuda_stream))

    def end(self, q, g, lr0):
        self.lib.dm_async_end(self.ct, self.mt, g, self.stats[q], q, self.n, self.numel, lr0, 1.0, 1, 16,
                              ctypes.c_void_p(self.streams[q].cuda_stream), None)

    def run(self, grads, lr0):
        """grads[q][j]: replica q's j-th gradient; every replica's iterations enqueued round robin on its own stream."""
        torch.cuda.synchronize()
        for j in range(len(grads[0])):
            for q in range(self.n):
                self.begin(q)
                self.end(q, grads[q][j], lr0)
        torch.cuda.synchronize()
        for q in range(self.n):
            self.begin(q)                  # the final pull
        torch.cuda.synchronize()

    def stats_of(self, q):
        from distributedmnist_b200.parallel.fused import FusedBackend
        return FusedBackend.async_stats(self.stats[q])

    def counter(self):
        from distributedmnist_b200.parallel.fused import FusedBackend
        off = int(self.lib.dm_sync_ctrl_offset(b"global_step"))
        return int(self.ctrl[0][off:off + 4].view(torch.int32).item())


def _check_protocol(R, U):
    T = R.n * U
    assert R.counter() == T
    tickets = []
    for q in range(R.n):
        st = R.stats_of(q)
        assert st["updates"] == U
        pairs = st["pairs"]
        tickets += pairs[:, 1].tolist()
        tau = pairs[:, 1] - pairs[:, 0]
        assert (tau >= 0).all()
        hist = np.bincount(np.minimum(tau, 63), minlength=64).tolist()
        assert st["hist"] == hist and st["tau_sum"] == int(tau.sum()) and st["tau_max"] == int(tau.max())
        assert (np.diff(pairs[:, 1]) > 0).all() and (np.diff(pairs[:, 0]) >= 0).all()
    assert sorted(tickets) == list(range(T))
    return tickets


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_replicas_on_one_gpu_exact(nranks):
    """Integer weights and gradients with a rate of 2^-3: every product and sum is exact in fp32, so every master copy is
    init - sum of all updates bit for bit, whatever order the reductions landed in."""
    from distributedmnist_b200.ops import aggrefs as A
    numel, U = 1 << 16, 24
    gen = torch.Generator(device="cuda").manual_seed(nranks)
    init = torch.randint(-64, 64, (numel,), generator=gen, device="cuda").float()
    grads = [[torch.randint(-32, 33, (numel,), generator=gen, device="cuda").float() for _ in range(U)]
             for _ in range(nranks)]
    R = _Replicas(nranks, numel, init)
    R.run(grads, 0.125)
    _check_protocol(R, U)
    want = A.f32(init).astype(np.float64) - 0.125 * sum(A.f32(g).astype(np.float64) for gq in grads for g in gq)
    for q in range(nranks):
        assert A.bits(R.master[q]).tolist() == A.bits(want.astype(np.float32)).tolist(), q
        assert torch.equal(R.params[q], R.master[q])


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_replicas_on_one_gpu_random(nranks):
    """Random data: every copy agrees with the float64 sum of the (exactly emulated) updates within T half-ulps of the
    largest magnitude a partial sum can reach, T the number of adds whose order the replicas decide."""
    from distributedmnist_b200.ops import aggrefs as A
    numel, U, lr = 1 << 16, 16, 0.01
    gen = torch.Generator(device="cuda").manual_seed(100 + nranks)
    init = torch.randn(numel, generator=gen, device="cuda") * 0.1
    grads = [[torch.randn(numel, generator=gen, device="cuda") for _ in range(U)] for _ in range(nranks)]
    R = _Replicas(nranks, numel, init)
    R.run(grads, lr)
    _check_protocol(R, U)
    scale = A.step_scale(lambda s: lr, 0, 1)
    xs = [A.async_update(A.f32(g), scale).astype(np.float64) for gq in grads for g in gq]
    exact = A.f32(init).astype(np.float64) + sum(xs)
    top = np.abs(A.f32(init)).astype(np.float64) + sum(np.abs(x) for x in xs)
    bound = len(xs) * 0.5 * np.spacing(top.astype(np.float32)).astype(np.float64)
    for q in range(nranks):
        got = A.f32(R.master[q]).astype(np.float64)
        assert np.all(np.abs(got - exact) <= bound), q


# ---- 3. engine steps, one replica ---------------------------------------------------------------------------------------
def _engine(model, B):
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
    eng.attach_optimizer(AsyncSGDOptimizer(be, sched, 1))
    assert eng._async and not eng._bucketed and not eng._interval
    be.set_global_step(STEP0)
    return eng, be, sched, StepRecorder(eng)


@pytest.mark.parametrize("model,B", [("lenet", 256), ("mlp3", 512)])
def test_engine_steps_stage_by_stage(model, B):
    from distributedmnist_b200.ops import trajectory as T
    eng, be, sched, rec = _engine(model, B)
    gen = torch.Generator().manual_seed(9)
    shape = (B, 28, 28) if model == "lenet" else (B, 784)
    batches = [(torch.rand(*shape, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen)) for _ in range(6)]
    for x, y in batches:
        eng.load_batch(x.numpy(), y.numpy())
        eng.train_step()
        rec.record()
    torch.cuda.synchronize()
    be.check_error()
    assert be.device_epoch == STEP0 + 5                 # the epoch word is the counter the last pull read
    assert eng.launches_per_step > 0
    upd = T.update_of(eng, sched, STEP0)
    assert upd["mode"] == "async"
    if model == "lenet":
        res = T.lenet_trajectory_results(model, eng.spec, rec.init, rec.records, batches, upd, eng.seed, eng.rank,
                                         eng.keep_prob, 0.0)
    else:
        res = T.mlp_trajectory_results(model, eng.spec, rec.init, rec.records, batches, upd)
    print("\nTRAJECTORY async.%s %s" % (model, json.dumps(T.worst_by_stage(model, res), sort_keys=True)))
    bad = T.failures(res)
    assert not bad, "%d of %d checks failed, first: %s" % (len(bad), len(res), bad[:20])
    assert eng.async_finish() == STEP0 + 6
    st = eng.async_staleness()
    assert st["updates"] == 6 and st["hist"][0] == 6


# ---- 4. train(), one replica --------------------------------------------------------------------------------------------
def _train(d, *extra, steps=120):
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import train
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % d, "--batch_size=128", "--max_steps=%d" % steps, "--eval_every_steps=20",
                 "--async_method", "--save_interval_secs=1000", "--log_every=20"] + list(extra))
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
    res = _train(d, "--target_accuracy=0.999", "--device_data", "--augment_max_shift=1.5", "--augment_max_rotation=8")
    st = res["staleness"]
    T = res["final_step"]
    assert st["updates"] == T and st["hist"][0] == T and st["max"] == 0
    assert 121 <= T <= 122 or res["time_to_accuracy"]["reached"]   # max_steps + 1, and at most one more in flight
    assert res["accepted"] == T and res["dropped"] == 0
    with open(os.path.join(d, "worker0_staleness.json")) as f:
        assert json.load(f) == st
    evals = res["evals"]
    steps = [int(r[0]) for r in evals]
    assert steps[:6] == [20, 40, 60, 80, 100, 120] and steps[-1] == T
    assert "time_to_accuracy" in res
    # the final checkpoint holds the weights of the final pass: a standalone pass over it reproduces the pass's count
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    state, step = Saver.restore(Saver.latest(d))
    assert step == T
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaLeNetEngine(128, be, use_graph=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True, synthetic_sizes=(8192, 2048))
    eng.arm_eval(ds.validation.images, ds.validation.labels)
    eng.params.copy_(eng.spec.from_state_dict(state).cuda())
    eng.params_updated()
    be.set_global_step(T)
    rec = eng.run_eval()
    assert rec[0] == T and rec[4] == int(evals[-1][4]) and rec[3] == 2048
    # ... and so does the polling evaluator (evaluator.py, as src/mnist_eval.py runs it) on the checkpoint directory
    from distributedmnist_b200 import evaluator
    capsys.readouterr()
    FLAGS.reset()
    FLAGS.parse(["--checkpoint_dir=%s" % d, "--eval_dir=%s" % str(tmp_path / "eval"), "--run_once=true"])
    try:
        assert int(evaluator.evaluate(ds.validation, FLAGS, torch.device("cuda", 0), max_evals=1)) == T
    finally:
        FLAGS.reset()
    m = re.search(r"Num examples: 2048  Precision @ 1: ([0-9.]+) Loss", capsys.readouterr().out)
    assert m and round(float(m.group(1)) * 2048) == int(evals[-1][4])


def test_train_restart_continues_the_counter(tmp_path, one_replica):
    from distributedmnist_b200.checkpoint import Saver
    d = str(tmp_path / "run")
    first = _train(d, steps=40)
    T1 = first["final_step"]
    second = _train(d, steps=90)
    T2 = second["final_step"]
    assert 91 <= T2 <= 92
    assert second["staleness"]["updates"] == T2 - T1     # the counter continued from the restored step
    assert second["steps"][0] == T1 + 1
    assert Saver.restore(Saver.latest(d))[1] == T2


# ---- 6. several GPUs (tests/_async_worker.py) ---------------------------------------------------------------------------
@pytest.mark.multigpu
@pytest.mark.parametrize("nvls", [False, True], ids=["p2p", "nvls"])
def test_multi_gpu_train_with_a_straggler(tmp_path, nvls):
    from distributedmnist_b200.parallel.launcher import run_replicas
    n = min(torch.cuda.device_count(), 8)
    if nvls and n < 4:
        pytest.skip("the NVLS case needs 4 GPUs")
    here = os.path.dirname(os.path.abspath(__file__))
    os.environ["DMNIST_NVLS"] = "1" if nvls else "0"       # inherited by the helper processes
    try:
        codes = run_replicas([os.path.join(here, "_async_worker.py"), str(tmp_path / "train"), str(tmp_path / "res_RANK.json"),
                              "400", "%d:1.0:2000" % (n - 1)], n, timeout=600, out_dir=str(tmp_path / "out"))
    finally:
        os.environ.pop("DMNIST_NVLS")
    logs = "\n".join(open(os.path.join(tmp_path, "out", f)).read()[-1500:] for f in sorted(os.listdir(tmp_path / "out")))
    assert codes == [0] * n, logs
    res = [json.load(open(tmp_path / ("res_%d.json" % r))) for r in range(n)]
    T = res[0]["final_step"]
    assert all(r["final_step"] == T for r in res)
    assert len({r["params"] for r in res}) == 1 and len({r["master"] for r in res}) == 1
    assert res[0]["params"] == res[0]["master"]
    assert sum(r["updates"] for r in res) == T                     # every ticket is one replica's update
    assert 401 <= T <= 400 + 2 * n
    assert all(r["nvls"] == nvls for r in res)
    slow, fast = res[n - 1], res[:n - 1]
    assert all(4 * slow["updates"] < f["updates"] for f in fast), [r["updates"] for r in res]
    assert slow["max_tau"] >= 1                                    # the straggler's updates are stale
