"""Learning-rate warmup and cosine decay on the GPU: the step size every aggregation kernel evaluates from its control
block, bit for bit against the host schedule (single kernel, bucketed kernels, interval and K > N applies, with and
without a cut table); graph-replayed LeNet and MLP steps bit for bit against the exact emulation; back-to-back LeNet
steps stage by stage against the float64 references; runs through ``train()`` in every mode with a restart mid-warmup;
and two replicas staying bit-identical."""
import importlib.util
import json
import logging
import os
import re

import numpy as np
import pytest
import torch

from distributedmnist_b200 import lr_plateau as lp
from distributedmnist_b200.ops import aggrefs as A
from distributedmnist_b200.schedule import LearningRateSchedule

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

# (lr0, decay_steps, decay_rate, W, f0, T, alpha)
SHAPES = {
    "warmup": (0.05, 1, 0.999, 100, 1.0 / 3, 0, 0.0),
    "cosine": (0.05, 1, 0.999, 0, 1.0 / 3, 1000, 0.0),
    "both": (0.1, 7, 0.95, 64, 0.1, 5000, 0.01),
    "short": (0.4, 1, 0.999, 3, 0.0, 10, 0.5),
}


def _sched(shape, factor=1.0, cuts=()):
    lr0, ds, rate, w, f0, t, alpha = SHAPES[shape]
    return LearningRateSchedule(lr0, ds, rate, factor=factor, cuts=cuts, warmup_steps=w, warmup_start=f0, cosine_steps=t,
                                cosine_alpha=alpha)


def probe_steps(shape):
    """Steps across the warmup, the cosine, its end and past it, increasing."""
    _lr0, _ds, _rate, w, _f0, t, _alpha = SHAPES[shape]
    s = {0, 1, 2, 77777}
    for x in (w - 1, w, w + 1, t // 3, t // 2, t - 2, t - 1, t, t + 1, 2 * t):
        if x >= 0:
            s.add(x)
    return sorted(s)


def cut_table_for(shape):
    _lr0, _ds, _rate, w, _f0, t, _alpha = SHAPES[shape]
    return sorted({1, max(w, 2), max(t // 2, 3)})


def _backend():
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    return FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))


def _table(cuts):
    words = np.full(lp.MAX_CUTS, lp.NO_CUT, dtype=np.uint32)
    words[:len(cuts)] = cuts
    return torch.from_numpy(words.view(np.int32)).cuda()


def _arm(be, sched):
    be.set_lr_schedule(sched.warmup_steps, sched.warmup_start, sched.cosine_steps, sched.cosine_alpha)


def _judge(sched, probes, got, count=1):
    """``got[i]``: the device step size at ``probes[i]`` with ``count`` gradients (fp32 values)."""
    checked, wrong = 0, []
    for s, x in zip(probes, got):
        host = sched(s) / count
        if host < A.FLT_MIN:
            assert x == 0.0, (s, x, host)
            continue
        # the device's double sin and pow may differ from the host's by a few double ulps: that never matters this far
        # from a rounding boundary
        assert A.midpoint_distance_ulps(host) > 16, (s, host)
        checked += 1
        if np.float32(x) != np.float32(host):
            wrong.append((s, x, float(np.float32(host))))
    assert not wrong, "%d of %d step sizes differ from the host schedule: %s" % (len(wrong), checked, wrong[:8])
    return checked


# ---- the step size of every aggregation kernel -------------------------------------------------------------------------
@pytest.mark.parametrize("cuts", [False, True])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_single_kernel_step_size_equals_host_schedule(shape, cuts):
    """fused_sync_sgd with weights 0 and gradients 1.0: the new weight is -scale exactly."""
    from distributedmnist_b200.ops.lib import load
    lib = load()
    table = cut_table_for(shape) if cuts else []
    sched = _sched(shape, 0.5, table)
    be = _backend()
    try:
        params, grads = be.allocate(1024), be.allocate(1024)
        grads.fill_(1.0)
        if cuts:
            t = _table(table)
            lib.dm_sync_set_lr_cuts(be.ctrl.local_ptr, t, 0.5)
        _arm(be, sched)
        got = []
        for s in probe_steps(shape):
            params.zero_()
            be.set_global_step(s)
            be.enqueue(params, grads, 1, sched.initial_learning_rate, sched.decay_rate, sched.decay_steps)
            got.append(-params[0].item())
        be.check_error()
        assert _judge(sched, probe_steps(shape), got) >= 6
        # disarmed again: the staircase alone
        be.set_lr_schedule(0, 1.0 / 3, 0, 0.0)
        lib.dm_sync_set_lr_cuts(be.ctrl.local_ptr, None, 0.0)
        params.zero_()
        be.set_global_step(5)
        be.enqueue(params, grads, 1, sched.initial_learning_rate, sched.decay_rate, sched.decay_steps)
        plain = LearningRateSchedule(sched.initial_learning_rate, sched.decay_steps, sched.decay_rate)
        assert np.float32(-params[0].item()) == np.float32(plain(5))
    finally:
        be.close()


@pytest.mark.parametrize("cuts", [False, True])
@pytest.mark.parametrize("shape", ["both", "short"])
def test_bucket_kernels_step_size_equals_host_schedule(shape, cuts):
    """The bf16-wire bucketed kernels (csrc/fused_bucket.cu) on one replica, lenet's layout: every weight of the early
    (fc1) and of the late bucket is -scale."""
    from distributedmnist_b200.models.lenet import lenet_spec
    from distributedmnist_b200.ops.lib import load
    lib = load()
    spec = lenet_spec()
    q = [p for p in spec.params if p.name == "fc1_weights"][0]
    b, e = q.offset, q.offset + q.numel
    n = spec.arena_numel
    table = cut_table_for(shape) if cuts else []
    sched = _sched(shape, 0.5, table)
    be = _backend()
    try:
        params, grads = be.allocate(n), be.allocate(n)
        g16 = be.allocate_buffer((e - b) * 2)
        grads.fill_(1.0)
        g16.view(torch.bfloat16, 0, e - b).fill_(1.0)
        be.attach_shadow(params)
        if cuts:
            t = _table(table)
            lib.dm_sync_set_lr_cuts(be.ctrl.local_ptr, t, 0.5)
        _arm(be, sched)
        got = []
        for s in probe_steps(shape):
            params.zero_()
            be.set_global_step(s)
            for phase in (1, 2):
                be.enqueue_bucket_v2(params, grads, g16, None, phase, b, e, sched.initial_learning_rate,
                                     sched.decay_rate, sched.decay_steps)
            w = params.cpu()
            assert float(w[b]) == float(w[0]) == float(w[n - 1]), s
            got.append(-float(w[0]))
        be.check_error()
        assert _judge(sched, probe_steps(shape), got) >= 8
    finally:
        be.close()


@pytest.mark.parametrize("mode", ["interval", "kgtn"])
@pytest.mark.parametrize("shape", ["both", "short"])
def test_interval_and_kgtn_apply_step_size_equals_host_schedule(shape, mode):
    """iv_apply_kernel reads the schedule from its own control block (no cut table in interval mode or with K > N).
    Interval: a 1 us tick commits every iteration, one gradient.  K = 2 > N = 1: two iterations commit a step of two
    gradients, each 1.0, so the new weight is -2 * fp32(lr / 2) = -2 * scale exactly."""
    sched = _sched(shape)
    n = 4096
    count = 1 if mode == "interval" else 2
    be = _backend()
    try:
        params, grads, acc = be.allocate(n), be.allocate(n), be.allocate(n)
        grads.fill_(1.0)
        be.attach_shadow(params)
        _arm(be, sched)
        args = (sched.initial_learning_rate, sched.decay_rate, sched.decay_steps)
        got = []
        for s in probe_steps(shape):        # increasing: no commit word of an earlier probe names a later step
            params.zero_()
            be.set_global_step(s)
            if mode == "interval":
                be.interval_arm(0.001)
                be.enqueue_interval_begin(params)
                be.enqueue_interval_end(params, grads, acc, *args)
                be.enqueue_interval_begin(params)
            else:
                be.kgtn_arm()
                for _ in range(2):
                    be.enqueue_kgtn_begin(params)
                    be.enqueue_kgtn_end(params, grads, acc, 2, *args)
                be.enqueue_kgtn_begin(params)
            torch.cuda.synchronize()
            st = be.read_status()
            assert st["epoch"] == s + 1, (s, st)
            got.append(-params[0].item() / count)
        be.check_error()
        assert _judge(sched, probe_steps(shape), got, count) >= 8
    finally:
        be.close()


def test_armed_block_refuses_host_evaluated_rates():
    be = _backend()
    try:
        params, grads = be.allocate(1024), be.allocate(1024)
        _arm(be, _sched("short"))
        with pytest.raises(RuntimeError, match="host evaluated"):
            be.sync_step(params, grads, 0.1, 0, 1)
        with pytest.raises(RuntimeError, match="host evaluated"):
            be.interval_tick(params, grads, 1, 0.1, 0)
        with pytest.raises(Exception):
            be.lib.dm_sync_set_lr_schedule(be.ctrl.local_ptr, 3, 1.0, 0, 0.0)      # f0 = 1 is refused
        with pytest.raises(Exception):
            be.lib.dm_sync_set_lr_schedule(be.ctrl.local_ptr, 0, 0.5, 2 ** 32 - 1, 0.0)
    finally:
        be.close()


# ---- graph-replayed engine steps against the exact emulation -----------------------------------------------------------
ENGINE_SCHED = dict(warmup_steps=2, warmup_start=0.25, cosine_steps=4, cosine_alpha=0.1)


def _engine_steps(make_engine, bucket, monkeypatch, alpha, steps=6):
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    monkeypatch.setenv("DMNIST_BUCKET", bucket)
    be = _backend()
    eng = make_engine(be)
    sched = LearningRateSchedule(0.05, 2, 0.999, **dict(ENGINE_SCHED, cosine_alpha=alpha))
    eng.attach_optimizer(SyncReplicasOptimizer(be, sched, 1, 1))
    assert be.lr_schedule_armed
    be.set_global_step(0)
    gen = torch.Generator().manual_seed(9)
    B, n = eng.batch_size, eng.spec.arena_numel
    b, e = eng._bucket_early
    rounds = A.late_bucket_rounds_bf16(n, e - b, be.late_ll, be.late_bf16)
    shape = (B, 28, 28) if hasattr(eng, "h_part") else (B, 784)
    for s in range(steps):
        torch.cuda.synchronize()
        step = be.device_epoch
        assert step == s
        w = A.f32(eng.params)
        eng.load_batch(torch.rand(*shape, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen))
        eng.train_step()
        torch.cuda.synchronize()
        scale = A.step_scale(sched, step, 1)
        if scale != 0:
            assert A.midpoint_distance_ulps(sched(step)) > 16, step
        grads = A.f32(eng.grads)
        if eng._bucket_v2:
            want = A.bucket_step(w, [grads], [A.f32(eng._g16_view.float()).reshape(-1)], (b, e), scale, rounds)
        else:
            want = A.fused_sync_step(w, [grads], 1, scale)
        got = A.bits(eng.params)
        bad = np.flatnonzero(got != A.bits(want))
        assert bad.size == 0, "bucket=%s step %d: %d weights differ" % (bucket, step, bad.size)
        sh = eng.shadow.view(torch.int16).cpu().numpy().view(np.uint16)
        assert (sh == A.bf16_bits(want)).all(), "bucket=%s step %d: shadow" % (bucket, step)
        if step >= 4 and alpha == 0.0:
            assert (got == A.bits(w)).all(), "alpha = 0: the weights stop at step T"
    be.check_error()


@pytest.mark.parametrize("bucket", ["2", "1", "0"])
def test_lenet_engine_steps_are_bit_exact(bucket, monkeypatch):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    _engine_steps(lambda be: CudaLeNetEngine(128, be, seed=3, rank=0, use_graph=True), bucket, monkeypatch, 0.1)


@pytest.mark.parametrize("bucket", ["2", "0"])
def test_mlp_engine_steps_are_bit_exact_and_stop_at_t(bucket, monkeypatch):
    from distributedmnist_b200.engine_cuda import CudaMlpEngine
    _engine_steps(lambda be: CudaMlpEngine("mlp3", 128, be, hidden=1024, seed=3, use_graph=True), bucket, monkeypatch,
                  0.0)


# ---- back-to-back steps against float64, through ops/trajectory.py ------------------------------------------------------
def _trajectory_module():
    spec = importlib.util.spec_from_file_location("_lr_traj", os.path.join(HERE, "test_step_trajectory_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("bucket", ["2", "0"])
def test_lenet_trajectory_with_warmup_and_cosine(bucket, monkeypatch):
    """Six back-to-back graph-replayed steps from global step S0 = 3001, with the warmup ending at S0 + 2 and the cosine
    at S0 + 4 (then its floor): every stage against float64 and every update bit for bit at the scheduled rate."""
    T = _trajectory_module()
    monkeypatch.setenv("DMNIST_BUCKET", bucket)
    s0 = T.STEP0
    sched = LearningRateSchedule(0.05, 1, 0.999, warmup_steps=s0 + 2, warmup_start=0.5, cosine_steps=s0 + 4,
                                 cosine_alpha=0.2)
    for s in range(s0, s0 + 6):
        assert A.midpoint_distance_ulps(sched(s)) > 16, s
    eng, be, rec = T._lenet(128, sched=sched)
    assert be.lr_schedule_armed
    batches = T._batches(eng, 6)
    T._feed(eng, rec, batches)
    T._check("lenet.B128.bucket%s.warmup.cosine" % bucket, eng, be, rec, batches, sched=sched)


# ---- through train() -----------------------------------------------------------------------------------------------------
SCHED_FLAGS = ("--lr_warmup_steps=6", "--lr_warmup_start_factor=0.2", "--lr_cosine_decay_steps=20",
               "--lr_cosine_alpha=0.05")
LINE = re.compile(r"Learning rate schedule: (.*); the update of global step #(\d+) is made at (\S+)$")


@pytest.fixture
def flags(monkeypatch):
    from distributedmnist_b200.flags import FLAGS
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    FLAGS.reset()
    yield FLAGS
    FLAGS.reset()


def _train(d, *extra, steps=12):
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import train
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % d, "--batch_size=128", "--max_steps=%d" % steps, "--initial_learning_rate=0.05",
                 "--log_every=1000", "--save_results_period=1000000", "--save_interval_secs=1000",
                 "--should_summarize", "--save_summaries_secs=0"] + list(extra))
    ctx = init_context(FLAGS)
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True, synthetic_sizes=(8192, 1000))
    return train(ctx, ds.train, ds.validation, FLAGS)


def _summary_rates(d):
    import glob
    from distributedmnist_b200.utils.summary import read_tfevents
    rates = {}
    for f in glob.glob(os.path.join(str(d), "events.out.tfevents.*")):
        rates.update({int(ev["step"]): ev["scalars"]["learning_rate"] for ev in read_tfevents(f)
                      if "learning_rate" in ev["scalars"]})
    return rates


MODES = {"k_eq_n": (), "k4_gt_n1": ("--num_replicas_to_aggregate=4",), "cdf": ("--worker_times_cdf_method",),
         "interval": ("--interval_method", "--interval_ms=1")}


class _Lines(logging.Handler):
    """The ``Learning rate schedule:`` lines of the "dmnist" logger, whatever its propagation."""

    def __init__(self):
        super().__init__(logging.INFO)
        self.found = []

    def emit(self, record):
        m = LINE.match(record.getMessage())
        if m:
            self.found.append(m)


def _train_logged(d, *extra, steps):
    h = _Lines()
    logger = logging.getLogger("dmnist")
    level = logger.level
    logger.addHandler(h)
    logger.setLevel(logging.INFO)
    try:
        res = _train(d, *extra, steps=steps)
    finally:
        logger.removeHandler(h)
        logger.setLevel(level)
    return res, h.found


@pytest.mark.parametrize("mode", list(MODES))
def test_train_runs_at_the_scheduled_rate_and_restarts_mid_warmup(tmp_path, flags, mode):
    d = str(tmp_path / "run")
    first, lines = _train_logged(d, *(SCHED_FLAGS + MODES[mode]), steps=3)
    sched = first["optimizer"].lr_schedule
    assert first["engine"].backend.lr_schedule_armed
    assert first["lr_schedule"] == dict(warmup_steps=6, warmup_start_factor=0.2, cosine_decay_steps=20,
                                        cosine_alpha=0.05)
    assert len(lines) == 1 and lines[0].group(2) == "0"
    assert float(lines[0].group(3)) == pytest.approx(0.05 * 0.2, rel=1e-5)
    assert "cosine decay over 20 global steps" in lines[0].group(1)
    rates = _summary_rates(d)
    assert rates and all(v == np.float32(sched(s)) for s, v in rates.items()), rates
    second, lines = _train_logged(d, *(SCHED_FLAGS + MODES[mode]), steps=24)
    # the final checkpoint holds the newest committed step, which interval mode may have moved past the last one the
    # loop consumed
    assert len(lines) == 1
    r = int(lines[0].group(2))
    assert first["final_step"] <= r < 6, (first["final_step"], r)          # the restart lands inside the warmup
    assert float(lines[0].group(3)) == pytest.approx(sched(r), rel=1e-5)
    assert second["final_step"] >= 24
    rates = _summary_rates(d)
    later = {s: v for s, v in rates.items() if s > r}
    assert later and all(v == np.float32(sched(s)) for s, v in later.items()), later
    assert any(s >= 20 for s in later) and min(later) <= r + 2


def test_train_without_the_flags_leaves_the_block_disarmed(tmp_path, flags):
    a = _train(str(tmp_path / "a"), "--pipeline_steps=false", steps=8)
    assert not a["engine"].backend.lr_schedule_armed
    sched = a["optimizer"].lr_schedule
    assert not sched.shaped and a["lr_schedule"]["warmup_steps"] == 0


# ---- two replicas --------------------------------------------------------------------------------------------------------
@pytest.mark.multigpu
@pytest.mark.parametrize("k", [2, 1])
def test_two_replicas_stay_bit_identical_through_warmup_and_cosine(tmp_path, k):
    """K = N = 2 on every aggregation path, and K = 1 of 2: the replicas end bit-identical, and every committed update
    of the probe (weights 0, gradients 1) is fp32(lr(step) / count) * count for the schedule the engine armed."""
    from distributedmnist_b200.parallel.launcher import run_replicas
    worker = os.path.join(HERE, "_lr_schedule_worker.py")
    for b in (("2", "1", "0") if k == 2 else ("0",)):
        d = tmp_path / ("k%d_bucket%s" % (k, b))
        codes = run_replicas([worker, str(d / "rank_RANK.json"), str(k)], 2, timeout=600, out_dir=str(d / "out"),
                             env={"DMNIST_BUCKET": b})
        logs = "\n".join(open(os.path.join(d, "out", f)).read()[-1500:] for f in sorted(os.listdir(d / "out")))
        assert codes == [0, 0], (b, logs)
        res = [json.load(open(str(d / ("rank_%d.json" % r)))) for r in range(2)]
        assert res[0]["params_fp"] == res[1]["params_fp"], "k=%d bucket %s: the replicas differ" % (k, b)
        for r in res:
            assert r["probe_wrong"] == [], (k, b, r["probe_wrong"])
            assert r["probe_checked"] >= 8
