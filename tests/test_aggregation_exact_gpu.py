"""The aggregation kernels (csrc/fused_sync.cu, csrc/fused_bucket.cu, csrc/fused_interval.cu) on one H100, bit for bit
against the exact emulation of ops/aggrefs.py: the fp32 weights and the bf16 shadow over the whole arena, after every
step, at the real learning-rate schedule (decay 0.999, p = step / decay_steps changing every step)."""
import json
import os
import time

import numpy as np
import pytest
import torch

from distributedmnist_b200.ops import aggrefs as A
from distributedmnist_b200.schedule import LearningRateSchedule

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

SCHED = LearningRateSchedule(0.05, 1, 0.999)
LENET_ARENA = 1665024


def _backend(ctas: int = 0):
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    return FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"), ctas=ctas)


def _enqueue(be, params, grads, sched=SCHED):
    be.enqueue(params, grads, 1, sched.initial_learning_rate, sched.decay_rate, sched.decay_steps)


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


def _randn(n, g, scale=1.0):
    return torch.randn(n, device="cuda", generator=g) * scale


# ---- learning rate ---------------------------------------------------------------------------------------------------
PROBE_P = sorted(set(range(65)) | {int(x) for x in np.geomspace(64, 1e5, 240)} | {99999, 100000})


@pytest.mark.parametrize("rate", [0.999, 0.95, 0.5, 1.0])
def test_device_step_size_equals_host_schedule(rate):
    """Solo step with weights 0 and gradients 1.0: the new weight is -scale exactly.  The device's scale must be
    fp32(LearningRateSchedule(step)) bit for bit wherever that is a normal fp32 number; below that the kernels flush it."""
    sched = LearningRateSchedule(0.05, 1, rate)
    be = _backend()
    try:
        params, grads = be.allocate(1024), be.allocate(1024)
        grads.fill_(1.0)
        got = []
        for p in PROBE_P:
            params.zero_()
            be.set_global_step(p)
            _enqueue(be, params, grads, sched)
            got.append(-params[0].item())
        be.check_error()
    finally:
        be.close()
    checked, wrong = 0, []
    for p, x in zip(PROBE_P, got):
        host = sched(p)
        if host < A.FLT_MIN:
            assert x == 0.0, (p, x, host)
            continue
        # the device's double pow may differ from the host's by a few double ulps: that never matters this far from a
        # rounding boundary
        assert A.midpoint_distance_ulps(host) > 16, (p, host)
        checked += 1
        if np.float32(x) != np.float32(host):
            wrong.append((p, x, float(np.float32(host))))
    assert not wrong, "rate %g: %d of %d step sizes differ from the host schedule: %s" % (rate, len(wrong), checked, wrong[:8])
    assert checked >= 60


# ---- fused_sync_sgd_kernel -------------------------------------------------------------------------------------------
def _mlp_arena(layers, hidden):
    from distributedmnist_b200.models.mlp import mlp_spec
    return mlp_spec(layers, hidden).arena_numel


ARENAS = {"lenet": lambda: LENET_ARENA, "mlp3_h4096": lambda: _mlp_arena(3, 4096),
          "ragged": lambda: 4 * (132 * 512 * 3 + 5)}      # numel4 not a multiple of any grid used here


@pytest.mark.parametrize("ctas", [0, 3])
@pytest.mark.parametrize("arena", list(ARENAS))
def test_fused_sync_sgd_solo_is_bit_exact(arena, ctas):
    n = ARENAS[arena]()
    be = _backend(ctas)
    try:
        params, grads = be.allocate(n), be.allocate(n)
        g = torch.Generator(device="cuda").manual_seed(n + ctas)
        params.copy_(_randn(n, g, 0.05))
        be.attach_shadow(params)
        be.set_global_step(4321)
        for s in range(2 if n > 10 ** 7 else 3):
            step = be.device_epoch
            w = A.f32(params)
            grads.copy_(_randn(n, g))
            _enqueue(be, params, grads)
            want = A.fused_sync_step(w, [A.f32(grads)], 1, A.step_scale(SCHED, step, 1))
            _assert_exact("%s ctas=%d step %d" % (arena, ctas, s), params, be.shadow, want)
        be.check_error()
    finally:
        be.close()


def test_fused_sync_sgd_solo_drop_connect_is_bit_exact():
    n = LENET_ARENA
    be = _backend()
    try:
        params, grads = be.allocate(n), be.allocate(n)
        g = torch.Generator(device="cuda").manual_seed(7)
        params.copy_(_randn(n, g, 0.05))
        be.attach_shadow(params)
        be.drop_connect_(grads, 0.9, 0)
        be.set_global_step(300)
        for s in range(3):
            step = be.device_epoch
            w = A.f32(params)
            grads.copy_(_randn(n, g))
            _enqueue(be, params, grads)
            want = A.fused_sync_step(w, [A.f32(grads)], 1, A.step_scale(SCHED, step, 1),
                                     drop=(be.drop_seed, step, be.drop_keep))
            _assert_exact("drop-connect step %d" % s, params, be.shadow, want)
    finally:
        be.close()


# ---- bucketed kernels (csrc/fused_bucket.cu) -------------------------------------------------------------------------
def _param(spec, name):
    q = [p for p in spec.params if p.name == name][0]
    return q.offset, q.offset + q.numel


def _bucket_run(spec, early, late_ll, late_bf16, split_phases, steps=3):
    n = spec.arena_numel
    b, e = early
    be = _backend()
    try:
        be.late_ll, be.late_bf16 = late_ll, late_bf16
        params, grads = be.allocate(n), be.allocate(n)
        g16 = be.allocate_buffer((e - b) * 2)
        g16v = g16.view(torch.bfloat16, 0, e - b)
        g = torch.Generator(device="cuda").manual_seed(11)
        params.copy_(_randn(n, g, 0.05))
        be.attach_shadow(params)
        be.set_global_step(2024)
        rounds = A.late_bucket_rounds_bf16(n, e - b, late_ll, late_bf16)
        for s in range(steps):
            step = be.device_epoch
            w = A.f32(params)
            grads.copy_(_randn(n, g))
            g16v.copy_(_randn(e - b, g).to(torch.bfloat16))
            for phase in ((3, 4, 2) if split_phases else (1, 2)):
                be.enqueue_bucket_v2(params, grads, g16, None, phase, b, e, SCHED.initial_learning_rate, SCHED.decay_rate,
                                     SCHED.decay_steps)
            want = A.bucket_step(w, [A.f32(grads)], [A.f32(g16v.float())], early, A.step_scale(SCHED, step, 1), rounds)
            _assert_exact("bucket step %d" % s, params, be.shadow, want)
            assert be.device_epoch == step + 1
        be.check_error()
    finally:
        be.close()
    return rounds


@pytest.mark.parametrize("late", ["ll_bf16", "ll_fp32", "flags_fp32"])
def test_bucket_kernels_solo_lenet_layout_are_bit_exact(late):
    from distributedmnist_b200.models.lenet import lenet_spec
    spec = lenet_spec()
    rounds = _bucket_run(spec, _param(spec, "fc1_weights"), late != "flags_fp32", late == "ll_bf16", False)
    assert rounds == (late == "ll_bf16")


def test_bucket_kernels_solo_mlp_layout_are_bit_exact():
    """The MLP engine's layout: the early bucket is fc2 (not fc1), exchanged (phase 3) and applied (phase 4) apart, and
    the 3.3 MB late bucket goes through the fp32 bucket_late_kernel even with LL lines on."""
    from distributedmnist_b200.models.mlp import mlp_spec
    spec = mlp_spec(3, 1024)
    early = _param(spec, "fc2_weights")
    assert (spec.arena_numel - (early[1] - early[0])) * 4 > (1 << 20)
    assert not _bucket_run(spec, early, True, True, True)


# ---- interval mode (csrc/fused_interval.cu) --------------------------------------------------------------------------
def test_interval_apply_solo_is_bit_exact():
    """T gradients accumulate inside one long tick; the T-th, after the deadline, commits it: w - fp32(lr / T) * sum, with
    the sum in iteration order.  The next iteration adopts the weights and its shadow is RNE of them."""
    n = LENET_ARENA
    be = _backend()
    try:
        params, grads, acc = be.allocate(n), be.allocate(n), be.allocate(n)
        g = torch.Generator(device="cuda").manual_seed(5)
        params.copy_(_randn(n, g, 0.05))
        be.attach_shadow(params)
        be.set_global_step(1234)
        interval_s = 1.5                  # the T - 1 early iterations must all land inside one tick
        be.interval_arm(interval_s * 1e3)
        for T in (3, 5, 7):
            step = be.device_epoch
            w = A.f32(params)
            gs = []
            for it in range(T):
                if it == T - 1:
                    torch.cuda.synchronize()
                    assert be.device_epoch == step, \
                        "T=%d: the tick committed before its last iteration (host stalled past the deadline)" % T
                    time.sleep(interval_s + 0.05)
                be.enqueue_interval_begin(params)
                grads.copy_(_randn(n, g))
                gs.append(A.f32(grads))
                be.enqueue_interval_end(params, grads, acc, SCHED.initial_learning_rate, SCHED.decay_rate, SCHED.decay_steps)
            be.enqueue_interval_begin(params)      # adopts the committed step and refreshes the shadow
            torch.cuda.synchronize()
            st = be.read_status()
            assert st["epoch"] == step + 1 and st["last_count"] == T, ("T=%d: committed step / divisor" % T, st)
            want = A.fused_sync_step(w, [A.interval_accumulate(gs)], 1, A.step_scale(SCHED, step, T))
            _assert_exact("interval T=%d" % T, params, be.shadow, want)
        be.check_error()
    finally:
        be.close()


# ---- whole engines, graph-replayed ---------------------------------------------------------------------------------------
def _engine_steps(make_engine, bucket, monkeypatch, steps=4):
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    monkeypatch.setenv("DMNIST_BUCKET", bucket)
    be = _backend()
    eng = make_engine(be)
    sched = LearningRateSchedule(0.05, 2, 0.999)
    eng.attach_optimizer(SyncReplicasOptimizer(be, sched, 1, 1))
    assert eng._bucket_v2 == (bucket == "2")
    be.set_global_step(3001)
    gen = torch.Generator().manual_seed(9)
    B = eng.batch_size
    n = eng.spec.arena_numel
    b, e = eng._bucket_early
    rounds = A.late_bucket_rounds_bf16(n, e - b, be.late_ll, be.late_bf16)
    for s in range(steps):
        torch.cuda.synchronize()
        step = be.device_epoch
        w = A.f32(eng.params)
        eng.load_batch(torch.rand(B, 28, 28, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen))
        eng.train_step()
        torch.cuda.synchronize()
        scale = A.step_scale(sched, step, 1)
        grads = A.f32(eng.grads)
        if bucket == "2":
            want = A.bucket_step(w, [grads], [A.f32(eng._g16_view.float()).reshape(-1)], (b, e), scale, rounds)
        else:
            want = A.fused_sync_step(w, [grads], 1, scale)
        _assert_exact("engine bucket=%s step %d" % (bucket, s), eng.params, eng.shadow, want)
    be.check_error()
    assert be.device_epoch == 3001 + steps


@pytest.mark.parametrize("bucket", ["2", "0"])
def test_lenet_engine_steps_are_bit_exact(bucket, monkeypatch):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    _engine_steps(lambda be: CudaLeNetEngine(128, be, seed=3, rank=0, use_graph=True), bucket, monkeypatch)


@pytest.mark.parametrize("bucket", ["2", "0"])
def test_mlp_engine_steps_are_bit_exact(bucket, monkeypatch):
    """mlp3 at hidden 1024: fc2 is the early bucket (phases 3 and 4), the late bucket takes the fp32 kernel."""
    from distributedmnist_b200.engine_cuda import CudaMlpEngine
    _engine_steps(lambda be: CudaMlpEngine("mlp3", 128, be, hidden=1024, seed=3, use_graph=True), bucket, monkeypatch)


# ---- several replicas (tests/_agg_exact_worker.py): every rank emulates each step from all-gathered gradients ----------
def _run_worker(tmp_path, n, cases):
    from distributedmnist_b200.parallel.launcher import run_replicas
    worker = os.path.join(HERE, "_agg_exact_worker.py")
    codes = run_replicas([worker, str(tmp_path / "res_RANK.json"), ",".join(cases)], n, timeout=600,
                         out_dir=str(tmp_path / "out"))
    logs = "\n".join(open(os.path.join(tmp_path, "out", f)).read()[-2000:] for f in sorted(os.listdir(tmp_path / "out")))
    assert codes == [0] * n, logs
    return [json.load(open(tmp_path / ("res_%d.json" % r)))["cases"] for r in range(n)]


def _assert_exact_everywhere(res, name):
    rows = [r[name] for r in res]
    assert all(x["bad_w"] == 0 and x["bad_sh"] == 0 for x in rows), (name, rows)
    assert len({x["fp"] for x in rows}) == 1, (name, "replicas differ")
    return rows


def test_exact_worker_single_replica(tmp_path):
    """The multi-replica worker's cases that exist on one replica, so that its emulation runs wherever there is a GPU."""
    cases = ["p2p", "drop", "v2_ll_bf16", "v2_ll_fp32", "v2_flags", "v2_mlp", "interval"]
    res = _run_worker(tmp_path, 1, cases)
    for name in cases:
        rows = _assert_exact_everywhere(res, name)
        assert rows[0]["steps"][-1] > 5000, (name, rows[0]["steps"])
    assert res[0]["interval"]["steps"][1] - res[0]["interval"]["steps"][0] >= 3


MULTI_CASES = ["p2p", "kofn", "drop", "nvls", "bucket1", "v2_ll_bf16", "v2_ll_fp32", "v2_flags", "v2_mlp", "interval"]


@pytest.mark.multigpu
@pytest.mark.parametrize("case", MULTI_CASES)
def test_multi_replica_aggregation_is_bit_exact(case, tmp_path):
    """N = min(GPUs, 8) replicas.  Bit-exact weights and shadow on every rank after every step, against the emulation of the
    rank-ordered sums.  NVLS at N >= 3 adds in the switch's own order: replicas identical and within the fp32 sum bound."""
    n = min(torch.cuda.device_count(), 8)
    if (case == "bucket1" or case.startswith("v2")) and n not in (2, 4, 8):
        pytest.skip("the bucketed kernels are built for 2, 4 and 8 replicas")
    res = _run_worker(tmp_path, n, [case])
    rows = [r[case] for r in res]
    if case == "nvls" and n >= 3 and rows[0]["nvls"]:
        assert all(x["bad_sh"] == 0 and x["bound_excess"] <= 0.0 for x in rows), rows
        assert len({x["fp"] for x in rows}) == 1
        return
    rows = _assert_exact_everywhere(res, case)
    if case == "kofn":
        for x in rows:
            assert all(c == max(n - 1, 1) for c in x["counts"]), x["counts"]
            assert all(not (m >> (n - 1)) & 1 for m in x["masks"]), x["masks"]       # the delayed rank is masked out
    elif case == "interval":
        assert any(m and not (m >> (n - 1)) & 1 for m in rows[0]["masks"]), rows[0]["masks"]
        assert rows[n - 1]["dropped"] > 0
    else:
        assert all(x["counts"] == [] or all(c == n for c in x["counts"]) for x in rows), rows
