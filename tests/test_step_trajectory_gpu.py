"""Back-to-back graph-replayed training steps, each checked stage by stage against the float64 references from its own
recorded buffers (ops/trajectory.py), and every update bit for bit.  The steps are enqueued without waiting for one
another, so the fork/join edges of the step graphs, the carrying of weights, shadow and epoch from one step to the next,
the clearing of atomically accumulated gradients and both slot graphs are all exercised as training runs them.

Every run starts at global step 3001 with a schedule whose rate changes every step, and has at least 6 steps unless
stated otherwise: the first two capture the two slot graphs, the rest replay them pipelined.

The L2 weight decay (``--weight_decay``) runs are checked the same way, with the fc gradients against the plain reference
+ lambda v of the weights the step read, R against float64 and the loss word against CE + lambda R.  Interval mode is not
among them: its commits follow a wall-clock deadline, which the update check has no model of, so it is covered by a
smoke run (tests/test_weight_decay_gpu.py) only.  Runs with more than one replica need more than one GPU."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

STEP0 = 3001
SEED = 3


def _sched():
    from distributedmnist_b200.schedule import LearningRateSchedule
    return LearningRateSchedule(0.05, 1, 0.999)


def _backend():
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    return FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))


def _start(eng, be, k=1, lam=0.0, drop=None, sched=None):
    from distributedmnist_b200.ops.trajectory import StepRecorder
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    eng.attach_optimizer(SyncReplicasOptimizer(be, sched or _sched(), k, 1, drop_connect_probability=drop))
    if lam:
        eng.arm_weight_decay(lam)
    be.set_global_step(STEP0)
    if k > 1:
        be.kgtn_arm()
    return StepRecorder(eng)


def _lenet(B, keep_prob=0.5, k=1, lam=0.0, drop=None, sched=None):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    be = _backend()
    eng = CudaLeNetEngine(B, be, seed=SEED, rank=0, keep_prob=keep_prob, use_graph=True)
    return eng, be, _start(eng, be, k, lam, drop, sched)


def _mlp(model, B, hidden, k=1):
    from distributedmnist_b200.engine_cuda import CudaMlpEngine
    be = _backend()
    eng = CudaMlpEngine(model, B, be, hidden=hidden, seed=SEED, use_graph=True)
    return eng, be, _start(eng, be, k)


def _batches(eng, n, seed=9):
    gen = torch.Generator().manual_seed(seed)
    B = eng.batch_size
    shape = (B, 28, 28) if hasattr(eng, "h_part") else (B, 784)
    return [(torch.rand(*shape, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen)) for _ in range(n)]


def _feed(eng, rec, batches, how="numpy", sleep_after=None):
    """Enqueue one step per batch, back to back, recording each.  ``how``: "numpy" (load_batch from numpy arrays: the
    page-locked staging path), "packed" (step_packed from page-locked packed buffers: the native runner once both slot
    graphs exist), "indices" (load_indices + train_step) or "step_indices" (step_indices with numpy indices, native runner
    from the third step) -- both on a training set armed with the batches' rows.  ``sleep_after``: after that many steps,
    put a spin of about 0.1 s on the training stream, so the host runs ahead of the device for the rest."""
    keep = []
    if how in ("indices", "step_indices"):
        x = torch.cat([b[0].reshape(-1, 784) for b in batches])
        y = torch.cat([b[1] for b in batches])
        eng.arm_train_data(x, y)
    B = eng.batch_size
    for t, (x, y) in enumerate(batches):
        if t == sleep_after:
            torch.cuda.synchronize()
            torch.cuda._sleep(200_000_000)
        if how == "numpy":
            eng.load_batch(x.numpy(), y.numpy())
            eng.train_step()
        elif how == "packed":
            keep.append(eng.pack_batch(x, y))
            eng.step_packed(keep[-1])
        elif how == "indices":
            eng.load_indices(np.arange(t * B, (t + 1) * B))
            eng.train_step()
        else:
            eng.step_indices(np.arange(t * B, (t + 1) * B))
        rec.record()
    torch.cuda.synchronize()
    return keep


def _check(tag, eng, be, rec, batches, lam=0.0, sched=None):
    """``lam``: the L2 weight decay the engine was armed with; ``sched``: the schedule it was attached with (default
    :func:`_sched`)."""
    from distributedmnist_b200.ops import trajectory as T
    be.check_error()
    upd = T.update_of(eng, sched or _sched(), STEP0)
    bucket = os.environ.get("DMNIST_BUCKET", "2") == "2" and be.drop_keep <= 0.0     # drop-connect: the single kernel
    assert upd["mode"] == ("kgtn" if eng._kgtn_k else ("bucket" if bucket else "fused"))
    assert getattr(eng, "_decay", 0.0) == float(np.float32(lam)) and (("decay_ws" in rec.records[0]) == bool(lam))
    if not eng._kgtn_k:
        assert be.device_epoch == STEP0 + len(batches)
    if hasattr(eng, "h_part"):
        res = T.lenet_trajectory_results(tag, eng.spec, rec.init, rec.records, batches, upd, eng.seed, eng.rank,
                                         eng.keep_prob, lam)
    else:
        res = T.mlp_trajectory_results(tag, eng.spec, rec.init, rec.records, batches, upd)
    worst = T.worst_by_stage(tag, res)
    print("\nTRAJECTORY %s %s" % (tag, json.dumps(worst, sort_keys=True)))
    bad = T.failures(res)
    assert not bad, "%d of %d checks failed, first: %s" % (len(bad), len(res), bad[:20])
    return worst


@pytest.mark.parametrize("B", [64, 128, 256, 1024])
def test_lenet_bucketed_trajectory(B, monkeypatch):
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    eng, be, rec = _lenet(B)
    batches = _batches(eng, 6, seed=B)
    _feed(eng, rec, batches)
    _check("lenet.B%d.bucket2" % B, eng, be, rec, batches)


def test_lenet_single_kernel_trajectory(monkeypatch):
    monkeypatch.setenv("DMNIST_BUCKET", "0")
    eng, be, rec = _lenet(128)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("lenet.B128.bucket0", eng, be, rec, batches)


def test_lenet_keep_08_trajectory(monkeypatch):
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    eng, be, rec = _lenet(128, keep_prob=0.8)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("lenet.B128.keep0.8", eng, be, rec, batches)


@pytest.mark.parametrize("how", ["packed", "step_indices"])
def test_lenet_native_runner_feeds(how, monkeypatch):
    """Steps 3 on run through the native runner (one C call per step), from packed batches or row indices."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    eng, be, rec = _lenet(256)
    batches = _batches(eng, 7)
    _feed(eng, rec, batches, how)
    assert eng._runner is not None
    _check("lenet.B256.%s" % how, eng, be, rec, batches)


def test_lenet_k4_trajectory():
    """K = 4 on one replica, 2 commits.  Every iteration computes on the weights of the commit it adopted, and its dropout
    mask is the one of the epoch word its fc2_fwd_bwd read: the committed global step.  So the 4 iterations of a commit
    share one mask (trajectory.epoch_of)."""
    eng, be, rec = _lenet(128, k=4)
    batches = _batches(eng, 8)
    _feed(eng, rec, batches)
    _check("lenet.B128.k4", eng, be, rec, batches)


@pytest.mark.parametrize("how", ["numpy", "indices", "step_indices"])
def test_staging_buffers_hold_until_their_copy_ran(how, monkeypatch):
    """The host enqueues eight steps while the device is still busy with an earlier one: each input's host staging buffer
    (load_batch's and load_indices' page-locked buffers, step_indices' copy of non-pinned indices) must not be refilled
    before its DMA has run, or a step trains on the batch of a later one."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    eng, be, rec = _lenet(128)
    warm = 3 if how == "step_indices" else 2          # both slot graphs (and the native runner) exist before the spin
    batches = _batches(eng, warm + 8, seed=77)
    _feed(eng, rec, batches, how, sleep_after=warm)
    _check("lenet.B128.staging.%s" % how, eng, be, rec, batches)


def test_mlp3_8192x4096_trajectory(monkeypatch):
    """The largest configured MLP shape, 3 steps (about 0.6 GB of records per step)."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    eng, be, rec = _mlp("mlp3", 8192, 4096)
    batches = _batches(eng, 3)
    _feed(eng, rec, batches)
    _check("mlp3.B8192.H4096", eng, be, rec, batches)


@pytest.mark.parametrize("bucket", ["2", "0"])
@pytest.mark.parametrize("model", ["mlp2", "mlp3"])
def test_mlp_trajectory(model, bucket, monkeypatch):
    """mlp3's early bucket is fc2: its data gradient must read the shadow before phase 4 rewrites it."""
    monkeypatch.setenv("DMNIST_BUCKET", bucket)
    eng, be, rec = _mlp(model, 128, 1024)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("%s.B128.H1024.bucket%s" % (model, bucket), eng, be, rec, batches)


def test_mlp2_k2_trajectory():
    eng, be, rec = _mlp("mlp2", 128, 1024, k=2)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("mlp2.B128.H1024.k2", eng, be, rec, batches)


# ---- L2 weight decay ----------------------------------------------------------------------------------------------------
LAM = 5e-4
LAM_LARGE = 0.25               # a decay read from the wrong weights differs from the right one far beyond the bound


@pytest.mark.parametrize("B,lam", [(37, LAM), (129, LAM), (256, LAM), (1024, LAM), (256, LAM_LARGE)])
def test_lenet_decayed_bucketed_trajectory(B, lam, monkeypatch):
    """fc1's decayed gradient leaves the GEMM as bf16 on the wire; the early bucket then updates fc1 on the same branch,
    after the decayed epilogue read it."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    eng, be, rec = _lenet(B, lam=lam)
    batches = _batches(eng, 6, seed=B)
    _feed(eng, rec, batches)
    _check("lenet.B%d.bucket2.decay%g" % (B, lam), eng, be, rec, batches, lam)


def test_lenet_decayed_single_kernel_trajectory(monkeypatch):
    monkeypatch.setenv("DMNIST_BUCKET", "0")
    eng, be, rec = _lenet(128, lam=LAM)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("lenet.B128.bucket0.decay", eng, be, rec, batches, LAM)


def test_lenet_decayed_keep_08_trajectory(monkeypatch):
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    eng, be, rec = _lenet(128, keep_prob=0.8, lam=LAM)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("lenet.B128.keep0.8.decay", eng, be, rec, batches, LAM)


@pytest.mark.parametrize("how", ["packed", "step_indices"])
def test_lenet_decayed_native_runner_feeds(how, monkeypatch):
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    eng, be, rec = _lenet(256, lam=LAM)
    batches = _batches(eng, 7)
    _feed(eng, rec, batches, how)
    assert eng._runner is not None
    _check("lenet.B256.%s.decay" % how, eng, be, rec, batches, LAM)


@pytest.mark.parametrize("lam", [LAM, LAM_LARGE])
def test_lenet_decayed_k4_trajectory(lam):
    """K = 4 on one replica, 2 commits: every iteration is decayed at the weights of the commit it adopted (DESIGN §4,
    which weights the decay term reads), which the previous record holds."""
    eng, be, rec = _lenet(128, k=4, lam=lam)
    batches = _batches(eng, 8)
    _feed(eng, rec, batches)
    _check("lenet.B128.k4.decay%g" % lam, eng, be, rec, batches, lam)


def test_lenet_decayed_drop_connect_trajectory():
    """--drop_connect runs the single fused kernel, which masks each gradient element, its lambda v included."""
    eng, be, rec = _lenet(128, lam=LAM, drop=0.8)
    assert be.drop_keep == pytest.approx(0.8) and not eng._bucket_v2
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("lenet.B128.drop0.8.decay", eng, be, rec, batches, LAM)


@pytest.mark.parametrize("bucket", ["2", "0"])
def test_lenet_decayed_trajectory_with_lr_cuts(bucket, monkeypatch):
    """A cut table with entries before, inside and at the end of the run: the step sizes are those of the schedule with
    the cuts, and the decay is unaffected."""
    from distributedmnist_b200.schedule import LearningRateSchedule
    monkeypatch.setenv("DMNIST_BUCKET", bucket)
    cuts = [2990, STEP0 + 2, STEP0 + 4, STEP0 + 4]
    sched = LearningRateSchedule(0.05, 1, 0.999, factor=0.5, cuts=cuts)
    eng, be, rec = _lenet(128, lam=LAM, sched=sched)
    eng.arm_lr_cuts(0.5, cuts)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("lenet.B128.bucket%s.cuts.decay" % bucket, eng, be, rec, batches, LAM, sched)
