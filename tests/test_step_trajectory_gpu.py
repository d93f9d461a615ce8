"""Back-to-back graph-replayed training steps, each checked stage by stage against the float64 references from its own
recorded buffers (ops/trajectory.py), and every update bit for bit.  The steps are enqueued without waiting for one
another, so the fork/join edges of the step graphs, the carrying of weights, shadow and epoch from one step to the next,
the clearing of atomically accumulated gradients and both slot graphs are all exercised as training runs them.  The
recorder's clones sit on the stream between two steps, though, and they do not trigger the next step's programmatic
launch, so a recorded step starts only once the previous one has completed: these runs check the ordering inside a step,
not the overlap of consecutive steps that PDL allows.

Every run starts at global step 3001 with a schedule whose rate changes every step, and has at least 6 steps unless
stated otherwise: the first two capture the two slot graphs, the rest replay them pipelined.

The L2 weight decay (``--weight_decay``) runs are checked the same way, with the fc gradients against the plain reference
+ lambda v of the weights the step read, R against float64 and the loss word against CE + lambda R.

Interval mode (``--interval_method``) runs the non-bucketed backward between the adoption of pushed weights and the
gate / accumulate / close / apply kernels, and commits a tick when its close finds the wall-clock deadline passed.  The
recorder clones the replica's control block after every step, so the checker reads which steps committed and with how
many gradients, judges every update bit for bit against those ticks and every stage on the weights and epoch word of the
commit the step adopted, and checks the decisions against the device's own %globaltimer stamps (trajectory.control_results).
The runs tick every step (a 1 us interval) or are paced by the host (ticks of 3, 4 and 2 gradients), with dropout keep
0.8, weight decay, augmentation with elastic distortion, the native runner, eager launches and the MLPs.  cdf mode
(``--worker_times_cdf_method``) computes what K = N computes, with the start and arrival stamp nodes (and a straggler's
delay) in the step graph; its runs are checked as K = N runs, and each step's stamps as its own.  Runs with more than one
replica need more than one GPU."""
import json
import os
import time

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


def _start(eng, be, k=1, lam=0.0, drop=None, sched=None, aug=None, mode=None, interval_ms=None, straggler=None):
    """``aug``: (ranges, first iteration[, elastic distortion]) of the random affine augmentation to arm, None for none.
    ``mode``: "interval" or "cdf" (TimeoutReplicasOptimizer, ``interval_ms``, ``straggler`` as parse_straggler_spec
    returns it), None for SyncReplicasOptimizer."""
    from distributedmnist_b200.ops.trajectory import StepRecorder
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer, TimeoutReplicasOptimizer
    if mode is None:
        opt = SyncReplicasOptimizer(be, sched or _sched(), k, 1, drop_connect_probability=drop)
    else:
        opt = TimeoutReplicasOptimizer(be, sched or _sched(), 1, mode=mode, interval_ms=interval_ms or 1000,
                                       straggler=straggler, seed=SEED)
    eng.attach_optimizer(opt)
    if lam:
        eng.arm_weight_decay(lam)
    if aug is not None:
        eng.arm_augment(*aug[0], start_iteration=aug[1], elastic=aug[2] if len(aug) > 2 else None)
    be.set_global_step(STEP0)
    if k > 1:
        be.kgtn_arm()
    if mode == "interval":
        be.interval_arm(interval_ms)    # after set_global_step, as train.py arms it: the clock's step half is STEP0 + 1
    return StepRecorder(eng)


def _lenet(B, keep_prob=0.5, k=1, lam=0.0, drop=None, sched=None, aug=None, use_graph=True, mode=None, interval_ms=None,
           straggler=None):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    be = _backend()
    eng = CudaLeNetEngine(B, be, seed=SEED, rank=0, keep_prob=keep_prob, use_graph=use_graph)
    return eng, be, _start(eng, be, k, lam, drop, sched, aug, mode, interval_ms, straggler)


def _mlp(model, B, hidden, k=1, aug=None, mode=None, interval_ms=None, straggler=None):
    from distributedmnist_b200.engine_cuda import CudaMlpEngine
    be = _backend()
    eng = CudaMlpEngine(model, B, be, hidden=hidden, seed=SEED, use_graph=True)
    return eng, be, _start(eng, be, k, aug=aug, mode=mode, interval_ms=interval_ms, straggler=straggler)


def _batches(eng, n, seed=9):
    gen = torch.Generator().manual_seed(seed)
    B = eng.batch_size
    shape = (B, 28, 28) if hasattr(eng, "h_part") else (B, 784)
    return [(torch.rand(*shape, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen)) for _ in range(n)]


def _feed(eng, rec, batches, how="numpy", sleep_after=None, after=None):
    """Enqueue one step per batch, back to back, recording each.  ``how``: "numpy" (load_batch from numpy arrays: the
    page-locked staging path), "packed" (step_packed from page-locked packed buffers: the native runner once both slot
    graphs exist), "indices" (load_indices + train_step) or "step_indices" (step_indices with numpy indices, native runner
    from the third step) -- both on a training set armed with the batches' rows.  ``sleep_after``: after that many steps,
    put a spin of about 0.1 s on the training stream, so the host runs ahead of the device for the rest.  ``after``:
    called with t after step t is enqueued and recorded.  ``rec`` None: nothing is recorded, so nothing is enqueued
    between two steps."""
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
        if rec is not None:
            rec.record()
        if after is not None:
            after(t)
    torch.cuda.synchronize()
    return keep


def _check(tag, eng, be, rec, batches, lam=0.0, sched=None, aug=None):
    """``lam``: the L2 weight decay the engine was armed with; ``sched``: the schedule it was attached with (default
    :func:`_sched`); ``aug``: the (ranges, first iteration) of the augmentation it was armed with."""
    from distributedmnist_b200 import augment as AU
    from distributedmnist_b200.ops import trajectory as T
    be.check_error()
    upd = T.update_of(eng, sched or _sched(), STEP0, aug[1] if aug is not None else 0)
    if aug is None:
        assert upd["aug"] is None and "aug_images" not in rec.records[0]
    else:
        assert upd["aug"] == (aug[0], AU.seed_mix(SEED, 0)) and "aug_images" in rec.records[0]
    # drop-connect: the single kernel; interval mode: its own kernels
    bucket = os.environ.get("DMNIST_BUCKET", "2") == "2" and be.drop_keep <= 0.0 and not eng._interval
    assert upd["mode"] == ("kgtn" if eng._kgtn_k else "interval" if eng._interval else "bucket" if bucket else "fused")
    assert getattr(eng, "_decay", 0.0) == float(np.float32(lam)) and (("decay_ws" in rec.records[0]) == bool(lam))
    assert ("ctrl" in rec.records[0]) == (eng._interval or eng._stamp)
    if not eng._interval:
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


# ---- random affine augmentation -----------------------------------------------------------------------------------------
# augment_affine writes the step's images into one engine-owned buffer that conv1 forward, conv1 wgrad and the MLP's x16
# conversion read instead of the input slot.  Each step's recorded buffer is checked against the float64 warp of the batch
# it was fed with the draws of its own iteration (the first step's plus t, in every mode), the counter after every step,
# and every image reader against the recorded buffer: a reader that saw another step's warp within its step, or a counter
# that skipped or repeated an iteration across capture, replay or the native runner, fails its stage.  The recorded steps
# run one after another (see the module docstring); test_lenet_augmented_unrecorded_run_matches_the_checked_one runs the
# same steps back to back with nothing between them, as training enqueues them, and compares the results bit for bit.
AUG = (3.0, 20.0, 0.15)
AUG_WIDE = (8.0, 180.0, 0.9)


def _aug(ranges=AUG, start=STEP0):
    from distributedmnist_b200 import augment as AU
    return AU.Ranges(*ranges), start


@pytest.mark.parametrize("B", [37, 129, 256, 1024])
def test_lenet_augmented_bucketed_trajectory(B, monkeypatch):
    """1024 rows are more than 4 CTAs per SM: the augment CTAs then get an uneven number of rows."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    aug = _aug()
    eng, be, rec = _lenet(B, aug=aug)
    batches = _batches(eng, 6, seed=B)
    _feed(eng, rec, batches)
    _check("lenet.B%d.bucket2.aug" % B, eng, be, rec, batches, aug=aug)


def test_lenet_augmented_single_kernel_keep_08_wide_trajectory(monkeypatch):
    """The single aggregation kernel, keep 0.8, and ranges that turn images about and zoom them out to a tenth, so that
    most of many rows is background."""
    monkeypatch.setenv("DMNIST_BUCKET", "0")
    aug = _aug(AUG_WIDE)
    eng, be, rec = _lenet(128, keep_prob=0.8, aug=aug)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("lenet.B128.bucket0.keep0.8.aug_wide", eng, be, rec, batches, aug=aug)


@pytest.mark.parametrize("how", ["packed", "step_indices"])
def test_lenet_augmented_native_runner_feeds(how, monkeypatch):
    """Graph replay through the native runner, from packed batches or gathered rows."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    aug = _aug()
    eng, be, rec = _lenet(256, aug=aug)
    batches = _batches(eng, 7)
    _feed(eng, rec, batches, how)
    assert eng._runner is not None
    _check("lenet.B256.%s.aug" % how, eng, be, rec, batches, aug=aug)


def test_lenet_augmented_staging_spin(monkeypatch):
    """The host enqueues eight augmented steps while the device is still busy with an earlier one."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    aug = _aug()
    eng, be, rec = _lenet(128, aug=aug)
    batches = _batches(eng, 10, seed=78)
    _feed(eng, rec, batches, "numpy", sleep_after=2)
    _check("lenet.B128.staging.numpy.aug", eng, be, rec, batches, aug=aug)


def test_lenet_augmented_eager_trajectory(monkeypatch):
    """use_graph=False: the step's kernels launched eagerly, each step's one PDL chain (the recorder's clones end the
    chain between steps)."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    aug = _aug()
    eng, be, rec = _lenet(128, aug=aug, use_graph=False)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("lenet.B128.eager.aug", eng, be, rec, batches, aug=aug)


def test_lenet_augmented_k4_trajectory():
    """K = 4 on one replica, 2 commits: the counter advances once per iteration, while the dropout mask stays that of the
    commit's global step."""
    aug = _aug()
    eng, be, rec = _lenet(128, k=4, aug=aug)
    batches = _batches(eng, 8)
    _feed(eng, rec, batches)
    _check("lenet.B128.k4.aug", eng, be, rec, batches, aug=aug)


def test_lenet_augmented_decayed_trajectory(monkeypatch):
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    aug = _aug()
    eng, be, rec = _lenet(256, lam=LAM, aug=aug)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("lenet.B256.bucket2.decay.aug", eng, be, rec, batches, LAM, aug=aug)


def test_lenet_augmented_counter_wraps_trajectory(monkeypatch):
    """From iteration 2^32 - 3: the u32 counter wraps through 0 in the replayed steps."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    aug = _aug(start=2 ** 32 - 3)
    eng, be, rec = _lenet(128, aug=aug)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("lenet.B128.wrap.aug", eng, be, rec, batches, aug=aug)


def test_lenet_augmented_with_evaluation_passes(monkeypatch):
    """In-training evaluation passes after the 2nd and 4th steps: a pass neither advances the counter nor writes the
    augmented buffer, and the steps after it draw on from where the last step left off."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    g = torch.Generator().manual_seed(3)
    vx, vy = torch.rand(3000, 28, 28, 1, generator=g) - 0.5, torch.randint(0, 10, (3000,), generator=g)
    aug = _aug()
    eng, be, rec = _lenet(128, aug=aug)
    eng.arm_eval(vx.numpy(), vy.numpy())
    after_eval = {}

    def evaluate(t):
        if t in (1, 3):
            eng.enqueue_eval()
            after_eval[t] = (eng._aug_images.clone(), eng._aug_counter.clone())
    batches = _batches(eng, 6)
    _feed(eng, rec, batches, after=evaluate)
    assert sorted(after_eval) == [1, 3]
    for t, (images, counter) in after_eval.items():
        assert torch.equal(images, rec.records[t]["aug_images"]), t
        assert torch.equal(counter, rec.records[t]["aug_counter"]), t
    _check("lenet.B128.eval.aug", eng, be, rec, batches, aug=aug)


@pytest.mark.parametrize("bucket", ["2", "0"])
@pytest.mark.parametrize("model", ["mlp2", "mlp3"])
def test_mlp_augmented_trajectory(model, bucket, monkeypatch):
    monkeypatch.setenv("DMNIST_BUCKET", bucket)
    aug = _aug()
    eng, be, rec = _mlp(model, 128, 1024, aug=aug)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("%s.B128.H1024.bucket%s.aug" % (model, bucket), eng, be, rec, batches, aug=aug)


def test_mlp2_augmented_k2_trajectory():
    aug = _aug()
    eng, be, rec = _mlp("mlp2", 128, 1024, k=2, aug=aug)
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("mlp2.B128.H1024.k2.aug", eng, be, rec, batches, aug=aug)


def test_mlp3_8192x4096_augmented_trajectory(monkeypatch):
    """The largest configured MLP shape, 3 steps: 8192 rows over 4 CTAs per SM, 15 or 16 rows per augment CTA on 132
    SMs."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    aug = _aug()
    eng, be, rec = _mlp("mlp3", 8192, 4096, aug=aug)
    batches = _batches(eng, 3)
    _feed(eng, rec, batches)
    _check("mlp3.B8192.H4096.aug", eng, be, rec, batches, aug=aug)


@pytest.mark.parametrize("how,use_graph", [("numpy", False), ("numpy", True), ("packed", True)],
                         ids=["eager", "graph", "native_runner"])
def test_lenet_augmented_unrecorded_run_matches_the_checked_one(how, use_graph, monkeypatch):
    """The same 6 augmented steps twice: once recorded and checked stage by stage, once enqueued back to back with
    nothing between two steps, as training enqueues them, so that consecutive steps overlap as far as their PDL edges
    allow.  A reader of step t that saw step t+1's warp (or augment_affine overwriting the buffer before step t's readers
    were done) would change that run's gradients and weights.  The lenet kernels reduce in a fixed order, so both runs
    must end with the same weights, gradients, augmented buffer and counter, bit for bit."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    aug = _aug()
    ends = []
    for recorded in (True, False):
        eng, be, rec = _lenet(128, aug=aug, use_graph=use_graph)
        batches = _batches(eng, 6)
        keep = _feed(eng, rec if recorded else None, batches, how)
        if recorded:
            _check("lenet.B128.%s.aug.recorded" % ("eager" if not use_graph else how), eng, be, rec, batches, aug=aug)
        be.check_error()
        ends.append([t.clone() for t in (eng.params, eng.grads, eng._aug_images, eng._aug_counter)])
        del keep
    for name, a, b in zip(("params", "grads", "aug_images", "aug_counter"), *ends):
        assert torch.equal(a, b), name


# ---- interval mode ------------------------------------------------------------------------------------------------------
# One replica: every tick's commit is its own (the mask is rank 0, the divisor its count).  Paced runs: the host enqueues
# the first T - 1 steps of a tick back to back, waits for them, sleeps past the deadline and enqueues the T-th, whose close
# commits the tick; the next step adopts it and re-arms the deadline.  The checker follows what the device recorded, so a
# host stall that let a tick commit early changes the ticks, not the verdict; each paced run still asserts that a tick of
# at least 3 gradients committed.
PACE_MS = 1000.0
PACED_TICKS = (3, 4, 2)


def _pace(be, ticks=PACED_TICKS, interval_ms=PACE_MS):
    """``(after, early)``: the ``after`` callback of :func:`_feed` that paces ``ticks``, and the list of the ticks' last
    steps before which the tick had already committed (a host stall past the deadline)."""
    last = set(np.cumsum(ticks) - 1)
    early = []
    base = be._read_u32("iv_ticks_committed")

    def after(t):
        if t + 1 in last:
            torch.cuda.synchronize()
            if be._read_u32("iv_ticks_committed") - base != sum(1 for s in last if s <= t):
                early.append(t + 1)
            time.sleep(interval_ms * 1e-3 + 0.05)
    return after, early


def _ticks(eng, rec):
    """Gradients of each committed tick, as the control blocks recorded them."""
    from distributedmnist_b200.ops import trajectory as T
    tr = T.interval_trace(T.update_of(eng, _sched(), STEP0), rec.init, rec.records)
    return [n for n, c in zip(tr["count"], tr["commit"]) if c], tr


def _paced(tag, eng, be, rec, how="numpy", lam=0.0, aug=None):
    after, early = _pace(be)
    batches = _batches(eng, sum(PACED_TICKS))
    _feed(eng, rec, batches, how, after=after)
    if how != "numpy":
        assert eng._runner is not None
    worst = _check(tag, eng, be, rec, batches, lam, aug=aug)
    sizes, _tr = _ticks(eng, rec)
    print("TICKS %s committed %s, paced %s, committed before their last step: %s" % (tag, sizes, PACED_TICKS, early))
    assert any(n >= 3 for n in sizes), sizes
    if not early:
        assert sizes == list(PACED_TICKS), sizes
    return batches, worst


def test_lenet_interval_every_step_commits():
    """A 1 us interval: every close comes after the deadline, so every step commits a tick of its own gradient."""
    eng, be, rec = _lenet(128, mode="interval", interval_ms=0.001)
    assert eng._interval and not eng._kgtn_k and not eng._bucketed
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check("lenet.B128.interval1us", eng, be, rec, batches)
    sizes, tr = _ticks(eng, rec)
    assert tr["commit"] == [True] * 6 and sizes == [1] * 6, tr
    assert be.device_epoch == STEP0 + 5               # the last commit is adopted by the next step


def test_lenet_interval_paced_trajectory():
    """Ticks of 3, 4 and 2 gradients.  Premise: judged as K = N steps (an update and a new epoch word every step) the
    same records fail."""
    from distributedmnist_b200.ops import trajectory as T
    eng, be, rec = _lenet(128, mode="interval", interval_ms=PACE_MS)
    batches, _ = _paced("lenet.B128.interval", eng, be, rec)
    upd = dict(T.update_of(eng, _sched(), STEP0), mode="fused")
    bad = T.failures(T.lenet_trajectory_results("kn", eng.spec, rec.init, rec.records, batches, upd, eng.seed, eng.rank,
                                                eng.keep_prob))
    stages = sorted({n.split(".", 2)[2] for n, _, _ in bad})
    print("K = N model on the interval records: %d checks fail, stages %s" % (len(bad), stages[:12]))
    assert any(n.endswith("update_bits_differ") for n, _, _ in bad) and any("fc2_fwd_bwd" in n for n, _, _ in bad)


def test_lenet_interval_keep_08_trajectory():
    eng, be, rec = _lenet(128, keep_prob=0.8, mode="interval", interval_ms=PACE_MS)
    _paced("lenet.B128.keep0.8.interval", eng, be, rec)


@pytest.mark.parametrize("lam", [LAM, LAM_LARGE])
def test_lenet_interval_decayed_trajectory(lam):
    """Every iteration of a tick is decayed at the weights it adopted, which the previous record holds."""
    eng, be, rec = _lenet(128, lam=lam, mode="interval", interval_ms=PACE_MS)
    _paced("lenet.B128.interval.decay%g" % lam, eng, be, rec, lam=lam)


def test_lenet_interval_elastic_trajectory():
    """The augmentation counter advances once per iteration (the first step's plus t), the epoch word once per commit."""
    from distributedmnist_b200 import augment as AU
    aug = _aug() + (AU.Elastic(34.0, 4.0),)
    eng, be, rec = _lenet(128, aug=aug, mode="interval", interval_ms=PACE_MS)
    assert eng._aug_elastic is not None
    _paced("lenet.B128.interval.elastic", eng, be, rec, aug=aug)


@pytest.mark.parametrize("how", ["packed", "step_indices"])
def test_lenet_interval_native_runner_feeds(how):
    eng, be, rec = _lenet(128, mode="interval", interval_ms=PACE_MS)
    _paced("lenet.B128.interval.%s" % how, eng, be, rec, how)


def test_lenet_interval_eager_trajectory():
    eng, be, rec = _lenet(128, use_graph=False, mode="interval", interval_ms=PACE_MS)
    _paced("lenet.B128.interval.eager", eng, be, rec)


@pytest.mark.parametrize("model", ["mlp2", "mlp3"])
def test_mlp_interval_trajectory(model):
    eng, be, rec = _mlp(model, 128, 1024, mode="interval", interval_ms=PACE_MS)
    _paced("%s.B128.H1024.interval" % model, eng, be, rec)


# ---- cdf mode -------------------------------------------------------------------------------------------------------------
# The updates are those of K = N; the step graph adds the start and arrival stamps and, with a straggler, the delay inside
# the stamped span.  Every step's stamps must be its own (trajectory.control_results) and span its delay.
def _straggler(form):
    from distributedmnist_b200.parallel.aggregators import parse_straggler_spec
    return None if form is None else parse_straggler_spec(form, 30000)


def _check_cdf(tag, eng, be, rec, batches, form):
    from distributedmnist_b200.ops import trajectory as T
    assert eng._stamp and not eng._interval
    _check(tag, eng, be, rec, batches)
    spans = np.array([(w["t_arrive"] - w["t_start"]) for w in
                      (T.ctrl_words(r["ctrl"], be._off, STEP0 + t) for t, r in enumerate(rec.records))], dtype=np.int64)
    if form is None:
        return
    if form.split(":")[1] == "exp":
        j, _drawn, spun = be.straggler_samples()
        assert np.array_equal(j, np.arange(len(batches))), j
        delay = spun.astype(np.int64)
    else:
        delay = np.full(len(batches), int(float(form.split(":")[2]) * 1000), dtype=np.int64)
    print("CDF %s compute span - delay (us): %s" % (tag, ((spans - delay) / 1e3).round(1).tolist()))
    assert (spans >= delay).all(), (spans, delay)


@pytest.mark.parametrize("form", [None, "0:1.0:50", "0:exp:20"], ids=["none", "fixed", "sampled"])
@pytest.mark.parametrize("bucket", ["2", "0"])
def test_lenet_cdf_trajectory(bucket, form, monkeypatch):
    """Bucketed, the delay sits in the compute chain after the start stamp (_delay_in_chain), and the arrival stamp
    waits for the small fc gradients' branch; with the single kernel both come after the backward pass."""
    monkeypatch.setenv("DMNIST_BUCKET", bucket)
    eng, be, rec = _lenet(256, mode="cdf", straggler=_straggler(form))
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    assert eng._bucketed == (bucket == "2") and eng._delay_in_chain == (bucket == "2" and form is not None)
    _check_cdf("lenet.B256.bucket%s.cdf.%s" % (bucket, form or "none"), eng, be, rec, batches, form)


@pytest.mark.parametrize("form", [None, "0:exp:20"], ids=["none", "sampled"])
def test_mlp2_cdf_trajectory(form, monkeypatch):
    """The MLP step graph's start stamp: without it read_timing hands the cdf telemetry t_start = 0, a compute time of
    the whole %globaltimer value."""
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    eng, be, rec = _mlp("mlp2", 128, 1024, mode="cdf", straggler=_straggler(form))
    batches = _batches(eng, 6)
    _feed(eng, rec, batches)
    _check_cdf("mlp2.B128.H1024.cdf.%s" % (form or "none"), eng, be, rec, batches, form)
