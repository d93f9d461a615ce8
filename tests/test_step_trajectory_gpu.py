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


def _start(eng, be, k=1, lam=0.0, drop=None, sched=None, aug=None):
    """``aug``: (ranges, first iteration) of the random affine augmentation to arm, None for none."""
    from distributedmnist_b200.ops.trajectory import StepRecorder
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    eng.attach_optimizer(SyncReplicasOptimizer(be, sched or _sched(), k, 1, drop_connect_probability=drop))
    if lam:
        eng.arm_weight_decay(lam)
    if aug is not None:
        eng.arm_augment(*aug[0], start_iteration=aug[1])
    be.set_global_step(STEP0)
    if k > 1:
        be.kgtn_arm()
    return StepRecorder(eng)


def _lenet(B, keep_prob=0.5, k=1, lam=0.0, drop=None, sched=None, aug=None, use_graph=True):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    be = _backend()
    eng = CudaLeNetEngine(B, be, seed=SEED, rank=0, keep_prob=keep_prob, use_graph=use_graph)
    return eng, be, _start(eng, be, k, lam, drop, sched, aug)


def _mlp(model, B, hidden, k=1, aug=None):
    from distributedmnist_b200.engine_cuda import CudaMlpEngine
    be = _backend()
    eng = CudaMlpEngine(model, B, be, hidden=hidden, seed=SEED, use_graph=True)
    return eng, be, _start(eng, be, k, aug=aug)


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
