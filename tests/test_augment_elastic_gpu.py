"""Elastic distortion on the GPU (csrc/augment_elastic.cu): the kernel's field against the float64 field within one fp32
ulp, its affine coefficients bit for bit against augment_affine's, its pixels within the derived bound, every row
written and the counter advanced once, at the batch sizes where the grid logic changes; its argument refusals; the wiring
of the augmented buffer into every reader of the training images (lenet and mlp2); host-fed and gathered slots, graph
replay, eager launch and the native runner; reproducibility; the counter under K > N; evaluation without augmentation;
and graph-replayed trajectories checked stage by stage (ops/trajectory.py).  One replica only."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from distributedmnist_b200 import augment as AU

pytestmark = pytest.mark.gpu

EL = AU.Elastic(34.0, 4.0)
R = AU.Ranges(2.0, 15.0, 0.1)
ZERO = AU.Ranges(0.0, 0.0, 0.0)
STEP0 = 3001
SEED = 3


def _lib():
    from distributedmnist_b200.ops.lib import load
    return load()


def _counter(it):
    return torch.from_numpy(np.array([it & 0xFFFFFFFF, 0], dtype=np.uint32).view(np.int32)).cuda()


def _taps(el):
    w = AU.gaussian_weights(el.sigma)
    return (ctypes.c_double * len(w))(*w), len(w) - 1


def _launch(src, mix, it, r, el):
    """One eager augment_elastic launch on ``src`` [B, 784] (device): (images, params_out, field_out [B, 2, 784],
    counter words) on the host."""
    from distributedmnist_b200.ops.lib import stream_ptr
    B = src.shape[0]
    dst = torch.full((B, 784), float("nan"), device="cuda")
    params = torch.full((B, 8), float("nan"), device="cuda")
    field = torch.full((B, 2, 784), float("nan"), device="cuda")
    ctr = _counter(it)
    w, radius = _taps(el)
    _lib().dm_augment_elastic(src, dst, B, ctr, mix, *(float(v) for v in r), el.alpha, w, radius, params, field,
                              stream_ptr())
    torch.cuda.synchronize()
    return dst.cpu().numpy(), params.cpu().numpy(), field.cpu().numpy(), ctr.cpu().numpy().view(np.uint32)


def _affine_params(src, mix, it, r):
    from distributedmnist_b200.ops.lib import stream_ptr
    B = src.shape[0]
    params = torch.full((B, 8), float("nan"), device="cuda")
    _lib().dm_augment_affine(src, torch.empty_like(src), B, _counter(it), mix, *(float(v) for v in r), params,
                             stream_ptr())
    torch.cuda.synchronize()
    return params.cpu().numpy()


def _images(B, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 784, generator=g) - 0.5


def _check_launch(B, mix, it, r, el, seed):
    """Field, coefficients, pixels, rows written and counter of one launch at batch B."""
    from distributedmnist_b200.ops.selfcheck import augment_pixel_bound, elastic_field_err
    src = _images(B, seed)
    got, p, f, ctr = _launch(src.cuda(), mix, it, r, el)
    assert ctr.tolist() == [(it + 1) & 0xFFFFFFFF, 0], (B, ctr)
    assert not np.isnan(got).any(), (B, np.flatnonzero(np.isnan(got).any(axis=1))[:10])
    assert np.array_equal(p, _affine_params(src.cuda(), mix, it, r)), B         # augment_affine's coefficients, bit for bit
    if r == ZERO:
        assert np.array_equal(p[:, 4:], np.tile(np.float32([1, 0, 0, 0]), (B, 1)))
    ref = AU.elastic_field(mix, it, B, el).reshape(B, 2, 784)
    ferr = np.abs(f.astype(np.float64) - ref)
    fbound = elastic_field_err(ref, el)
    assert np.all(ferr <= fbound), (B, float((ferr / fbound).max()))
    want = AU.warp(src.numpy(), *(p[:, k].astype(np.float64) for k in range(4, 8)), field=f).reshape(B, 784)
    err, bound = np.abs(got.astype(np.float64) - want), augment_pixel_bound(p[:, 4:8], field=f)
    assert np.all(err <= bound), (B, float((err / bound).max()))
    return got, f


# ---- the kernel --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 96, 256, 8192])
def test_field_coefficients_pixels_rows_and_counter(B):
    for r, el, (seed, rank, it) in ((AU.Ranges(8.0, 180.0, 0.5), EL, (66478, 0, 0)), (R, AU.Elastic(64.0, 8.0), (7, 3, 12345)),
                                    (ZERO, AU.Elastic(8.0, 0.5), (1, 1, 2 ** 32 - 1))):
        _got, f = _check_launch(B, AU.seed_mix(seed, rank), it, r, el, B + seed)
        assert np.abs(f).max() > 0.01 * el.alpha


def _grid_edge_batches():
    """augment_affine's grid edges: one row; around 4 CTAs per SM; 32 rows in every CTA of 4 per SM and one more; 40000."""
    sms = int(_lib().dm_num_sms())
    return [1, 4 * sms - 1, 4 * sms, 4 * sms + 1, 128 * sms, 128 * sms + 1, 40000]


def test_grid_edges():
    mix = AU.seed_mix(11, 1)
    for B in _grid_edge_batches():
        _check_launch(B, mix, 2 ** 32 - 1 if B % 2 else 4321, AU.Ranges(8.0, 180.0, 0.5), EL, 1000 + B)


def test_alpha_zero_is_the_affine_warp():
    from distributedmnist_b200.ops.lib import stream_ptr
    src = _images(300, 5).cuda()
    got, _p, f, _c = _launch(src, AU.seed_mix(2, 0), 9, R, AU.Elastic(0.0, 4.0))
    want = torch.empty_like(src)
    _lib().dm_augment_affine(src, want, 300, _counter(9), AU.seed_mix(2, 0), *R, None, stream_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(got, want.cpu().numpy()) and not np.any(f)


def test_argument_checks():
    from distributedmnist_b200.ops.lib import KernelLibraryError, stream_ptr
    lib, src = _lib(), torch.zeros(4, 784, device="cuda")
    dst, ctr = torch.zeros_like(src), _counter(0)
    w, radius = _taps(EL)
    nan_w = (ctypes.c_double * 17)(*([float("nan")] * 17))
    good = [src, dst, 4, ctr, 1, 1.0, 1.0, 0.1, 34.0, w, radius]
    bad = [dict(batch=0), dict(batch=AU.MAX_ELASTIC_BATCH + 1), dict(counter=None), dict(src=None), dict(dst=None),
           dict(weights=None), dict(scale=1.0), dict(shift=float("nan")), dict(alpha=-1.0), dict(alpha=64.5),
           dict(alpha=float("inf")), dict(radius=33), dict(radius=-1), dict(weights=nan_w)]
    keys = ["src", "dst", "batch", "counter", "mix", "shift", "rotation", "scale", "alpha", "weights", "radius"]
    for change in bad:
        args = list(good)
        for k, v in change.items():
            args[keys.index(k)] = v
        with pytest.raises(KernelLibraryError):
            lib.dm_augment_elastic(*args, None, None, stream_ptr())
    torch.cuda.synchronize()
    assert ctr.cpu().tolist() == [0, 0] and not torch.any(dst)


# ---- engines -----------------------------------------------------------------------------------------------------------
def _engine(kind, B=256, seed=5, use_graph=True, k=1, hidden=1024):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine, CudaMlpEngine
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    if kind == "lenet":
        eng = CudaLeNetEngine(B, be, seed=seed, use_graph=use_graph)
    else:
        eng = CudaMlpEngine(kind, B, be, hidden=hidden, seed=seed, use_graph=use_graph)
    eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 20, 0.7), k, 1))
    return eng


def _batch(eng, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(*eng.images[0].shape, generator=g) - 0.5, torch.randint(0, 10, (eng.batch_size,), generator=g)


def test_engine_draws_start_at_the_armed_iteration_and_match_the_kernel():
    eng = _engine("lenet")
    eng.arm_augment(*R, start_iteration=1234, elastic=EL)
    x, y = _batch(eng, 1)
    eng.load_batch(x, y)
    eng.forward_backward(0)                         # captures the graph: its warm-up launch must not consume draws
    got = eng.augmented_batch().cpu().numpy()
    assert eng.augment_iteration() == 1235
    want, _p, _f, _c = _launch(x.reshape(256, 784).cuda(), AU.seed_mix(5, 0), 1234, R, EL)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("kind", ["lenet", "mlp2"])
def test_every_reader_sees_the_distorted_batch(kind):
    a, b, c = _engine(kind), _engine(kind), _engine(kind)
    a.arm_augment(*R, start_iteration=3, elastic=EL)
    c.arm_augment(*R, start_iteration=3)
    x, y = _batch(a, 2)
    a.load_batch(x, y)
    a.train_step()
    aug = a.augmented_batch()
    b.load_batch(aug.view(a.images[0].shape), y.cuda())
    b.train_step()
    torch.cuda.synchronize()
    ga, gb = a.spec.views(a.grads.cpu()), b.spec.views(b.grads.cpu())
    for q in a.spec.params:
        if kind == "lenet" or q.name.endswith("weights"):
            assert torch.equal(ga[q.name], gb[q.name]), q.name
        else:                                         # accumulated with fp32 atomics in no fixed order
            assert torch.allclose(ga[q.name], gb[q.name], rtol=1e-5, atol=1e-7), q.name
    if kind == "lenet":
        assert torch.equal(a.params, b.params) and a.loss_acc() == b.loss_acc()
    assert a.launches_per_step == b.launches_per_step + 1
    c.load_batch(x, y)
    c.train_step()
    assert a.launches_per_step == c.launches_per_step                 # the same node in the same place
    a.backend.check_error()


@pytest.mark.parametrize("kind", ["lenet", "mlp2"])
def test_host_fed_gathered_eager_and_graph_agree(kind):
    n, B = 2000, 256
    g = torch.Generator().manual_seed(8)
    table = torch.rand(n, 784, generator=g) - 0.5
    labels = torch.randint(0, 10, (n,), generator=g)
    idx = np.random.RandomState(1).randint(0, n, size=B)
    outs = []
    for feed, graph in (("host", True), ("gather", True), ("host", False), ("gather", False)):
        eng = _engine(kind, use_graph=graph)
        eng.arm_augment(*R, start_iteration=50, elastic=EL)
        if feed == "gather":
            eng.arm_train_data(table.numpy(), labels.numpy())
            eng.load_indices(idx)
        else:
            eng.load_batch(table[idx].reshape(eng.images[0].shape), labels[idx])
        eng.train_step()
        outs.append((eng.augmented_batch().cpu(), eng.params.cpu() if kind == "lenet" else None))
    want, _p, _f, _c = _launch(table[idx].cuda(), AU.seed_mix(5, 0), 50, R, EL)
    assert np.array_equal(outs[0][0].numpy(), want)
    for o in outs[1:]:
        assert torch.equal(o[0], outs[0][0])
        if kind == "lenet":
            assert torch.equal(o[1], outs[0][1])


def _run(steps, ranges, elastic, seed=9):
    """The native runner over ``steps`` packed batches: (weights, launches per step, next iteration)."""
    eng = _engine("lenet", seed=seed)
    eng.arm_augment(*ranges, elastic=elastic)
    g = torch.Generator().manual_seed(12)
    for _ in range(steps):
        ev, _lb, _s = eng.step_packed(eng.pack_batch(torch.rand(256, 784, generator=g) - 0.5,
                                                     torch.randint(0, 10, (256,), generator=g)))
        ev.synchronize()
    torch.cuda.synchronize()
    eng.backend.check_error()
    eng._leave_native_runner()
    return eng.params.cpu(), eng.launches_per_step, (eng.augment_iteration() if eng._aug is not None else None)


def test_native_runner_runs_are_reproducible():
    w1, n1, it1 = _run(30, R, EL)
    w2, n2, it2 = _run(30, R, EL)
    assert torch.equal(w1, w2) and it1 == it2 == 30 and n1 == n2
    wa, na, _ = _run(30, R, None)
    w0, n0, _ = _run(30, ZERO, AU.Elastic(0.0, 4.0))               # alpha 0 and no affine range: off
    assert na == n1 == n0 + 1 and not torch.equal(wa, w1)
    we, ne, ite = _run(30, ZERO, EL)                               # alpha alone turns augmentation on
    assert ne == n1 and ite == 30 and not torch.equal(we, w0)


def test_counter_advances_once_per_iteration_with_k_greater_than_n():
    eng = _engine("lenet", k=4)
    assert eng._kgtn_k == 4
    eng.arm_augment(*R, start_iteration=100, elastic=EL)
    x, y = _batch(eng, 6)
    seen = []
    for _ in range(8):
        eng.load_batch(x, y)
        eng.train_step()
        seen.append(eng.augmented_batch().cpu())
    assert eng.augment_iteration() == 108
    for i in range(8):
        for j in range(i):
            assert not torch.equal(seen[i], seen[j]), (i, j)
    want, _p, _f, _c = _launch(x.reshape(256, 784).cuda(), AU.seed_mix(5, 0), 107, R, EL)
    assert np.array_equal(seen[-1].numpy(), want)
    eng.backend.check_error()


def test_evaluation_is_never_augmented():
    eng = _engine("lenet")
    g = torch.Generator().manual_seed(3)
    vx, vy = torch.rand(3000, 28, 28, 1, generator=g) - 0.5, torch.randint(0, 10, (3000,), generator=g)
    eng.arm_eval(vx.numpy(), vy.numpy())
    eng.arm_augment(8.0, 90.0, 0.5, elastic=EL)
    for s in range(5):
        eng.load_batch(*_batch(eng, 10 + s))
        eng.train_step()
    eng.enqueue_eval()
    torch.cuda.synchronize()
    rec = eng.eval_record()
    ev = eng.evaluate(vx, vy)
    eng.arm_augment(0.0, 0.0, 0.0)
    plain = eng.run_eval()
    assert rec[3:] == plain[3:] and rec[0] == plain[0]
    assert ev == eng.evaluate(vx, vy)


# ---- trajectories ------------------------------------------------------------------------------------------------------
def _trajectory(eng, be, B, steps, k=1, ranges=R, elastic=EL, start=STEP0):
    from distributedmnist_b200.ops import trajectory as T
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.schedule import LearningRateSchedule
    sched = LearningRateSchedule(0.05, 1, 0.999)
    eng.attach_optimizer(SyncReplicasOptimizer(be, sched, k, 1))
    eng.arm_augment(*ranges, start_iteration=start, elastic=elastic)
    be.set_global_step(STEP0)
    if k > 1:
        be.kgtn_arm()
    rec = T.StepRecorder(eng)
    gen = torch.Generator().manual_seed(B)
    shape = (B, 28, 28) if hasattr(eng, "h_part") else (B, 784)
    batches = [(torch.rand(*shape, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen)) for _ in range(steps)]
    for x, y in batches:
        eng.load_batch(x.numpy(), y.numpy())
        eng.train_step()
        rec.record()
    torch.cuda.synchronize()
    be.check_error()
    upd = T.update_of(eng, sched, STEP0, start)
    assert upd["elastic"] == elastic and upd["aug"] == (ranges, AU.seed_mix(SEED, 0))
    if hasattr(eng, "h_part"):
        res = T.lenet_trajectory_results("t", eng.spec, rec.init, rec.records, batches, upd, eng.seed, eng.rank,
                                         eng.keep_prob)
    else:
        res = T.mlp_trajectory_results("t", eng.spec, rec.init, rec.records, batches, upd)
    worst = T.worst_by_stage("t", res)
    print("\nTRAJECTORY B%d k%d %s" % (B, k, json.dumps(worst, sort_keys=True)))
    for p in ("iteration_minus_1", "iteration_plus_1", "next_rank", "swapped_components", "no_field", "sigma_1.25"):
        assert "augment.premise.%s_detectable" % p in worst
    bad = T.failures(res)
    assert not bad, "%d of %d checks failed, first: %s" % (len(bad), len(res), bad[:20])


def _backend():
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    return FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))


@pytest.mark.parametrize("B,k", [(37, 1), (256, 1), (128, 4)])
def test_lenet_elastic_trajectory(B, k, monkeypatch):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    be = _backend()
    eng = CudaLeNetEngine(B, be, seed=SEED, rank=0, keep_prob=0.5, use_graph=True)
    _trajectory(eng, be, B, 8 if k > 1 else 6, k=k)


def test_lenet_elastic_only_counter_wrapping_trajectory(monkeypatch):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    be = _backend()
    eng = CudaLeNetEngine(128, be, seed=SEED, rank=0, keep_prob=0.5, use_graph=True)
    _trajectory(eng, be, 128, 6, ranges=ZERO, elastic=AU.Elastic(8.0, 2.0), start=2 ** 32 - 3)


def test_mlp2_elastic_trajectory(monkeypatch):
    from distributedmnist_b200.engine_cuda import CudaMlpEngine
    monkeypatch.setenv("DMNIST_BUCKET", "2")
    be = _backend()
    eng = CudaMlpEngine("mlp2", 128, be, hidden=1024, seed=SEED, use_graph=True)
    _trajectory(eng, be, 128, 6)
