"""Random affine augmentation on the GPU (csrc/augment.cu): the kernel's draws against the numpy emulation bit for bit, its
pixels against the float64 warp within a derived bound, the wiring of the augmented buffer into every reader of the training
images (lenet and mlp2), host-fed and gathered slots, graph replay and eager launch, reproducibility, the iteration counter
(K > N and restarts), evaluation without augmentation, and the step graph with augmentation off.  One replica only."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from distributedmnist_b200 import augment as AU

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _lib():
    from distributedmnist_b200.ops.lib import load
    return load()


def _counter(it):
    return torch.from_numpy(np.array([it & 0xFFFFFFFF, 0], dtype=np.uint32).view(np.int32)).cuda()


def _launch(src, mix, it, r):
    """One eager launch on ``src`` [B, 784] (device): (images, params_out, counter words) on the host."""
    from distributedmnist_b200.ops.lib import stream_ptr
    B = src.shape[0]
    dst = torch.full((B, 784), float("nan"), device="cuda")
    params = torch.full((B, 8), float("nan"), device="cuda")
    ctr = _counter(it)
    _lib().dm_augment_affine(src, dst, B, ctr, mix, *(float(v) for v in r), params, stream_ptr())
    torch.cuda.synchronize()
    return dst.cpu().numpy(), params.cpu().numpy(), ctr.cpu().numpy().view(np.uint32)


def _images(B, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 784, generator=g) - 0.5


# ---- the kernel --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [1, 96, 256, 8192])
def test_draws_equal_the_numpy_emulation(B):
    src = _images(B, B).cuda()
    r = AU.Ranges(8.0, 180.0, 0.5)
    for seed, rank, it in ((66478, 0, 0), (7, 3, 12345), (1, 1, 2 ** 32 - 1), (99, 7, 2 ** 31)):
        mix = AU.seed_mix(seed, rank)
        _img, p, ctr = _launch(src, mix, it, r)
        u = AU.uniforms(mix, it, B)
        assert np.array_equal(p[:, :4], u.astype(np.float32)), (seed, rank, it)
        assert ctr[0] == (it + 1) & 0xFFFFFFFF and ctr[1] == 0                 # advanced once, ticket left at 0
        # the coefficients: the float64 ones rounded once to fp32 (sin / cos may differ in the last double bits)
        want = np.stack(AU.coefficients(u, r), axis=1)
        assert np.all(np.abs(p[:, 4:].astype(np.float64) - want) <= 2.0 ** -23 * np.abs(want) + 1e-300)


def _pixel_bound(p):
    """Per-pixel bound on |kernel - float64 warp of the kernel's own fp32 coefficients| (params_out columns 4..7),
    [B, 784]: see ``selfcheck.augment_pixel_bound``."""
    from distributedmnist_b200.ops.selfcheck import augment_pixel_bound
    return augment_pixel_bound(p[:, 4:8])


@pytest.mark.parametrize("r", [AU.Ranges(8.0, 180.0, 0.9), AU.Ranges(30.0, 10.0, 0.5), AU.Ranges(2.0, 15.0, 0.1),
                               AU.Ranges(0.0, 0.0, 0.0)], ids=["wide", "off-image", "typical", "zero"])
def test_pixels_are_the_float64_warp_within_the_bound(r):
    B = 4096
    src = _images(B, 3)
    mix = AU.seed_mix(5, 2)
    got, p, _ = _launch(src.cuda(), mix, 77, r)
    want = AU.warp(src.numpy(), *(p[:, k].astype(np.float64) for k in range(4, 8))).reshape(B, 784)
    err = np.abs(got.astype(np.float64) - want)
    bound = _pixel_bound(p)
    worst = np.unravel_index(np.argmax(err / bound), err.shape)
    assert np.all(err <= bound), "row %d pixel %d: error %g > bound %g" % (worst[0], worst[1], err[worst], bound[worst])
    theta, s = np.degrees(np.arctan2(p[:, 5], p[:, 4])), 1.0 / np.hypot(p[:, 4], p[:, 5])
    if r == AU.Ranges(0.0, 0.0, 0.0):
        assert np.array_equal(got, src.numpy())
    if r.max_rotation == 180.0:                     # the draws reach rotations near +-180 degrees and zooms near 1 +- S
        assert np.abs(theta).max() > 179.0 and s.min() < 0.11 and s.max() > 1.89
    if r.max_shift == 30.0:                         # shifts that move the whole image off: background everywhere
        full = np.all(got == AU.BACKGROUND, axis=1)
        assert full.sum() > 50 and np.array_equal(full, np.all(want == AU.BACKGROUND, axis=1))


def _grid_edge_batches():
    """The batch sizes where the grid logic changes: one row; around 4 CTAs per SM (grid = min(4 SMs, B)); 32 rows in
    every CTA of 4 per SM and one row more, where the grid grows to ceil(B / 32); and 40000 rows."""
    sms = int(_lib().dm_num_sms())
    return [1, 4 * sms - 1, 4 * sms, 4 * sms + 1, 128 * sms, 128 * sms + 1, 40000]


def test_grid_edges_draws_pixels_rows_and_counter():
    """At each grid edge: the draws bit for bit, the pixels within the bound, every row of the NaN-filled output written,
    and the counter advanced once with the ticket back at 0."""
    r = AU.Ranges(8.0, 180.0, 0.5)
    mix = AU.seed_mix(11, 1)
    for B in _grid_edge_batches():
        src = _images(B, 1000 + B)
        it = 2 ** 32 - 1 if B % 2 else 4321
        got, p, ctr = _launch(src.cuda(), mix, it, r)
        assert np.array_equal(p[:, :4], AU.uniforms(mix, it, B).astype(np.float32)), B
        assert not np.isnan(got).any(), (B, np.flatnonzero(np.isnan(got).any(axis=1))[:10])
        want = AU.warp(src.numpy(), *(p[:, k].astype(np.float64) for k in range(4, 8))).reshape(B, 784)
        err, bound = np.abs(got.astype(np.float64) - want), _pixel_bound(p)
        assert np.all(err <= bound), (B, float((err / bound).max()))
        assert ctr.tolist() == [(it + 1) & 0xFFFFFFFF, 0], (B, ctr)


def test_argument_checks():
    from distributedmnist_b200.ops.lib import KernelLibraryError, stream_ptr
    lib, src = _lib(), torch.zeros(4, 784, device="cuda")
    dst, ctr = torch.zeros_like(src), _counter(0)
    for args in ((src, dst, 0, ctr, 1, 1.0, 1.0, 0.1), (src, dst, 4, None, 1, 1.0, 1.0, 0.1),
                 (src, dst, 4, ctr, 1, 1.0, 1.0, 1.0), (src, dst, 4, ctr, 1, -1.0, 1.0, 0.1),
                 (src, dst, 4, ctr, 1, float("nan"), 1.0, 0.1), (src, dst, 4, ctr, 1, 1.0, float("inf"), 0.1)):
        with pytest.raises(KernelLibraryError):
            lib.dm_augment_affine(*args, None, stream_ptr())
    torch.cuda.synchronize()
    assert ctr.cpu().tolist() == [0, 0]


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
    B = eng.batch_size
    return torch.rand(*eng.images[0].shape, generator=g) - 0.5, torch.randint(0, 10, (B,), generator=g)


R = AU.Ranges(3.0, 20.0, 0.15)


def test_engine_draws_start_at_the_armed_iteration():
    eng = _engine("lenet")
    eng.arm_augment(*R, start_iteration=1234)
    x, y = _batch(eng, 1)
    eng.load_batch(x, y)
    eng.forward_backward(0)                         # captures the graph: its warm-up launch must not consume draws
    got = eng.augmented_batch().cpu().numpy()
    assert eng.augment_iteration() == 1235
    want, _p, _c = _launch(x.reshape(256, 784).cuda(), AU.seed_mix(5, 0), 1234, R)
    assert np.array_equal(got, want)


def test_lenet_every_reader_sees_the_augmented_batch():
    a, b = _engine("lenet"), _engine("lenet")
    a.arm_augment(*R, start_iteration=3)
    x, y = _batch(a, 2)
    a.load_batch(x, y)
    a.forward_backward(0)
    aug = a.augmented_batch()
    assert not torch.equal(aug.cpu(), x.reshape(256, 784))
    b.load_batch(aug.view(256, 28, 28), y.cuda())
    b.forward_backward(0)
    torch.cuda.synchronize()
    assert torch.equal(a.grads, b.grads)                  # conv1 forward and conv1 wgrad both read the augmented images
    # one full training step each: the same update
    a.load_batch(x, y)
    a.train_step()
    b.load_batch(a.augmented_batch().view(256, 28, 28), y.cuda())
    b.train_step()
    torch.cuda.synchronize()
    assert torch.equal(a.params, b.params) and torch.equal(a.grads, b.grads)
    assert a.loss_acc() == b.loss_acc()
    assert a.launches_per_step == b.launches_per_step + 1
    a.backend.check_error()


def test_mlp2_reads_the_augmented_batch():
    a, b = _engine("mlp2"), _engine("mlp2")
    a.arm_augment(*R, start_iteration=3)
    x, y = _batch(a, 4)
    a.load_batch(x, y)
    a.forward_backward(0)
    b.load_batch(a.augmented_batch(), y.cuda())
    b.forward_backward(0)
    torch.cuda.synchronize()
    ga, gb = a.spec.views(a.grads.cpu()), b.spec.views(b.grads.cpu())
    for q in a.spec.params:
        if q.name.endswith("weights"):
            assert torch.equal(ga[q.name], gb[q.name]), q.name
        else:                                         # accumulated with fp32 atomics in no fixed order
            assert torch.allclose(ga[q.name], gb[q.name], rtol=1e-5, atol=1e-7), q.name
    assert a.launches_per_step == b.launches_per_step + 1


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
        eng.arm_augment(*R, start_iteration=50)
        if feed == "gather":
            eng.arm_train_data(table.numpy(), labels.numpy())
            eng.load_indices(idx)
        else:
            eng.load_batch(table[idx].reshape(eng.images[0].shape), labels[idx])
        eng.train_step()
        outs.append((eng.augmented_batch().cpu(), eng.params.cpu() if kind == "lenet" else None))
    for o in outs[1:]:
        assert torch.equal(o[0], outs[0][0])
        if kind == "lenet":
            assert torch.equal(o[1], outs[0][1])


def _run(steps, ranges, seed=9):
    eng = _engine("lenet", seed=seed)
    if ranges is not None:
        eng.arm_augment(*ranges)
    g = torch.Generator().manual_seed(12)
    for _ in range(steps):
        buf = eng.pack_batch(torch.rand(256, 784, generator=g) - 0.5, torch.randint(0, 10, (256,), generator=g))
        ev, _lb, _s = eng.step_packed(buf)          # the native runner replays the graphs
        ev.synchronize()
    torch.cuda.synchronize()
    eng.backend.check_error()
    eng._leave_native_runner()
    return eng.params.cpu(), eng.launches_per_step, (eng.augment_iteration() if eng._aug is not None else None)


def test_runs_are_reproducible_and_off_changes_nothing():
    w1, n1, it1 = _run(50, R)
    w2, n2, it2 = _run(50, R)
    assert torch.equal(w1, w2) and it1 == it2 == 50
    w0, n0, _ = _run(50, None)
    wz, nz, _ = _run(50, AU.Ranges(0.0, 0.0, 0.0))
    assert torch.equal(w0, wz) and n0 == nz and n1 == n0 + 1
    assert not torch.equal(w0, w1)


def test_counter_advances_once_per_iteration_with_k_greater_than_n():
    eng = _engine("lenet", k=4)
    assert eng._kgtn_k == 4
    eng.arm_augment(*R, start_iteration=100)
    x, y = _batch(eng, 6)
    seen = []
    for _ in range(8):                              # two global steps of four iterations each
        eng.load_batch(x, y)
        eng.train_step()
        seen.append(eng.augmented_batch().cpu())
    assert eng.augment_iteration() == 108
    for i in range(8):
        for j in range(i):
            assert not torch.equal(seen[i], seen[j]), (i, j)      # the same batch, never the same draws
    want, _p, _c = _launch(x.reshape(256, 784).cuda(), AU.seed_mix(5, 0), 107, R)
    assert np.array_equal(seen[-1].numpy(), want)
    eng.backend.check_error()


def test_evaluation_is_never_augmented():
    eng = _engine("lenet")
    g = torch.Generator().manual_seed(3)
    vx, vy = torch.rand(3000, 28, 28, 1, generator=g) - 0.5, torch.randint(0, 10, (3000,), generator=g)
    eng.arm_eval(vx.numpy(), vy.numpy())
    eng.arm_augment(8.0, 90.0, 0.5)
    for s in range(5):
        eng.load_batch(*_batch(eng, 10 + s))
        eng.train_step()
    eng.enqueue_eval()                              # the in-training pass (graph) after augmented steps
    torch.cuda.synchronize()
    rec = eng.eval_record()
    ev = eng.evaluate(vx, vy)
    eng.arm_augment(0.0, 0.0, 0.0)
    plain = eng.run_eval()
    assert rec[3:] == plain[3:] and rec[0] == plain[0]
    assert ev == eng.evaluate(vx, vy)


def _train_twice(tmp_path, *extra):
    """A 12-step lenet run with augmentation and its restart to 20 steps: (first log, restart log, restored step)."""
    train_dir = str(tmp_path / "train")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="0")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    logs = []
    for steps in (12, 20):
        tr = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_distributed_train.py"), "--job_name=worker",
                             "--task_id=0", "--worker_hosts=localhost:1234", "--batch_size=128", "--max_steps=%d" % steps,
                             "--augment_max_shift=2", "--augment_max_rotation=10", "--save_interval_secs=1000",
                             "--train_dir=" + train_dir] + list(extra), env=env, capture_output=True, text=True,
                            timeout=600)
        logs.append(tr.stdout + tr.stderr)
        assert tr.returncode == 0, logs[-1][-3000:]
    assert "draws from iteration 0;" in logs[0]
    m = re.search(r"Restored model from \S+ at step=(\d+)", logs[1])
    assert m and int(m.group(1)) > 0, logs[1][-2000:]
    losses = [float(x) for x in re.findall(r"loss = ([0-9.]+),", logs[1])]
    assert losses and np.all(np.isfinite(losses))
    return logs[0], logs[1], int(m.group(1))


def test_restart_draws_from_the_restored_step(tmp_path):
    _first, restart, g = _train_twice(tmp_path)
    assert "draws from iteration %d;" % g in restart


def test_restart_with_k4_draws_past_the_restored_iterations(tmp_path):
    """K = 4 on one replica: the global step g the restart restores took iterations 0 .. 4g - 1, so it draws from 4g."""
    _first, restart, g = _train_twice(tmp_path, "--num_replicas_to_aggregate=4")
    assert "draws from iteration %d;" % (4 * g) in restart
