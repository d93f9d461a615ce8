"""L2 weight decay on the GPU (``--weight_decay``): the decayed epilogues of the fc1 weight-gradient GEMM (fp32 and bf16
stores) and of fc2_wgrad against an exact single-rounding emulation of ``fma(lambda, w, plain)``, the W^2 partials and the
loss word, the lenet engine's arena after ``forward_backward`` and a bucketed / single-kernel ``train_step``, graph size and
bit-identical training with the decay off, and short one-replica runs in the cdf, K > N and interval modes.  No run with
more than one replica is made here."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from distributedmnist_b200.ops import aggrefs as A
from distributedmnist_b200.ops import refs as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LAMS = (np.float32(5e-4), np.float32(0.0123))
FC = ("fc1_weights", "fc1_biases", "fc2_weights", "fc2_biases")


def _lib():
    from distributedmnist_b200.ops.lib import load
    return load()


def _fma_bits(lam, w, plain):
    return A.bits(A.fma_f32(np.float32(lam), A.f32(w), A.f32(plain)))


def _assert_bits(what, got, want_bits):
    got = A.bits(got)
    bad = np.flatnonzero(got.reshape(-1) != want_bits.reshape(-1))
    assert bad.size == 0, "%s: %d of %d differ, first at %d" % (what, bad.size, got.size, bad[0])


def _sumsq(*arrays):
    return float(sum((A.f32(a).astype(np.float64) ** 2).sum() for a in arrays))


# ---- kernels -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["grid", "rand"])
def test_fc1_wgrad_epilogues_are_fma_of_the_plain_accumulator(kind):
    from distributedmnist_b200.ops import gemm as G
    from distributedmnist_b200.ops.lib import stream_ptr
    lib, B = _lib(), 256
    g = torch.Generator().manual_seed(31)
    if kind == "grid":             # the exact input grid of ops/refs.py: every sum is exact in fp32
        a2, dh = R.grid(g, (B, 3136), 0, 2), R.grid(g, (B, 512), -64, 64, 64)
    else:
        a2, dh = torch.rand(B, 3136, generator=g), torch.randn(B, 512, generator=g) * 0.01
    a2, dh = a2.to(torch.bfloat16).cuda(), dh.to(torch.bfloat16).cuda()
    w = (torch.randn(3136, 512, generator=g) * 0.1).cuda()
    plain = torch.empty(3136, 512, device="cuda")
    G.gemm_bf16_raw(a2, dh, plain, 3136, 512, B, 3136, 512, 512, True, True, G.EPI_STORE_F32, bn=128)
    n = int(lib.dm_gemm_decay_ctas(3136, 512))
    assert n == 25 * 4
    want_r = _sumsq(w.cpu())
    for lam in LAMS:
        out = torch.full((3136, 512), float("nan"), device="cuda")
        out16 = torch.zeros(3136, 512, dtype=torch.bfloat16, device="cuda")
        ws = torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")
        lib.dm_gemm_bf16_decay(a2, dh, out, 3136, 512, B, 3136, 512, 512, 0, w, float(lam), ws, stream_ptr())
        torch.cuda.synchronize()
        want = A.fma_f32(lam, A.f32(w), A.f32(plain))
        _assert_bits("fp32 epilogue lambda=%g" % lam, out, A.bits(want))
        assert abs(float(ws.sum().item()) - want_r) <= 1e-12 * want_r
        ws.fill_(float("nan"))
        lib.dm_gemm_bf16_decay(a2, dh, out16, 3136, 512, B, 3136, 512, 512, 1, w, float(lam), ws, stream_ptr())
        torch.cuda.synchronize()
        got16 = out16.view(torch.int16).cpu().numpy().view(np.uint16)
        assert np.array_equal(got16, A.bf16_bits(want)), "bf16 epilogue lambda=%g" % lam
        assert abs(float(ws.sum().item()) - want_r) <= 1e-12 * want_r


def test_fc2_wgrad_variant_is_fma_of_the_plain_gradients():
    from distributedmnist_b200.ops.lib import stream_ptr
    lib, B = _lib(), 256
    g = torch.Generator().manual_seed(32)
    h = torch.relu(torch.randn(B, 512, generator=g)).cuda()
    dl = torch.zeros(B, 12)
    dl[:, :10] = torch.randn(B, 10, generator=g) * 0.01
    dl = dl.cuda()
    dh = (torch.randn(B, 512, generator=g) * 0.01).to(torch.bfloat16).cuda()
    w2, b2, b1 = ((torch.randn(*s, generator=g) * 0.1).cuda() for s in ((512, 10), (10,), (512,)))
    outs = [[torch.zeros(512, 10, device="cuda"), torch.zeros(10, device="cuda"), torch.zeros(512, device="cuda")]
            for _ in range(2)]
    lib.dm_fc2_wgrad(h, dl, dh, *outs[0], B, stream_ptr())
    n = int(lib.dm_fc2_wgrad_decay_ctas())
    want_r = _sumsq(w2.cpu(), b2.cpu(), b1.cpu())
    for lam in LAMS:
        ws = torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")
        lib.dm_fc2_wgrad_decay(h, dl, dh, *outs[1], B, w2, b2, b1, float(lam), ws, stream_ptr())
        torch.cuda.synchronize()
        for name, got, plain, v in zip(("g_w2", "g_b2", "g_b1"), outs[1], outs[0], (w2, b2, b1)):
            _assert_bits("%s lambda=%g" % (name, lam), got, _fma_bits(lam, v.cpu(), plain.cpu()))
        assert abs(float(ws.sum().item()) - want_r) <= 1e-12 * want_r


# ---- the lenet engine --------------------------------------------------------------------------------------------------
def _engine(B=256, seed=5, lr=0.05):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaLeNetEngine(B, be, seed=seed, use_graph=True)
    sched = LearningRateSchedule(lr, 4, 0.7)
    eng.attach_optimizer(SyncReplicasOptimizer(be, sched, 1, 1))
    return eng, be, sched


def _batch(eng, seed):
    g = torch.Generator().manual_seed(seed)
    B = eng.batch_size
    return torch.rand(B, 28, 28, generator=g) - 0.5, torch.randint(0, 10, (B,), generator=g)


def _views(eng, flat):
    return eng.spec.views(flat.cpu())


def _device_r(eng, w):
    v = eng.spec.views(w)
    return _sumsq(*(v[n] for n in FC)) / 2


def test_forward_backward_arena_and_loss_word():
    lam = LAMS[0]
    eng, be, _ = _engine()
    eng.load_batch(*_batch(eng, 1))
    eng.forward_backward(0)
    plain, plain_loss = eng.grads.cpu(), eng.loss_acc()
    w = eng.params.cpu()
    eng.arm_weight_decay(float(lam))
    runs = []
    for _ in range(2):
        eng.forward_backward(0)
        runs.append((eng.grads.cpu(), eng.loss_acc(), eng.weight_decay_r()))
    (got, loss, r), (got2, loss2, r2) = runs
    assert A.bits(got).tobytes() == A.bits(got2).tobytes()
    assert np.float32(loss[0]).tobytes() == np.float32(loss2[0]).tobytes() and r == r2       # two runs, the same words
    pv, gv, wv = _views(eng, plain), _views(eng, got), _views(eng, w)
    for q in eng.spec.params:
        if q.name in FC:
            _assert_bits(q.name, gv[q.name], _fma_bits(lam, wv[q.name], pv[q.name]))
        else:
            assert torch.equal(gv[q.name], pv[q.name]), q.name
    want_r = _device_r(eng, w)
    assert abs(r - want_r) <= 1e-12 * want_r
    want_loss = np.float32(plain_loss[0]) + np.float32(float(lam) * r)
    assert np.float32(loss[0]).tobytes() == want_loss.tobytes()
    assert loss[1] == plain_loss[1]                                   # training accuracy unchanged
    be.check_error()


@pytest.mark.parametrize("bucket", ["2", "0"])
def test_train_step_applies_the_decayed_gradient(bucket, monkeypatch):
    lam = LAMS[0]
    monkeypatch.setenv("DMNIST_BUCKET", bucket)
    eng, be, sched = _engine()
    assert eng._bucket_v2 == (bucket == "2")
    be.set_global_step(40)
    eng.load_batch(*_batch(eng, 2))
    eng.forward_backward(0)                      # the plain gradient of the batch and weights train_step will see
    torch.cuda.synchronize()
    plain, w = eng.grads.cpu(), eng.params.cpu()
    eng.arm_weight_decay(float(lam))
    step = be.device_epoch
    eng.train_step()
    torch.cuda.synchronize()
    scale = A.step_scale(sched, step, 1)
    grads = eng.grads.cpu()
    b, e = eng._bucket_early
    pv, gv, wv = _views(eng, plain), _views(eng, grads), _views(eng, w)
    for name in FC:
        if name == "fc1_weights" and bucket == "2":
            continue                             # exchanged through the bf16 wire buffer instead
        _assert_bits(name, gv[name], _fma_bits(lam, wv[name], pv[name]))
    if bucket == "2":
        wire = eng._g16_view.view(torch.int16).cpu().numpy().view(np.uint16).reshape(-1)
        dec = A.fma_f32(lam, A.f32(wv["fc1_weights"]), A.f32(pv["fc1_weights"])).reshape(-1)
        assert np.array_equal(wire, A.bf16_bits(dec))
        rounds = A.late_bucket_rounds_bf16(eng.spec.arena_numel, e - b, be.late_ll, be.late_bf16)
        want = A.bucket_step(A.f32(w), [A.f32(grads)], [A.f32(eng._g16_view.float()).reshape(-1)], (b, e), scale, rounds)
    else:
        want = A.fused_sync_step(A.f32(w), [A.f32(grads)], 1, scale)
    _assert_bits("weights after the step", eng.params.cpu(), A.bits(want))
    be.check_error()


def _trajectory(steps, lam):
    eng, be, _ = _engine(seed=9)
    if lam is not None:
        eng.arm_weight_decay(lam)
    g = torch.Generator().manual_seed(12)
    losses = []
    for _ in range(steps):
        buf = eng.pack_batch(torch.rand(256, 784, generator=g) - 0.5, torch.randint(0, 10, (256,), generator=g))
        ev, lb, _s = eng.step_packed(buf)
        ev.synchronize()
        losses.append(float(lb[0]))
    torch.cuda.synchronize()
    be.check_error()
    n = eng.launches_per_step
    eng._leave_native_runner()
    return eng.params.cpu(), losses, n


def test_off_is_bit_identical_and_on_adds_one_launch():
    w_ref, l_ref, n_ref = _trajectory(20, None)
    w0, l0, n0 = _trajectory(20, 0.0)
    assert n0 == n_ref and A.bits(w0).tobytes() == A.bits(w_ref).tobytes() and l0 == l_ref
    w1, l1, n1 = _trajectory(20, float(LAMS[0]))
    assert n1 == n_ref + 1
    assert np.all(np.isfinite(l1)) and not torch.equal(w1, w_ref)


def test_mlp_engine_refuses():
    from distributedmnist_b200.engine_cuda import CudaMlpEngine
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaMlpEngine("mlp2", 64, be, hidden=64, use_graph=False)
    eng.arm_weight_decay(0.0)
    with pytest.raises(ValueError, match="implemented for lenet"):
        eng.arm_weight_decay(1e-4)


# ---- short runs of the training driver in the modes whose weights peers may rewrite ------------------------------------
@pytest.mark.parametrize("mode", [["--worker_times_cdf_method"], ["--num_replicas_to_aggregate=4"],
                                  ["--interval_method", "--interval_ms=2"]], ids=["cdf", "k4", "interval"])
def test_one_replica_modes_run_and_checkpoint_scores(mode, tmp_path):
    train_dir = str(tmp_path / "train")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="0")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    tr = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_distributed_train.py"), "--job_name=worker",
                         "--task_id=0", "--worker_hosts=localhost:1234", "--batch_size=128", "--max_steps=30",
                         "--weight_decay=5e-4", "--save_interval_secs=1000", "--train_dir=" + train_dir] + mode,
                        env=env, capture_output=True, text=True, timeout=600)
    log = tr.stdout + tr.stderr
    assert tr.returncode == 0, log[-3000:]
    assert "L2 weight decay 0.0005" in log
    losses = [float(x) for x in re.findall(r"loss = ([0-9.]+),", log)]
    assert losses and np.all(np.isfinite(losses)), log[-2000:]
    ev = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_eval.py"), "--run_once=true",
                         "--checkpoint_dir=" + train_dir, "--eval_dir=" + str(tmp_path / "eval")], env=env,
                        capture_output=True, text=True, timeout=600)
    out = ev.stdout + ev.stderr
    assert ev.returncode == 0, out[-3000:]
    assert re.search(r"Num examples: 10000  Precision @ 1: ([0-9.]+) Loss: ([0-9.]+)", out), out[-2000:]
