"""Moving average of the weights on the GPU (csrc/moving_average.cu, ``_CudaEngine.arm_moving_average``): the kernel bit for
bit against the float32 emulation, graph-replayed lenet and mlp2 steps (training unperturbed, the shadow after every step
equal to the emulation over the recorded weights), a lenet pass on the average, a device checkpoint carrying the average,
``train()`` with ``--eval_moving_average --target_accuracy``, and two replicas at K = N."""
import json
import os

import numpy as np
import pytest
import torch

from distributedmnist_b200 import moving_average as ema

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VAL = 1000


def _bits(a):
    return (a.numpy() if isinstance(a, torch.Tensor) else a).view(np.int32)


def _launch(shadow, w, g, decay, bf16=None, ranges=(0, 0, 0, 0), step_out=None):
    from distributedmnist_b200.ops.lib import load, stream_ptr
    epoch = torch.tensor([g], dtype=torch.int64, device="cuda").view(torch.int32)[:1]   # low word, little endian
    load().dm_moving_average(shadow, w, shadow.numel(), epoch, decay, step_out, bf16, *ranges, stream_ptr())
    torch.cuda.synchronize()


def _numel(model):
    from distributedmnist_b200.models import get_model
    return get_model(model)[0].arena_numel


@pytest.mark.parametrize("numel", [_numel("lenet"), _numel("mlp2"), 1001, 3, 4099], ids=["lenet", "mlp2", "1001", "3", "4099"])
def test_kernel_bit_exact_against_the_emulation(numel):
    rng = np.random.default_rng(numel)
    s = (rng.standard_normal(numel) * 0.1).astype(np.float32)
    r = (0, 0, 0, 0) if numel < 8 else (4, 4 * (numel // 8), 4 * (numel // 4) - 4 * (numel // 16), 4 * (numel // 4) - 4)
    if numel >= 16:
        s[-4:] = [0.0, -0.0, 1e-40, -3e-39]            # subnormals in the tail, outside the bf16 ranges
    shadow = torch.from_numpy(s).cuda()
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    bf = torch.zeros(numel, dtype=torch.bfloat16, device="cuda")
    for decay in (0.9, 0.999):
        for g in (0, 1, 3, 9, 10, 89, 90, 1000, 123456, 2 ** 32 - 1):
            w = (s + rng.standard_normal(numel).astype(np.float32) * 0.01).astype(np.float32)
            if numel >= 16:
                w[-4:] = [1e-40, 0.0, 2e-40, -1e-40]
            bf.zero_()
            _launch(shadow, torch.from_numpy(w).cuda(), g, decay, bf, r, step)
            s = ema.emulate(s, w, decay, g)
            got = shadow.cpu()
            assert np.array_equal(_bits(got), _bits(s)), (numel, decay, g)
            assert int(step.item()) & 0xFFFFFFFF == g
            want = torch.zeros(numel, dtype=torch.bfloat16)
            for b, e in ((r[0], r[1]), (r[2], r[3])):
                want[b:e] = torch.from_numpy(s[b:e]).to(torch.bfloat16)
            assert torch.equal(bf.cpu().view(torch.int16), want.view(torch.int16)), (numel, g)
    # without weights the call only converts, and leaves the shadow and the step untouched
    bf.zero_()
    _launch(shadow, None, 7, 0.0, bf, r, step)
    assert np.array_equal(_bits(shadow.cpu()), _bits(s)) and int(step.item()) & 0xFFFFFFFF == 2 ** 32 - 1
    assert torch.equal(bf.cpu()[r[0]:r[1]].view(torch.int16), torch.from_numpy(s[r[0]:r[1]]).to(torch.bfloat16).view(torch.int16))


def test_kernel_raises_on_bad_arguments():
    from distributedmnist_b200.ops.lib import KernelLibraryError, load, stream_ptr
    lib = load()
    t = torch.zeros(64, device="cuda")
    e = torch.zeros(1, dtype=torch.int32, device="cuda")
    b = torch.zeros(64, dtype=torch.bfloat16, device="cuda")
    for decay, rg in ((1.0, (0, 0, 0, 0)), (0.0, (0, 0, 0, 0)), (0.5, (2, 8, 0, 0)), (0.5, (0, 68, 0, 0)), (0.5, (8, 4, 0, 0))):
        with pytest.raises(KernelLibraryError, match=r"code -1\b"):
            lib.dm_moving_average(t, t, 64, e, decay, None, b, *rg, stream_ptr())


def _engine(model="lenet", B=256, seed=5, decay=None):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine, CudaMlpEngine
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaLeNetEngine(B, be, seed=seed, use_graph=True) if model == "lenet" else \
        CudaMlpEngine(model, B, be, seed=seed, use_graph=True)
    eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 4, 0.7), 1, 1))
    if decay is not None:
        eng.arm_moving_average(decay)
    return eng, be


def _packed(eng, n, seed):
    g = torch.Generator().manual_seed(seed)
    B = eng.batch_size
    return [eng.pack_batch(torch.rand(B, 784, generator=g) - 0.5, torch.randint(0, 10, (B,), generator=g)) for _ in range(n)]


def _trajectory(model, steps, decay):
    eng, be = _engine(model, decay=decay)
    w0 = eng.params.cpu()
    weights, shadows = [], []
    for buf in _packed(eng, steps, 11):
        ev, _l, _s = eng.step_packed(buf)
        ev.synchronize()
        torch.cuda.synchronize()
        weights.append(eng.params.cpu())
        if decay is not None:
            shadows.append(eng.moving_average())
    be.check_error()
    n = eng.launches_per_step
    eng._leave_native_runner()
    return w0, weights, shadows, n


@pytest.mark.parametrize("model", ["lenet", "mlp2"])
def test_graph_replayed_steps_average_bit_exact_and_training_unperturbed(model):
    steps, decay = 40, 0.9
    _w0, ref, _none, n_ref = _trajectory(model, steps, None)
    w0, got, shadows, n_avg = _trajectory(model, steps, decay)
    assert n_avg == n_ref + 1                               # one node more in the step graph
    for i in range(steps):
        if model == "lenet":
            assert np.array_equal(_bits(got[i]), _bits(ref[i])), "step %d: the average perturbed training" % (i + 1)
        else:
            # mlp2 sums its bias gradients with fp32 atomics: two runs agree to rounding, not bit for bit
            assert float((got[i] - ref[i]).abs().max()) < 1e-4, (i + 1, float((got[i] - ref[i]).abs().max()))
    s = w0.numpy().copy()
    for i in range(steps):
        s = ema.emulate(s, got[i].numpy(), decay, i + 1)
        avg, step = shadows[i]
        assert step == i + 1
        assert np.array_equal(_bits(avg.cpu()), _bits(s)), "shadow after step %d differs from the emulation" % (i + 1)


def _validation():
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.flags import FLAGS
    FLAGS.reset()
    return mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True, synthetic_sizes=(4096, 2500)).validation


def test_lenet_pass_on_the_average_equals_a_pass_on_an_arena_holding_it():
    val = _validation()
    eng, be = _engine(decay=0.95)
    for buf in _packed(eng, 25, 3):
        eng.step_packed(buf)
    torch.cuda.synchronize()
    eng._leave_native_runner()
    eng.arm_eval(val.images, val.labels, moving_average=True)
    rec = eng.run_eval()
    avg, step = eng.moving_average()
    live = eng.params.clone()
    del eng
    ref, _ = _engine()
    ref.params.copy_(avg)
    ref.params_updated()
    ref.arm_eval(val.images, val.labels)
    want = ref.run_eval()
    assert rec[0] == step == 25
    assert (rec[3], rec[4], rec[5]) == (want[3], want[4], want[5]), (rec, want)
    ref.params.copy_(live)
    ref.params_updated()
    other = ref.run_eval()
    print("\naverage: %d of %d correct, loss_sum %.4f; live weights: %d correct, loss_sum %.4f"
          % (rec[4], rec[3], rec[5], other[4], other[5]))


def test_device_checkpoint_carries_the_average_of_the_same_step():
    eng, be = _engine(decay=0.9)
    eng.arm_checkpoint(snapshot=False)
    for i, buf in enumerate(_packed(eng, 12, 9)):
        eng.step_packed(buf)
        eng.enqueue_checkpoint(i & 1)
        seq, b, step = eng.checkpoint_wait()
        avg, avg_step = eng.moving_average()
        assert step == avg_step == i + 1
        assert np.array_equal(_bits(eng.ckpt_host[b]), _bits(eng.params.cpu()))
        assert np.array_equal(_bits(eng.ckpt_ema_host[b]), _bits(avg.cpu()))
    be.check_error()
    eng._leave_native_runner()


@pytest.fixture
def flags(monkeypatch):
    from distributedmnist_b200.flags import FLAGS
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    FLAGS.reset()
    yield FLAGS
    FLAGS.reset()


def _train(d, *extra, steps=300):
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import train
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % d, "--batch_size=128", "--max_steps=%d" % steps, "--eval_every_steps=10",
                 "--initial_learning_rate=0.05", "--log_every=1000", "--save_results_period=1000000",
                 "--save_interval_secs=1000", "--device_data=true", "--moving_average_decay=0.99",
                 "--eval_moving_average"] + list(extra))
    ctx = init_context(FLAGS)
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True, synthetic_sizes=(8192, VAL))
    return train(ctx, ds.train, ds.validation, FLAGS)


def test_train_eval_moving_average_target_stops_and_reports(tmp_path, flags):
    from distributedmnist_b200.checkpoint import Saver
    from distributedmnist_b200.train import STOP_MARGIN
    _train(tmp_path / "ref")
    rows = np.load(str(tmp_path / "ref" / "worker0_eval.npy"))
    early = rows[rows[:, 0] <= 250]
    best = int(early[:, 4].max())
    g = int(early[early[:, 4] == best][0, 0])
    res = _train(tmp_path / "armed", "--target_accuracy=%r" % (best / VAL))
    s = g + STOP_MARGIN
    assert res["final_step"] == s + 1
    rep = res["time_to_accuracy"]
    assert rep["reached"] and rep["global_step"] == g and rep["correct"] == best and rep["weights"] == "moving_average"
    with open(str(tmp_path / "armed" / "worker0_time_to_accuracy.json")) as f:
        assert json.load(f) == rep
    a = np.load(str(tmp_path / "armed" / "worker0_eval.npy"))
    np.testing.assert_array_equal(a[a[:, 0] <= g][:, [0, 3, 4, 5]], rows[rows[:, 0] <= g][:, [0, 3, 4, 5]])
    # the final file: weights and averages of the step in its name
    eng = res["engine"]
    state, step = Saver.restore(Saver.latest(str(tmp_path / "armed")))
    avg, avg_step = eng.moving_average()
    assert step == avg_step == s + 1
    spec = eng.spec
    m = spec.valid_mask()
    assert np.array_equal(_bits(spec.from_state_dict(state)[m]), _bits(res["params"].cpu()[m]))
    assert np.array_equal(_bits(ema.from_state_dict(spec, state)[m]), _bits(avg.cpu()[m]))
    print("\naveraged weights: target %d/%d reached at step %d, train time %.4f s" % (best, VAL, g, rep["train_time_s"]))


@pytest.mark.multigpu
def test_two_replicas_only_the_chief_averages(tmp_path):
    from distributedmnist_b200.parallel.launcher import run_replicas
    worker = os.path.join(ROOT, "tests", "_moving_average_worker.py")
    d = tmp_path / "run"
    codes = run_replicas([worker, str(d / "rank_RANK"), "--train_dir=%s" % (d / "train_dir"), "--batch_size=128",
                          "--max_steps=60", "--initial_learning_rate=0.05", "--save_interval_secs=1000", "--log_every=50",
                          "--moving_average_decay=0.99"], 2, timeout=600, out_dir=str(d / "out"))
    assert codes == [0, 0]
    meta = [json.load(open(str(d / ("rank_%d.json" % r)))) for r in range(2)]
    params = [np.load(str(d / ("rank_%d.npy" % r))) for r in range(2)]
    assert meta[0]["average"] and not meta[1]["average"]
    assert meta[0]["launches_per_step"] == meta[1]["launches_per_step"] + 1
    assert meta[0]["average_step"] == meta[0]["final_step"] == meta[1]["final_step"]
    assert np.array_equal(params[0].view(np.uint32), params[1].view(np.uint32))
