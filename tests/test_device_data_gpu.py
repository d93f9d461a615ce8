"""--device_data on the GPU: the training set lives in device memory and a step's input slot is gathered from B row indices
(csrc/batch_gather.cu).  The gathered slot is byte for byte the packed batch of the same rows, the native runner and the
torch-dispatched path fill identical slots, and training through ``train.train`` computes bit for bit what the host-fed
loop computes."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _backend():
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    return FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))


def _engine(kind, B, use_graph=False):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine, CudaMlpEngine
    if kind == "lenet":
        return CudaLeNetEngine(B, _backend(), seed=7, use_graph=use_graph)
    return CudaMlpEngine("mlp2", B, _backend(), seed=7, use_graph=use_graph)


def _table(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 28, 28, 1, generator=g) - 0.5, torch.randint(0, 10, (n,), generator=g)


def _indices(n, B, seed):
    """Random rows of [0, n) that include 0 and n - 1 and (for B > 2) a repeated row."""
    rng = np.random.RandomState(seed)
    idx = rng.randint(0, n, size=B)
    idx[0] = n - 1
    if B > 1:
        idx[-1] = 0
    if B > 2:
        idx[B // 2] = idx[1]
    return idx


@pytest.mark.parametrize("kind", ["lenet", "mlp2"])
@pytest.mark.parametrize("B", [1, 64, 256, 1000])
def test_gathered_slot_equals_the_packed_batch_byte_for_byte(kind, B):
    n = 3001
    images, labels = _table(n, B)
    eng = _engine(kind, B)
    eng.arm_train_data(images.numpy(), labels.numpy())
    for k in range(3):                                       # both slots, the first one twice
        idx = _indices(n, B, 100 * B + k)
        eng.load_indices(idx)
        torch.cuda.synchronize()
        ref = eng.pack_batch(images[torch.from_numpy(idx)], labels[torch.from_numpy(idx)], pin=False)
        got = eng.in_dev[eng._slot].cpu()
        assert got.dtype == ref.dtype == torch.uint8 and torch.equal(got, ref), (kind, B, k)
        assert tuple(eng.images[eng._slot].shape) == ((B, 28, 28) if kind == "lenet" else (B, 784))


def test_out_of_range_rows_are_refused_before_anything_is_enqueued():
    eng = _engine("lenet", 8)
    images, labels = _table(100, 1)
    eng.arm_train_data(images, labels)
    loaded = eng._loaded
    for bad in ([0] * 7 + [100], [-1] + [0] * 7, [0] * 7):
        with pytest.raises(ValueError):
            eng.load_indices(np.array(bad))
        with pytest.raises(ValueError):
            eng.step_indices(np.array(bad))
    with pytest.raises(ValueError):
        eng.load_indices(np.zeros(8, np.float32))
    assert eng._loaded == loaded


def _train_steps(kind, monkeypatch, native: bool, steps=12):
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.schedule import LearningRateSchedule
    monkeypatch.setenv("DMNIST_NATIVE_RUNNER", "1" if native else "0")
    B, n = 256, 2000
    images, labels = _table(n, 5)
    eng = _engine(kind, B, use_graph=True)
    eng.attach_optimizer(SyncReplicasOptimizer(eng.backend, LearningRateSchedule(0.05, 20, 0.7), 1, 1))
    eng.arm_train_data(images, labels)
    slots, losses = [], []
    for s in range(steps):
        idx = torch.from_numpy(_indices(n, B, s).astype(np.int32)).pin_memory()
        ev, buf, _seq = eng.step_indices(idx)
        ev.synchronize()
        torch.cuda.synchronize()
        slots.append(eng.in_dev[eng._slot].clone())
        losses.append((float(buf[0]), float(buf[1])))
    eng.backend.check_error()
    runner = eng._runner is not None
    out = (slots, losses, eng.params.clone(), runner)
    eng._leave_native_runner()
    return out


@pytest.mark.parametrize("kind", ["lenet", "mlp2"])
def test_native_runner_and_torch_dispatched_path_fill_identical_slots(kind, monkeypatch):
    s1, l1, p1, r1 = _train_steps(kind, monkeypatch, native=True)
    s0, l0, p0, r0 = _train_steps(kind, monkeypatch, native=False)
    assert r1 and not r0
    assert len(s1) == len(s0) and all(torch.equal(a, b) for a, b in zip(s1, s0))
    if kind == "lenet":            # the MLP kernels sum loss and bias gradients with fp32 atomics: not bit-reproducible
        assert l1 == l0 and torch.equal(p1, p0)


# ---- training through train.train (tests/_device_data_worker.py) -------------------------------------------------------
def _train_runs(tmp_path, name, n, extra, rows=4096):
    from distributedmnist_b200.parallel.launcher import run_replicas
    d = tmp_path / name
    codes = run_replicas([os.path.join(ROOT, "tests", "_device_data_worker.py"), str(d / "rank_RANK"), str(rows),
                          "--train_dir=%s" % (d / "train_dir"), "--batch_size=256", "--initial_learning_rate=0.05",
                          "--save_interval_secs=1000", "--save_results_period=1", "--log_every=100", "--seed=11"]
                         + list(extra), n, timeout=900, out_dir=str(d / "out"))
    logs = "\n".join(open(os.path.join(d, "out", f)).read()[-2000:] for f in sorted(os.listdir(d / "out")))
    assert codes == [0] * n, (name, logs)
    out = []
    for r in range(n):
        with open(str(d / ("rank_%d.json" % r))) as f:
            meta = json.load(f)
        out.append((np.load(str(d / ("rank_%d.npy" % r))), meta))
    return out


def _assert_same(a, b, what):
    (pa, ma), (pb, mb) = a, b
    assert ma["final_step"] == mb["final_step"], what
    assert ma["steps"] == mb["steps"] and ma["losses"] == mb["losses"], what
    assert ma["rows"] == mb["rows"], what
    assert np.array_equal(pa.view(np.uint32), pb.view(np.uint32)), what + ": final parameters differ"


@pytest.mark.parametrize("flags", [
    ("--model=lenet", "--max_steps=300"),                                       # K = N = 1: bucketed aggregation
    ("--model=lenet", "--max_steps=75", "--num_replicas_to_aggregate=4"),       # K > N: count trigger, 300 batches
    ("--model=lenet", "--max_steps=300", "--pipeline_steps=false"),             # load_indices instead of step_indices
], ids=["lenet", "lenet_k4", "lenet_unpipelined"])
def test_training_is_bit_identical_to_the_host_fed_loop(tmp_path, flags):
    host = _train_runs(tmp_path, "host", 1, flags)
    dev = _train_runs(tmp_path, "device", 1, list(flags) + ["--device_data=true"])
    assert len(host[0][1]["losses"]) >= 290
    _assert_same(host[0], dev[0], "--device_data vs host-fed")


def test_mlp2_training_matches_the_host_fed_loop(tmp_path):
    """mlp2 sums its loss and bias gradients with fp32 atomics, so two host-fed runs already differ in the last bits: the
    runs agree to a tolerance here (the slots they train on are byte-identical, see above)."""
    flags = ("--model=mlp2", "--max_steps=300")
    (ph, mh), = _train_runs(tmp_path, "host", 1, flags)
    (pd, md), = _train_runs(tmp_path, "device", 1, list(flags) + ["--device_data=true"])
    assert mh["final_step"] == md["final_step"] and mh["steps"] == md["steps"]
    lh, ld = np.array(mh["losses"]), np.array(md["losses"])
    assert np.allclose(lh, ld, rtol=1e-3, atol=1e-4), float(np.abs(lh - ld).max())
    ah, ad = np.array(mh["rows"])[:, 0], np.array(md["rows"])[:, 0]
    assert np.abs(ah - ad).max() <= 2.0 / 256, float(np.abs(ah - ad).max())
    diff = float(np.abs(ph - pd).max())
    assert diff <= 1e-3 * float(np.abs(ph).max()), diff


@pytest.mark.multigpu
def test_two_replicas_stay_bit_identical_and_match_the_host_fed_run(tmp_path):
    flags = ("--model=lenet", "--max_steps=200")
    host = _train_runs(tmp_path, "host", 2, flags)
    dev = _train_runs(tmp_path, "device", 2, list(flags) + ["--device_data=true"])
    assert np.array_equal(dev[0][0].view(np.uint32), dev[1][0].view(np.uint32)), "the replicas diverged"
    for r in range(2):
        _assert_same(host[r], dev[r], "rank %d" % r)
