"""``--weight_decay`` on the CPU: the flag and its refusals, the decayed-variable set, one torch-engine step against
CE + lambda * R, ``train()`` unchanged with the decay off, and a short decayed run whose checkpoint the evaluator scores."""
import math
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200 import weight_decay as W
from distributedmnist_b200.engine import TorchEngine
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.models import get_model
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.train import train

STEP_LINE = re.compile(r"Worker 0: .*: step (\d+), loss = ([0-9.]+), train_acc = ([0-9.]+)")


@pytest.fixture
def clean_flags():
    FLAGS.reset()
    saved = {k: os.environ.pop(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") if k in os.environ}
    yield FLAGS
    FLAGS.reset()
    os.environ.update(saved)


def _flags(**kw):
    d = dict(weight_decay=0.0, model="lenet", backend="auto")
    d.update(kw)
    return SimpleNamespace(**d)


def _ctx(on_gpu):
    return SimpleNamespace(on_gpu=on_gpu, world_size=1, rank=0)


def test_flag_default_and_parsing(clean_flags):
    assert FLAGS.weight_decay == 0.0 and W.value(FLAGS) == 0.0
    FLAGS.parse(["--weight_decay=5e-4"])
    assert W.value(FLAGS) == float(np.float32(5e-4))
    FLAGS.parse(["--weight_decay", "0.1"])
    assert W.value(FLAGS) == float(np.float32(0.1))


@pytest.mark.parametrize("lam", [-1e-4, 1.0, 2.0, float("inf"), float("nan"), 0.99999999, 1e-50])
def test_out_of_range_values_are_refused(lam):
    with pytest.raises(ValueError, match="--weight_decay"):
        W.check_flags(_flags(weight_decay=lam), _ctx(False))


def test_gpu_path_refuses_the_mlps_and_torch_engine_takes_them():
    for model in ("mlp2", "mlp3"):
        with pytest.raises(ValueError, match="implemented for lenet, not --model=%s" % model):
            W.check_flags(_flags(weight_decay=1e-4, model=model), _ctx(True))
        W.check_flags(_flags(weight_decay=1e-4, model=model, backend="nccl"), _ctx(True))
        W.check_flags(_flags(weight_decay=1e-4, model=model), _ctx(False))
    W.check_flags(_flags(weight_decay=1e-4), _ctx(True))
    W.check_flags(_flags(weight_decay=0.0, model="mlp2"), _ctx(True))


def test_decayed_variables():
    assert [q.name for q in W.decayed(get_model("lenet")[0])] == ["fc1_weights", "fc1_biases", "fc2_weights",
                                                                  "fc2_biases"]
    assert [q.name for q in W.decayed(get_model("mlp2", 64)[0])] == ["fc1_weights", "fc1_biases", "fc2_weights",
                                                                     "fc2_biases"]
    assert [q.name for q in W.decayed(get_model("mlp3", 64)[0])] == ["fc1_weights", "fc1_biases", "fc2_weights",
                                                                     "fc2_biases", "fc3_weights", "fc3_biases"]


@pytest.mark.parametrize("model", ["lenet", "mlp2", "mlp3"])
def test_torch_engine_step_is_the_decayed_gradient(model):
    lam = float(np.float32(5e-4))
    B = 16
    g = torch.Generator().manual_seed(3)
    x, y = torch.rand(B, 28, 28, 1, generator=g) - 0.5, torch.randint(0, 10, (B,), generator=g)
    eng = TorchEngine(model, B, torch.device("cpu"), lambda n: torch.zeros(n), mlp_hidden=64)
    eng.load_batch(x, y)
    eng.forward_backward(0)
    g0, (ce, acc0) = eng.grads.clone(), eng.loss_acc()
    eng.arm_weight_decay(lam)
    eng.forward_backward(0)
    g1, (loss, acc1) = eng.grads.clone(), eng.loss_acc()
    assert acc1 == acc0
    v0, v1, w = eng.spec.views(g0), eng.spec.views(g1), eng.spec.views(eng.params)
    names = {q.name for q in W.decayed(eng.spec)}
    r = 0.0
    for q in eng.spec.params:
        if q.name in names:
            want = v0[q.name].double() + lam * w[q.name].double()
            tol = 4 * torch.finfo(torch.float32).eps * (v0[q.name].double().abs() + lam * w[q.name].double().abs()) + 1e-30
            assert bool(((v1[q.name].double() - want).abs() <= tol).all()), q.name
            r += float((w[q.name].double() ** 2).sum()) / 2
        else:
            assert torch.equal(v1[q.name], v0[q.name]), q.name
    want_loss = ce + lam * r
    assert math.isclose(loss, want_loss, rel_tol=1e-5), (loss, want_loss)


def _train(train_dir, *extra, steps=12):
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=32", "--max_steps=%d" % steps, "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000", "--initial_learning_rate=0.05"]
                + list(extra))
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    return train(ctx, ds.train, ds.validation, FLAGS)


def _outputs(d):
    out = {}
    for f in sorted(os.listdir(d)):
        with open(os.path.join(d, f), "rb") as fh:
            out[f] = fh.read()
    return out


def _step_lines(caplog):
    return [m.groups() for m in (STEP_LINE.match(r.getMessage()) for r in caplog.records) if m]


def test_off_leaves_logs_and_outputs_unchanged(tmp_path, clean_flags, caplog):
    runs = []
    for i, extra in enumerate(([], ["--weight_decay=0"])):
        caplog.clear()
        d = tmp_path / str(i)
        _train(str(d), *extra)
        runs.append((_step_lines(caplog), _outputs(d)))
    assert runs[0][0] and runs[0][0] == runs[1][0]
    a, b = runs[0][1], runs[1][1]
    assert sorted(a) == sorted(b)
    for f in a:
        if f.endswith(".npy") and "time_acc" in f:
            x, y = np.load(tmp_path / "0" / f), np.load(tmp_path / "1" / f)
            assert np.array_equal(x[:, 1:], y[:, 1:]), f          # column 0 is the wall clock
        elif f != "checkpoint" and not f.endswith(".index"):       # these two name paths and times
            assert a[f] == b[f], f


def test_decayed_run_logs_the_term_and_its_checkpoint_evaluates(tmp_path, clean_flags, caplog, capsys):
    from distributedmnist_b200.evaluator import evaluate
    caplog.clear()
    d0, d1 = tmp_path / "plain", tmp_path / "decay"
    _train(str(d0), steps=5)
    plain = _step_lines(caplog)
    caplog.clear()
    res = _train(str(d1), "--weight_decay=0.01", steps=5)
    dec = _step_lines(caplog)
    # step 1 starts from the same weights: the logged loss adds lambda * R of the initial weights
    spec = get_model("mlp2", 32)[0]
    w = spec.init_flat(FLAGS.seed)
    r = sum(float((w[q.offset:q.offset + q.numel].double() ** 2).sum()) / 2 for q in W.decayed(spec))
    assert float(dec[0][1]) == pytest.approx(float(plain[0][1]) + float(np.float32(0.01)) * r, rel=1e-4, abs=1e-4)
    assert dec[0][2] == plain[0][2]
    acc = np.load(d1 / "worker0_time_acc.npy")
    assert acc[0, 3] == pytest.approx(float(dec[0][1]), rel=1e-5)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    FLAGS.parse(["--checkpoint_dir=%s" % d1, "--eval_dir=%s" % (tmp_path / "eval"), "--run_once=true"])
    assert evaluate(ds.validation, FLAGS, device=torch.device("cpu")) == str(res["final_step"])
    out = capsys.readouterr().out
    m = re.search(r"Num examples: 64  Precision @ 1: ([0-9.]+) Loss: ([0-9.]+) Time: ", out)
    assert m and 0.0 <= float(m.group(1)) <= 1.0
    assert float(m.group(2)) < float(dec[0][1])      # the evaluator scores cross entropy only
