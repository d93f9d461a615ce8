"""``--eval_every_steps`` on the CPU: the driver logic (which steps are scored, what is logged and saved, which combinations
are refused) with the torch engine, which evaluates synchronously with ``engine.evaluate``."""
import logging
import os
import re
import sys
from types import SimpleNamespace

import numpy as np
import pytest

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.train import check_eval_flags, train

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEP_LINE = re.compile(r"Worker 0: .*: step (\d+), loss = ([0-9.]+), train_acc = ([0-9.]+), test_acc = ([0-9.]+)\(")


@pytest.fixture
def clean_flags():
    FLAGS.reset()
    saved = {k: os.environ.pop(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") if k in os.environ}
    yield FLAGS
    FLAGS.reset()
    os.environ.update(saved)


def _train(train_dir, *extra, steps=12, with_test=True):
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=32", "--max_steps=%d" % steps, "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000", "--initial_learning_rate=0.05"]
                + list(extra))
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    return train(ctx, ds.train, ds.validation if with_test else None, FLAGS), ds


def _step_lines(caplog):
    out = []
    for r in caplog.records:
        m = STEP_LINE.match(r.getMessage())
        if m:
            out.append((int(m.group(1)), m.group(2), m.group(3), float(m.group(4))))
    return out


def test_default_off_leaves_logs_and_outputs_unchanged(tmp_path, clean_flags, caplog, monkeypatch):
    """E = 0 (the default, and explicitly): nothing is evaluated, and the log lines, worker0_time_acc.npy and the train_dir
    listing are exactly what the driver wrote before the flag existed."""
    from distributedmnist_b200.engine import TorchEngine

    def no_eval(*a, **k):
        raise AssertionError("evaluate() called with --eval_every_steps=0")
    monkeypatch.setattr(TorchEngine, "evaluate", no_eval)
    # save_interval_secs = 1000: the final checkpoint is the only one
    expected_files = ["checkpoint", "model.ckpt-13.data-00000-of-00001", "model.ckpt-13.index", "worker0_time_acc.npy"]
    runs = []
    for i, extra in enumerate([(), ("--eval_every_steps=0",)]):
        caplog.clear()
        d = tmp_path / ("run%d" % i)
        with caplog.at_level(logging.INFO, logger="dmnist"):
            res, _ = _train(str(d), *extra)
        msgs = [r.getMessage() for r in caplog.records if STEP_LINE.match(r.getMessage())]
        acc = np.load(os.path.join(str(d), "worker0_time_acc.npy"))
        files = sorted(os.listdir(str(d)))
        assert res["final_step"] == 13 and "evals" not in res
        # the log line of every step: steps 1..12, test_acc printed as the reference's hard-wired 0 (`%f`)
        assert [int(STEP_LINE.match(m).group(1)) for m in msgs] == list(range(1, 13))
        assert all(", test_acc = 0.000000(" in m for m in msgs)
        # worker0_time_acc.npy: one (time, train_acc, test_acc, loss) row per logged step, saved at step 10 and never
        # rewritten after it (save_results_period = 5, last logged step 12); test_acc exactly 0, the others as logged
        assert acc.shape == (10, 4) and acc.dtype == np.float64 and not acc[:, 2].any()
        for row, m in zip(acc, msgs):
            g = STEP_LINE.match(m)
            assert "%f" % row[3] == g.group(2) and "%f" % row[1] == g.group(3)
        assert files == expected_files, files
        runs.append((msgs, acc))
    (m0, a0), (m1, a1) = runs
    strip = [re.sub(r": .*?: step", ": step", re.sub(r"\(.*\)$", "", m)) for m in m0]
    assert strip == [re.sub(r": .*?: step", ": step", re.sub(r"\(.*\)$", "", m)) for m in m1]
    np.testing.assert_array_equal(a0[:, 1:], a1[:, 1:])     # column 0 is the wall-clock time


def test_mlp2_run_writes_eval_rows_and_reports_test_acc(tmp_path, clean_flags, caplog):
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res, ds = _train(str(tmp_path / "t"), "--eval_every_steps=5", steps=12)
    assert res["final_step"] == 13
    rows = np.load(str(tmp_path / "t" / "worker0_eval.npy"))
    assert rows.shape == (3, 6)
    assert rows[:, 0].tolist() == [5, 10, 13]                    # every 5th global step and the final one
    n = ds.validation.num_examples
    assert (rows[:, 3] == n).all()
    assert ((rows[:, 4] >= 0) & (rows[:, 4] <= n)).all() and (rows[:, 4] == np.round(rows[:, 4])).all()
    assert (rows[:, 2] >= 0).all() and (rows[:, 5] > 0).all()
    lines = _step_lines(caplog)
    before = [t for s, _l, _a, t in lines if s < 5]
    after = [t for s, _l, _a, t in lines if s >= 5]
    assert before and all(t == 0.0 for t in before)
    assert after and all(t > 0.0 for t in after)
    # the log's test_acc is the newest evaluation's correct / examples
    by_step = {s: t for s, _l, _a, t in lines}
    assert by_step[12] == pytest.approx(rows[1, 4] / n, abs=1e-6)
    acc = np.load(str(tmp_path / "t" / "worker0_time_acc.npy"))
    assert acc[-1, 2] == pytest.approx(rows[1, 4] / n, abs=1e-6)


def test_missing_validation_set_is_refused(tmp_path, clean_flags):
    with pytest.raises(ValueError, match="needs the validation set"):
        _train(str(tmp_path / "t"), "--eval_every_steps=5", with_test=False)
    assert not (tmp_path / "t").exists()                          # refused before anything was set up


@pytest.mark.parametrize("extra, msg", [
    (dict(model="mlp2"), "implemented for lenet"),
    (dict(model="mlp3"), "implemented for lenet"),
    (dict(interval_method=True), "interval commits push weights"),
    (dict(k=1), "K < N"),
])
def test_gpu_path_rejections_give_their_reason(extra, msg):
    flags = SimpleNamespace(eval_every_steps=10, backend="auto", model=extra.get("model", "lenet"),
                            interval_method=extra.get("interval_method", False))
    ctx = SimpleNamespace(on_gpu=True, world_size=2)
    with pytest.raises(ValueError, match=msg):
        check_eval_flags(flags, ctx, extra.get("k", 2), dataset_test=object())


def test_gpu_path_accepts_lenet_with_full_aggregation_and_cpu_path_accepts_everything():
    gpu = SimpleNamespace(on_gpu=True, world_size=2)
    cpu = SimpleNamespace(on_gpu=False, world_size=2)
    ok = SimpleNamespace(eval_every_steps=10, backend="auto", model="lenet", interval_method=False)
    check_eval_flags(ok, gpu, 2, dataset_test=object())
    # cdf mode aggregates all N behind a full barrier whatever --num_replicas_to_aggregate says
    cdf = SimpleNamespace(eval_every_steps=10, backend="auto", model="lenet", interval_method=False,
                          worker_times_cdf_method=True)
    check_eval_flags(cdf, gpu, 1, dataset_test=object())
    cdf.interval_method = True                       # interval wins when both are set
    with pytest.raises(ValueError, match="interval commits push weights"):
        check_eval_flags(cdf, gpu, 1, dataset_test=object())
    anything = SimpleNamespace(eval_every_steps=10, backend="auto", model="mlp3", interval_method=True)
    check_eval_flags(anything, cpu, 1, dataset_test=object())
    off = SimpleNamespace(eval_every_steps=0, backend="auto", model="mlp3", interval_method=True)
    check_eval_flags(off, gpu, 1, dataset_test=None)
    with pytest.raises(ValueError, match=">= 0"):
        check_eval_flags(SimpleNamespace(eval_every_steps=-1), gpu, 2, dataset_test=object())


def test_plot_device_time_precision_renders(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import benchmark as bm
    d = tmp_path / "train"
    d.mkdir()
    rows = np.array([(100, 1000.0, 0.002, 10000, 9000, 0.35), (200, 1000.5, 0.002, 10000, 9500, 0.2),
                     (301, 1001.0, 0.002, 10000, 9700, 0.1)])
    np.save(str(d / "worker0_eval.npy"), rows)
    out = bm.plot_device_time_precision(str(d), str(tmp_path))
    assert out.endswith("device_time_precision.png") and os.path.getsize(out) > 0
    with open(out, "rb") as f:
        assert f.read(8) == b"\x89PNG\r\n\x1a\n"
