"""``--target_accuracy`` on the CPU: the flag and its refusals, the exact correct-count threshold, a torch-engine run that
stops at S = g + STOP_MARGIN and ends exactly as a run with ``--max_steps=S``, and the host-loop model of N lock-step
replicas against the stop word."""
import json
import logging
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.parallel.protocol import ProtocolHazard, TargetStopModel, run_random
from distributedmnist_b200.train import STOP_MARGIN, check_target_flags, need_count, train

TTA_LINE = re.compile(r"Time to accuracy: target ([0-9.]+) reached by the evaluation of global step #(\d+) \(accuracy "
                      r"([0-9.]+), (\d+) of (\d+) correct\); training time ([0-9.]+) s")
SCRAPERS = [r".*step ([0-9]*),.*", r"Num examples: ([0-9]*)  Precision @ 1: ([\.0-9]*) Loss: ([\.0-9]*) Time: ([\.0-9]*)",
            r".* step=([0-9]*)", r".*ELAPSED TIMES (.*)", r".*ITERATION TIMES (.*)"]       # tools/benchmark.py


@pytest.fixture
def clean_flags():
    FLAGS.reset()
    saved = {k: os.environ.pop(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") if k in os.environ}
    yield FLAGS
    FLAGS.reset()
    os.environ.update(saved)


def _train(train_dir, *extra, steps=40):
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=32", "--max_steps=%d" % steps, "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000", "--initial_learning_rate=0.05",
                 "--eval_every_steps=2"] + list(extra))
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    return train(ctx, ds.train, ds.validation, FLAGS)


def test_flag_is_registered_and_off_by_default(clean_flags):
    assert "target_accuracy" in FLAGS and FLAGS.target_accuracy == 0.0
    FLAGS.parse(["--target_accuracy=0.99"])
    assert FLAGS.target_accuracy == 0.99


@pytest.mark.parametrize("flags, ctx, msg", [
    (dict(target_accuracy=-0.1), {}, r"must lie in \(0, 1\]"),
    (dict(target_accuracy=1.5), {}, r"must lie in \(0, 1\]"),
    (dict(target_accuracy=float("nan")), {}, r"must lie in \(0, 1\]"),
    (dict(target_accuracy=0.9, eval_every_steps=0), {}, "needs --eval_every_steps > 0"),
    (dict(target_accuracy=0.9), dict(on_gpu=False, world_size=2), "torch engine .* one replica, not 2"),
    (dict(target_accuracy=0.9, backend="nccl"), dict(world_size=4), "torch engine .* one replica, not 4"),
], ids=["negative", "above_one", "nan", "no_eval", "cpu_two_replicas", "nccl_four_replicas"])
def test_refusals_name_their_reason(flags, ctx, msg):
    f = SimpleNamespace(**dict(dict(eval_every_steps=10, backend="auto"), **flags))
    c = SimpleNamespace(**dict(dict(on_gpu=True, world_size=1), **ctx))
    with pytest.raises(ValueError, match=msg):
        check_target_flags(f, c)


def test_accepted_combinations():
    for ctx in (SimpleNamespace(on_gpu=True, world_size=8), SimpleNamespace(on_gpu=False, world_size=1)):
        check_target_flags(SimpleNamespace(target_accuracy=1.0, eval_every_steps=5, backend="auto"), ctx)
    check_target_flags(SimpleNamespace(target_accuracy=0.0, eval_every_steps=0, backend="gloo"),
                       SimpleNamespace(on_gpu=False, world_size=4))                     # off: nothing is checked


def test_refused_before_any_work(tmp_path, clean_flags):
    with pytest.raises(ValueError, match="needs --eval_every_steps > 0"):
        _train(str(tmp_path / "t"), "--target_accuracy=0.5", "--eval_every_steps=0")
    assert not (tmp_path / "t").exists()


@pytest.mark.parametrize("a, n, need", [(0.99, 10000, 9900), (1.0, 10000, 10000), (1.0, 64, 64), (0.3, 10, 3),
                                        (0.7, 10, 7), (0.1, 3, 1), (0.9871, 10000, 9871), (0.98715, 10000, 9872),
                                        (1e-9, 10000, 1)])
def test_need_is_exact(a, n, need):
    assert need_count(a, n) == need
    assert need / n >= a or abs(need / n - a) < 1e-15
    assert (need - 1) / n < a


def _rows(d):
    return np.load(os.path.join(d, "worker0_eval.npy"))


def _ckpt(d, step):
    with open(os.path.join(d, "model.ckpt-%d.data-00000-of-00001" % step), "rb") as f:
        return f.read()


def test_torch_engine_run_stops_at_g_plus_margin_like_max_steps(tmp_path, clean_flags, caplog):
    """A reference run without a target finds a reachable count; the armed run stops at S = g + STOP_MARGIN and writes the
    same final checkpoint, the same evaluation rows and the same step lines as a run with --max_steps=S."""
    ref = _train(str(tmp_path / "ref"))
    rows = _rows(str(tmp_path / "ref"))
    early = rows[rows[:, 0] <= 30]
    best = int(early[:, 4].max())
    g = int(early[early[:, 4] == best][0, 0])
    assert (early[early[:, 0] < g, 4] < best).all()
    n = int(rows[0, 3])
    target = best / n                                     # n = 64: exact in binary and in its decimal repr
    assert need_count(target, n) == best
    s = g + STOP_MARGIN
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(str(tmp_path / "armed"), "--target_accuracy=%r" % target)
    msgs = [r.getMessage() for r in caplog.records]
    with caplog.at_level(logging.INFO, logger="dmnist"):
        cut = _train(str(tmp_path / "cut"), steps=s)
    assert ref["final_step"] == 41
    assert res["final_step"] == cut["final_step"] == s + 1
    assert res["steps"] == cut["steps"] and res["losses"] == cut["losses"]
    assert _ckpt(str(tmp_path / "armed"), s + 1) == _ckpt(str(tmp_path / "cut"), s + 1)
    a, c = _rows(str(tmp_path / "armed")), _rows(str(tmp_path / "cut"))
    np.testing.assert_array_equal(a[:, [0, 3, 4, 5]], c[:, [0, 3, 4, 5]])
    assert (a[a[:, 0] < g, 4] < best).all() and int(a[a[:, 0] == g, 4][0]) == best
    # the report: results, JSON file and one log line
    rep = res["time_to_accuracy"]
    with open(str(tmp_path / "armed" / "worker0_time_to_accuracy.json")) as f:
        assert json.load(f) == rep
    assert rep["reached"] and rep["global_step"] == g and rep["correct"] == best and rep["need"] == best
    assert rep["examples"] == n and rep["accuracy"] == best / n and rep["clock"] == "host"
    assert 0 < rep["train_time_s"] <= rep["wall_time_s"]
    lines = [m for m in msgs if m.startswith("Time to accuracy")]
    assert len(lines) == 1
    m = TTA_LINE.match(lines[0])
    assert m and int(m.group(2)) == g and int(m.group(4)) == best and int(m.group(5)) == n, lines[0]
    assert not any(re.match(p, lines[0]) for p in SCRAPERS)
    assert not os.path.exists(str(tmp_path / "cut" / "worker0_time_to_accuracy.json"))
    assert "time_to_accuracy" not in cut


def test_target_reached_only_by_the_final_pass_is_only_reported(tmp_path, clean_flags):
    ref = _train(str(tmp_path / "ref"), steps=9)
    rows = _rows(str(tmp_path / "ref"))
    assert rows[-1, 0] == 10
    last, before = int(rows[-1, 4]), rows[:-1, 4]
    if (before >= last).any():
        pytest.skip("the final pass is not a new best on this data")
    res = _train(str(tmp_path / "armed"), "--target_accuracy=%r" % (last / float(rows[-1, 3])), steps=9)
    assert res["final_step"] == ref["final_step"] == 10
    assert res["time_to_accuracy"]["global_step"] == 10


def test_unreached_target_changes_nothing_but_the_report(tmp_path, clean_flags):
    ref = _train(str(tmp_path / "ref"), steps=12)
    res = _train(str(tmp_path / "armed"), "--target_accuracy=1.0", steps=12)
    assert res["final_step"] == ref["final_step"] == 13 and res["losses"] == ref["losses"]
    assert _ckpt(str(tmp_path / "armed"), 13) == _ckpt(str(tmp_path / "ref"), 13)
    assert res["time_to_accuracy"]["reached"] is False and res["time_to_accuracy"]["global_step"] is None


@pytest.mark.parametrize("pipelined", [True, False], ids=["pipelined", "non_pipelined"])
@pytest.mark.parametrize("n", [1, 2, 3])
def test_model_every_replica_stops_at_the_same_step(n, pipelined):
    for every, reach, max_steps in ((3, 1, 1000), (2, 3, 1000), (1, 4, 1000), (3, 1, 4), (2, 100, 7)):
        run_random(lambda: TargetStopModel(n, every, reach, STOP_MARGIN, max_steps=max_steps, pipelined=pipelined),
                   range(400))


def test_model_margin_one_is_too_small_for_the_pipelined_loop():
    """With S = g + 1 the pipelined chief decides its pass after step S + 1 before it has read S: the run differs from
    --max_steps=S (the final pass is missing) under some completion orders."""
    with pytest.raises(ProtocolHazard, match="enqueued passes"):
        run_random(lambda: TargetStopModel(2, 3, 1, 1), range(400))


def test_new_kernels_are_listed_by_ptxas_report_without_spills():
    """The in-tree build compiles csrc/eval_target.cu for sm_90a; its -Xptxas -v log lists the three kernels, none spilling."""
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    log = os.path.join(root, "build", "obj", "eval_target.log")
    if not os.path.exists(log):
        pytest.skip("no in-tree build log (build() has not run)")
    spec = importlib.util.spec_from_file_location("ptxas_report", os.path.join(root, "tools", "ptxas_report.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rows = {r["name"]: r for r in mod.parse(log)}
    names = [n for n in rows if any(k in n for k in ("eval_target_kernel", "stop_publish_kernel", "tta_stamp_kernel"))]
    assert len(names) == 3, sorted(rows)
    for n in names:
        assert rows[n]["arch"] == "sm_90a" and rows[n]["spill_st"] == rows[n]["spill_ld"] == rows[n]["stack"] == 0, rows[n]
