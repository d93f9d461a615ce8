"""``--keep_best_checkpoint`` on the CPU: the flag and its refusal, the shared selection rule, a torch-engine run whose best
checkpoint holds the weights of the first best-scoring evaluation (the same bytes as the final checkpoint of a run cut at
that step) and scores the same in the evaluator, restarted runs that keep or replace an earlier best, unchanged logs and
files with the flag off, and the new kernels in the ptxas report."""
import json
import logging
import os
import re

import numpy as np
import pytest
import torch

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.best import emulate_decide, improves
from distributedmnist_b200.checkpoint import Saver, get_checkpoint_state
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.train import train

SCRAPERS = [r".*step ([0-9]*),.*", r"Num examples: ([0-9]*)  Precision @ 1: ([\.0-9]*) Loss: ([\.0-9]*) Time: ([\.0-9]*)",
            r".* step=([0-9]*)", r".*ELAPSED TIMES (.*)", r".*ITERATION TIMES (.*)"]       # tools/benchmark.py
# fields of the log that depend on the clock
CLOCK_FIELDS = [(re.compile(r"\d{4}-\d\d-\d\d \d\d:\d\d:\d\d\.\d+"), "<date>"),
                (re.compile(r"\([0-9.e+-]+ examples/sec; [0-9.e+-]+  sec/batch\)"), "(<rate>)"),
                (re.compile(r"RUNNING SESSION\.\.\. [0-9.]+"), "RUNNING SESSION... <t>"),
                (re.compile(r"Elapsed Time: [0-9.]+"), "Elapsed Time: <t>")]


@pytest.fixture
def clean_flags():
    FLAGS.reset()
    saved = {k: os.environ.pop(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") if k in os.environ}
    yield FLAGS
    FLAGS.reset()
    os.environ.update(saved)


def _data():
    return mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                                 synthetic_sizes=(256, 64))


def _train(train_dir, *extra, steps=40):
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=32", "--max_steps=%d" % steps, "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000", "--initial_learning_rate=0.05",
                 "--eval_every_steps=2"] + list(extra))
    ctx = init_context(FLAGS, want_gpu=False)
    ds = _data()
    return train(ctx, ds.train, ds.validation, FLAGS)


def _rows(d):
    return np.load(os.path.join(str(d), "worker0_eval.npy"))


def _best_json(d):
    with open(os.path.join(str(d), "worker0_best.json")) as f:
        return json.load(f)


def _data_file(d, step):
    with open(os.path.join(str(d), "model.ckpt-%d.data-00000-of-00001" % step), "rb") as f:
        return f.read()


def _first_argmax(rows):
    best = int(rows[:, 4].max())
    return int(rows[rows[:, 4] == best][0, 0]), best


def _messages(caplog):
    out = []
    for r in caplog.records:
        m = r.getMessage()
        for pat, rep in CLOCK_FIELDS:
            m = pat.sub(rep, m)
        out.append(m)
    return out


def test_flag_is_registered_and_off_by_default(clean_flags):
    assert "keep_best_checkpoint" in FLAGS and FLAGS.keep_best_checkpoint is False
    FLAGS.parse(["--keep_best_checkpoint"])
    assert FLAGS.keep_best_checkpoint is True


def test_refused_without_eval_before_any_work(tmp_path, clean_flags):
    with pytest.raises(ValueError, match="--keep_best_checkpoint needs --eval_every_steps > 0"):
        _train(str(tmp_path / "t"), "--keep_best_checkpoint", "--eval_every_steps=0")
    assert not (tmp_path / "t").exists()


@pytest.mark.parametrize("correct, examples, n, best, status, want", [
    (10, 64, 64, 9, None, True),          # live pass, one more correct row
    (10, 64, 64, 10, None, False),        # tie: the earlier pass stays
    (9, 64, 64, 10, None, False),         # worse
    (10, 32, 64, 0, None, False),         # incomplete pass
    (64, 64, 64, 63, 1, True),            # snapshot accepted on the first attempt
    (64, 64, 64, 63, 4, True),            # ... on the last one
    (64, 64, 64, 0, 0, False),            # no attempt settled
    (64, 64, 64, 0, -1, False),           # dropped snapshot: its count is meaningless
])
def test_selection_rule(correct, examples, n, best, status, want):
    assert improves(correct, examples, n, best, status) is want
    old = (7, best, n, 1.5, 1)
    new, decision = emulate_decide(correct, examples, 2.5, 12, n, old, status)
    assert decision == int(want)
    assert new == ((12, correct, examples, 2.5, 1) if want else old)


def test_torch_engine_run_keeps_the_first_best_weights(tmp_path, clean_flags, caplog):
    from distributedmnist_b200.engine import TorchEngine
    from distributedmnist_b200.evaluator import do_eval
    d = tmp_path / "armed"
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(str(d), "--keep_best_checkpoint")
    rows = _rows(d)
    g, best = _first_argmax(rows)
    rep = _best_json(d)
    assert rep == res["best"]
    n = int(rows[0, 3])
    assert rep["global_step"] == g and rep["correct"] == best and rep["examples"] == n and rep["weights"] == "live"
    assert rep["accuracy"] == best / n
    assert abs(rep["mean_loss"] - float(rows[rows[:, 0] == g][0, 5])) < 1e-12
    # the best checkpoint is the final checkpoint of a run cut at g (the loop stops once step > max_steps)
    cut = _train(str(tmp_path / "cut"), steps=g - 1)
    assert cut["final_step"] == g
    assert _data_file(d / "best", g) == _data_file(tmp_path / "cut", g)
    st = get_checkpoint_state(str(d / "best"))
    assert st.model_checkpoint_path == "model.ckpt-%d" % g and st.all_model_checkpoint_paths == [st.model_checkpoint_path]
    # one log line, which no scraper of the reference's logs picks up
    lines = [m for m in _messages(caplog) if m.startswith("Best weights")]
    assert len(lines) == 1 and ("global step #%d" % g) in lines[0] and ("%d of %d correct" % (best, n)) in lines[0]
    assert not any(re.match(p, lines[0]) for p in SCRAPERS)
    # the evaluator scores the best directory as it is
    ds = _data()
    FLAGS.reset()
    FLAGS.parse(["--checkpoint_dir=%s" % (d / "best"), "--model=mlp2", "--mlp_hidden=32", "--run_once"])
    eng = TorchEngine("mlp2", 1, torch.device("cpu"), lambda k: torch.zeros(k), mlp_hidden=32)
    assert do_eval(eng, None, ds.validation, FLAGS) == str(g)
    _loss, acc = eng.evaluate(ds.validation.images, ds.validation.labels)
    assert int(round(acc * n)) == best


def test_moving_average_best_is_the_scored_average(tmp_path, clean_flags):
    from distributedmnist_b200 import moving_average as ema
    d = tmp_path / "avg"
    res = _train(str(d), "--keep_best_checkpoint", "--moving_average_decay=0.9", "--eval_moving_average")
    g, _best = _first_argmax(_rows(d))
    assert res["best"]["global_step"] == g and res["best"]["weights"] == "moving_average"
    _train(str(tmp_path / "cut"), "--moving_average_decay=0.9", steps=g - 1)
    spec = res["engine"].spec
    state_cut, _ = Saver.restore(os.path.join(str(tmp_path / "cut"), "model.ckpt-%d" % g))
    state_best, step = Saver.restore(os.path.join(str(d / "best"), "model.ckpt-%d" % g))
    assert step == g and sorted(state_best) == sorted(p.ckpt_name for p in spec.params)   # plain names only
    assert torch.equal(spec.from_state_dict(state_best), ema.from_state_dict(spec, state_cut))


def _snapshot(d):
    out = {}
    for root, _dirs, files in os.walk(str(d)):
        for f in files:
            if f == "worker0_best.json" or os.path.basename(root) == "best":
                p = os.path.join(root, f)
                with open(p, "rb") as fh:
                    out[os.path.relpath(p, str(d))] = (fh.read(), os.stat(p).st_mtime_ns)
    return out


def test_restarted_run_replaces_the_best_only_when_better(tmp_path, clean_flags, caplog):
    d = tmp_path / "run"
    first = _train(str(d), "--keep_best_checkpoint", steps=6)["best"]
    # a better later history: the restarted run trains on to step 40 and beats the early best
    res = _train(str(d), "--keep_best_checkpoint", steps=40)
    rows = _rows(d)
    later = rows[rows[:, 0] > 7]
    assert int(later[:, 4].max()) > first["correct"]
    g, best = _first_argmax(later)
    assert res["best"]["global_step"] == g and res["best"]["correct"] == best and _best_json(d) == res["best"]
    assert sorted(os.listdir(str(d / "best"))) == ["checkpoint", "model.ckpt-%d.data-00000-of-00001" % g,
                                                   "model.ckpt-%d.index" % g]
    # a worse later history: a learning rate that wrecks the weights; the files stay exactly as they are
    before = _snapshot(d)
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(str(d), "--keep_best_checkpoint", "--initial_learning_rate=500", steps=60)
    rows = _rows(d)
    assert int(rows[rows[:, 0] > 41][:, 4].max()) <= best
    assert res["best"] is None
    assert _snapshot(d) == before
    assert sum(m.startswith("Best weights: an earlier run kept the evaluation of global step #%d" % g)
               for m in _messages(caplog)) == 1


def test_flag_off_writes_nothing_and_logs_the_same(tmp_path, clean_flags, caplog):
    logs = {}
    for tag, extra in (("absent", []), ("off", ["--keep_best_checkpoint=false"]), ("on", ["--keep_best_checkpoint"])):
        caplog.clear()
        with caplog.at_level(logging.INFO, logger="dmnist"):
            res = _train(str(tmp_path / tag), *extra, steps=12)
        logs[tag] = _messages(caplog)
        assert ("best" in res) == (tag == "on")
        assert os.path.exists(str(tmp_path / tag / "best")) == (tag == "on")
        assert os.path.exists(str(tmp_path / tag / "worker0_best.json")) == (tag == "on")
    assert logs["absent"] == logs["off"]
    assert [m for m in logs["on"] if not m.startswith("Best weights")] == logs["off"]
    assert _data_file(tmp_path / "off", 13) == _data_file(tmp_path / "on", 13)


def test_new_kernels_are_listed_by_ptxas_report_without_spills():
    """The in-tree build compiles csrc/eval_best.cu for sm_90a; its -Xptxas -v log lists both kernels, none spilling."""
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    log = os.path.join(root, "build", "obj", "eval_best.log")
    if not os.path.exists(log):
        pytest.skip("no in-tree build log (build() has not run)")
    spec = importlib.util.spec_from_file_location("ptxas_report", os.path.join(root, "tools", "ptxas_report.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rows = {r["name"]: r for r in mod.parse(log)}
    names = [n for n in rows if any(k in n for k in ("eval_best_decide_kernel", "eval_best_copy_kernel"))]
    assert len(names) == 2, sorted(rows)
    for n in names:
        assert rows[n]["arch"] == "sm_90a" and rows[n]["spill_st"] == rows[n]["spill_ld"] == rows[n]["stack"] == 0, rows[n]
