"""``--early_stopping_patience`` on the CPU: the flags and their refusals, the exact min_delta row count, the rule of
early_stopping.advance on hand-written pass sequences, and torch-engine runs that stop at S = g + STOP_MARGIN and end
exactly as a run with ``--max_steps=S``."""
import dataclasses
import json
import logging
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200 import early_stopping as es
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.train import STOP_MARGIN, check_early_stopping_flags, train

SCRAPERS = [r".*step ([0-9]*),.*", r"Num examples: ([0-9]*)  Precision @ 1: ([\.0-9]*) Loss: ([\.0-9]*) Time: ([\.0-9]*)",
            r".* step=([0-9]*)", r".*ELAPSED TIMES (.*)", r".*ITERATION TIMES (.*)"]       # tools/benchmark.py
LINE = re.compile(r"Early stopping: patience (\d+) exhausted by the evaluation of global step #(\d+), the best being "
                  r"that of global step #(\d+) \((\d+) of (\d+) correct, min_delta (\d+) rows\); the run ends as "
                  r"--max_steps=(\d+) would end it$")


@pytest.fixture
def clean_flags():
    FLAGS.reset()
    saved = {k: os.environ.pop(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") if k in os.environ}
    yield FLAGS
    FLAGS.reset()
    os.environ.update(saved)


def _train(train_dir, *extra, steps=40, world_size=None):
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=32", "--max_steps=%d" % steps, "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000", "--initial_learning_rate=0.05",
                 "--eval_every_steps=2"] + list(extra))
    ctx = init_context(FLAGS, want_gpu=False)
    if world_size is not None:
        ctx = dataclasses.replace(ctx, world_size=world_size)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    return train(ctx, ds.train, ds.validation, FLAGS)


def _rows(d):
    return np.load(os.path.join(str(d), "worker0_eval.npy"))


def _ckpt(d, step):
    with open(os.path.join(str(d), "model.ckpt-%d.data-00000-of-00001" % step), "rb") as f:
        return f.read()


def _replay(rows, patience, delta_rows, n):
    """early_stopping.advance over the rows of a run: the step that exhausts the patience, or None, and the final state."""
    state = es.State()
    for r in rows:
        state, fired = es.advance(state, int(r[0]), int(r[4]), int(r[3]), n, patience, delta_rows)
        if fired:
            return int(r[0]), state
    return None, state


# ---- flags -------------------------------------------------------------------------------------------------------------
def test_flags_are_registered_and_off_by_default(clean_flags):
    assert FLAGS.early_stopping_patience == 0 and FLAGS.early_stopping_min_delta == 0.0
    FLAGS.parse(["--early_stopping_patience=3", "--early_stopping_min_delta=0.001"])
    assert FLAGS.early_stopping_patience == 3 and FLAGS.early_stopping_min_delta == 0.001


REFUSALS = [
    (dict(early_stopping_patience=-1), {}, r"must be >= 1 \(0 = off\), got -1"),
    (dict(early_stopping_patience=2, eval_every_steps=0), {}, "needs --eval_every_steps > 0"),
    (dict(early_stopping_patience=2, early_stopping_min_delta=1.0), {}, r"min_delta must lie in \[0, 1\)"),
    (dict(early_stopping_patience=2, early_stopping_min_delta=-0.01), {}, r"min_delta must lie in \[0, 1\)"),
    (dict(early_stopping_patience=2, early_stopping_min_delta=float("nan")), {}, r"min_delta must lie in \[0, 1\)"),
    (dict(early_stopping_min_delta=0.01), {}, "min_delta needs --early_stopping_patience >= 1"),
    (dict(early_stopping_patience=2), dict(on_gpu=False, world_size=2), "torch engine .* one replica, not 2"),
    (dict(early_stopping_patience=2, backend="nccl"), dict(world_size=4), "torch engine .* one replica, not 4"),
]
REFUSAL_IDS = ["negative", "no_eval", "delta_one", "delta_negative", "delta_nan", "delta_without_patience",
               "cpu_two_replicas", "nccl_four_replicas"]


@pytest.mark.parametrize("flags, ctx, msg", REFUSALS, ids=REFUSAL_IDS)
def test_refusals_name_their_reason(flags, ctx, msg):
    f = SimpleNamespace(**dict(dict(eval_every_steps=10, backend="auto", early_stopping_patience=0,
                                    early_stopping_min_delta=0.0), **flags))
    c = SimpleNamespace(**dict(dict(on_gpu=True, world_size=1), **ctx))
    with pytest.raises(ValueError, match=msg):
        check_early_stopping_flags(f, c)


def test_accepted_combinations():
    for ctx in (SimpleNamespace(on_gpu=True, world_size=8), SimpleNamespace(on_gpu=False, world_size=1)):
        check_early_stopping_flags(SimpleNamespace(early_stopping_patience=1, early_stopping_min_delta=0.999,
                                                   eval_every_steps=5, backend="auto"), ctx)
    check_early_stopping_flags(SimpleNamespace(early_stopping_patience=0, early_stopping_min_delta=0.0,
                                               eval_every_steps=0, backend="gloo"),
                               SimpleNamespace(on_gpu=False, world_size=4))            # off: nothing is checked


@pytest.mark.parametrize("args, world_size, msg", [
    (["--early_stopping_patience=-2"], None, "must be >= 1"),
    (["--early_stopping_patience=2", "--eval_every_steps=0"], None, "needs --eval_every_steps > 0"),
    (["--early_stopping_patience=2", "--early_stopping_min_delta=1"], None, r"must lie in \[0, 1\)"),
    (["--early_stopping_min_delta=0.5"], None, "needs --early_stopping_patience"),
    (["--early_stopping_patience=2"], 2, "one replica, not 2"),
], ids=["negative", "no_eval", "delta_one", "delta_without_patience", "two_replicas"])
def test_refused_before_any_work(tmp_path, clean_flags, args, world_size, msg):
    with pytest.raises(ValueError, match=msg):
        _train(str(tmp_path / "t"), *args, world_size=world_size)
    assert not (tmp_path / "t").exists()


@pytest.mark.parametrize("d, n, rows", [(0.001, 10000, 10), (0.0, 10000, 0), (0.29, 100, 29), (0.57, 100, 57),
                                        (0.3, 10, 3), (0.1, 3, 0), (0.015625, 64, 1), (0.0156, 64, 0),
                                        (0.999, 1000, 999), (0.9999, 10000, 9999), (1e-9, 10000, 0)])
def test_min_delta_rows_is_exact(d, n, rows):
    assert es.min_delta_rows(d, n) == rows
    assert rows <= d * n + 1e-9 and (rows + 1) / n > d


# ---- the rule ---------------------------------------------------------------------------------------------------------
def _run(passes, patience, delta_rows, n=100):
    """``passes``: (step, correct, examples, status); returns the states after each pass and the firing passes."""
    state, states, fired = es.State(), [], []
    for step, correct, examples, status in passes:
        state, f = es.advance(state, step, correct, examples, n, patience, delta_rows, status)
        states.append(state)
        if f:
            fired.append(step)
    return states, fired


def test_first_counting_pass_sets_the_baseline_even_when_low():
    states, fired = _run([(1, 90, 99, None), (2, 5, 100, -1), (3, 5, 100, 0), (4, 3, 100, None)], patience=2, delta_rows=0)
    assert states[0] == states[1] == states[2] == es.State()            # partial, dropped, unsettled: nothing
    assert states[3] == es.State(best=3, since=0, best_step=4, trigger_step=0, baseline=True)
    assert fired == []


def test_ties_and_the_min_delta_boundary():
    # m = 2: best + 2 does not beat the best, best + 3 does
    states, fired = _run([(1, 50, 100, None), (2, 50, 100, None), (3, 52, 100, None), (4, 53, 100, None)],
                         patience=3, delta_rows=2)
    assert [(s.best, s.since, s.best_step) for s in states] == [(50, 0, 1), (50, 1, 1), (50, 2, 1), (53, 0, 4)]
    assert fired == []
    # m = 0: a tie counts against the patience, one row more resets it
    states, fired = _run([(1, 50, 100, None), (2, 50, 100, None), (3, 51, 100, None)], patience=5, delta_rows=0)
    assert [(s.best, s.since) for s in states] == [(50, 0), (50, 1), (51, 0)]


def test_passes_that_do_not_count_neither_reset_nor_advance():
    passes = [(10, 60, 100, 2), (20, 55, 100, 1), (30, 99, 100, -1), (40, 99, 80, 3), (50, 61, 100, 4)]
    states, fired = _run(passes, patience=3, delta_rows=1)
    assert [(s.best, s.since) for s in states] == [(60, 0), (60, 1), (60, 1), (60, 1), (60, 2)]
    assert fired == []


def test_patience_is_exhausted_once_and_the_state_then_stays():
    passes = [(5, 40, 100, None), (10, 45, 100, None), (15, 44, 100, None), (20, 45, 100, None), (25, 90, 100, None),
              (30, 10, 100, None)]
    states, fired = _run(passes, patience=2, delta_rows=0)
    assert fired == [20]
    want = es.State(best=45, since=2, best_step=10, trigger_step=20, baseline=True)
    assert states[3] == states[4] == states[5] == want
    assert es.exhausted(want, 2) and not es.exhausted(states[2], 2)


def test_patience_one_fires_on_the_first_pass_after_the_baseline():
    states, fired = _run([(3, 70, 100, None), (6, 70, 100, None)], patience=1, delta_rows=0)
    assert fired == [6] and states[-1].trigger_step == 6 and states[-1].best_step == 3


# ---- torch-engine runs ------------------------------------------------------------------------------------------------
def _pick(rows, n, max_step):
    """(patience, min_delta, delta rows, g): the first setting, by host emulation, whose patience runs out at a step g
    with g + STOP_MARGIN < max_step."""
    for patience in (3, 2, 4, 1):
        for d in (1.0 / n, 0.0):
            m = es.min_delta_rows(d, n)
            g, _s = _replay(rows, patience, m, n)
            if g is not None and g + STOP_MARGIN < max_step:
                return patience, d, m, g
    pytest.fail("no patience runs out inside the run: %s" % rows[:, [0, 4]].tolist())


def test_torch_engine_run_stops_at_g_plus_margin_like_max_steps(tmp_path, clean_flags, caplog):
    _train(str(tmp_path / "ref"))
    rows = _rows(tmp_path / "ref")
    n = int(rows[0, 3])
    patience, d, m, g = _pick(rows, n, 40)
    s = g + STOP_MARGIN
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(str(tmp_path / "armed"), "--early_stopping_patience=%d" % patience,
                     "--early_stopping_min_delta=%r" % d)
    msgs = [r.getMessage() for r in caplog.records]
    cut = _train(str(tmp_path / "cut"), steps=s)
    assert res["final_step"] == cut["final_step"] == s + 1
    assert res["steps"] == cut["steps"] and res["losses"] == cut["losses"]
    assert _ckpt(tmp_path / "armed", s + 1) == _ckpt(tmp_path / "cut", s + 1)
    a, c = _rows(tmp_path / "armed"), _rows(tmp_path / "cut")
    np.testing.assert_array_equal(a[:, [0, 3, 4, 5]], c[:, [0, 3, 4, 5]])
    rep = res["early_stopping"]
    with open(str(tmp_path / "armed" / "worker0_early_stopping.json")) as f:
        assert json.load(f) == rep
    _g, state = _replay(a, patience, m, n)
    counted = sum(1 for r in a if r[0] <= g)
    assert rep == dict(patience=patience, min_delta=d, min_delta_rows=m, examples=n, triggered=True, trigger_step=g,
                       stop_step=s, best_step=state.best_step, best_correct=state.best, counted_passes=counted,
                       weights="live")
    lines = [x for x in msgs if x.startswith("Early stopping")]
    assert len(lines) == 1
    mt = LINE.match(lines[0])
    assert mt and [int(x) for x in mt.groups()] == [patience, g, state.best_step, state.best, n, m, s], lines[0]
    assert not any(re.match(p, lines[0]) for p in SCRAPERS)
    assert "early_stopping" not in cut and not os.path.exists(str(tmp_path / "cut" / "worker0_early_stopping.json"))
    print("\npatience %d, min_delta %d rows: exhausted at step %d, run ended at %d" % (patience, m, g, s + 1))


def test_unexhausted_patience_changes_nothing_but_the_report(tmp_path, clean_flags):
    ref = _train(str(tmp_path / "ref"), steps=12)
    res = _train(str(tmp_path / "armed"), "--early_stopping_patience=1000", steps=12)
    assert res["final_step"] == ref["final_step"] == 13 and res["losses"] == ref["losses"]
    assert _ckpt(tmp_path / "armed", 13) == _ckpt(tmp_path / "ref", 13)
    np.testing.assert_array_equal(_rows(tmp_path / "armed")[:, [0, 3, 4, 5]], _rows(tmp_path / "ref")[:, [0, 3, 4, 5]])
    assert sorted(os.listdir(str(tmp_path / "armed"))) == sorted(os.listdir(str(tmp_path / "ref")) +
                                                                 ["worker0_early_stopping.json"])
    rep = res["early_stopping"]
    assert rep["triggered"] is False and rep["trigger_step"] is None and rep["stop_step"] is None
    assert rep["counted_passes"] == len(_rows(tmp_path / "armed"))


def test_target_and_patience_whichever_fires_first_sets_the_stop(tmp_path, clean_flags):
    """A target reached before the patience runs out stops the run at the target's S; both reports are written."""
    _train(str(tmp_path / "ref"))
    rows = _rows(tmp_path / "ref")
    n = int(rows[0, 3])
    patience, d, _m, g = _pick(rows, n, 40)
    first = rows[0]
    target = int(first[4]) / n                                      # reached by the very first pass
    res = _train(str(tmp_path / "both"), "--early_stopping_patience=%d" % patience, "--early_stopping_min_delta=%r" % d,
                 "--target_accuracy=%r" % target)
    s = int(first[0]) + STOP_MARGIN
    assert s <= g + STOP_MARGIN
    assert res["final_step"] == s + 1
    assert res["time_to_accuracy"]["global_step"] == int(first[0])
    for name in ("worker0_time_to_accuracy.json", "worker0_early_stopping.json"):
        assert os.path.exists(str(tmp_path / "both" / name))
    trig, state = _replay(_rows(tmp_path / "both"), patience, es.min_delta_rows(d, n), n)
    rep = res["early_stopping"]
    assert (rep["trigger_step"], rep["best_step"], rep["best_correct"]) == (trig, state.best_step, state.best)


def test_new_kernel_is_sm_90a_without_spills_or_stack():
    """The in-tree build compiles csrc/eval_patience.cu for sm_90a; its -Xptxas -v log lists eval_patience_kernel."""
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    log = os.path.join(root, "build", "obj", "eval_patience.log")
    if not os.path.exists(log):
        pytest.skip("no in-tree build log (build() has not run)")
    spec = importlib.util.spec_from_file_location("ptxas_report", os.path.join(root, "tools", "ptxas_report.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rows = [r for r in mod.parse(log) if "eval_patience_kernel" in r["name"]]
    assert len(rows) == 1, [r["name"] for r in mod.parse(log)]
    r = rows[0]
    assert r["arch"] == "sm_90a" and r["spill_st"] == r["spill_ld"] == r["stack"] == 0, r
