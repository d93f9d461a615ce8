"""``--lr_plateau_patience`` on the CPU: the rule of lr_plateau.advance on hand-written pass sequences, the schedule with
cuts bit for bit against a direct double evaluation, the flags' refusals, and torch-engine runs whose cuts fall at steps
known in advance, with restarts."""
import dataclasses
import json
import logging
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200 import lr_plateau as lp
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.ops import aggrefs
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.schedule import LearningRateSchedule
from distributedmnist_b200.train import STOP_MARGIN, check_lr_plateau_flags, train

SCRAPERS = [r".*step ([0-9]*),.*", r"Num examples: ([0-9]*)  Precision @ 1: ([\.0-9]*) Loss: ([\.0-9]*) Time: ([\.0-9]*)",
            r".* step=([0-9]*)", r".*ELAPSED TIMES (.*)", r".*ITERATION TIMES (.*)"]       # tools/benchmark.py
LINE = re.compile(r"Learning rate plateau: cut (\d+) after the evaluation of global step #(\d+) \((\d+) of (\d+) correct, "
                  r"best (\d+), patience (\d+), min_delta (\d+) rows\); from global step #(\d+) the learning rate is (\S+)$")


@pytest.fixture
def clean_flags():
    FLAGS.reset()
    saved = {k: os.environ.pop(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") if k in os.environ}
    yield FLAGS
    FLAGS.reset()
    os.environ.update(saved)


def _train(train_dir, *extra, steps=24, world_size=None):
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


def _file(d):
    with open(os.path.join(str(d), "worker0_lr_plateau.json")) as f:
        return json.load(f)


def _cut_steps(rows):
    """With --lr_plateau_min_delta=0.5 and --lr_plateau_patience=1: the first pass sets the best, and no later pass can
    beat it by more than half the validation set at the accuracies of these short runs, so every later pass cuts."""
    return [(int(r[0]), int(r[0]) + STOP_MARGIN) for r in rows[1:]]


# ---- the rule ---------------------------------------------------------------------------------------------------------
def _run(passes, patience, delta_rows, n=100, state=None):
    """``passes``: (step, correct, examples, status); returns the states after each pass and the triggering steps."""
    state, states, fired = state or lp.State(), [], []
    for step, correct, examples, status in passes:
        state, f = lp.advance(state, step, correct, examples, n, patience, delta_rows, status)
        states.append(state)
        if f:
            fired.append(step)
    return states, fired


def test_first_counting_pass_sets_the_baseline():
    states, fired = _run([(1, 90, 99, None), (2, 5, 100, -1), (3, 5, 100, 0), (4, 3, 100, None)], patience=1, delta_rows=0)
    assert states[0] == states[1] == states[2] == lp.State()            # partial, dropped, unsettled: nothing
    assert states[3] == lp.State(best=3, since=0, baseline=True, cuts=0, trigger_step=0)
    assert fired == []


def test_min_delta_boundary():
    # m = 2: best + 2 does not improve, best + 3 does
    states, fired = _run([(1, 50, 100, None), (2, 52, 100, None), (3, 53, 100, None)], patience=5, delta_rows=2)
    assert [(s.best, s.since) for s in states] == [(50, 0), (50, 1), (53, 0)]
    assert fired == []


def test_cut_at_the_patience_resets_since_and_keeps_best():
    passes = [(5, 40, 100, None), (10, 45, 100, None), (15, 44, 100, None), (20, 45, 100, None), (25, 44, 100, None),
              (30, 43, 100, None), (35, 46, 100, None)]
    states, fired = _run(passes, patience=2, delta_rows=0)
    assert fired == [20, 30]
    assert states[3] == lp.State(best=45, since=0, baseline=True, cuts=1, trigger_step=20)
    assert states[4] == lp.State(best=45, since=1, baseline=True, cuts=1, trigger_step=20)
    assert states[5] == lp.State(best=45, since=0, baseline=True, cuts=2, trigger_step=30)
    assert states[6] == lp.State(best=46, since=0, baseline=True, cuts=2, trigger_step=30)


def test_passes_that_do_not_count_change_nothing():
    passes = [(10, 60, 100, 2), (20, 55, 100, 1), (30, 99, 100, -1), (40, 99, 80, 3), (50, 10, 100, 0), (60, 61, 100, 4)]
    states, fired = _run(passes, patience=2, delta_rows=1)
    assert [(s.best, s.since, s.cuts) for s in states] == [(60, 0, 0), (60, 1, 0), (60, 1, 0), (60, 1, 0), (60, 1, 0),
                                                           (60, 0, 1)]
    assert fired == [60]


def test_at_most_max_cuts_and_later_triggers_cut_nothing():
    passes = [(1, 50, 100, None)] + [(2 + i, 50, 100, None) for i in range(lp.MAX_CUTS + 3)]
    states, fired = _run(passes, patience=1, delta_rows=0)
    assert len(fired) == lp.MAX_CUTS + 3
    assert [s.cuts for s in states[1:]] == list(range(1, lp.MAX_CUTS + 1)) + [lp.MAX_CUTS] * 3
    assert states[-1] == lp.State(best=50, since=0, baseline=True, cuts=lp.MAX_CUTS, trigger_step=passes[-1][0])


def test_seeded_cut_count_carries_on():
    states, fired = _run([(10, 50, 100, None), (20, 50, 100, None)], patience=1, delta_rows=0, state=lp.State(cuts=3))
    assert fired == [20] and states[-1].cuts == 4


# ---- the schedule -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lr0, decay, decay_steps, factor", [(0.1, 0.95, 7, 0.1), (0.05, 0.5, 3, 0.3),
                                                             (0.01, 0.999, 1000, 0.7), (0.2, 1.0, 1, 0.25)])
def test_schedule_with_cuts_is_the_double_product(lr0, decay, decay_steps, factor):
    cuts = [12, 15, 15, 40]
    s = LearningRateSchedule(lr0, decay_steps, decay, factor=factor, cuts=cuts)
    plain = LearningRateSchedule(lr0, decay_steps, decay)
    for step in list(range(0, 50)) + [1000, 123456]:
        c = sum(1 for x in cuts if x <= step)
        want = float(lr0) * (float(decay) ** float(step // decay_steps)) * (float(factor) ** float(c))
        got = s(step)
        assert np.float64(got).view(np.uint64) == np.float64(want).view(np.uint64), (step, got, want)
        if c == 0:
            assert np.float64(got).view(np.uint64) == np.float64(plain(step)).view(np.uint64)
        for count in (1, 2, 3, 8):
            assert aggrefs.bits(aggrefs.step_scale(s, step, count)) == aggrefs.bits(np.float32(want / count))
    # before, at and after a cut's step
    assert s(11) == plain(11) and s(12) == plain(12) * factor and s(13) == plain(13) * factor
    assert s(14) == plain(14) * factor and s(15) == plain(15) * factor ** 3.0


def test_schedule_without_cuts_is_unchanged():
    a, b = LearningRateSchedule(0.1, 5, 0.9), LearningRateSchedule(0.1, 5, 0.9, factor=0.1, cuts=[])
    assert all(a(s) == b(s) for s in range(100))
    assert a.cuts == [] and a.factor == 1.0


# ---- flags ------------------------------------------------------------------------------------------------------------
def test_flags_are_registered_and_off_by_default(clean_flags):
    assert FLAGS.lr_plateau_patience == 0 and FLAGS.lr_plateau_factor == 0.1 and FLAGS.lr_plateau_min_delta == 0.0
    FLAGS.parse(["--lr_plateau_patience=3", "--lr_plateau_factor=0.5", "--lr_plateau_min_delta=0.001"])
    assert FLAGS.lr_plateau_patience == 3 and FLAGS.lr_plateau_factor == 0.5 and FLAGS.lr_plateau_min_delta == 0.001


_ON = dict(lr_plateau_patience=2)
REFUSALS = [
    (dict(lr_plateau_patience=-1), {}, r"--lr_plateau_patience must be >= 1 \(0 = off\), got -1"),
    (dict(_ON, eval_every_steps=0), {}, "--lr_plateau_patience needs --eval_every_steps > 0"),
    (dict(_ON, lr_plateau_factor=1.0), {}, r"--lr_plateau_factor must lie in \(0, 1\), got 1.0"),
    (dict(_ON, lr_plateau_factor=0.0), {}, r"--lr_plateau_factor must lie in \(0, 1\), got 0.0"),
    (dict(_ON, lr_plateau_factor=float("nan")), {}, r"--lr_plateau_factor must lie in \(0, 1\)"),
    (dict(_ON, lr_plateau_min_delta=1.0), {}, r"--lr_plateau_min_delta must lie in \[0, 1\)"),
    (dict(_ON, lr_plateau_min_delta=-0.01), {}, r"--lr_plateau_min_delta must lie in \[0, 1\)"),
    (dict(lr_plateau_min_delta=0.01), {}, "need --lr_plateau_patience >= 1"),
    (dict(lr_plateau_factor=0.5), {}, "need --lr_plateau_patience >= 1"),
    (dict(_ON), dict(on_gpu=False, world_size=2), "torch engine .* one replica, not 2"),
    (dict(_ON, backend="nccl"), dict(world_size=4), "torch engine .* one replica, not 4"),
    (dict(_ON, interval_method=True), dict(world_size=4), "cannot be combined with --interval_method: .*not in lock step"),
    (dict(_ON, interval_method=True, worker_times_cdf_method=True), dict(world_size=4), "--interval_method"),
    (dict(_ON), dict(world_size=4, k=3), r"needs --num_replicas_to_aggregate = number of replicas \(4\), got 3 \(K < N\)"),
    (dict(_ON), dict(world_size=4, k=8), r"got 8 \(K > N\): its replicas are not in lock step"),
]
REFUSAL_IDS = ["negative", "no_eval", "factor_one", "factor_zero", "factor_nan", "delta_one", "delta_negative",
               "delta_without_patience", "factor_without_patience", "cpu_two_replicas", "nccl_four_replicas", "interval",
               "interval_and_cdf", "k_below_n", "k_above_n"]


def _check(flags, ctx):
    f = SimpleNamespace(**dict(dict(eval_every_steps=10, backend="auto", lr_plateau_patience=0, lr_plateau_factor=0.1,
                                    lr_plateau_min_delta=0.0, interval_method=False, worker_times_cdf_method=False),
                               **flags))
    ctx = dict(dict(on_gpu=True, world_size=1), **ctx)
    k = ctx.pop("k", ctx["world_size"])
    check_lr_plateau_flags(f, SimpleNamespace(**ctx), k)


@pytest.mark.parametrize("flags, ctx, msg", REFUSALS, ids=REFUSAL_IDS)
def test_refusals_name_their_reason(flags, ctx, msg):
    with pytest.raises(ValueError, match=msg):
        _check(flags, ctx)


def test_accepted_combinations():
    _check(dict(lr_plateau_patience=1, lr_plateau_factor=0.999, lr_plateau_min_delta=0.999), dict(world_size=8))
    _check(dict(_ON, worker_times_cdf_method=True), dict(world_size=4, k=2))          # cdf: every step waits for all N
    _check(dict(_ON, interval_method=True), dict(on_gpu=False, world_size=1))         # torch engine, one replica
    _check(dict(eval_every_steps=0, backend="gloo"), dict(on_gpu=False, world_size=4))  # off: nothing is checked


@pytest.mark.parametrize("args, world_size, msg", [
    (["--lr_plateau_patience=-2"], None, "must be >= 1"),
    (["--lr_plateau_patience=2", "--eval_every_steps=0"], None, "needs --eval_every_steps > 0"),
    (["--lr_plateau_patience=2", "--lr_plateau_factor=2"], None, r"must lie in \(0, 1\)"),
    (["--lr_plateau_min_delta=0.5"], None, "need --lr_plateau_patience"),
    (["--lr_plateau_patience=2"], 2, "one replica, not 2"),
], ids=["negative", "no_eval", "factor_two", "delta_without_patience", "two_replicas"])
def test_refused_before_any_work(tmp_path, clean_flags, args, world_size, msg):
    with pytest.raises(ValueError, match=msg):
        _train(str(tmp_path / "t"), *args, world_size=world_size)
    assert not (tmp_path / "t").exists()


# ---- torch-engine runs ------------------------------------------------------------------------------------------------
ARMED = ("--lr_plateau_patience=1", "--lr_plateau_min_delta=0.5")


def _summary_rates(d):
    import glob
    from distributedmnist_b200.utils.summary import read_tfevents
    files = glob.glob(os.path.join(str(d), "events.out.tfevents.*"))
    assert len(files) == 1
    return {int(ev["step"]): ev["scalars"]["learning_rate"] for ev in read_tfevents(files[0])
            if "learning_rate" in ev["scalars"]}


def test_torch_engine_cuts_at_the_known_steps(tmp_path, clean_flags, caplog):
    summ = ("--should_summarize=true", "--save_summaries_secs=0")
    ref = _train(str(tmp_path / "ref"), *summ)
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(str(tmp_path / "armed"), *(ARMED + summ))
    msgs = [r.getMessage() for r in caplog.records]
    rows = _rows(tmp_path / "armed")
    n = int(rows[0, 3])
    want = _cut_steps(rows)
    assert len(want) >= 5
    rep = res["lr_plateau"]
    assert rep == _file(tmp_path / "armed")
    assert rep == dict(patience=1, factor=0.1, min_delta=0.5, min_delta_rows=n // 2, examples=n, weights="live",
                       cuts=[dict(trigger_step=g, from_step=s) for g, s in want])
    sched = res["optimizer"].lr_schedule
    assert sched.cuts == [s for _g, s in want] and sched.factor == 0.1
    # one log line per cut, none a reference log scraper matches
    lines = [x for x in msgs if x.startswith("Learning rate plateau")]
    assert len(lines) == len(want)
    for k, (line, (g, s)) in enumerate(zip(lines, want)):
        mt = LINE.match(line)
        assert mt, line
        row = rows[rows[:, 0] == g][0]
        assert [int(x) for x in mt.groups()[:8]] == [k + 1, g, int(row[4]), n, int(rows[0, 4]), 1, n // 2, s]
        assert float(mt.group(9)) == pytest.approx(sched(s), rel=1e-5)
        assert not any(re.match(p, line) for p in SCRAPERS)
    # the summary's rate has the cuts in it
    rates = _summary_rates(tmp_path / "armed")
    plain = LearningRateSchedule.from_flags(FLAGS, 256, 1)
    assert rates and all(v == np.float32(sched(st)) for st, v in rates.items())
    assert any(v != np.float32(plain(st)) for st, v in rates.items())
    assert all(v == np.float32(plain(st)) for st, v in _summary_rates(tmp_path / "ref").items())
    # the same run as without the flag up to the first cut's step: the loss of step s is computed on the weights of step
    # s - 1, and the weights of step S_1 are the last ones the first cut does not touch
    s1 = want[0][1]
    k = [i for i, st in enumerate(res["steps"]) if st <= s1 + 1]
    assert res["steps"] == ref["steps"]
    assert [res["losses"][i] for i in k] == [ref["losses"][i] for i in k]
    assert res["losses"] != ref["losses"]
    ra = _rows(tmp_path / "ref")
    np.testing.assert_array_equal(rows[rows[:, 0] <= s1][:, [0, 3, 4, 5]], ra[ra[:, 0] <= s1][:, [0, 3, 4, 5]])


def test_flags_off_leave_logs_and_files_unchanged(tmp_path, clean_flags, caplog):
    def run(name, *args):
        caplog.clear()
        with caplog.at_level(logging.INFO, logger="dmnist"):
            r = _train(str(tmp_path / name), *args, steps=10)
        return r, [re.sub(r"[0-9.]+", "#", m.getMessage()) for m in caplog.records]
    a, la = run("a")
    b, lb = run("b", "--lr_plateau_patience=0")
    assert la == lb and a["losses"] == b["losses"] and "lr_plateau" not in a and "lr_plateau" not in b
    assert sorted(os.listdir(str(tmp_path / "a"))) == sorted(os.listdir(str(tmp_path / "b")))
    assert not os.path.exists(str(tmp_path / "a" / "worker0_lr_plateau.json"))
    assert not any("plateau" in m for m in la)


def test_restart_keeps_the_cuts_up_to_the_restored_step(tmp_path, clean_flags, caplog):
    d = str(tmp_path / "run")
    first = _train(d, *ARMED, steps=12)
    r = first["final_step"]
    cuts1 = _file(d)["cuts"]
    assert any(c["from_step"] > r for c in cuts1) and any(c["from_step"] <= r for c in cuts1)
    kept = [c for c in cuts1 if c["from_step"] <= r]
    # a different factor while cuts are kept is refused, and the file stays as it was
    with pytest.raises(ValueError, match=r"--lr_plateau_factor=0\.5 differs from the factor 0\.1 of the %d learning-rate"
                                         % len(kept)):
        _train(d, *ARMED, "--lr_plateau_factor=0.5", steps=20)
    assert _file(d)["cuts"] == cuts1
    # a restart without the flag ignores the file and leaves it alone
    d2 = str(tmp_path / "copy")
    import shutil
    shutil.copytree(d, d2)
    _train(d2, steps=14)
    assert _file(d2)["cuts"] == cuts1
    # a restart with the flag keeps the earlier cuts with from_step <= r, drops the rest, and starts the patience afresh
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="dmnist"):
        second = _train(d, *ARMED, steps=24)
    sched = second["optimizer"].lr_schedule
    rows = [x for x in _rows(d) if x[0] > r]                     # the second run's passes
    new = [dict(trigger_step=int(x[0]), from_step=int(x[0]) + STOP_MARGIN) for x in rows[1:]]
    assert second["lr_plateau"]["cuts"] == kept + new == _file(d)["cuts"]
    assert sched.cuts == [c["from_step"] for c in kept + new]
    msgs = [m.getMessage() for m in caplog.records]
    assert any(m.startswith("Learning rate plateau: %d cut(s) up to the restored global step #%d kept" % (len(kept), r))
               for m in msgs)
    # the second run's first update is made at the rate with the kept cuts
    plain = LearningRateSchedule.from_flags(FLAGS, 256, 1)
    assert sched(r) == plain(r) * 0.1 ** float(len(kept))


def test_new_kernel_is_sm_90a_without_spills_or_stack():
    """The in-tree build compiles csrc/eval_plateau.cu for sm_90a; its -Xptxas -v log lists eval_plateau_kernel."""
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    log = os.path.join(root, "build", "obj", "eval_plateau.log")
    if not os.path.exists(log):
        pytest.skip("no in-tree build log (build() has not run)")
    spec = importlib.util.spec_from_file_location("ptxas_report", os.path.join(root, "tools", "ptxas_report.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rows = [r for r in mod.parse(log) if "eval_plateau_kernel" in r["name"]]
    assert len(rows) == 1, [r["name"] for r in mod.parse(log)]
    r = rows[0]
    assert r["arch"] == "sm_90a" and r["spill_st"] == r["spill_ld"] == r["stack"] == 0, r
