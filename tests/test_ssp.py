"""Stale synchronous parallel (``--ssp_staleness`` with ``--async_method``) on the CPU: the refusals and accepted
combinations of ``check_async_flags``, the word-level model of the wait, the clock publication and retirement under every
schedule of small instances (and three mutants that must fail), the torch engine with one replica against a plain
asynchronous run, the report, JSON file and log line, and the generated configurations."""
import json
import logging
import os
import re
from types import SimpleNamespace

import pytest
import torch

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.parallel.protocol import ProtocolHazard, SSPModel, explore_schedules
from distributedmnist_b200.train import SSP_JSON, STALENESS_JSON, check_async_flags, train

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRAPERS = [r".*step ([0-9]*),.*", r"Num examples: ([0-9]*)  Precision @ 1: ([\.0-9]*) Loss: ([\.0-9]*) Time: ([\.0-9]*)",
            r".* step=([0-9]*)", r".*ELAPSED TIMES (.*)", r".*ITERATION TIMES (.*)"]       # tools/benchmark.py


def _flags(*args):
    FLAGS.reset()
    FLAGS.parse(list(args))
    return FLAGS


def _ctx(n, gpu=True, rank=0):
    return SimpleNamespace(world_size=n, on_gpu=gpu, rank=rank, is_chief=rank == 0)


# ---- flags ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("args,n,gpu,msg", [
    (["--ssp_staleness=0"], 4, True, r"--ssp_staleness bounds asynchronous SGD and needs --async_method"),
    (["--ssp_staleness=3", "--local_sgd_steps=4"], 4, True, r"needs --async_method"),
    (["--async_method", "--ssp_staleness=-2"], 4, True, r"0 <= s < 2\^31, or -1 for off; got -2"),
    (["--async_method", "--ssp_staleness=2147483648"], 4, True, r"got 2147483648"),
    (["--async_method", "--ssp_staleness=1", "--interval_method"], 4, True,
     r"--async_method cannot be combined with --interval_method"),
    (["--async_method", "--ssp_staleness=1", "--worker_times_cdf_method"], 4, True, r"--worker_times_cdf_method"),
    (["--async_method", "--ssp_staleness=1", "--num_replicas_to_aggregate=2"], 4, True, r"got 2"),
    (["--async_method", "--ssp_staleness=0", "--drop_connect"], 1, True, r"cannot be combined with --drop_connect"),
    (["--async_method", "--ssp_staleness=0", "--lr_plateau_patience=2", "--eval_every_steps=10"], 1, True,
     r"--lr_plateau_patience"),
    (["--async_method", "--ssp_staleness=0", "--moving_average_decay=0.99"], 1, True, r"--moving_average_decay"),
    (["--async_method", "--ssp_staleness=0", "--backend=gloo"], 2, True, r"implemented for one replica, not 2"),
    (["--async_method", "--ssp_staleness=4"], 2, False, r"no GPU\) is implemented for one replica, not 2"),
])
def test_refusals_name_their_reason(args, n, gpu, msg):
    try:
        with pytest.raises(ValueError, match=msg):
            check_async_flags(_flags(*args), _ctx(n, gpu))
    finally:
        FLAGS.reset()


@pytest.mark.parametrize("value", ["1.5", "x", "true"])
def test_non_integer_values_are_refused_by_the_parser(value):
    try:
        with pytest.raises(Exception):
            _flags("--async_method", "--ssp_staleness=%s" % value)
            check_async_flags(FLAGS, _ctx(2))
    finally:
        FLAGS.reset()


@pytest.mark.parametrize("value", [1.5, True])
def test_non_integer_values_are_refused(value):
    try:
        f = _flags("--async_method")
        f.ssp_staleness = value
        with pytest.raises(ValueError, match=r"--ssp_staleness must be an integer"):
            check_async_flags(f, _ctx(2))
    finally:
        FLAGS.reset()


@pytest.mark.parametrize("args,n,gpu", [
    (["--ssp_staleness=0"], 8, True),
    (["--ssp_staleness=4", "--inject_straggler=*:lognormal:100:1.0"], 8, True),
    (["--ssp_staleness=2147483647"], 2, True),
    (["--ssp_staleness=-1"], 8, True),
    (["--ssp_staleness=1", "--device_data", "--augment_max_shift=2", "--augment_max_rotation=10"], 4, True),
    (["--ssp_staleness=2", "--lr_warmup_steps=10", "--lr_cosine_decay_steps=100", "--weight_decay=0.0005"], 2, True),
    (["--ssp_staleness=0", "--eval_every_steps=50", "--target_accuracy=0.98", "--early_stopping_patience=3",
      "--keep_best_checkpoint"], 4, True),
    (["--ssp_staleness=0", "--backend=gloo"], 1, True),
    (["--ssp_staleness=3"], 1, False),
])
def test_accepted_combinations(args, n, gpu):
    from distributedmnist_b200.train import (check_best_flags, check_early_stopping_flags, check_eval_flags,
                                             check_lr_schedule_flags, check_target_flags)
    try:
        f = _flags("--async_method", *args)
        ctx = _ctx(n, gpu)
        check_async_flags(f, ctx)
        check_eval_flags(f, ctx, n, dataset_test=object())
        check_target_flags(f, ctx)
        check_early_stopping_flags(f, ctx)
        check_lr_schedule_flags(f)
        check_best_flags(f)
    finally:
        FLAGS.reset()


def test_off_by_default():
    try:
        f = _flags("--async_method")
        assert f.ssp_staleness == -1
        check_async_flags(f, _ctx(4))
        check_async_flags(_flags(), _ctx(4))
    finally:
        FLAGS.reset()


# ---- the protocol model ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,iters", [(2, (4, 2)), (2, (3, 1)), (3, (4, 4, 2)), (3, (3, 4, 1))])
@pytest.mark.parametrize("s", [0, 1])
def test_model_every_schedule_keeps_b1_to_b4(n, iters, s):
    """Every state reachable under any schedule, one replica stopping early: B1-B4 hold at every step, and every copy
    ends with every update."""
    runs = explore_schedules(lambda: SSPModel(n, s, iters), max_runs=2000000, dedup=True)
    assert runs > 10, runs


@pytest.mark.parametrize("n,s,iters,max_steps", [(2, 0, (6, 6), 4), (2, 1, (6, 6), 5), (3, 0, (4, 4, 4), 5),
                                                 (3, 1, (5, 5, 5), 6), (3, 1, (5, 5, 2), 6)])
def test_model_every_schedule_with_the_stop_rule(n, s, iters, max_steps):
    """The pipelined loop's stop rule decides how many iterations each replica runs: B1-B4 hold, and two replicas that
    stopped by the rule differ by at most s + 3 updates (DESIGN.md §4)."""
    runs = explore_schedules(lambda: SSPModel(n, s, iters, max_steps=max_steps), max_runs=2000000, dedup=True)
    assert runs > 10, runs


@pytest.mark.parametrize("n,s", [(2, 0), (2, 1), (3, 0), (3, 1)])
def test_model_mutant_publishing_before_the_apply_fails(n, s):
    with pytest.raises(ProtocolHazard, match=r"B1: replica \d pulled \d of replica \d's updates"):
        explore_schedules(lambda: SSPModel(n, s, (4,) * (n - 1) + (2,), publish_before_apply=True), dedup=True)


@pytest.mark.parametrize("n,s", [(2, 0), (2, 1), (3, 0), (3, 1)])
def test_model_mutant_without_retirement_deadlocks(n, s):
    with pytest.raises(ProtocolHazard, match=r"B4: deadlock"):
        explore_schedules(lambda: SSPModel(n, s, (4,) * (n - 1) + (1,), retire=False), dedup=True)


@pytest.mark.parametrize("n,s", [(2, 0), (2, 1), (3, 0), (3, 1)])
def test_model_mutant_waiting_for_c_minus_s_minus_1_fails(n, s):
    with pytest.raises(ProtocolHazard, match=r"B1|B2"):
        explore_schedules(lambda: SSPModel(n, s, (4,) * (n - 1) + (2,), slack=1), dedup=True)


def test_dedup_visits_what_plain_exploration_visits():
    """On an instance small enough for both, the deduplicated exploration and the plain one see the same mutant fail and
    the same correct model pass."""
    plain = explore_schedules(lambda: SSPModel(2, 0, (3, 2)))
    assert plain > explore_schedules(lambda: SSPModel(2, 0, (3, 2)), dedup=True) > 1
    for kw in (dict(publish_before_apply=True), dict(slack=1)):
        with pytest.raises(ProtocolHazard):
            explore_schedules(lambda: SSPModel(2, 0, (3, 2), **kw))


# ---- the torch engine, one replica ------------------------------------------------------------------------------------
def _train(train_dir, *extra, steps=7):
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=32", "--max_steps=%d" % steps, "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000", "--initial_learning_rate=0.05",
                 "--backend=gloo", "--dropout_keep_prob=1.0", "--log_every=1", "--async_method"] + list(extra))
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    return train(ctx, ds.train, ds.validation, FLAGS)


@pytest.fixture
def one_replica(monkeypatch):
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    yield
    FLAGS.reset()


@pytest.mark.parametrize("s", [0, 3])
def test_torch_engine_one_replica_equals_plain_async(tmp_path, one_replica, caplog, s):
    plain = _train(str(tmp_path / "plain"), "--lr_warmup_steps=3")
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(str(tmp_path / "ssp"), "--lr_warmup_steps=3", "--ssp_staleness=%d" % s)
    assert torch.equal(plain["params"].view(torch.int32), res["params"].view(torch.int32))
    assert res["final_step"] == plain["final_step"] == 8 and res["steps"] == plain["steps"]
    assert res["staleness"] == plain["staleness"]
    assert "ssp" not in plain
    rep = res["ssp"]
    assert rep == dict(s=s, waits=0, wait_total_ns=0, wait_max_ns=0, lead_max=0, updates=8)
    with open(str(tmp_path / "ssp" / (SSP_JSON % 0))) as f:
        assert json.load(f) == rep
    with open(str(tmp_path / "ssp" / (STALENESS_JSON % 0))) as f, open(str(tmp_path / "plain" / (STALENESS_JSON % 0))) as g:
        assert f.read() == g.read()
    assert not os.path.exists(str(tmp_path / "plain" / (SSP_JSON % 0)))
    msgs = [m.getMessage() for m in caplog.records]
    line = [m for m in msgs if m.startswith("Stale synchronous: ")]
    assert line == ["Stale synchronous: worker 0 ran at most %d update(s) ahead of the slowest running replica; 0 of its "
                    "8 update(s) waited, 0.000000 s in total, longest 0.000000 s; largest lead seen 0; final global "
                    "step 8" % s]
    assert not any(re.match(p, line[0]) for p in SCRAPERS)
    assert len([m for m in msgs if m.startswith("Staleness: ")]) == 1


def test_async_log_parses_with_the_benchmark_scrapers(tmp_path, one_replica):
    import sys
    log = tmp_path / "out_worker_0"
    handler = logging.FileHandler(str(log))
    handler.setFormatter(logging.Formatter("%(message)s"))
    logger = logging.getLogger("dmnist")
    logger.addHandler(handler)
    try:
        _train(str(tmp_path / "ssp"), "--ssp_staleness=1", steps=5)
    finally:
        logger.removeHandler(handler)
        handler.close()
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        import benchmark
        assert benchmark.current_iteration(str(log)) == 5
    finally:
        sys.path.remove(os.path.join(ROOT, "tools"))


# ---- configurations -------------------------------------------------------------------------------------------------
def test_generated_ssp_cfgs_are_committed(tmp_path, monkeypatch):
    monkeypatch.syspath_prepend(os.path.join(ROOT, "tools"))
    import make_cfgs
    monkeypatch.setattr(make_cfgs, "ROOT", str(tmp_path))
    make_cfgs.main()
    for s in (0, 4):
        name = "8_gpus_ssp_%d_lognormal" % s
        with open(os.path.join(tmp_path, "cfg", "8_gpus", name)) as f, open(os.path.join(ROOT, "cfg", "8_gpus", name)) as g:
            text = g.read()
            assert f.read() == text
        cfg = eval(text, {"Cfg": dict})
        assert cfg["num_replicas_to_aggregate"] == "8"
        assert cfg["extra_flags"].endswith(" --async_method=true --ssp_staleness=%d --inject_straggler=*:lognormal:100:1.0"
                                           % s)
