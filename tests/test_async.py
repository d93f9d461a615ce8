"""Asynchronous SGD (``--async_method``) on the CPU: the refusals and accepted combinations of ``check_async_flags``, the
exact emulation of the device update against float64 arithmetic, the torch engine with one replica (plain SGD bit for
bit, every staleness 0), the staleness report, JSON file and log line, the parsing of an async log, and the generated
configurations."""
import json
import logging
import os
import re
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.ops import aggrefs as A
from distributedmnist_b200.parallel.aggregators import STALENESS_BUCKETS, staleness_report
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.train import STALENESS_JSON, check_async_flags, train

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
    (["--interval_method"], 4, True, r"--async_method cannot be combined with --interval_method"),
    (["--worker_times_cdf_method"], 4, True, r"--async_method cannot be combined with --worker_times_cdf_method"),
    (["--num_replicas_to_aggregate=2"], 4, True, r"--num_replicas_to_aggregate must be left unset or equal the number "
                                                 r"of replicas \(4\), got 2"),
    (["--num_replicas_to_aggregate=8"], 4, True, r"got 8"),
    (["--drop_connect"], 1, True, r"--async_method cannot be combined with --drop_connect"),
    (["--lr_plateau_patience=2", "--eval_every_steps=10"], 1, True, r"cannot be combined with --lr_plateau_patience"),
    (["--moving_average_decay=0.99"], 1, True, r"cannot be combined with --moving_average_decay"),
    (["--backend=gloo"], 2, True, r"torch engine \(--backend=gloo\) is implemented for one replica, not 2"),
    ([], 2, False, r"torch engine \(--backend=auto, no GPU\) is implemented for one replica, not 2"),
])
def test_refusals_name_their_reason(args, n, gpu, msg):
    try:
        with pytest.raises(ValueError, match=msg):
            check_async_flags(_flags("--async_method", *args), _ctx(n, gpu))
    finally:
        FLAGS.reset()


@pytest.mark.parametrize("args,n,gpu", [
    ([], 8, True),
    (["--num_replicas_to_aggregate=8"], 8, True),
    (["--inject_straggler=*:lognormal:100:1.0"], 8, True),
    (["--device_data", "--augment_max_shift=2", "--augment_max_rotation=10", "--augment_elastic_alpha=8"], 4, True),
    (["--weight_decay=0.0005"], 2, True),
    (["--lr_warmup_steps=10", "--lr_cosine_decay_steps=100"], 2, True),
    (["--eval_every_steps=50", "--target_accuracy=0.98", "--early_stopping_patience=3", "--keep_best_checkpoint"], 4, True),
    (["--eval_every_steps=50", "--eval_snapshot"], 4, True),
    (["--backend=gloo"], 1, True),
    ([], 1, False),
])
def test_accepted_combinations(args, n, gpu):
    from distributedmnist_b200.train import (check_best_flags, check_early_stopping_flags, check_eval_flags,
                                             check_lr_schedule_flags, check_target_flags)
    try:
        f = _flags("--async_method", *args)
        ctx = _ctx(n, gpu)
        check_async_flags(f, ctx)
        k = n if f.num_replicas_to_aggregate == -1 else f.num_replicas_to_aggregate
        check_eval_flags(f, ctx, k, dataset_test=object())
        check_target_flags(f, ctx)
        check_early_stopping_flags(f, ctx)
        check_lr_schedule_flags(f)
        check_best_flags(f)
    finally:
        FLAGS.reset()


def test_off_by_default_changes_nothing():
    try:
        f = _flags("--interval_method", "--num_replicas_to_aggregate=2", "--drop_connect")
        assert f.async_method is False
        check_async_flags(f, _ctx(4))
    finally:
        FLAGS.reset()


# ---- the update's arithmetic ----------------------------------------------------------------------------------------
def test_emulation_against_float64():
    """-fl(scale * g) is the float64 product rounded once to fp32, and each add the float64 sum of two fp32 numbers rounded
    once: the emulation equals that arithmetic exactly, away from subnormals, where it flushes them to signed zeros."""
    rng = np.random.default_rng(1)
    w = (rng.standard_normal(4096) * 0.1).astype(np.float32)
    scale = np.float32(0.0173)
    xs = []
    want = w.astype(np.float64)
    want32 = w.copy()
    for _ in range(5):
        g = (rng.standard_normal(4096) * 3).astype(np.float32)
        x = A.async_update(g, scale)
        prod = np.float32(float(scale)) * g.astype(np.float64)               # exact in float64
        assert A.bits(x).tolist() == A.bits(-(prod.astype(np.float32))).tolist()
        xs.append(x)
        want32 = (want32.astype(np.float64) + x.astype(np.float64)).astype(np.float32)   # exact sum, one rounding
        want = want + x.astype(np.float64)
    got = A.async_apply(w, xs)
    assert A.bits(got).tolist() == A.bits(want32).tolist()
    # five rounded adds stay within 5 half-ulps (at the largest magnitude the sum can pass through) of the exact float64
    # sum of the rounded updates
    top = np.abs(w).astype(np.float64) + sum(np.abs(x).astype(np.float64) for x in xs)
    assert np.all(np.abs(got - want) <= 2.5 * np.spacing(top.astype(np.float32)).astype(np.float64))


def test_emulation_flushes_subnormals():
    tiny = np.float32(2.0 ** -130)                                           # subnormal
    assert A.ftz(np.array([tiny, -tiny, 1.0], np.float32)).tolist() == [0.0, 0.0, 1.0]
    assert np.signbit(A.ftz(np.array([-tiny], np.float32)))[0]
    # a product that lands below FLT_MIN is flushed; an add that lands there too
    x = A.async_update(np.array([2.0 ** -70], np.float32), np.float32(2.0 ** -60))
    assert x[0] == 0.0
    w = A.async_apply(np.array([2.0 ** -125], np.float32), [np.array([-0.75 * 2.0 ** -125], np.float32)])
    assert w[0] == 0.0


def test_exact_updates_are_order_free():
    """Small integers times a power of two: every product and sum is exact, so any order of the adds gives init - sum."""
    rng = np.random.default_rng(2)
    w = rng.integers(-64, 64, 512).astype(np.float32)
    scale = np.float32(2.0 ** -3)
    xs = [A.async_update(rng.integers(-32, 32, 512).astype(np.float32), scale) for _ in range(12)]
    want = w.astype(np.float64) + sum(x.astype(np.float64) for x in xs)
    for perm in (range(12), reversed(range(12)), rng.permutation(12)):
        got = A.async_apply(w, [xs[i] for i in perm])
        assert A.bits(got).tolist() == A.bits(want.astype(np.float32)).tolist()


# ---- staleness report -----------------------------------------------------------------------------------------------
def test_staleness_report():
    hist = [0] * STALENESS_BUCKETS
    taus = [0] * 40 + [1] * 30 + [2] * 29 + [70]
    for t in taus:
        hist[min(t, 63)] += 1
    rep = staleness_report(hist, sum(taus), max(taus))
    assert rep["updates"] == 100 and rep["max"] == 70 and rep["hist"] == hist
    assert rep["mean"] == pytest.approx(sum(taus) / 100.0)
    assert rep["p50"] == 1 and rep["p99"] == 2
    hist[63] += 5
    assert staleness_report(hist, sum(taus) + 5 * 80, 80)["p99"] == 63      # 63: >= 63
    assert staleness_report([0] * 64, 0, 0) == dict(updates=0, hist=[0] * 64, mean=0.0, max=0, p50=0, p99=0)


# ---- the torch engine, one replica ------------------------------------------------------------------------------------
def _train(train_dir, *extra, steps=7):
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=32", "--max_steps=%d" % steps, "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=5", "--save_interval_secs=1000", "--initial_learning_rate=0.05",
                 "--backend=gloo", "--dropout_keep_prob=1.0", "--log_every=1"] + list(extra))
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


def test_torch_engine_is_plain_sgd_with_staleness_zero(tmp_path, one_replica, caplog):
    plain = _train(str(tmp_path / "plain"), "--lr_warmup_steps=3")
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(str(tmp_path / "async"), "--lr_warmup_steps=3", "--async_method")
    assert torch.equal(plain["params"].view(torch.int32), res["params"].view(torch.int32))
    assert res["final_step"] == plain["final_step"] == 8 and res["steps"] == plain["steps"]
    st = res["staleness"]
    assert st["updates"] == 8 and st["hist"][0] == 8 and sum(st["hist"]) == 8
    assert st["mean"] == 0.0 and st["max"] == 0 and st["p50"] == 0 and st["p99"] == 0
    assert res["accepted"] == 8 and res["dropped"] == 0
    with open(str(tmp_path / "async" / (STALENESS_JSON % 0))) as f:
        assert json.load(f) == st
    msgs = [m.getMessage() for m in caplog.records]
    line = [m for m in msgs if m.startswith("Staleness: ")]
    assert line == ["Staleness: worker 0 applied 8 update(s); staleness of its updates (global steps between pull and "
                    "update) mean 0.000, p50 0, p99 0, max 0; final global step 8"]
    assert not any(re.match(p, line[0]) for p in SCRAPERS)
    attained = [int(m.split(": ")[1]) for m in msgs if m.startswith("Global step attained: ")]
    assert attained == list(range(1, 9))


def test_async_log_parses_with_the_benchmark_scrapers(tmp_path, one_replica):
    """The log lines an async run writes keep their format: tools/benchmark.py reads the step of the last one."""
    log = tmp_path / "out_worker_0"
    handler = logging.FileHandler(str(log))
    handler.setFormatter(logging.Formatter("%(message)s"))
    logger = logging.getLogger("dmnist")
    logger.addHandler(handler)
    try:
        _train(str(tmp_path / "async"), "--async_method", steps=5)
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
def test_generated_cfgs_are_committed(tmp_path, monkeypatch):
    """tools/make_cfgs.py writes the two async configurations, and they are the committed files."""
    monkeypatch.syspath_prepend(os.path.join(ROOT, "tools"))
    import make_cfgs
    monkeypatch.setattr(make_cfgs, "ROOT", str(tmp_path))
    make_cfgs.main()
    for name in sorted(os.listdir(os.path.join(ROOT, "cfg", "8_gpus"))):
        with open(os.path.join(tmp_path, "cfg", "8_gpus", name)) as f, open(os.path.join(ROOT, "cfg", "8_gpus", name)) as g:
            assert f.read() == g.read(), name
    def cfg(name):
        with open(os.path.join(ROOT, "cfg", "8_gpus", name)) as f:
            return eval(f.read(), {"Cfg": dict})
    plain, lognormal = cfg("8_gpus_async"), cfg("8_gpus_async_lognormal")
    assert plain["extra_flags"].endswith(" --async_method=true") and plain["num_replicas_to_aggregate"] == "8"
    assert lognormal["extra_flags"].endswith(" --async_method=true --inject_straggler=*:lognormal:100:1.0")
    assert cfg("8_gpus_8_aggregate_sync_lognormal")["extra_flags"].endswith(" --inject_straggler=*:lognormal:100:1.0")
