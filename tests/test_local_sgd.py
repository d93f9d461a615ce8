"""Local SGD (``--local_sgd_steps``) on the CPU: the refusals and accepted combinations of ``check_local_sgd_flags``, the
exact emulation of the average against float64 arithmetic, the stop margin S = g + 2H, the torch engine with one replica
(plain SGD bit for bit), two gloo replicas (different weights between averages, bit-identical ones after each, the
average equal to the mean of the recorded copies, H = 1 against the K = N run), the report, JSON file and log line, and
the generated configurations."""
import json
import logging
import os
import re
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.flags import FLAGS, FlagError
from distributedmnist_b200.ops import aggrefs as A
from distributedmnist_b200.parallel.aggregators import local_sgd_report
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.parallel.launcher import run_replicas
from distributedmnist_b200.train import (LOCAL_SGD_JSON, STOP_MARGIN, _EarlyStopping, check_local_sgd_flags, stop_margin,
                                         train)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "_local_sgd_gloo_worker.py")


def _flags(*args):
    FLAGS.reset()
    FLAGS.parse(list(args))
    return FLAGS


def _ctx(n, gpu=True, rank=0):
    return SimpleNamespace(world_size=n, on_gpu=gpu, rank=rank, is_chief=rank == 0)


# ---- flags ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("args,n,msg", [
    (["--interval_method"], 4, r"--local_sgd_steps cannot be combined with --interval_method"),
    (["--worker_times_cdf_method"], 4, r"--local_sgd_steps cannot be combined with --worker_times_cdf_method"),
    (["--async_method"], 4, r"--local_sgd_steps cannot be combined with --async_method"),
    (["--num_replicas_to_aggregate=2"], 4, r"--num_replicas_to_aggregate must be left unset or equal the number of "
                                           r"replicas \(4\), got 2"),
    (["--num_replicas_to_aggregate=8"], 4, r"got 8"),
    (["--drop_connect"], 1, r"--local_sgd_steps cannot be combined with --drop_connect"),
    (["--moving_average_decay=0.99"], 1, r"cannot be combined with --moving_average_decay: between two averages"),
    (["--lr_plateau_patience=2", "--eval_every_steps=8"], 1, r"cannot be combined with --lr_plateau_patience"),
    (["--eval_every_steps=6"], 2, r"--eval_every_steps \(6\) must be a multiple of --local_sgd_steps \(4\)"),
])
def test_refusals_name_their_reason(args, n, msg):
    try:
        with pytest.raises(ValueError, match=msg):
            check_local_sgd_flags(_flags("--local_sgd_steps=4", *args), _ctx(n))
    finally:
        FLAGS.reset()


@pytest.mark.parametrize("h", ["-1", str(-2 ** 31), str(2 ** 31), str(2 ** 40)])
def test_period_out_of_range(h):
    try:
        with pytest.raises(ValueError, match=r"1 <= H < 2\^31, or 0 for off"):
            check_local_sgd_flags(_flags("--local_sgd_steps=" + h), _ctx(2))
    finally:
        FLAGS.reset()


@pytest.mark.parametrize("h", ["1.5", "four", "2e3"])
def test_period_not_an_integer(h):
    try:
        with pytest.raises(FlagError, match="is not an integer"):
            _flags("--local_sgd_steps=" + h)
    finally:
        FLAGS.reset()


@pytest.mark.parametrize("args,n,gpu", [
    ([], 8, True),
    (["--num_replicas_to_aggregate=8"], 8, True),
    (["--inject_straggler=*:lognormal:100:1.0"], 8, True),
    (["--inject_straggler=1:0.5:200"], 2, True),
    (["--inject_straggler=*:exp:50"], 4, True),
    (["--device_data", "--augment_max_shift=2", "--augment_max_rotation=10", "--augment_elastic_alpha=8"], 4, True),
    (["--weight_decay=0.0005"], 2, True),
    (["--lr_warmup_steps=10", "--lr_cosine_decay_steps=100"], 2, True),
    (["--eval_every_steps=40", "--target_accuracy=0.98", "--early_stopping_patience=3", "--keep_best_checkpoint"], 4, True),
    (["--eval_every_steps=8", "--eval_snapshot"], 4, True),
    (["--backend=gloo"], 2, False),
    ([], 2, False),
])
def test_accepted_combinations(args, n, gpu):
    from distributedmnist_b200.train import (check_best_flags, check_early_stopping_flags, check_eval_flags,
                                             check_lr_schedule_flags, check_target_flags)
    try:
        f = _flags("--local_sgd_steps=4", *args)
        ctx = _ctx(n, gpu)
        check_local_sgd_flags(f, ctx)
        check_eval_flags(f, ctx, n, dataset_test=object())
        check_target_flags(f, ctx)
        check_early_stopping_flags(f, ctx)
        check_lr_schedule_flags(f)
        check_best_flags(f)
    finally:
        FLAGS.reset()


def test_off_by_default_changes_nothing():
    try:
        f = _flags("--interval_method", "--num_replicas_to_aggregate=2", "--drop_connect", "--eval_every_steps=7")
        assert f.local_sgd_steps == 0
        check_local_sgd_flags(f, _ctx(4))
        assert stop_margin(f) == STOP_MARGIN == 2
    finally:
        FLAGS.reset()


# ---- the average's arithmetic ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
def test_average_against_float64(n):
    """The rank-order sum from +0.0 is one float64 add rounded once to fp32 per copy, and the division the float64 quotient
    of the two fp32 numbers rounded once (a correctly rounded fp32 division)."""
    rng = np.random.default_rng(n)
    ws = [(rng.standard_normal(4096) * 0.1).astype(np.float32) for _ in range(n)]
    s = np.zeros(4096, np.float32)
    for w in ws:
        s = (s.astype(np.float64) + w.astype(np.float64)).astype(np.float32)
    want = (s.astype(np.float64) / n).astype(np.float32)
    got = A.local_average(ws)
    assert A.bits(got).tolist() == A.bits(want).tolist()
    exact = sum(w.astype(np.float64) for w in ws) / n
    top = sum(np.abs(w).astype(np.float64) for w in ws)
    assert np.all(np.abs(got - exact) <= n * np.spacing(top.astype(np.float32)).astype(np.float64))


def test_average_exact_cases_and_ftz():
    w = np.array([1.0, -3.0, 2.0 ** -20, 0.0], np.float32)
    assert A.bits(A.local_average([w])).tolist() == A.bits(w).tolist()                # N = 1: the identity
    assert A.bits(A.local_average([w] * 8)).tolist() == A.bits(w).tolist()            # equal copies, N a power of 2
    tiny = np.array([2.0 ** -126], np.float32)
    assert A.local_average([tiny, np.zeros(1, np.float32)])[0] == 0.0                # the quotient is subnormal: flushed
    assert A.local_average([np.array([2.0 ** -130], np.float32)] * 2)[0] == 0.0      # subnormal operands: flushed


# ---- stop margin ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,g", [(1, 10), (3, 12), (4, 40), (16, 160)])
def test_stop_margin_is_two_periods(h, g):
    try:
        f = _flags("--local_sgd_steps=%d" % h)
        s = g + stop_margin(f)
        assert s == g + 2 * h
        assert s % h == 0 and s >= g + h + 1            # an averaging step, after the host has waited for step g + H
        es = _EarlyStopping(1, 0.0, 100, "live", stop_margin(f))
        es.add(g, 100, 90)
        es.add(g + h, 100, 50)
        assert es.report()["stop_step"] == g + h + 2 * h
    finally:
        FLAGS.reset()


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


@pytest.mark.parametrize("h", [1, 3])
def test_torch_engine_one_replica_is_plain_sgd(tmp_path, one_replica, caplog, h):
    plain = _train(str(tmp_path / "plain"), "--lr_warmup_steps=3")
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(str(tmp_path / "local"), "--lr_warmup_steps=3", "--local_sgd_steps=%d" % h)
    assert torch.equal(plain["params"].view(torch.int32), res["params"].view(torch.int32))
    assert res["final_step"] == plain["final_step"] == 8 and res["steps"] == plain["steps"]
    rounds = 8 // h + (1 if 8 % h else 0)            # the averaging steps, and the final average after step 8
    rep = res["local_sgd"]
    assert rep == local_sgd_report(h, rounds, 0, 0) and rep["rounds"] == rounds and rep["wait_total_s"] == 0.0
    with open(str(tmp_path / "local" / (LOCAL_SGD_JSON % 0))) as f:
        assert json.load(f) == rep
    msgs = [m.getMessage() for m in caplog.records]
    line = [m for m in msgs if m.startswith("Local SGD: ")]
    assert line == ["Local SGD: worker 0 averaged every %d step(s); %d averaging round(s), 0.000000 s in their barriers "
                    "(mean 0.000000 s, max 0.000000 s); final global step 8" % (h, rounds)]
    assert not re.match(r".*step ([0-9]*),.*", line[0])        # tools/benchmark.py's step scraper skips it
    attained = [int(m.split(": ")[1]) for m in msgs if m.startswith("Global step attained: ")]
    assert attained == list(range(1, 9))


def test_torch_engine_eval_and_target(tmp_path, one_replica):
    """With evaluation every 2H steps and a target the run reaches, the run ends as --max_steps = g + 2H would end it, and
    the final pass scores the final average."""
    res = _train(str(tmp_path / "local"), "--local_sgd_steps=2", "--eval_every_steps=4", "--target_accuracy=0.01",
                 steps=40)
    tta = res["time_to_accuracy"]
    assert tta["reached"] and tta["global_step"] == 4
    assert res["final_step"] == 4 + 2 * 2 + 1
    assert [r[0] for r in res["evals"]] == [4, 8, 9]


# ---- two gloo replicas ----------------------------------------------------------------------------------------------
COMMON = ["--model=mlp2", "--mlp_hidden=32", "--batch_size=16", "--backend=gloo", "--initial_learning_rate=0.05",
          "--save_interval_secs=1000", "--dropout_keep_prob=1.0"]


def _run(tmp_path, extra, n=2, timeout=180):
    out = str(tmp_path / "out")
    argv = [WORKER, str(tmp_path / "res_RANK.npz")] + COMMON + ["--train_dir=%s" % (tmp_path / "train_dir")] + extra
    codes = run_replicas(["-c", "import os,sys,runpy; sys.argv=[a.replace('RANK', os.environ['RANK']) for a in sys.argv[1:]];"
                          " runpy.run_path(sys.argv[0], run_name='__main__')"] + argv, n, timeout=timeout, out_dir=out)
    logs = [open(os.path.join(out, f)).read() for f in sorted(os.listdir(out))]
    assert codes == [0] * n, "\n".join(l[-2000:] for l in logs)
    return [dict(np.load(str(tmp_path / ("res_%d.npz" % r)))) for r in range(n)], logs


def test_gloo_replicas_differ_between_averages_and_agree_after(tmp_path):
    (a, b), logs = _run(tmp_path, ["--max_steps=10", "--local_sgd_steps=3"])
    assert a["steps"].tolist() == b["steps"].tolist() == list(range(1, 12))
    for t, s in enumerate(a["steps"].tolist()):
        same = A.bits(a["after"][t]).tolist() == A.bits(b["after"][t]).tolist()
        assert same == (s % 3 == 0), s
    # every average, the final one after step 11 included, is the mean of the copies the two workers held before it
    assert len(a["before"]) == len(b["before"]) == 4
    for r in range(4):
        want = A.local_average([a["before"][r], b["before"][r]])
        ta = 3 * r + 2
        got = a["after"][ta] if ta < 11 else a["final"]
        assert A.bits(got).tolist() == A.bits(want).tolist()
    assert A.bits(a["final"]).tolist() == A.bits(b["final"]).tolist()
    assert int(a["final_step"]) == int(b["final_step"]) == 11
    for r, (res, log) in enumerate(zip((a, b), logs)):
        rep = json.loads(str(res["report"]))
        assert rep["period"] == 3 and rep["rounds"] == 4 and rep["wait_total_s"] > 0.0
        assert rep["wait_max_s"] <= rep["wait_total_s"]
        assert "Local SGD: worker %d averaged every 3 step(s); 4 averaging round(s)" % r in log
        with open(str(tmp_path / "train_dir" / (LOCAL_SGD_JSON % r))) as f:
            assert json.load(f) == rep


def test_gloo_period_one_matches_k_equals_n(tmp_path):
    """H = 1: mean of (w - lr g_q) against w - lr mean(g_q), equal in exact arithmetic; in fp32 they differ by rounding."""
    (a, b), _ = _run(tmp_path / "local", ["--max_steps=12", "--local_sgd_steps=1"])
    (c, d), _ = _run(tmp_path / "sync", ["--max_steps=12"])
    assert A.bits(a["final"]).tolist() == A.bits(b["final"]).tolist() and int(a["final_step"]) == 13
    assert A.bits(c["final"]).tolist() == A.bits(d["final"]).tolist() and int(c["final_step"]) == 13
    diff = np.abs(a["final"].astype(np.float64) - c["final"].astype(np.float64))
    scale = np.maximum(np.abs(c["final"]).astype(np.float64), 1e-3)
    assert float((diff / scale).max()) < 1e-4
    assert not np.array_equal(a["final"], np.zeros_like(a["final"]))


# ---- configurations -------------------------------------------------------------------------------------------------
def test_generated_cfgs():
    def cfg(name):
        with open(os.path.join(ROOT, "cfg", "8_gpus", name)) as f:
            return eval(f.read(), {"Cfg": dict})
    for name, flags in (("8_gpus_local_4", " --local_sgd_steps=4"), ("8_gpus_local_16", " --local_sgd_steps=16"),
                        ("8_gpus_local_16_lognormal", " --local_sgd_steps=16 --inject_straggler=*:lognormal:100:1.0")):
        c = cfg(name)
        assert c["name"] == name and c["num_replicas_to_aggregate"] == "8" and c["n_gpus"] == 8
        assert c["extra_flags"] == "--save_interval_secs=0.05 --log_every=500" + flags
