"""Gossip SGD (``--gossip_method``) on the CPU: the refusals and accepted combinations of ``check_gossip_flags``, the exact
emulation of the mix against float64 arithmetic and against the local-SGD average for N <= 3, the word-level model
(``parallel/protocol.py::GossipModel``) explored exhaustively over three iterations with its mutants, and under random
schedules with the stop rule, the stop margin, the torch engine (one
replica bit for bit plain SGD; four gloo replicas against the emulation of their recorded half steps; three gloo
replicas against ``--local_sgd_steps=1``), the report, JSON file and log line, and the configurations."""
import json
import logging
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.ops import aggrefs as A
from distributedmnist_b200.parallel.aggregators import gossip_report
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.parallel.launcher import run_replicas
from distributedmnist_b200.parallel.protocol import GossipModel, ProtocolHazard, explore_schedules, run_random
from distributedmnist_b200.train import GOSSIP_JSON, STOP_MARGIN, _EarlyStopping, check_gossip_flags, stop_margin, train

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "_gossip_gloo_worker.py")


def _flags(*args):
    FLAGS.reset()
    FLAGS.parse(list(args))
    return FLAGS


def _ctx(n, gpu=True, rank=0):
    return SimpleNamespace(world_size=n, on_gpu=gpu, rank=rank, is_chief=rank == 0)


# ---- flags ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("args,n,msg", [
    (["--interval_method"], 4, r"--gossip_method cannot be combined with --interval_method"),
    (["--worker_times_cdf_method"], 4, r"--gossip_method cannot be combined with --worker_times_cdf_method"),
    (["--async_method"], 4, r"--gossip_method cannot be combined with --async_method"),
    (["--async_method", "--ssp_staleness=2"], 4, r"--gossip_method cannot be combined with --async_method \(or "
                                                 r"--ssp_staleness\)"),
    (["--local_sgd_steps=4"], 4, r"--gossip_method cannot be combined with --local_sgd_steps"),
    (["--num_replicas_to_aggregate=2"], 4, r"--num_replicas_to_aggregate must be left unset or equal the number of "
                                           r"replicas \(4\), got 2"),
    (["--num_replicas_to_aggregate=8"], 4, r"got 8"),
    (["--drop_connect"], 1, r"--gossip_method cannot be combined with --drop_connect"),
    (["--moving_average_decay=0.99"], 1, r"cannot be combined with --moving_average_decay: the replicas are not in lock"),
    (["--lr_plateau_patience=2", "--eval_every_steps=8"], 1, r"cannot be combined with --lr_plateau_patience"),
])
def test_refusals_name_their_reason(args, n, msg):
    try:
        with pytest.raises(ValueError, match=msg):
            check_gossip_flags(_flags("--gossip_method", *args), _ctx(n))
    finally:
        FLAGS.reset()


@pytest.mark.parametrize("args,n,gpu", [
    ([], 8, True),
    (["--num_replicas_to_aggregate=8"], 8, True),
    (["--model=mlp2"], 4, True),
    (["--model=mlp3"], 4, True),
    (["--inject_straggler=*:lognormal:100:1.0"], 8, True),
    (["--inject_straggler=1:0.5:200"], 2, True),
    (["--device_data", "--augment_max_shift=2", "--augment_max_rotation=10", "--augment_elastic_alpha=8"], 4, True),
    (["--weight_decay=0.0005"], 2, True),
    (["--lr_warmup_steps=10", "--lr_cosine_decay_steps=100"], 2, True),
    (["--eval_every_steps=7", "--target_accuracy=0.98", "--early_stopping_patience=3", "--keep_best_checkpoint"], 4, True),
    (["--eval_every_steps=8", "--eval_snapshot"], 4, True),
    (["--backend=gloo"], 4, False),
    ([], 3, False),
])
def test_accepted_combinations(args, n, gpu):
    from distributedmnist_b200.train import (check_async_flags, check_best_flags, check_early_stopping_flags,
                                             check_eval_flags, check_local_sgd_flags, check_lr_schedule_flags,
                                             check_target_flags)
    try:
        f = _flags("--gossip_method", *args)
        ctx = _ctx(n, gpu)
        check_async_flags(f, ctx)
        check_local_sgd_flags(f, ctx)
        check_gossip_flags(f, ctx)
        check_eval_flags(f, ctx, n, dataset_test=object())
        check_target_flags(f, ctx)
        check_early_stopping_flags(f, ctx)
        check_lr_schedule_flags(f)
        check_best_flags(f)
    finally:
        FLAGS.reset()


def test_off_by_default_changes_nothing():
    try:
        f = _flags("--interval_method", "--num_replicas_to_aggregate=2", "--drop_connect", "--local_sgd_steps=3")
        assert f.gossip_method is False
        check_gossip_flags(f, _ctx(4))
        assert stop_margin(f, 8) == STOP_MARGIN * 3
    finally:
        FLAGS.reset()


# ---- the mix's arithmetic -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 8])
def test_mix_against_float64(n):
    """The rank-order sum from +0.0 over N(i) is one float64 add rounded once to fp32 per term, and the division the
    float64 quotient rounded once; the result is within m roundings of the exact mean."""
    rng = np.random.default_rng(n)
    hs = [(rng.standard_normal(4096) * 0.1).astype(np.float32) for _ in range(n)]
    for i in range(n):
        nb = A.ring_neighbours(i, n)
        assert nb == sorted({(i - 1) % n, i, (i + 1) % n}) and len(nb) == min(n, 3)
        s = np.zeros(4096, np.float32)
        for q in nb:
            s = (s.astype(np.float64) + hs[q].astype(np.float64)).astype(np.float32)
        want = (s.astype(np.float64) / len(nb)).astype(np.float32)
        got = A.gossip_mix(hs, i)
        assert A.bits(got).tolist() == A.bits(want).tolist()
        exact = sum(hs[q].astype(np.float64) for q in nb) / len(nb)
        top = sum(np.abs(hs[q]).astype(np.float64) for q in nb)
        assert np.all(np.abs(got - exact) <= len(nb) * np.spacing(top.astype(np.float32)).astype(np.float64))


@pytest.mark.parametrize("n", [1, 2, 3])
def test_mix_is_the_local_average_up_to_three_replicas(n):
    rng = np.random.default_rng(10 + n)
    hs = [(rng.standard_normal(4096) * (q + 1)).astype(np.float32) for q in range(n)]
    for i in range(n):
        assert A.bits(A.gossip_mix(hs, i)).tolist() == A.bits(A.local_average(hs)).tolist()


def test_mix_is_sparse_from_four_replicas():
    hs = [np.full(4, float(q), np.float32) for q in range(8)]
    assert A.gossip_mix(hs, 0).tolist() == [np.float32(8.0) / np.float32(3.0)] * 4
    assert A.gossip_mix(hs, 4).tolist() == [4.0] * 4


# ---- the protocol model ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [3, 4])
def test_model_explored_over_three_iterations(n):
    """G1-G3 in every reachable state of three iterations of every replica (the devices alone, every step launched)."""
    assert explore_schedules(lambda: GossipModel(n, 2, hosts=False), dedup=True) > 1


@pytest.mark.parametrize("n", [3, 4, 6, 8])
def test_model_with_the_stop_rule(n):
    """G1-G4 with the host loops and a pass after step 2 that reaches the target, S = 2 + stop_margin, under random
    schedules."""
    f = SimpleNamespace(gossip_method=True)
    assert run_random(lambda: GossipModel(n, 100, every=2, reach=2, margin=stop_margin(f, n)), range(150)) == 150


@pytest.mark.parametrize("kw,n", [
    (dict(parities=1), 3), (dict(parities=1), 4),                 # a single send buffer
    (dict(skip=True), 3), (dict(skip=True), 4),                   # a barrier that skips one neighbour
    (dict(parity_offset=1), 3), (dict(parity_offset=1), 4),       # a mix reading send[(s + 1) % 2]
])
def test_model_mutants_fail(kw, n):
    with pytest.raises(ProtocolHazard, match="G1|G2"):
        explore_schedules(lambda: GossipModel(n, 2, hosts=False, **kw), dedup=True)


@pytest.mark.parametrize("n,every", [(3, 3), (8, 2)])
def test_model_margin_one_below_fails(n, every):
    """One step less than stop_margin: for N <= 5 the chief decides on its final pass before it can know S; for N = 8
    the replica opposite the chief learns S only after it launched step S + 1."""
    f = SimpleNamespace(gossip_method=True)
    with pytest.raises(ProtocolHazard, match="G3|G4"):
        run_random(lambda: GossipModel(n, 100, every=every, reach=every, margin=stop_margin(f, n) - 1), range(150))


# ---- stop margin ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,want", [(1, 2), (2, 2), (3, 2), (4, 2), (5, 2), (6, 3), (7, 3), (8, 4)])
def test_stop_margin(n, want):
    try:
        f = _flags("--gossip_method")
        assert stop_margin(f, n) == want == max(STOP_MARGIN, n // 2)
        es = _EarlyStopping(1, 0.0, 100, "live", stop_margin(f, n))
        es.add(10, 100, 90)
        es.add(20, 100, 50)
        assert es.report()["stop_step"] == 20 + want
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


def test_torch_engine_one_replica_is_plain_sgd(tmp_path, one_replica, caplog):
    plain = _train(str(tmp_path / "plain"), "--lr_warmup_steps=3")
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(str(tmp_path / "gossip"), "--lr_warmup_steps=3", "--gossip_method")
    assert torch.equal(plain["params"].view(torch.int32), res["params"].view(torch.int32))
    assert res["final_step"] == plain["final_step"] == 8 and res["steps"] == plain["steps"]
    rep = res["gossip"]
    assert rep == gossip_report(1, 8, 0, 0, 0) and rep["neighbourhood"] == 1 and rep["wait_total_s"] == 0.0
    with open(str(tmp_path / "gossip" / (GOSSIP_JSON % 0))) as f:
        assert json.load(f) == rep
    line = [m.getMessage() for m in caplog.records if m.getMessage().startswith("Gossip SGD: ")]
    assert line == ["Gossip SGD: worker 0 mixed with 1 replica(s) of a ring of 1; 8 iteration(s), 0 of whose barriers "
                    "waited for a neighbour, 0.000000 s in them (mean 0.000000 s, max 0.000000 s); final global step 8"]


def test_torch_engine_eval_and_target(tmp_path, one_replica):
    """The run ends as --max_steps = g + stop_margin would end it, and the final pass scores the closing average."""
    res = _train(str(tmp_path / "gossip"), "--gossip_method", "--eval_every_steps=4", "--target_accuracy=0.01", steps=40)
    tta = res["time_to_accuracy"]
    assert tta["reached"] and tta["global_step"] == 4
    assert res["final_step"] == 4 + 2 + 1
    assert [r[0] for r in res["evals"]] == [4, 7]


# ---- gloo replicas --------------------------------------------------------------------------------------------------
COMMON = ["--model=mlp2", "--mlp_hidden=32", "--batch_size=16", "--backend=gloo", "--initial_learning_rate=0.05",
          "--save_interval_secs=1000", "--dropout_keep_prob=1.0"]


def _run(tmp_path, extra, n, timeout=240):
    out = str(tmp_path / "out")
    argv = [WORKER, str(tmp_path / "res_RANK.npz")] + COMMON + ["--train_dir=%s" % (tmp_path / "train_dir")] + extra
    codes = run_replicas(["-c", "import os,sys,runpy; sys.argv=[a.replace('RANK', os.environ['RANK']) for a in sys.argv[1:]];"
                          " runpy.run_path(sys.argv[0], run_name='__main__')"] + argv, n, timeout=timeout, out_dir=out)
    logs = [open(os.path.join(out, f)).read() for f in sorted(os.listdir(out))]
    assert codes == [0] * n, "\n".join(l[-2000:] for l in logs)
    return [dict(np.load(str(tmp_path / ("res_%d.npz" % r)))) for r in range(n)], logs


def test_gloo_four_replicas_against_the_emulation(tmp_path):
    n = 4
    res, logs = _run(tmp_path, ["--max_steps=9", "--gossip_method"], n)
    steps = res[0]["steps"].tolist()
    assert steps == list(range(1, 11)) and all(r["steps"].tolist() == steps for r in res)
    for t in range(len(steps)):
        hs = [r["half"][t] for r in res]
        for q in range(n):
            assert A.bits(res[q]["after"][t]).tolist() == A.bits(A.gossip_mix(hs, q)).tolist(), (t, q)
        assert len({A.bits(r["after"][t]).tobytes() for r in res}) == n          # the replicas differ
    want = A.local_average([r["after"][-1] for r in res])                        # the closing average
    assert all(A.bits(r["final"]).tolist() == A.bits(want).tolist() for r in res)
    assert all(int(r["final_step"]) == 10 for r in res)
    for r, (x, log) in enumerate(zip(res, logs)):
        rep = json.loads(str(x["report"]))
        assert rep["replicas"] == 4 and rep["neighbourhood"] == 3 and rep["iterations"] == 10
        assert "Gossip SGD: worker %d mixed with 3 replica(s) of a ring of 4; 10 iteration(s)" % r in log
        with open(str(tmp_path / "train_dir" / (GOSSIP_JSON % r))) as f:
            assert json.load(f) == rep


def test_gloo_three_replicas_against_local_sgd(tmp_path):
    """With three replicas every neighbourhood is the whole ring: every replica's mix is the rank-order local average of
    every half step, bit for bit, and the replicas agree.  The torch engine's --local_sgd_steps=1 averages with gloo's
    all_reduce, which associates the three-term sum in its own order, so against it the runs agree to rounding; the
    device kernels, which both sum in rank order, are compared bit for bit in tests/test_gossip_gpu.py."""
    g, _ = _run(tmp_path / "gossip", ["--max_steps=9", "--gossip_method"], 3)
    loc, _ = _run(tmp_path / "local", ["--max_steps=9", "--local_sgd_steps=1"], 3)
    for t in range(10):
        want = A.local_average([a["half"][t] for a in g])
        assert all(A.bits(a["after"][t]).tolist() == A.bits(want).tolist() for a in g), t
    for a, b in zip(g, loc):
        assert a["steps"].tolist() == b["steps"].tolist() == list(range(1, 11))
        diff = np.abs(a["final"].astype(np.float64) - b["final"].astype(np.float64))
        scale = np.maximum(np.abs(b["final"]).astype(np.float64), 1e-3)
        assert float((diff / scale).max()) < 1e-4


# ---- configurations -------------------------------------------------------------------------------------------------
def test_generated_cfgs():
    def cfg(name):
        with open(os.path.join(ROOT, "cfg", "8_gpus", name)) as f:
            return eval(f.read(), {"Cfg": dict})
    for name, flags in (("8_gpus_gossip", " --gossip_method=true"),
                        ("8_gpus_gossip_lognormal", " --gossip_method=true --inject_straggler=*:lognormal:100:1.0")):
        c = cfg(name)
        assert c["name"] == name and c["num_replicas_to_aggregate"] == "8" and c["n_gpus"] == 8
        assert c["extra_flags"] == "--save_interval_secs=0.05 --log_every=500" + flags
