"""Straggler delays drawn per replica from a distribution or a measured profile (``--inject_straggler``): the spec grammar
and its refusals, the quantile tables, the host emulation of the device sampler (distribution, independence across
replicas), the profile tool, and a 2-process gloo run whose ranks sleep exactly what the emulation draws."""
import json
import os
import random
import sys
import types

import numpy as np
import pytest
from scipy import stats

from distributedmnist_b200.parallel import straggler as S
from distributedmnist_b200.parallel.aggregators import StragglerSpec, _AggregatorBase, parse_straggler_spec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tests")


def _opt(rank, straggler, seed):
    backend = types.SimpleNamespace(ctx=types.SimpleNamespace(rank=rank))
    return _AggregatorBase(backend, lambda step: 0.1, 4, straggler, seed)


# ---- the rank:prob:usec form is unchanged ----------------------------------------------------------------------------------
def test_fixed_form_parses_as_before():
    assert parse_straggler_spec("3:0.5:2000,5:1:500") == {3: StragglerSpec(0.5, 2000.0), 5: StragglerSpec(1.0, 500.0)}
    assert parse_straggler_spec("7:0.2:300,6:0.2:300") == {7: StragglerSpec(0.2, 300.0), 6: StragglerSpec(0.2, 300.0)}
    assert parse_straggler_spec("") == {}
    s = parse_straggler_spec("1:0.3:700")[1]
    assert not s.sampled and s.dist == "fixed" and s.table is None
    assert parse_straggler_spec("1:0.3:700").get(0) is None


def test_fixed_form_draws_the_same_sequence():
    opt = _opt(1, parse_straggler_spec("1:0.3:500"), seed=5)
    rng = random.Random(5 * 7919 + 1)
    want = [500e-6 if rng.random() < 0.3 else 0.0 for _ in range(500)]
    assert [opt._delay_s() for _ in range(500)] == want
    assert opt.straggler_delays_ns == []
    assert _opt(0, parse_straggler_spec("1:0.3:500"), seed=5)._delay_s() == 0.0


# ---- new forms -------------------------------------------------------------------------------------------------------------
def test_sampled_forms_parse(tmp_path):
    m = parse_straggler_spec("2:exp:50, 3:lognormal:100:1.0")
    assert m[2].dist == "exp" and m[2].params == (50.0,) and m[2].sampled
    assert m[3].dist == "lognormal" and m[3].params == (100.0, 1.0)
    w = parse_straggler_spec("*:exp:50")
    assert set(w) == {"*"} and w.get(0) is w.get(7) is w["*"]
    d = tmp_path / "a:b"                                 # a path may contain ':'
    d.mkdir()
    np.save(str(d / "p.npy"), np.array([1.0, 2.0, 3.0]))
    p = parse_straggler_spec("1:profile:%s" % (d / "p.npy"))[1]
    assert p.dist == "profile" and p.params == (str(d / "p.npy"),)
    for s in (m[2], m[3], p):
        assert s.table.shape == (1025,) and s.table.dtype == np.uint32


@pytest.mark.parametrize("text,why", [
    ("0:gamma:5", "unknown distribution"),
    ("0:exp:abc", "not a number"),
    ("0:exp:5:6", "wants rank:exp:MEAN_US"),
    ("0:lognormal:100", "wants rank:lognormal:MEDIAN_US:SIGMA"),
    ("0:exp:-5", "positive"),
    ("0:exp:nan", "positive"),
    ("0:lognormal:100:-1", "positive"),
    ("0:lognormal:-100:1", "positive"),
    ("x:exp:5", "rank must be an integer or *"),
    ("0:profile:/nonexistent/delays.npy", "no such file"),
    ("1:exp:5,1:0.5:10", "given twice"),
    ("*:exp:5,2:exp:3", "given twice"),
    ("2:exp:3,*:exp:5", "given twice"),
    ("3:0.5:100,3:0.2:100", "given twice"),
    ("0:exp:1000000", "exceeds the limit"),             # mean 1 s: the table reaches ~7.6 s > 4 s
    ("0:1:2:3", "wants rank:prob:usec"),
])
def test_refusals_name_their_reason(text, why):
    with pytest.raises(ValueError, match=why):
        parse_straggler_spec(text)


def test_table_limit_follows_the_watchdog(tmp_path):
    parse_straggler_spec("0:exp:2000", 30000)                  # ~15 ms max: fine
    with pytest.raises(ValueError, match="exceeds the limit of 25000 us"):
        parse_straggler_spec("0:exp:5000", 100)                # ~38 ms max > 100 ms / 4
    bad = tmp_path / "p.txt"
    bad.write_text("1 2 -3\n")
    with pytest.raises(ValueError, match="non-negative"):
        parse_straggler_spec("0:profile:%s" % bad)
    empty = tmp_path / "e.npy"
    np.save(str(empty), np.zeros(0))
    with pytest.raises(ValueError, match="non-empty"):
        parse_straggler_spec("0:profile:%s" % empty)


@pytest.mark.parametrize("text,law", [("0:exp:50", stats.expon(scale=50.0)),
                                      ("0:lognormal:100:1.0", stats.lognorm(s=1.0, scale=100.0))])
def test_tables_are_monotone_quantiles(text, law):
    t = parse_straggler_spec(text)[0].table
    assert t.shape == (1025,) and (np.diff(t.astype(np.int64)) >= 0).all()
    assert np.abs(t.astype(np.float64) - law.ppf(S.table_probs()) * 1e3).max() <= 1.0


def test_profile_table_is_numpy_quantile(tmp_path):
    prof = np.random.default_rng(3).gamma(2.0, 40.0, size=5000)
    path = tmp_path / "prof.txt"
    np.savetxt(str(path), prof)
    t = parse_straggler_spec("0:profile:%s" % path)[0].table
    want = np.rint(np.quantile(np.loadtxt(str(path)), S.table_probs()) * 1e3)
    assert np.array_equal(t, want.astype(np.uint32))


# ---- host emulation --------------------------------------------------------------------------------------------------------
def test_sampler_integer_arithmetic():
    t = np.arange(1025, dtype=np.uint32) * 1024          # linear table: segment * 1024 + position * 1024 / 65536
    j = np.arange(1000)
    u = S.hash_mix(7, j).astype(np.int64)
    assert np.array_equal(S.sample_ns(t, 7, j), ((u >> 22) * 1024 + (((u >> 6) & 0xFFFF) >> 6)).astype(np.uint32))
    # the murmur finaliser of dropout_keep (models/lenet.py), full 32 bits
    from distributedmnist_b200.models.lenet import dropout_keep_mask
    keep = dropout_keep_mask(7, 1, 1000, 0.5).view(-1).numpy()
    assert np.array_equal(keep, (u >> 8) < (1 << 23))


@pytest.mark.parametrize("text,law", [("0:exp:2000", stats.expon(scale=2000.0)),
                                      ("0:lognormal:100:1.0", stats.lognorm(s=1.0, scale=100.0))])
def test_host_draws_follow_the_distribution(text, law):
    n = 200_000
    t = parse_straggler_spec(text)[0].table
    x = S.sample_ns(t, S.seed_mix(66478, 0), np.arange(n)).astype(np.float64) / 1e3
    ks = stats.kstest(x, law.cdf).statistic
    crit = np.sqrt(-np.log(1e-3 / 2) / 2) / np.sqrt(n)    # alpha = 1e-3
    assert ks <= 1.0 / 1025 + crit, (ks, crit)


def test_replica_streams_are_independent():
    n = 200_000
    t = parse_straggler_spec("*:exp:100")["*"].table
    a = S.sample_ns(t, S.seed_mix(66478, 6), np.arange(n)).astype(np.float64)
    b = S.sample_ns(t, S.seed_mix(66478, 7), np.arange(n)).astype(np.float64)
    assert not np.array_equal(a, b)
    assert abs(np.corrcoef(a, b)[0, 1]) < 0.02
    both = np.mean((a > np.quantile(a, 0.9)) & (b > np.quantile(b, 0.9)))
    assert 0.009 <= both <= 0.011, both                   # independent: 0.1 * 0.1


def test_aggregator_delay_is_the_emulation_per_replica():
    m = parse_straggler_spec("*:lognormal:100:1.0")
    for rank in (0, 1):
        opt = _opt(rank, m, seed=17)
        got = [opt._delay_s() for _ in range(300)]
        want = S.sample_ns(m["*"].table, S.seed_mix(17, rank), np.arange(300))
        assert got == [int(v) * 1e-9 for v in want]
        assert opt.straggler_delays_ns == [int(v) for v in want]
        assert opt._straggler.seed_mix == S.seed_mix(17, rank) and m["*"].seed_mix == 0


# ---- profile tool ----------------------------------------------------------------------------------------------------------
def test_profile_tool_round_trip(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import straggler_profile as SP
    times = {1: [100e-6, 110e-6, 130e-6, 400e-6], 2: [105e-6, 120e-6, 90e-6, 1000e-6]}
    entries = [(t, w, i) for w, ts in times.items() for i, t in enumerate(ts)] + [(5e-3, 0, 0)]   # the chief is left out
    log = tmp_path / "run_out_master"
    log.write_text("some line\nELAPSED TIMES %r\n" % entries)
    prof = SP.profile_from_logs([str(log)])
    raw = np.array([t for t, w, _i in entries if w != 0]) * 1e6
    want = np.maximum(raw - np.median(raw), 0.0)
    assert np.allclose(prof, want) and np.median(raw) == pytest.approx(115.0)
    assert np.allclose(np.quantile(prof, [0.5, 1.0]), np.quantile(want, [0.5, 1.0]))
    assert np.allclose(SP.profile_from_logs([str(log)], absolute=True), raw)
    assert len(SP.profile_from_logs([str(log)], with_master=True)) == len(entries)
    out = tmp_path / "x:y" / "prof.npy"
    out.parent.mkdir()
    assert SP.main([str(out), str(log)]) == 0
    t = parse_straggler_spec("0:profile:%s" % out)[0].table
    assert np.array_equal(t, np.rint(np.quantile(np.load(str(out)), S.table_probs()) * 1e3).astype(np.uint32))
    assert t[0] == 0 and t[-1] <= int(round(want.max() * 1e3))


# ---- gloo: 2 processes, K = 1 of 2 -----------------------------------------------------------------------------------------
def test_gloo_ranks_sleep_the_emulated_delays(tmp_path):
    from distributedmnist_b200.parallel.launcher import run_replicas
    out = str(tmp_path / "out")
    argv = [os.path.join(HERE, "_straggler_gloo_worker.py"), str(tmp_path / "res_RANK.json"), "--model=mlp2",
            "--mlp_hidden=32", "--batch_size=16", "--backend=gloo", "--initial_learning_rate=0.05",
            "--save_interval_secs=1000", "--train_dir=%s" % (tmp_path / "train_dir"), "--max_steps=20", "--seed=7",
            "--num_replicas_to_aggregate=1", "--inject_straggler=*:exp:2000"]
    codes = run_replicas(argv, 2, timeout=180, out_dir=out)
    logs = [open(os.path.join(out, f)).read() for f in sorted(os.listdir(out))]
    assert codes == [0, 0], "\n".join(l[-2000:] for l in logs)
    res = [json.load(open(tmp_path / ("res_%d.json" % r))) for r in range(2)]
    table = parse_straggler_spec("*:exp:2000")["*"].table
    for r, got in enumerate(res):
        assert got["final_fp"] == res[0]["final_fp"]
        n = len(got["slept"])
        assert n >= 20
        want = S.sample_ns(table, S.seed_mix(7, r), np.arange(n))
        assert got["slept"] == [int(v) * 1e-9 for v in want], r
        assert got["recorded_ns"] == [int(v) for v in want]
    assert res[0]["slept"][:20] != res[1]["slept"][:20]
