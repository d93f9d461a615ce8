"""``--early_stopping_patience`` on the GPU: eval_patience (csrc/eval_patience.cu) word for word against the host rule on
hand-written pass records, with the stop word after every pass; lenet runs through ``train()`` that stop at
S = g + STOP_MARGIN and end exactly as a run with ``--max_steps=S`` (pipelined and non-pipelined loop, with the best
weights kept); the moving average; snapshot passes (a dropped pass changes nothing; K > N and interval end at
min(max_steps, S)); the node order of the pass; the synchronise count per step; and two replicas stopping together."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_OF_N, INTERVAL = 0, 1
VAL = 1000


@pytest.fixture
def flags(monkeypatch):
    from distributedmnist_b200.flags import FLAGS
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    FLAGS.reset()
    yield FLAGS
    FLAGS.reset()


def _train(d, *extra, steps=150):
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import train
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % d, "--batch_size=128", "--max_steps=%d" % steps, "--eval_every_steps=5",
                 "--initial_learning_rate=0.05", "--log_every=1000", "--save_results_period=1000000",
                 "--save_interval_secs=1000"] + list(extra))
    ctx = init_context(FLAGS)
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True, synthetic_sizes=(8192, VAL))
    return train(ctx, ds.train, ds.validation, FLAGS)


def _rows(d):
    return np.load(os.path.join(str(d), "worker0_eval.npy"))


def _ckpt(d, step):
    with open(os.path.join(str(d), "model.ckpt-%d.data-00000-of-00001" % step), "rb") as f:
        return f.read()


def _replay(rows, patience, delta_rows, n):
    """early_stopping.advance over a run's rows (every row a counting pass): the exhausting step or None, final state."""
    from distributedmnist_b200 import early_stopping as es
    state, trig = es.State(), None
    for r in rows:
        state, fired = es.advance(state, int(r[0]), int(r[4]), int(r[3]), n, patience, delta_rows)
        if fired:
            trig = int(r[0])
    return trig, state


def _pick(rows, n, max_step):
    """(patience, min_delta, delta rows, g): the first setting whose patience runs out, by host emulation of a reference
    run's rows, at a step g with g + STOP_MARGIN < max_step."""
    from distributedmnist_b200 import early_stopping as es
    from distributedmnist_b200.train import STOP_MARGIN
    for patience in (3, 2, 4, 1):
        for d in (0.01, 0.005, 0.0):
            m = es.min_delta_rows(d, n)
            g, _s = _replay(rows, patience, m, n)
            if g is not None and g + STOP_MARGIN < max_step:
                return patience, d, m, g
    pytest.fail("no patience runs out inside the run: %s" % rows[:, [0, 4]].tolist())


# ---- the kernel on hand-written records --------------------------------------------------------------------------------
def test_kernel_matches_the_host_rule_word_for_word():
    """Passes of hand-written EvalState records through dm_eval_patience, with two stop words standing for two replicas:
    after every pass the PatienceState words equal early_stopping.advance, and the stop words hold S = g + margin from the
    exhausting pass on -- unless a target had set them first, which is never overwritten."""
    from distributedmnist_b200 import early_stopping as es
    from distributedmnist_b200.ops.lib import load, stream_ptr
    lib = load()
    n, margin = 1000, 2
    # (step, correct, examples, status); status None: a live pass
    seq = [(1, 500, 999, None), (2, 400, 1000, -1), (3, 410, 1000, 0), (4, 420, 1000, None), (5, 420, 1000, None),
           (6, 423, 1000, None), (7, 424, 1000, None), (8, 700, 1000, -1), (9, 600, 900, None), (10, 422, 1000, 2),
           (11, 999, 1000, None), (12, 1, 1000, 1)]
    for patience, delta, preset in ((3, 4, 0), (3, 3, 0), (1, 0, 0), (2, 3, 9), (50, 0, 0)):
        ev = torch.zeros(int(lib.dm_eval_state_bytes()), dtype=torch.uint8, device="cuda")
        ps = torch.zeros(int(lib.dm_patience_state_bytes()) // 4, dtype=torch.int32, device="cuda")
        stop = torch.full((2, 64), 0, dtype=torch.int32, device="cuda")          # two words on separate 256-byte lines
        stop[:, 0] = preset
        table = (ctypes.c_void_p * 2)(stop[0].data_ptr(), stop[1].data_ptr())
        step_t = torch.zeros(1, dtype=torch.int32, device="cuda")
        status_t = torch.zeros(1, dtype=torch.int32, device="cuda")
        state, want_stop = es.State(), preset
        for step, correct, examples, status in seq:
            ev[16:24].view(torch.int32).copy_(torch.tensor([correct, examples], dtype=torch.int32))
            step_t.fill_(step)
            if status is not None:
                status_t.fill_(status)
            lib.dm_eval_patience(ev, step_t, None if status is None else status_t, n, patience, delta, margin, ps,
                                 table, 0, 2, stream_ptr())
            torch.cuda.synchronize()
            state, fired = es.advance(state, step, correct, examples, n, patience, delta, status)
            if fired and want_stop == 0:
                want_stop = step + margin
            u = ps.cpu().numpy().view(np.uint32)
            got = es.State(int(u[es.PAT_BEST_WORD]), int(u[es.PAT_SINCE_WORD]), int(u[es.PAT_BEST_STEP_WORD]),
                           int(u[es.PAT_TRIGGER_WORD]), bool(u[es.PAT_BASELINE_WORD]))
            assert got == state, (patience, delta, step)
            assert stop[:, 0].tolist() == [want_stop] * 2, (patience, delta, step)
            assert int(stop[:, 1:].abs().sum()) == 0
        if patience == 3 and delta == 4:
            assert state.trigger_step == 7 and want_stop == 9          # 4 sets the baseline, 5 6 7 do not beat 424
        if patience == 3 and delta == 3:
            assert state.best_step == 11 and want_stop == 0            # 7 beats 423 and resets, as 11 does later
        if preset:
            assert es.exhausted(state, patience) and want_stop == preset


# ---- lenet through train() --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pipelined", [True, False], ids=["pipelined", "non_pipelined"])
def test_lenet_stops_at_g_plus_margin_like_max_steps(tmp_path, flags, pipelined):
    from distributedmnist_b200.train import STOP_MARGIN
    # --device_data: the index feed draws batches on the training thread, so every run trains on the same batch sequence
    loop = ["--pipeline_steps=%s" % ("true" if pipelined else "false"), "--device_data=true"]
    _train(tmp_path / "ref", *loop)
    patience, d, m, g = _pick(_rows(tmp_path / "ref"), VAL, 150)
    s = g + STOP_MARGIN
    res = _train(tmp_path / "armed", *loop, "--early_stopping_patience=%d" % patience,
                 "--early_stopping_min_delta=%r" % d, "--keep_best_checkpoint")
    cut = _train(tmp_path / "cut", *loop, steps=s)
    rep = res["early_stopping"]
    assert rep["triggered"] and rep["trigger_step"] == g and rep["stop_step"] == s, rep
    assert res["final_step"] == cut["final_step"] == s + 1
    assert _ckpt(tmp_path / "armed", s + 1) == _ckpt(tmp_path / "cut", s + 1)
    a, c = _rows(tmp_path / "armed"), _rows(tmp_path / "cut")
    np.testing.assert_array_equal(a[:, [0, 3, 4, 5]], c[:, [0, 3, 4, 5]])
    with open(str(tmp_path / "armed" / "worker0_early_stopping.json")) as f:
        assert json.load(f) == rep
    trig, state = _replay(a, patience, m, VAL)
    assert trig == g and res["engine"].patience_state() == state
    assert (rep["best_step"], rep["best_correct"], rep["min_delta_rows"], rep["weights"]) == \
        (state.best_step, state.best, m, "live")
    # the best file holds the best-scoring pass of the run, not its last weights
    best = int(a[:, 4].max())
    best_step = int(a[a[:, 4] == best][0, 0])
    assert res["best"]["global_step"] == best_step and res["best"]["correct"] == best
    assert os.path.exists(str(tmp_path / "armed" / "best" / ("model.ckpt-%d.index" % best_step)))
    print("\n%s: patience %d, min_delta %d rows: exhausted at step %d (best %d/%d at step %d), S = %d"
          % ("pipelined" if pipelined else "non-pipelined", patience, m, g, state.best, VAL, state.best_step, s))


def test_moving_average_report_names_its_weights(tmp_path, flags):
    """min_delta 0.999: no pass beats the baseline, so the third counting pass (step 15) exhausts a patience of 2."""
    from distributedmnist_b200.train import STOP_MARGIN
    res = _train(tmp_path / "avg", "--device_data=true", "--moving_average_decay=0.9", "--eval_moving_average",
                 "--early_stopping_patience=2", "--early_stopping_min_delta=0.999", steps=100)
    rep = res["early_stopping"]
    assert rep["weights"] == "moving_average" and rep["min_delta_rows"] == 999
    assert rep["triggered"] and rep["trigger_step"] == 15 and rep["best_step"] == 5 and rep["counted_passes"] == 3
    assert res["final_step"] == 15 + STOP_MARGIN + 1
    assert res["engine"].patience_state().trigger_step == 15


def _emulate(eng, g, mode, phases=7):
    from distributedmnist_b200.ops.lib import stream_ptr
    eng.lib.dm_snap_test_emulate(eng.backend.ctrl.local_ptr, eng.params, eng.params.numel(), g, mode, 1, phases, stream_ptr())


def _stop_word(eng):
    torch.cuda.synchronize()
    return int(eng._stop.view(torch.int32, 0, 1).cpu()[0])


@pytest.mark.parametrize("mode", [K_OF_N, INTERVAL], ids=["k_of_n", "interval"])
def test_dropped_snapshot_pass_neither_resets_nor_advances(mode):
    """An emulated peer on one stream.  Patience 1 and min_delta n - 1 rows: after the baseline, the next counting pass
    exhausts the patience.  A dropped pass before the baseline and one after it change nothing."""
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.ops.selfcheck import mnist_like
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200 import early_stopping as es
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaLeNetEngine(256, be, seed=5, use_graph=True)
    eng._interval = mode == INTERVAL
    n = 2500
    g = torch.Generator().manual_seed(6)
    eng.arm_eval(mnist_like(g, n), torch.randint(0, 10, (n,), generator=g), snapshot=True)
    eng.arm_stop()
    eng.arm_patience(1, n - 1, 2)

    def one_pass():
        eng.enqueue_eval()
        torch.cuda.synchronize()
        (rec, status), = eng.eval_records_with_status()
        return rec, status

    _emulate(eng, 1, mode, phases=1 | 2)                 # committed and pushed, done never released: every attempt fails
    assert one_pass()[1] == -1
    assert eng.patience_state() == es.State() and _stop_word(eng) == 0
    _emulate(eng, 1, mode, phases=4)                     # the next pass scores the snapshot of step 1: the baseline
    rec1, st1 = one_pass()
    assert st1 > 0 and rec1[0] == 1
    base = es.State(rec1[4], 0, 1, 0, True)
    assert eng.patience_state() == base and _stop_word(eng) == 0
    _emulate(eng, 2, mode, phases=1 | 2)                 # dropped again: the count stays at 0, no stop
    assert one_pass()[1] == -1
    assert eng.patience_state() == base and _stop_word(eng) == 0
    _emulate(eng, 2, mode, phases=4)                     # an accepted pass of step 2 exhausts the patience
    rec2, st2 = one_pass()
    assert st2 > 0 and rec2[0] == 2
    assert eng.patience_state() == base._replace(since=1, trigger_step=2) and _stop_word(eng) == 2 + 2


@pytest.mark.parametrize("extra", [["--num_replicas_to_aggregate=4"], ["--interval_method=true", "--interval_ms=2"]],
                         ids=["k4_of_1", "interval"])
def test_snapshot_runs_end_at_min_max_steps_and_s(tmp_path, flags, extra):
    """min_delta 0.999 and patience 2: the third accepted pass exhausts the patience, whichever steps timing makes the
    snapshot passes score."""
    from distributedmnist_b200.train import STOP_MARGIN
    res = _train(tmp_path / "run", "--eval_snapshot=true", "--pipeline_steps=true", "--early_stopping_patience=2",
                 "--early_stopping_min_delta=0.999", *extra, steps=200)
    rep = res["early_stopping"]
    rows = _rows(tmp_path / "run")
    assert rep["triggered"] and rep["weights"] == "snapshot", (rep, rows[:, [0, 4]].tolist())
    assert (rep["best_step"], rep["trigger_step"]) == (int(rows[0, 0]), int(rows[2, 0]))
    assert res["engine"].patience_state().trigger_step == rep["trigger_step"]
    s = min(200, rep["trigger_step"] + STOP_MARGIN)
    assert max(res["steps"]) <= s < res["final_step"], (res["steps"][-5:], res["final_step"], s)
    print("\n%s: exhausted at snapshot step %d, S = %d, final step %d, %d pass(es) dropped"
          % (extra[0], rep["trigger_step"], s, res["final_step"], res["engine"].eval_dropped))


# ---- the pass graph and the step loop ---------------------------------------------------------------------------------
class _Recorder:
    """Stands in for the kernel library: records which entry points a launch sequence calls, in order."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)

        def call(*a):
            self.calls.append(name)
            return fn(*a)
        return call


def test_patience_is_the_last_node_of_the_pass_and_absent_when_off():
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.ops.selfcheck import mnist_like
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaLeNetEngine(256, be, seed=5, use_graph=True)
    g = torch.Generator().manual_seed(6)
    eng.arm_eval(mnist_like(g, 3000), torch.randint(0, 10, (3000,), generator=g))

    def pass_calls():
        rec, lib = _Recorder(eng.lib), eng.lib
        eng.lib = rec
        try:
            eng._launch_eval(publish=True)
        finally:
            eng.lib = lib
        torch.cuda.synchronize()
        return rec.calls

    off = pass_calls()
    assert not any("patience" in c or "target" in c or "best" in c for c in off)
    eng.arm_stop()
    eng.arm_best()
    eng.arm_target(3000, 2)
    eng.arm_patience(2, 0, 2)
    on = pass_calls()
    assert on[:len(off)] == off
    assert on[len(off):] == ["dm_eval_best_decide", "dm_eval_best_copy", "dm_eval_target", "dm_eval_patience"]


def test_armed_run_adds_no_synchronisation_per_step(tmp_path, flags, monkeypatch):
    """An armed run whose patience never runs out makes as many synchronise calls per step as an unarmed one: the
    difference between a 100-step and a 200-step run is the same with and without the patience.  Its step graph gains
    only stop_publish; with the flag off nothing is armed."""
    from distributedmnist_b200.train import _AsyncCheckpointer
    calls = {"sync": 0, "at_final_save": None}

    def counted(fn):
        def wrapper(*a, **k):
            calls["sync"] += 1
            return fn(*a, **k)
        return wrapper
    monkeypatch.setattr(torch.cuda, "synchronize", counted(torch.cuda.synchronize))
    monkeypatch.setattr(torch.cuda.Stream, "synchronize", counted(torch.cuda.Stream.synchronize))
    monkeypatch.setattr(torch.cuda.Event, "synchronize", counted(torch.cuda.Event.synchronize))
    real_save = _AsyncCheckpointer.save

    def save(self, *a, **k):
        calls["at_final_save"] = calls["sync"]
        return real_save(self, *a, **k)
    monkeypatch.setattr(_AsyncCheckpointer, "save", save)
    counts, launches = {}, {}
    for tag, extra in (("armed", ["--early_stopping_patience=1000"]), ("off", [])):
        for steps in (100, 200):
            calls.update(sync=0, at_final_save=None)
            res = _train(tmp_path / ("%s_%d" % (tag, steps)), *extra, steps=steps)
            assert res["final_step"] == steps + 1
            counts[(tag, steps)] = calls["at_final_save"]
            launches[tag] = res["engine"].launches_per_step
            if tag == "off":
                assert res["engine"]._patience is None and res["engine"]._stop is None
                assert "early_stopping" not in res
            else:
                assert res["early_stopping"]["triggered"] is False
    per_armed = counts[("armed", 200)] - counts[("armed", 100)]
    per_off = counts[("off", 200)] - counts[("off", 100)]
    assert per_armed == per_off, counts
    assert launches["armed"] == launches["off"] + 1, launches


# ---- two replicas ------------------------------------------------------------------------------------------------------
def _replica_runs(tmp_path, name, extra, steps, n=2):
    from distributedmnist_b200.parallel.launcher import run_replicas
    worker = os.path.join(ROOT, "tests", "_snapshot_eval_worker.py")
    d = tmp_path / name
    codes = run_replicas([worker, str(d / "rank_RANK"), "--train_dir=%s" % (d / "train_dir"), "--batch_size=128",
                          "--max_steps=%d" % steps, "--initial_learning_rate=0.05", "--save_interval_secs=1000",
                          "--log_every=50", "--eval_every_steps=10"] + extra, n, timeout=600, out_dir=str(d / "out"))
    logs = "\n".join(open(os.path.join(d, "out", f)).read()[-1500:] for f in sorted(os.listdir(d / "out")))
    assert codes == [0] * n, (name, logs)
    ranks = []
    for r in range(n):
        with open(str(d / ("rank_%d.json" % r))) as f:
            ranks.append((np.load(str(d / ("rank_%d.npy" % r))), json.load(f)))
    return ranks, d / "train_dir"


@pytest.mark.multigpu
def test_two_replicas_k_equals_n_stop_at_the_same_step(tmp_path):
    from distributedmnist_b200.train import STOP_MARGIN
    _ranks, ref_dir = _replica_runs(tmp_path, "ref", [], 300)
    rows = _rows(ref_dir)
    patience, d, _m, g = _pick(rows, int(rows[0, 3]), 300)
    ranks, train_dir = _replica_runs(tmp_path, "armed", ["--early_stopping_patience=%d" % patience,
                                                         "--early_stopping_min_delta=%r" % d], 300)
    with open(str(train_dir / "worker0_early_stopping.json")) as f:
        rep = json.load(f)
    assert rep["trigger_step"] == g
    assert [m["final_step"] for _p, m in ranks] == [g + STOP_MARGIN + 1] * 2
    assert np.array_equal(ranks[0][0].view(np.uint32), ranks[1][0].view(np.uint32))
