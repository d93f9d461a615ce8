"""``--lr_plateau_patience`` on the GPU: eval_plateau (csrc/eval_plateau.cu) word for word against lr_plateau.advance on
hand-written pass records, with two replicas' cut tables after every pass; the aggregation kernels' step size with a cut
table, bit for bit against the host schedule and the exact emulation of ops/aggrefs.py on every K = N path; lenet runs
through ``train()`` whose device table equals the host replay and the file; and two replicas staying bit-identical
through several cuts."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from distributedmnist_b200 import lr_plateau as lp
from distributedmnist_b200.ops import aggrefs as A
from distributedmnist_b200.schedule import LearningRateSchedule

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VAL = 1000
ARMED = ("--lr_plateau_patience=1", "--lr_plateau_min_delta=0.5")


@pytest.fixture
def flags(monkeypatch):
    from distributedmnist_b200.flags import FLAGS
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)
    FLAGS.reset()
    yield FLAGS
    FLAGS.reset()


def _backend():
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    return FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))


def _table(cuts):
    words = np.full(lp.MAX_CUTS, lp.NO_CUT, dtype=np.uint32)
    words[:len(cuts)] = cuts
    return torch.from_numpy(words.view(np.int32)).cuda()


# ---- eval_plateau on hand-written records ------------------------------------------------------------------------------
def test_kernel_matches_the_host_rule_word_for_word():
    """Passes of hand-written EvalState records through dm_eval_plateau, with two cut tables standing for two replicas:
    after every pass the PlateauState words equal lr_plateau.advance, and both tables hold S = g + margin for exactly
    the cuts made so far, 0xFFFFFFFF elsewhere -- up to the cap, after which triggers store nothing."""
    from distributedmnist_b200.ops.lib import load, stream_ptr
    lib = load()
    n, margin = 1000, 2
    # (step, correct, examples, status); status None: a live pass
    seq = [(1, 500, 999, None), (2, 400, 1000, -1), (3, 410, 1000, 0), (4, 420, 1000, None), (5, 420, 1000, None),
           (6, 423, 1000, None), (7, 424, 1000, None), (8, 700, 1000, -1), (9, 600, 900, None), (10, 422, 1000, 2),
           (11, 999, 1000, None), (12, 1, 1000, 1), (13, 999, 1000, 3), (14, 5, 1000, None)]
    long_run = [(100 + i, 300, 1000, None) for i in range(lp.MAX_CUTS + 4)]
    for patience, delta, restored, passes in ((3, 4, 0, seq), (2, 3, 0, seq), (1, 0, 0, seq), (1, 0, 5, seq),
                                              (2, 0, 30, seq), (1, 0, 0, long_run)):
        ev = torch.zeros(int(lib.dm_eval_state_bytes()), dtype=torch.uint8, device="cuda")
        ps = torch.zeros(int(lib.dm_plateau_state_bytes()) // 4, dtype=torch.int32)
        ps[lp.PL_CUTS_WORD] = restored
        ps = ps.cuda()
        pre = [50 + 2 * k for k in range(restored)]
        tables = torch.stack([_table(pre), _table(pre)])
        ptrs = (ctypes.c_void_p * 2)(tables[0].data_ptr(), tables[1].data_ptr())
        step_t = torch.zeros(1, dtype=torch.int32, device="cuda")
        status_t = torch.zeros(1, dtype=torch.int32, device="cuda")
        state, want = lp.State(cuts=restored), list(pre)
        for step, correct, examples, status in passes:
            ev[16:24].view(torch.int32).copy_(torch.tensor([correct, examples], dtype=torch.int32))
            step_t.fill_(step)
            if status is not None:
                status_t.fill_(status)
            lib.dm_eval_plateau(ev, step_t, None if status is None else status_t, n, patience, delta, margin, ps, ptrs, 2,
                                stream_ptr())
            torch.cuda.synchronize()
            before = state.cuts
            state, fired = lp.advance(state, step, correct, examples, n, patience, delta, status)
            if fired and state.cuts > before:
                want.append(step + margin)
            u = ps.cpu().numpy().view(np.uint32)
            got = lp.State(int(u[lp.PL_BEST_WORD]), int(u[lp.PL_SINCE_WORD]), bool(u[lp.PL_BASELINE_WORD]),
                           int(u[lp.PL_CUTS_WORD]), int(u[lp.PL_TRIGGER_WORD]))
            assert got == state, (patience, delta, restored, step)
            t = tables.cpu().numpy().view(np.uint32)
            exp = np.full(lp.MAX_CUTS, lp.NO_CUT, dtype=np.uint32)
            exp[:len(want)] = want
            assert (t == exp).all(), (patience, delta, restored, step, t[0].tolist())
        if (patience, delta, restored) == (3, 4, 0):
            # 4 sets the baseline, 5 6 7 do not beat 424 by more than 4; after the cut 11 becomes the best and 12 13 14
            # (a dropped pass between them) do not beat it
            assert want == [9, 16]
        if passes is long_run:
            assert len(want) == lp.MAX_CUTS and state.trigger_step == passes[-1][0]


# ---- the aggregation kernels with a cut table --------------------------------------------------------------------------
PROBE = [(0, []), (7, [7]), (7, [8]), (9, [1, 2, 3]), (9, [9, 9]), (40, list(range(1, 33))), (40, list(range(30, 62)))]


@pytest.mark.parametrize("factor", [0.1, 0.5, 0.3])
def test_device_step_size_with_cuts_equals_host_schedule(factor):
    """Solo fused_sync_sgd with weights 0 and gradients 1.0: the new weight is -scale exactly.  With a cut table the scale
    is fp32(LearningRateSchedule(step)) with the table's cuts, bit for bit, for entries below, at and above the step."""
    from distributedmnist_b200.ops.lib import load
    lib = load()
    be = _backend()
    try:
        params, grads = be.allocate(1024), be.allocate(1024)
        grads.fill_(1.0)
        checked = 0
        for base in (0, 1000, 77777):
            for off, cuts in PROBE:
                step = base + off
                cuts = [base + c for c in cuts]
                table = _table(cuts)
                lib.dm_sync_set_lr_cuts(be.ctrl.local_ptr, table, factor)
                sched = LearningRateSchedule(0.05, 1, 0.999, factor=factor, cuts=cuts)
                params.zero_()
                be.set_global_step(step)
                be.enqueue(params, grads, 1, 0.05, 0.999, 1)
                got = -params[0].item()
                host = sched(step)
                if host < A.FLT_MIN:
                    assert got == 0.0, (step, cuts, got, host)
                    continue
                assert A.midpoint_distance_ulps(host) > 16, (step, host)
                assert np.float32(got) == np.float32(host), (factor, step, cuts, got, host)
                checked += 1
        lib.dm_sync_set_lr_cuts(be.ctrl.local_ptr, None, 0.0)
        params.zero_()
        be.set_global_step(5)
        be.enqueue(params, grads, 1, 0.05, 0.999, 1)
        assert np.float32(-params[0].item()) == np.float32(LearningRateSchedule(0.05, 1, 0.999)(5))
        be.check_error()
        assert checked >= 15
    finally:
        be.close()


@pytest.mark.parametrize("bucket", ["2", "1", "0"])
def test_engine_steps_with_cut_table_are_bit_exact(bucket, monkeypatch):
    """Graph-replayed lenet steps at K = N = 1 with a preloaded table (entries below, equal to and above the steps):
    weights and shadow bit for bit against the exact emulation at the schedule with the same cuts.  On one replica
    DMNIST_BUCKET=1 runs the single kernel, as the engine selects it."""
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    monkeypatch.setenv("DMNIST_BUCKET", bucket)
    be = _backend()
    eng = CudaLeNetEngine(128, be, seed=3, rank=0, use_graph=True)
    cuts = [2990, 3001, 3003, 3003, 4000]
    sched = LearningRateSchedule(0.05, 2, 0.999, factor=0.5, cuts=cuts)
    eng.attach_optimizer(SyncReplicasOptimizer(be, sched, 1, 1))
    assert eng._bucket_v2 == (bucket == "2") and eng._bucketed == (bucket == "2")
    eng.arm_lr_cuts(0.5, cuts)
    assert eng.lr_cut_table() == cuts + [lp.NO_CUT] * (lp.MAX_CUTS - len(cuts))
    be.set_global_step(3000)
    gen = torch.Generator().manual_seed(9)
    B, n = eng.batch_size, eng.spec.arena_numel
    b, e = eng._bucket_early
    rounds = A.late_bucket_rounds_bf16(n, e - b, be.late_ll, be.late_bf16)
    seen = set()
    for s in range(5):
        torch.cuda.synchronize()
        step = be.device_epoch
        seen.add(sum(1 for c in cuts if c <= step))
        w = A.f32(eng.params)
        eng.load_batch(torch.rand(B, 28, 28, generator=gen) - 0.5, torch.randint(0, 10, (B,), generator=gen))
        eng.train_step()
        torch.cuda.synchronize()
        scale = A.step_scale(sched, step, 1)
        grads = A.f32(eng.grads)
        if bucket == "2":
            want = A.bucket_step(w, [grads], [A.f32(eng._g16_view.float()).reshape(-1)], (b, e), scale, rounds)
        else:
            want = A.fused_sync_step(w, [grads], 1, scale)
        torch.cuda.synchronize()
        got = A.bits(eng.params)
        bad = np.flatnonzero(got != A.bits(want))
        assert bad.size == 0, "bucket=%s step %d: %d weights differ" % (bucket, step, bad.size)
        sh = eng.shadow.view(torch.int16).cpu().numpy().view(np.uint16)
        assert (sh == A.bf16_bits(want)).all()
    be.check_error()
    assert seen == {1, 2, 4}


# ---- lenet runs through train() ---------------------------------------------------------------------------------------
def _train(d, *extra, steps=60):
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


def _replay(rows, patience, delta_rows, n):
    state, cuts = lp.State(), []
    for r in rows:
        before = state.cuts
        state, fired = lp.advance(state, int(r[0]), int(r[4]), int(r[3]), n, patience, delta_rows)
        if fired and state.cuts > before:
            cuts.append(dict(trigger_step=int(r[0]), from_step=int(r[0]) + 2))
    return state, cuts


@pytest.mark.parametrize("pipelined", [True, False])
def test_lenet_run_device_table_equals_replay_and_file(tmp_path, flags, pipelined, caplog):
    import logging
    pipe = "--pipeline_steps=%s" % ("true" if pipelined else "false")
    ref = _train(str(tmp_path / "ref"), pipe)
    with caplog.at_level(logging.WARNING, logger="dmnist"):
        res = _train(str(tmp_path / "armed"), pipe, *ARMED)
    assert not [r for r in caplog.records if "differs" in r.getMessage()]
    rows = _rows(tmp_path / "armed")
    state, cuts = _replay(rows, 1, VAL // 2, VAL)
    assert len(cuts) >= 3, rows[:, [0, 4]].tolist()
    rep = res["lr_plateau"]
    with open(str(tmp_path / "armed" / "worker0_lr_plateau.json")) as f:
        assert json.load(f) == rep
    assert rep["cuts"] == cuts and rep["min_delta_rows"] == VAL // 2 and rep["weights"] == "live"
    eng = res["engine"]
    assert eng.lr_plateau_state() == state
    assert eng.lr_cut_table() == [c["from_step"] for c in cuts] + [lp.NO_CUT] * (lp.MAX_CUTS - len(cuts))
    ra = _rows(tmp_path / "ref")
    assert rows[:, 0].tolist() == ra[:, 0].tolist() and res["final_step"] == ref["final_step"]
    if pipelined:
        return                 # the batch packer's threads draw batches in no fixed order: the two runs see other inputs
    # the evaluations score bit-identical weights up to the first cut's step, and different ones after it
    s1 = cuts[0]["from_step"]
    early = rows[:, 0] <= s1
    np.testing.assert_array_equal(rows[early][:, [0, 3, 4, 5]], ra[early][:, [0, 3, 4, 5]])
    assert not np.array_equal(rows[~early][:, 5], ra[~early][:, 5])


def test_lenet_run_with_cuts_follows_the_emulated_rate(tmp_path, flags):
    """A flag-armed run cut short at --max_steps = S_1 - 1 ends with the weights of step S_1, bit-identical to the run
    without the flag, and its schedule already holds the cut from S_1."""
    full = _train(str(tmp_path / "full"), *ARMED, "--pipeline_steps=false")
    s1 = full["lr_plateau"]["cuts"][0]["from_step"]
    a = _train(str(tmp_path / "a"), *ARMED, "--pipeline_steps=false", steps=s1 - 1)
    b = _train(str(tmp_path / "b"), "--pipeline_steps=false", steps=s1 - 1)
    assert a["final_step"] == b["final_step"] == s1
    assert np.array_equal(a["params"].cpu().numpy().view(np.uint32), b["params"].cpu().numpy().view(np.uint32))
    assert a["optimizer"].lr_schedule(s1) == b["optimizer"].lr_schedule(s1) * 0.1


# ---- two replicas -----------------------------------------------------------------------------------------------------
@pytest.mark.multigpu
def test_two_replicas_stay_bit_identical_through_cuts(tmp_path):
    """K = N on 2 GPUs with cuts after every pass but the first: on every aggregation path both replicas end with the same
    parameters, and the chief's file lists the cuts of the host replay of its evaluations."""
    from distributedmnist_b200.parallel.launcher import run_replicas
    worker = os.path.join(ROOT, "tests", "_device_eval_worker.py")
    for b in ("2", "1", "0"):
        d = tmp_path / ("bucket" + b)
        codes = run_replicas([worker, str(d / "rank_RANK"), "--train_dir=%s" % (d / "train_dir"), "--batch_size=128",
                              "--max_steps=120", "--initial_learning_rate=0.05", "--save_interval_secs=1000",
                              "--log_every=50", "--eval_every_steps=10"] + list(ARMED), 2, timeout=600,
                             out_dir=str(d / "out"), env={"DMNIST_BUCKET": b})
        logs = "\n".join(open(os.path.join(d, "out", f)).read()[-1500:] for f in sorted(os.listdir(d / "out")))
        assert codes == [0, 0], (b, logs)
        p = [np.load(str(d / ("rank_%d.npy" % r))) for r in range(2)]
        assert np.array_equal(p[0].view(np.uint32), p[1].view(np.uint32)), "bucket %s: the replicas differ" % b
        rows = np.load(str(d / "train_dir" / "worker0_eval.npy"))
        n = int(rows[0, 3])
        _state, cuts = _replay(rows, 1, n // 2, n)
        with open(str(d / "train_dir" / "worker0_lr_plateau.json")) as f:
            assert json.load(f)["cuts"] == cuts
        assert len(cuts) >= 3
