"""``--keep_best_checkpoint`` on the GPU: eval_best_decide / eval_best_copy (csrc/eval_best.cu) on crafted device words
against the host emulation and bit for bit on the lenet and mlp2 arena sizes; lenet runs through ``train()`` whose best
checkpoint is bit-identical to the step-g checkpoint of a run cut at g and scores the same in the standalone evaluator,
with unchanged weights, rows and step graph; the moving average; K > N and interval snapshot runs; a dropped snapshot pass
that never becomes the best; and a run stopped by --target_accuracy."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
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


def _data():
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.flags import FLAGS
    return mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True, synthetic_sizes=(8192, VAL))


def _train(d, *extra, steps=60):
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import train
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % d, "--batch_size=128", "--max_steps=%d" % steps, "--eval_every_steps=5",
                 "--initial_learning_rate=0.05", "--log_every=1000", "--save_results_period=1000000",
                 "--save_interval_secs=1000"] + list(extra))
    ctx = init_context(FLAGS)
    ds = _data()
    return train(ctx, ds.train, ds.validation, FLAGS)


def _rows(d):
    return np.load(os.path.join(str(d), "worker0_eval.npy"))


def _data_file(d, step):
    with open(os.path.join(str(d), "model.ckpt-%d.data-00000-of-00001" % step), "rb") as f:
        return f.read()


def _first_argmax(rows):
    best = int(rows[:, 4].max())
    return int(rows[rows[:, 4] == best][0, 0]), best


def _standalone_eval(best_dir, capsys):
    """The evaluator (src/mnist_eval.py's do_eval) on ``best_dir``: (printed precision, correct count)."""
    from distributedmnist_b200.evaluator import _make_eval_engine, do_eval
    from distributedmnist_b200.flags import FLAGS
    ds = _data()
    FLAGS.reset()
    FLAGS.parse(["--checkpoint_dir=%s" % best_dir, "--run_once"])
    eng = _make_eval_engine(FLAGS, torch.device("cuda", 0))
    capsys.readouterr()
    do_eval(eng, None, ds.validation, FLAGS)
    out = capsys.readouterr().out
    prec = out.split("Precision @ 1: ")[1].split(" ")[0]
    _loss, acc = eng.evaluate(ds.validation.images, ds.validation.labels)
    return prec, int(round(acc * ds.validation.num_examples))


# ---- the kernels on crafted words -------------------------------------------------------------------------------------
def _lib():
    from distributedmnist_b200.ops.lib import load
    return load()


def _decide(correct, examples, loss_sum, step, n, best, status):
    """One eval_best_decide launch: (BestState tuple, decision word) as the device left them."""
    from distributedmnist_b200.best import BEST_CORRECT_WORD, BEST_EXAMPLES_WORD, BEST_STEP_WORD, BEST_VALID_WORD
    from distributedmnist_b200.ops.lib import stream_ptr
    lib = _lib()
    ev = torch.zeros(int(lib.dm_eval_state_bytes()), dtype=torch.uint8)
    ev[0:8].view(torch.float64)[0] = loss_sum
    ev[16:24].view(torch.int32)[:] = torch.tensor([correct, examples], dtype=torch.int32)
    w = torch.zeros(int(lib.dm_best_state_bytes()) // 4, dtype=torch.int32)
    w[0:2].view(torch.float64)[0] = best[3]
    w[BEST_STEP_WORD], w[BEST_CORRECT_WORD], w[BEST_EXAMPLES_WORD], w[BEST_VALID_WORD] = best[0], best[1], best[2], best[4]
    ev, w = ev.cuda(), w.cuda()
    step_t = torch.tensor([step], dtype=torch.int32, device="cuda")
    st_t = None if status is None else torch.tensor([status], dtype=torch.int32, device="cuda")
    word = torch.full((1,), 7, dtype=torch.int32, device="cuda")
    lib.dm_eval_best_decide(ev, step_t, st_t, n, w, word, stream_ptr())
    torch.cuda.synchronize()
    h = w.cpu()
    return ((int(h[BEST_STEP_WORD]), int(h[BEST_CORRECT_WORD]), int(h[BEST_EXAMPLES_WORD]),
             float(h[0:2].view(torch.float64)[0]), int(h[BEST_VALID_WORD])), int(word.cpu()[0]))


@pytest.mark.parametrize("correct, examples, best_correct, status", [
    (600, 1000, 599, None),     # improve
    (600, 1000, 600, None),     # tie
    (599, 1000, 600, None),     # worse
    (900, 999, 0, None),        # incomplete pass
    (1000, 1000, 10, -1),       # dropped snapshot, highest count
    (1000, 1000, 10, 0),        # snapshot with no settled attempt
    (700, 1000, 10, 3),         # accepted snapshot
], ids=["improve", "tie", "worse", "incomplete", "dropped", "status0", "accepted"])
def test_decide_matches_the_emulation(correct, examples, best_correct, status):
    from distributedmnist_b200.best import emulate_decide
    best = (17, best_correct, 1000, 123.25, 1)
    got = _decide(correct, examples, 456.5, 42, 1000, best, status)
    assert got == emulate_decide(correct, examples, 456.5, 42, 1000, best, status)


def test_copy_is_bit_exact_and_skipped_on_a_zero_decision():
    from distributedmnist_b200.models import get_model
    from distributedmnist_b200.ops.lib import stream_ptr
    lib = _lib()
    mlp2 = get_model("mlp2", 1024)[0].arena_numel
    sizes = [get_model("lenet")[0].arena_numel, mlp2, mlp2 + 3, 1, 7]    # odd lengths take the scalar tail
    g = torch.Generator(device="cuda").manual_seed(1)
    for n in sizes:
        src = torch.randn(n, device="cuda", generator=g)
        src.view(torch.int32)[::97] = 0x7FC00001               # NaN payloads survive: a bit copy, not arithmetic
        dst = torch.full((n,), -3.0, device="cuda")
        for decision in (0, 1):
            word = torch.tensor([decision], dtype=torch.int32, device="cuda")
            lib.dm_eval_best_copy(word, src, dst, n, stream_ptr())
            torch.cuda.synchronize()
            want = src if decision else torch.full((n,), -3.0, device="cuda")
            assert torch.equal(dst.view(torch.int32), want.view(torch.int32)), (n, decision)


# ---- lenet through train() --------------------------------------------------------------------------------------------
def test_lenet_best_checkpoint_is_the_step_g_weights(tmp_path, flags, capsys):
    loop = ["--device_data=true"]
    res = _train(tmp_path / "armed", *loop, "--keep_best_checkpoint")
    off = _train(tmp_path / "off", *loop)
    rows = _rows(tmp_path / "armed")
    g, best = _first_argmax(rows)
    rep = res["best"]
    with open(str(tmp_path / "armed" / "worker0_best.json")) as f:
        assert json.load(f) == rep
    assert rep["global_step"] == g and rep["correct"] == best and rep["examples"] == VAL and rep["weights"] == "live"
    assert rep["mean_loss"] == rows[rows[:, 0] == g][0, 5]
    # the flag changes neither the training, nor the rows, nor the step graph
    assert torch.equal(res["params"].view(torch.int32), off["params"].view(torch.int32))
    np.testing.assert_array_equal(rows[:, [0, 3, 4, 5]], _rows(tmp_path / "off")[:, [0, 3, 4, 5]])
    assert res["engine"].launches_per_step == off["engine"].launches_per_step
    assert not os.path.exists(str(tmp_path / "off" / "best"))
    # the weights of step g, as the final checkpoint of a run cut at g holds them
    cut = _train(tmp_path / "cut", *loop, steps=g - 1)
    assert cut["final_step"] == g
    assert _data_file(tmp_path / "armed" / "best", g) == _data_file(tmp_path / "cut", g)
    prec, correct = _standalone_eval(str(tmp_path / "armed" / "best"), capsys)
    assert prec == "%f" % (best / VAL) and correct == best
    print("\nlenet K = N: best pass at step %d of %d, %d/%d correct" % (g, res["final_step"], best, VAL))


def test_moving_average_best_equals_the_checkpointed_average(tmp_path, flags):
    from distributedmnist_b200 import moving_average as ema
    from distributedmnist_b200.checkpoint import Saver
    avg = ["--device_data=true", "--moving_average_decay=0.9", "--eval_moving_average"]
    res = _train(tmp_path / "armed", *avg, "--keep_best_checkpoint")
    g, best = _first_argmax(_rows(tmp_path / "armed"))
    assert res["best"]["global_step"] == g and res["best"]["correct"] == best
    assert res["best"]["weights"] == "moving_average"
    cut = _train(tmp_path / "cut", *avg, steps=g - 1)
    assert cut["final_step"] == g
    spec = res["engine"].spec
    state_cut, _ = Saver.restore(os.path.join(str(tmp_path / "cut"), "model.ckpt-%d" % g))
    state_best, step = Saver.restore(os.path.join(str(tmp_path / "armed" / "best"), "model.ckpt-%d" % g))
    assert step == g
    want = ema.from_state_dict(spec, state_cut)
    for p in spec.params:
        assert torch.equal(state_best[p.ckpt_name].view(torch.int32),
                           want[p.offset:p.offset + p.numel].view(p.shape).view(torch.int32)), p.ckpt_name


@pytest.mark.parametrize("extra", [["--num_replicas_to_aggregate=4"], ["--interval_method=true", "--interval_ms=2"]],
                         ids=["k4_of_1", "interval"])
def test_snapshot_runs_best_file_scores_its_row(tmp_path, flags, capsys, extra):
    res = _train(tmp_path / "run", "--eval_snapshot=true", "--keep_best_checkpoint", *extra, steps=100)
    rows = _rows(tmp_path / "run")
    rep = res["best"]
    assert rep is not None and rep["weights"] == "snapshot"
    g, best = _first_argmax(rows)
    assert (rep["global_step"], rep["correct"]) == (g, best)
    prec, correct = _standalone_eval(str(tmp_path / "run" / "best"), capsys)
    assert correct == best and prec == "%f" % (best / VAL)
    print("\n%s: best snapshot pass at step %d, %d/%d correct" % (extra[0], g, best, VAL))


def _emulate(eng, g, mode, phases=7):
    from distributedmnist_b200.ops.lib import stream_ptr
    eng.lib.dm_snap_test_emulate(eng.backend.ctrl.local_ptr, eng.params, eng.params.numel(), g, mode, 1, phases, stream_ptr())


@pytest.mark.parametrize("mode", [K_OF_N, INTERVAL], ids=["k_of_n", "interval"])
def test_dropped_snapshot_pass_never_becomes_the_best(mode):
    """An emulated peer on one stream.  The validation labels are the predictions of the initial weights W0, so a pass over
    W0 scores every row.  Step 1's pushes (garbage weights) are accepted and become the best.  Then a snapshot attempt
    copies W0 -- pushed as step 2 -- and is rejected because step 3 commits during the copy; the pass scores W0 (the
    highest count there is) with status -1 and must leave the best at step 1."""
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.ops.lib import stream_ptr
    from distributedmnist_b200.ops.selfcheck import mnist_like
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaLeNetEngine(256, be, seed=5, use_graph=True)
    eng._interval = mode == INTERVAL
    n = 2000
    x = mnist_like(torch.Generator().manual_seed(6), n)
    w0 = eng.params.clone()
    eng.arm_eval(x, torch.zeros(n, dtype=torch.int64))
    logits = torch.zeros(n, 10, device="cuda")
    eng.run_eval(logits_out=logits)
    y = logits.argmax(1).cpu()
    eng.arm_eval(x, y, snapshot=True)
    eng.arm_best()
    _emulate(eng, 1, mode)                                       # step 1: committed, pushed, done
    eng.enqueue_eval()
    torch.cuda.synchronize()
    (rec1, st1), = eng.eval_records_with_status()
    assert st1 > 0 and rec1[0] == 1 and rec1[4] < n
    w1 = eng.params.clone()
    # step 2 pushes W0; an attempt copies it, step 3 commits before validate: the pass is dropped
    _emulate(eng, 2, mode, phases=1)
    eng.params.copy_(w0)
    _emulate(eng, 2, mode, phases=4)
    lib, ctrl, st = eng.lib, be.ctrl.local_ptr, eng._snap_state
    lib.dm_snap_select(ctrl, st, 0, int(eng._interval), eng.SNAP_WATCHDOG_MS, stream_ptr())
    lib.dm_snap_copy(st, eng.params, eng._snap, eng._snap16, eng.params.numel(), *eng._snap_bf_ranges, stream_ptr())
    _emulate(eng, 3, mode, phases=1)
    lib.dm_snap_validate(ctrl, st, eng.SNAP_ATTEMPTS - 1, eng.SNAP_ATTEMPTS, stream_ptr())
    p, pb = eng._ev_views
    eng._launch_eval(publish=True, p=p, pb=pb)                   # the pass's chunks, then decide and copy
    torch.cuda.synchronize()
    (rec2, st2), = eng.eval_records_with_status()
    assert st2 == -1 and rec2[3] == n and rec2[4] == n           # the highest count, from a dropped pass
    arena, step, correct, examples, _loss = eng.best_weights()
    assert (step, correct, examples) == (1, rec1[4], n)
    assert torch.equal(arena.view(torch.int32), w1.view(torch.int32))


def test_target_run_keeps_the_scored_step(tmp_path, flags):
    """A reference run scores every step (evaluation does not change training).  The target is the count of a step g,
    a multiple of E = 5, that beats every earlier multiple of 5 and the final pass's step g + 3 of a run stopped by that
    target: the stopped run's best file then holds step g, not its final weights."""
    from distributedmnist_b200.train import STOP_MARGIN
    loop = ["--device_data=true"]
    _train(tmp_path / "ref", *loop, "--eval_every_steps=1", steps=100)
    count = {int(r[0]): int(r[4]) for r in _rows(tmp_path / "ref")}
    final = STOP_MARGIN + 1
    cands = [g for g in range(5, 101 - final, 5)
             if all(count[k] < count[g] for k in range(5, g, 5)) and count[g + final] < count[g]]
    assert cands, count
    g = cands[-1]
    res = _train(tmp_path / "armed", *loop, "--target_accuracy=%r" % (count[g] / VAL), "--keep_best_checkpoint", steps=100)
    assert res["time_to_accuracy"]["global_step"] == g and res["final_step"] == g + final
    rows = _rows(tmp_path / "armed")
    assert int(rows[-1, 0]) == g + final and int(rows[-1, 4]) == count[g + final]
    assert (res["best"]["global_step"], res["best"]["correct"]) == (g, count[g])
    best_dir = str(tmp_path / "armed" / "best")
    assert sorted(os.listdir(best_dir)) == ["checkpoint", "model.ckpt-%d.data-00000-of-00001" % g, "model.ckpt-%d.index" % g]
    assert _data_file(best_dir, g) != _data_file(tmp_path / "armed", g + final)
    print("\ntarget %d/%d reached at step %d, run ended at %d (%d correct), best file holds step %d"
          % (count[g], VAL, g, g + final, count[g + final], g))
