"""``--moving_average_decay`` / ``--eval_moving_average`` on the CPU: every refusal and the accepted combinations, the float32
emulation against a float64 evaluation of the formula, the torch engine's average in the final checkpoint against a replay
over the weights of every global step, unchanged files with the flag off, and the evaluator scoring the averages."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200 import moving_average as ema
from distributedmnist_b200.checkpoint import Saver
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.train import check_moving_average_flags, train


@pytest.fixture
def clean_flags():
    FLAGS.reset()
    saved = {k: os.environ.pop(k) for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK") if k in os.environ}
    yield FLAGS
    FLAGS.reset()
    os.environ.update(saved)


def _flags(**kw):
    base = dict(moving_average_decay=0.99, eval_moving_average=False, eval_every_steps=0, interval_method=False,
                worker_times_cdf_method=False)
    return SimpleNamespace(**dict(base, **kw))


@pytest.mark.parametrize("flags, n, k, msg", [
    (dict(moving_average_decay=1.0), 1, 1, r"must lie in \(0, 1\)"),
    (dict(moving_average_decay=1.5), 1, 1, r"must lie in \(0, 1\)"),
    (dict(moving_average_decay=-0.5), 1, 1, r"must lie in \(0, 1\)"),
    (dict(moving_average_decay=float("nan")), 1, 1, r"must lie in \(0, 1\)"),
    (dict(), 4, 2, r"K < N.*cannot name the global steps"),
    (dict(), 2, 6, r"K > N.*cannot name the global steps"),
    (dict(interval_method=True), 2, 2, "cannot be combined with --interval_method"),
    (dict(interval_method=True, worker_times_cdf_method=True), 2, 2, "cannot be combined with --interval_method"),
    (dict(moving_average_decay=0.0, eval_moving_average=True, eval_every_steps=5), 1, 1, "needs --moving_average_decay"),
    (dict(eval_moving_average=True, eval_every_steps=0), 1, 1, "needs --eval_every_steps > 0"),
], ids=["one", "above_one", "negative", "nan", "k_lt_n", "k_gt_n", "interval", "interval_and_cdf", "eval_without_decay",
        "eval_without_eval_every"])
def test_refusals_name_their_reason(flags, n, k, msg):
    with pytest.raises(ValueError, match=msg):
        check_moving_average_flags(_flags(**flags), SimpleNamespace(world_size=n), k)


def test_accepted_combinations():
    for n in (1, 2, 8):
        check_moving_average_flags(_flags(), SimpleNamespace(world_size=n), n)                                 # K = N
        for k in (1, n, 3 * n):                                                                            # cdf, any K
            check_moving_average_flags(_flags(worker_times_cdf_method=True), SimpleNamespace(world_size=n), k)
    check_moving_average_flags(_flags(eval_moving_average=True, eval_every_steps=10, moving_average_decay=1e-6),
                               SimpleNamespace(world_size=1), 1)
    check_moving_average_flags(_flags(moving_average_decay=0.0, interval_method=True), SimpleNamespace(world_size=4), 1)


def test_flags_are_registered_and_off_by_default(clean_flags):
    assert FLAGS.moving_average_decay == 0.0 and FLAGS.eval_moving_average is False
    FLAGS.parse(["--moving_average_decay=0.999", "--eval_moving_average"])
    assert FLAGS.moving_average_decay == 0.999 and FLAGS.eval_moving_average is True


def _f64_step(s, w, decay, g):
    """The formula with the same roundings, each operation in float64 and rounded to float32 by hand."""
    d = min(decay, (1.0 + g) / (10.0 + g))
    m = np.float32(1.0 - d).astype(np.float64)
    f32 = lambda x: np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)   # noqa: E731
    s64, w64 = s.astype(np.float64), w.astype(np.float64)
    diff = f32(s64 - w64)
    return f32(s64 - f32(diff * m)).astype(np.float32)


@pytest.mark.parametrize("decay", [0.5, 0.9, 0.999, 0.9999])
def test_emulation_against_float64(decay):
    rng = np.random.default_rng(3)
    n = 4099
    s = rng.standard_normal(n).astype(np.float32) * 0.1
    s[:8] = [0.0, -0.0, 1e-40, -1e-40, 3e-39, 1e30, -1e-30, 0.5]      # zeros, subnormals, large and tiny values
    for g in [0, 1, 2, 5, 8, 9, 10, 50, 100, 999, 10 ** 4, 10 ** 6, 2 ** 32 - 1]:
        w = (s + rng.standard_normal(n).astype(np.float32) * 0.01).astype(np.float32)
        w[:8] = [1e-40, 0.0, -1e-40, 1e-40, 0.0, 1e30, 2e-30, 0.25]
        got = ema.emulate(s, w, decay, g)
        want = _f64_step(s, w, decay, g)
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), (decay, g)
        # early steps: (1 + g) / (10 + g) < D, the ramp TF's num_updates gives
        r = (1.0 + g) / (10.0 + g)
        assert float(ema.multiplier(decay, g)) == float(np.float32(1.0 - min(decay, r)))
        if r < decay:
            assert float(ema.multiplier(decay, g)) > float(np.float32(1.0 - decay))
        s = got
    # the real-number value it approximates: close in float64
    s0 = np.float32(0.3)
    w0 = np.float32(0.1)
    assert abs(float(ema.emulate(np.array([s0]), np.array([w0]), 0.9, 1000)[0]) - (0.3 - 0.2 * 0.1)) < 1e-7


def _train(train_dir, *extra, steps=20):
    FLAGS.reset()
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=32", "--max_steps=%d" % steps, "--model=mlp2",
                 "--mlp_hidden=32", "--save_results_period=1000", "--save_interval_secs=1000",
                 "--initial_learning_rate=0.05"] + list(extra))
    ctx = init_context(FLAGS, want_gpu=False)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    return train(ctx, ds.train, ds.validation, FLAGS)


def _recorded_weights(train_dir, steps, monkeypatch):
    """The weights after every global step of a run without the flag, recorded where the trainer applies them."""
    from distributedmnist_b200.engine import TorchEngine
    rec = {}
    real = TorchEngine.forward_backward

    def fb(self, step):
        rec[int(step)] = self.params.detach().clone()         # the weights of global step `step`
        return real(self, step)
    monkeypatch.setattr(TorchEngine, "forward_backward", fb)
    res = _train(train_dir, steps=steps)
    monkeypatch.undo()
    rec[res["final_step"]] = res["params"].detach().clone()
    return rec, res


def test_torch_engine_final_checkpoint_holds_the_replayed_average(tmp_path, clean_flags, monkeypatch):
    steps, decay = 20, 0.9
    rec, ref = _recorded_weights(str(tmp_path / "ref"), steps, monkeypatch)
    res = _train(str(tmp_path / "avg"), "--moving_average_decay=%r" % decay, steps=steps)
    final = res["final_step"]
    assert final == ref["final_step"] and res["losses"] == ref["losses"]
    assert torch.equal(res["params"], ref["params"])                       # the average never perturbs training
    s = rec[0].numpy().copy()
    for g in range(1, final + 1):
        s = ema.emulate(s, rec[g].numpy(), decay, g)
    state, step = Saver.restore(Saver.latest(str(tmp_path / "avg")))
    assert step == final
    spec = res["engine"].spec
    assert sorted(state) == sorted(spec.ckpt_names() + ema.names(spec))
    got = ema.from_state_dict(spec, state).numpy()
    mask = spec.valid_mask().numpy()
    assert np.array_equal(got[mask].view(np.int32), s[mask].view(np.int32))
    avg, avg_step = res["engine"].moving_average()
    assert avg_step == final and np.array_equal(avg.numpy().view(np.int32), s.view(np.int32))
    # the weights in the same file are those of the run without the flag
    assert torch.equal(spec.from_state_dict(state)[spec.valid_mask()], ref["params"][spec.valid_mask()])


def test_flag_off_files_hold_exactly_the_variables(tmp_path, clean_flags):
    res = _train(str(tmp_path / "off"), steps=6)
    state, _ = Saver.restore(Saver.latest(str(tmp_path / "off")))
    assert sorted(state) == sorted(res["engine"].spec.ckpt_names())
    assert res["engine"]._ema is None


def test_restore_loads_the_averages_or_starts_from_the_weights(tmp_path, clean_flags, caplog):
    import logging
    d = str(tmp_path / "run")
    _train(d, "--moving_average_decay=0.9", steps=6)
    first, step0 = Saver.restore(Saver.latest(d))
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(d, "--moving_average_decay=0.9", steps=6)             # restores step 7: nothing left to run but one
    spec = res["engine"].spec
    assert not any("holds no complete set of averages" in r.getMessage() for r in caplog.records)
    # the average restored, then one more update with the weights of the step after the restore
    assert res["final_step"] == step0 + 1
    state, _ = Saver.restore(Saver.latest(d))
    w = spec.from_state_dict(state).numpy()
    want = ema.emulate(ema.from_state_dict(spec, first).numpy(), w, 0.9, step0 + 1)
    mask = spec.valid_mask().numpy()
    assert np.array_equal(ema.from_state_dict(spec, state).numpy()[mask].view(np.int32), want[mask].view(np.int32))
    # a checkpoint without averages (flag off): the average starts from the restored weights, with one log line
    d2 = str(tmp_path / "plain")
    _train(d2, steps=6)
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="dmnist"):
        _train(d2, "--moving_average_decay=0.9", steps=6)
    assert sum("holds no complete set of averages" in r.getMessage() for r in caplog.records) == 1
    # restore with the flag off: the averages are ignored and not carried into the new file
    res = _train(d, steps=10)
    state, _ = Saver.restore(Saver.latest(d))
    assert sorted(state) == sorted(spec.ckpt_names())


def test_eval_moving_average_scores_the_average_in_training(tmp_path, clean_flags, caplog):
    import logging
    with caplog.at_level(logging.INFO, logger="dmnist"):
        res = _train(str(tmp_path / "a"), "--moving_average_decay=0.9", "--eval_moving_average", "--eval_every_steps=5",
                     "--target_accuracy=1.0", steps=10)
    assert sum("the in-training evaluation scores the averaged weights" in r.getMessage() for r in caplog.records) == 1
    eng = res["engine"]
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    loss, acc = eng.evaluate(ds.validation.images, ds.validation.labels, moving_average=True)
    last = res["evals"][-1]
    assert last[0] == res["final_step"] and last[4] == int(round(acc * last[3])) and abs(last[5] - loss) < 1e-12
    assert res["time_to_accuracy"]["weights"] == "moving_average"
    ref = _train(str(tmp_path / "b"), "--eval_every_steps=5", "--target_accuracy=1.0", steps=10)
    assert "weights" not in ref["time_to_accuracy"]


def test_evaluator_scores_the_averages_and_skips_a_checkpoint_without_them(tmp_path, clean_flags, capsys):
    from distributedmnist_b200.engine import TorchEngine
    from distributedmnist_b200.evaluator import do_eval
    d = str(tmp_path / "avg")
    res = _train(d, "--moving_average_decay=0.9", steps=8)
    spec = res["engine"].spec
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=0, n_workers=1, seed=FLAGS.seed, synthetic=True,
                               synthetic_sizes=(256, 64))
    state, step = Saver.restore(Saver.latest(d))
    probe = TorchEngine("mlp2", 1, torch.device("cpu"), lambda n: torch.zeros(n), mlp_hidden=32)
    probe.params.copy_(ema.from_state_dict(spec, state))
    want = probe.evaluate(ds.validation.images, ds.validation.labels)
    probe.params.copy_(spec.from_state_dict(state))
    live = probe.evaluate(ds.validation.images, ds.validation.labels)
    assert want != live
    for average, expect in ((True, want), (False, live)):
        FLAGS.reset()
        FLAGS.parse(["--checkpoint_dir=%s" % d, "--model=mlp2", "--mlp_hidden=32"] +
                    (["--eval_moving_average"] if average else []))
        eng = TorchEngine("mlp2", 1, torch.device("cpu"), lambda n: torch.zeros(n), mlp_hidden=32)
        capsys.readouterr()
        assert do_eval(eng, None, ds.validation, FLAGS) == str(step)
        out = capsys.readouterr().out
        assert "Precision @ 1: %f Loss: %f" % (expect[1], expect[0]) in out, out
    # a checkpoint written without the flag is reported and skipped, and the poller goes on
    d2 = str(tmp_path / "plain")
    _train(d2, steps=4)
    FLAGS.reset()
    FLAGS.parse(["--checkpoint_dir=%s" % d2, "--model=mlp2", "--mlp_hidden=32", "--eval_moving_average"])
    eng = TorchEngine("mlp2", 1, torch.device("cpu"), lambda n: torch.zeros(n), mlp_hidden=32)
    capsys.readouterr()
    assert do_eval(eng, None, ds.validation, FLAGS, prev_global_step="3") == "3"
    out = capsys.readouterr().out
    assert "Could not restore" in out and "no moving averages" in out and "Precision" not in out


def test_kernel_is_listed_by_ptxas_report_without_spills():
    """The in-tree build compiles csrc/moving_average.cu for sm_90a; its -Xptxas -v log lists the kernel, not spilling."""
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    log = os.path.join(root, "build", "obj", "moving_average.log")
    if not os.path.exists(log):
        pytest.skip("no in-tree build log (build() has not run)")
    spec = importlib.util.spec_from_file_location("ptxas_report", os.path.join(root, "tools", "ptxas_report.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rows = [r for r in mod.parse(log) if "moving_average_kernel" in r["name"]]
    assert len(rows) == 1, rows
    r = rows[0]
    assert r["arch"] == "sm_90a" and r["spill_st"] == r["spill_ld"] == r["stack"] == 0, r
