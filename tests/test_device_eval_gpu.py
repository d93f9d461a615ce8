"""In-training evaluation on the GPU (``CudaLeNetEngine.arm_eval`` / ``enqueue_eval``, csrc/eval_head.cu): exact logits, exact
counts against a float64 forward, bit-reproducible records, no effect on training, and records of exactly the weights of the
step they follow."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHUNK = 2048


def _engine(B, seed, use_graph):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    return CudaLeNetEngine(B, be, seed=seed, use_graph=use_graph), be


def _valset(n, seed):
    from distributedmnist_b200.ops.selfcheck import mnist_like
    g = torch.Generator().manual_seed(seed)
    return mnist_like(g, n), torch.randint(0, 10, (n,), generator=g)


def _fields(rec):
    gs, _t0, _t1, n, correct, loss = rec
    return gs, n, correct, float(loss)


def test_logits_bit_identical_to_forward_logits_chunk_by_chunk():
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    assert CudaLeNetEngine.EVAL_CHUNK == CHUNK
    eng, _ = _engine(CHUNK, 7, use_graph=False)      # engine batch = chunk, so forward_logits can run a whole chunk
    x, y = _valset(2500, 8)
    eng.arm_eval(x, y)
    lg = torch.full((2500, 10), float("nan"), device="cuda")
    rec = eng.run_eval(logits_out=lg)
    assert rec is not None and rec[3] == 2500
    xd, yd = x.cuda(), y.cuda()
    for s in range(0, 2500, CHUNK):                   # 2048 + a partial chunk of 452
        ref = eng.forward_logits(xd[s:s + CHUNK], yd[s:s + CHUNK], False)
        assert torch.equal(lg[s:s + CHUNK], ref), "chunk at row %d differs from forward_logits(train=False)" % s
    # the head's count is the first-maximum argmax of exactly these logits
    first = (lg == lg.max(dim=1, keepdim=True).values).to(torch.int8).argmax(dim=1)
    assert rec[4] == int((first == yd).sum())


# Loss bound.  A row's loss is log(sum_c exp(l_c - m)) - (l_label - m), computed in fp32 from the kernel's logits with the
# fast-math __expf / __logf (as fc2_fwd_bwd computes it).  If every logit of the row is within d of the float64 logit, the
# exact loss of the kernel's logits is within 2 d of the reference (the log-sum-exp and l_label each move by at most d).
# The intrinsics add an absolute error: __expf's relative error grows with |argument| (ex2.approx of a rounded product,
# about |x| 2^-23 for |x| <= 30 here) and __logf's absolute error is about 2^-21, so a row's loss is off by at most
# 2 d + 2^-16 (a generous envelope), and the mean by at most 2 mean(d) + 2^-16.  The fold into a double adds nothing
# measurable at 10 000 rows.
LOSS_ABS_SLACK = 2.0 ** -16


@pytest.mark.parametrize("n", [2500, 10000])
def test_counts_exact_and_loss_bounded_against_float64(n):
    from distributedmnist_b200.ops.selfcheck import EVAL_LOGIT_BOUND, EVAL_MAX_NEAR_TIES, lenet_eval_f64
    eng, _ = _engine(256, 9, use_graph=True)
    x, y = _valset(n, 10 + n)
    eng.arm_eval(x, y)
    lg = torch.zeros(n, 10, device="cuda")
    gs, _t0, _t1, examples, correct, loss_sum = eng.run_eval(logits_out=lg)
    assert examples == n and n % CHUNK != 0
    xd, yd = x.cuda(), y.cuda()
    ref = lenet_eval_f64(eng.p, eng.pb, xd, yd)
    rl = ref["logits"]
    dev = (lg.double() - rl).abs().max(dim=1).values
    assert float((dev / (1.0 + rl.abs().max(dim=1).values)).max()) <= EVAL_LOGIT_BOUND
    near = ref["gap"] <= 2 * float(dev.max())        # the argmax may differ from the reference only here
    assert float(near.sum()) / n <= EVAL_MAX_NEAR_TIES
    hits = (rl.argmax(dim=1) == yd) & ~near
    lo, hi = int(hits.sum()), int((hits | near).sum())
    assert lo <= correct <= hi, (lo, correct, hi)
    bound = 2 * float(dev.mean()) + LOSS_ABS_SLACK
    assert abs(loss_sum / n - float(ref["loss"])) <= bound, (loss_sum / n, float(ref["loss"]), bound)


def test_two_passes_give_identical_records():
    eng, _ = _engine(256, 12, use_graph=True)
    x, y = _valset(2500, 13)
    eng.arm_eval(x, y)
    eng.enqueue_eval()                                 # the captured graph
    torch.cuda.synchronize()
    a = eng.eval_record()
    b = eng.run_eval()                                 # eager launches of the same pass
    eng.enqueue_eval()
    torch.cuda.synchronize()
    c = eng.eval_record()
    assert a is not None and _fields(a) == _fields(b) == _fields(c)
    assert a[1] < a[2] and b[1] < b[2] and a[2] <= b[1]          # %globaltimer: begin < end, passes in order


def _batches(n, B, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.rand(B, 28, 28, 1, generator=g) - 0.5, torch.randint(0, 10, (B,), generator=g)) for _ in range(n)]


def _run(batches, val, packed, every):
    """60 graph-replayed steps at B = 256.  every > 0: a pass after every `every`-th step.  Returns parameters, shadow,
    losses, the records and the parameters saved after every 10th step."""
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.schedule import LearningRateSchedule
    eng, be = _engine(256, 21, use_graph=True)
    eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 20, 0.7), 1, 1))
    if every:
        eng.arm_eval(*val)
    bufs = [eng.pack_batch(x, y) for x, y in batches] if packed else None
    losses, saved, records = [], {}, []
    for s, (x, y) in enumerate(batches):
        if packed:
            ev, buf, _ = eng.step_packed(bufs[s])
        else:
            eng.load_batch(x.numpy(), y.numpy())
            eng.train_step()
            ev, buf = eng.read_loss_async()
        if every and (s + 1) % every == 0:
            eng.enqueue_eval()                         # between two native-runner steps, no host synchronisation
        ev.synchronize()
        losses.append((float(buf[0]), float(buf[1])))
        if every:
            records += eng.eval_records()
        elif (s + 1) % 10 == 0:
            torch.cuda.synchronize()
            saved[s + 1] = (eng.params.clone(), eng.shadow.clone())
    torch.cuda.synchronize()
    be.check_error()
    if every:
        records += eng.eval_records()
    out = (eng.params.clone(), eng.shadow.clone(), losses, records, saved, eng.step_info().global_step)
    eng._leave_native_runner()
    return out


@pytest.mark.parametrize("packed", [False, True], ids=["load_batch+train_step", "pack_batch+step_packed"])
def test_training_unperturbed_and_records_score_the_step_they_follow(packed):
    batches = _batches(60, 256, 31)
    val = _valset(2500, 32)
    p0, s0, l0, _r0, saved, g0 = _run(batches, val, packed, every=0)
    p1, s1, l1, recs, _s1, g1 = _run(batches, val, packed, every=10)
    assert g0 == g1 == 60
    assert torch.equal(p0, p1) and torch.equal(s0, s1), "the evaluation pass changed the training trajectory"
    assert l0 == l1
    assert [r[0] for r in recs] == [10, 20, 30, 40, 50, 60]
    # a standalone pass over the parameters saved at step s reproduces the record enqueued after step s
    eng, be = _engine(256, 21, use_graph=False)
    eng.arm_eval(*val)
    for r in recs:
        params, shadow = saved[r[0]]
        eng.params.copy_(params)
        eng.shadow.copy_(shadow)
        be.set_global_step(r[0])
        ref = eng.run_eval()
        assert _fields(ref) == _fields(r), (r, ref)


def test_end_to_end_eval_rows_match_the_standalone_evaluator(tmp_path):
    train_dir, eval_dir = str(tmp_path / "train_dir"), str(tmp_path / "eval_dir")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="0")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    tr = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_distributed_train.py"), "--job_name=worker",
                         "--task_id=0", "--worker_hosts=localhost:1234", "--batch_size=128", "--max_steps=300",
                         "--eval_every_steps=100", "--initial_learning_rate=0.05", "--learning_rate_decay_factor=1",
                         "--train_dir=" + train_dir, "--log_every=50"], env=env, capture_output=True, text=True, timeout=600)
    log = tr.stdout + tr.stderr
    assert tr.returncode == 0, log[-3000:]
    test_accs = [float(v) for v in re.findall(r"Worker 0: .*: step [0-9]+, loss = .*test_acc = ([0-9.]+)\(", log)]
    assert test_accs and max(test_accs) > 0.5, log[-2000:]
    rows = np.load(os.path.join(train_dir, "worker0_eval.npy"))
    assert rows[:, 0].tolist() == [100, 200, 300, 301], rows
    assert (rows[:, 3] == 10000).all() and (rows[:, 2] > 0).all()
    ev = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_eval.py"), "--run_once=true",
                         "--checkpoint_dir=" + train_dir, "--eval_dir=" + eval_dir], env=env, capture_output=True,
                        text=True, timeout=600)
    out = ev.stdout + ev.stderr
    assert ev.returncode == 0, out[-3000:]
    m = re.search(r"Num examples: 10000  Precision @ 1: ([0-9.]+) Loss: ([0-9.]+) Time", out)
    assert m and "model.ckpt-301 at step=301." in out, out[-2000:]
    assert int(rows[-1, 4]) == round(float(m.group(1)) * 10000)
    # the evaluator sums fp32 loss / 1000 terms per batch: relative agreement to 2^-10 (selfcheck.EVAL_LOSS_REL)
    assert abs(rows[-1, 5] - float(m.group(2))) <= 2.0 ** -10 * float(m.group(2)) + 1e-6


def replica_runs(tmp_path, n, max_steps=200, every=50):
    """n replicas (K = N) through train.train, each run in a fresh train_dir.  Pipelined loop with the pass on, on each
    aggregation path (DMNIST_BUCKET: 2 = bucketed bf16 wire, 1 = bucketed fp32, 0 = single kernel); non-pipelined loop with
    the pass on and off (its input order is deterministic, so the two runs can be compared with each other)."""
    import json

    from distributedmnist_b200.parallel.launcher import run_replicas
    worker = os.path.join(ROOT, "tests", "_device_eval_worker.py")
    runs = [("pipelined_bucket%s" % b, {"DMNIST_BUCKET": b}, ["--eval_every_steps=%d" % every]) for b in ("2", "1", "0")]
    runs += [("sync_eval", {}, ["--eval_every_steps=%d" % every, "--pipeline_steps=false"]),
             ("sync_off", {}, ["--pipeline_steps=false"])]
    out = {}
    for name, env, extra in runs:
        d = tmp_path / name
        codes = run_replicas([worker, str(d / "rank_RANK"), "--train_dir=%s" % (d / "train_dir"), "--batch_size=128",
                              "--max_steps=%d" % max_steps, "--initial_learning_rate=0.05", "--save_interval_secs=1000",
                              "--log_every=50"] + extra, n, timeout=600, out_dir=str(d / "out"), env=env)
        logs = "\n".join(open(os.path.join(d, "out", f)).read()[-1500:] for f in sorted(os.listdir(d / "out")))
        assert codes == [0] * n, (name, logs)
        ranks = []
        for r in range(n):
            with open(str(d / ("rank_%d.json" % r))) as f:
                meta = json.load(f)
            ranks.append((np.load(str(d / ("rank_%d.npy" % r))), meta))
        out[name] = (ranks, sorted(f for f in os.listdir(d / "train_dir") if f.endswith("_eval.npy")), d / "train_dir")
    return out


def check_replica_runs(out, n, max_steps=200, every=50):
    expected = list(range(every, max_steps + 1, every)) + [max_steps + 1]
    for name, (ranks, eval_files, train_dir) in out.items():
        p0 = ranks[0][0]
        for r in range(1, n):
            assert np.array_equal(p0.view(np.uint32), ranks[r][0].view(np.uint32)), "%s: rank %d differs from rank 0" % (name, r)
        assert all(meta["final_step"] == max_steps + 1 for _p, meta in ranks), name
        if name == "sync_off":
            assert eval_files == [] and all(meta["evals"] == [] for _p, meta in ranks)
            continue
        assert eval_files == ["worker0_eval.npy"], (name, eval_files)        # the chief only
        rows = np.load(str(train_dir / "worker0_eval.npy"))
        assert rows[:, 0].tolist() == expected, (name, rows)
        assert (rows[:, 3] == 10000).all() and (rows[:, 4] > 0).all()
        assert all(meta["evals"] == [] for _p, meta in ranks[1:])
    # the pass does not change what the replicas compute
    assert np.array_equal(out["sync_eval"][0][0][0].view(np.uint32), out["sync_off"][0][0][0].view(np.uint32))


@pytest.mark.multigpu
def test_two_replicas_stay_bit_identical_with_eval_on(tmp_path):
    """K = N on 2 GPUs: the chief runs the pass after every 50th step (about 1 ms longer than its peer there).  Both replicas
    end with the same parameters on every aggregation path, and with the same parameters as without the pass."""
    check_replica_runs(replica_runs(tmp_path, 2), 2)
