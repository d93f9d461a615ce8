#!/usr/bin/env python
"""Cost of the in-training evaluation (``--eval_every_steps``) on one GPU, synthetic data.  Prints one JSON line.

The training loop is driven as ``train.py``'s pipelined loop drives it: ``step_packed`` (native runner, one CUDA graph per
step), the pass enqueued on the training stream after every E-th step, the host waiting for step i while step i+1 is queued.
Step time is device time (CUDA events around a window of steps, divided by the steps).  The configurations E = off, 100
and 20 alternate over several rounds so the spread between rounds shows.  The cost of one 10k pass is read two ways: from
the pass's own %globaltimer stamps (records) and from CUDA events around passes enqueued between steps.  If the pass adds
only its own device time, the measured overhead matches ``t_eval / (E * t_step)``; a larger one means a pipeline bubble or
a host stall.

    python tools/eval_overhead.py [--steps 2000] [--rounds 3] [--batch 256] [--snapshot] [--out results/eval_overhead.json]

``--snapshot`` adds the cost of the weight snapshot that K < N and interval runs score (``--eval_snapshot``): the pass
with and without it, and the snapshot attempts alone (one accepted attempt and three that exit at once), CUDA events
between steps, quiescent weights.
"""
import argparse
import sys

import gpu_timing
import numpy as np
import torch
from distributedmnist_b200.data import make_synthetic_mnist
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
from distributedmnist_b200.schedule import LearningRateSchedule


def window(eng, bufs, steps, every, first):
    """Device time per step over `steps` steps, a pass after every `every`-th (0: none).  Returns (seconds per step,
    records completed in the window)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    eng.eval_records()
    pending = None
    e0.record()
    for i in range(steps):
        tok = eng.step_packed(bufs[(first + i) % len(bufs)])
        if every and (first + i + 1) % every == 0:
            eng.enqueue_eval()
        if pending is not None:
            pending[0].synchronize()
        pending = tok
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / steps, eng.eval_records()


def _event_median(eng, bufs, done, fn, reps=20):
    """Median device time of fn() enqueued between two training steps (CUDA events on the training stream)."""
    times = []
    for i in range(reps):
        tok = eng.step_packed(bufs[(done + i) % len(bufs)])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        tok[0].synchronize()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e-3)
    return float(np.median(times)), done + reps


def snapshot_cost(eng, tex, tey, bufs, done):
    eng.arm_eval(tex, tey)
    live, done = _event_median(eng, bufs, done, eng.enqueue_eval)
    eng.arm_eval(tex, tey, snapshot=True)
    snap, done = _event_median(eng, bufs, done, eng.enqueue_eval)
    attempts, done = _event_median(eng, bufs, done, lambda: eng._launch_snapshot(eng.SNAP_ATTEMPTS))
    eng.eval_records()
    st = eng.eval_snapshot_stats()
    eng._leave_native_runner()
    arena = eng.spec.arena_numel
    bf = sum(e - b for b, e in zip(eng._snap_bf_ranges[0::2], eng._snap_bf_ranges[1::2]))
    return {"pass_live_us": live * 1e6, "pass_snapshot_us": snap * 1e6, "snapshot_attempts_us": attempts * 1e6,
            "snapshot_share_of_pass": (snap - live) / snap, "bytes_read": 4 * arena, "bytes_written_f32": 4 * arena,
            "bytes_written_bf16": 2 * bf, "stats": st}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--snapshot", action="store_true", help="also measure the weight snapshot of --eval_snapshot")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("eval_overhead.py measures on a GPU; none found")
    B = a.batch
    eng = gpu_timing.one_replica_engine(
        "lenet", B, 0, lambda be: SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 10 ** 6, 1.0), 1, 1))
    trx, try_, tex, tey = make_synthetic_mnist(B * 16, 10000, seed=5)
    eng.arm_eval(tex, tey)
    bufs = [eng.pack_batch(trx[i * B:(i + 1) * B], try_[i * B:(i + 1) * B]) for i in range(16)]
    done = 0
    for e in (0, 20):                                   # warm-up: graphs, native runner, eval graph
        window(eng, bufs, 200, e, done)
        done += 200
    configs = (0, 100, 20)
    t_step = {e: [] for e in configs}
    stamps = []
    for _ in range(a.rounds):
        for e in configs:
            # start every window on a multiple of 100 steps so each E sees steps / E passes
            done += (-done) % 100
            t, recs = window(eng, bufs, a.steps, e, done)
            done += a.steps
            t_step[e].append(t)
            stamps += [(r[2] - r[1]) * 1e-9 for r in recs]
    # one pass between two steps, bracketed by CUDA events on the training stream
    ev_times = []
    for _ in range(20):
        tok = eng.step_packed(bufs[done % len(bufs)])
        done += 1
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.enqueue_eval()
        e1.record()
        tok[0].synchronize()
        torch.cuda.synchronize()
        ev_times.append(e0.elapsed_time(e1) * 1e-3)
    eng._leave_native_runner()
    eng.backend.check_error()
    base = float(np.mean(t_step[0]))
    t_eval = float(np.median(stamps)) if stamps else float("nan")
    res = dict(gpu_timing.card(), batch=B, steps_per_window=a.steps, rounds=a.rounds, eval_examples=10000,
               step_us={("off" if e == 0 else "E=%d" % e): {"mean": float(np.mean(v)) * 1e6, "min": float(np.min(v)) * 1e6,
                                                          "max": float(np.max(v)) * 1e6} for e, v in t_step.items()},
               eval_pass_us={"globaltimer_median": t_eval * 1e6, "globaltimer_min": float(np.min(stamps)) * 1e6,
                             "globaltimer_max": float(np.max(stamps)) * 1e6, "passes": len(stamps),
                             "cuda_events_median": float(np.median(ev_times)) * 1e6},
               overhead={})
    for e in (100, 20):
        res["overhead"]["E=%d" % e] = {"implied": t_eval / (e * base), "measured": float(np.mean(t_step[e])) / base - 1.0,
                                       "measured_min": float(np.min(t_step[e])) / float(np.max(t_step[0])) - 1.0,
                                       "measured_max": float(np.max(t_step[e])) / float(np.min(t_step[0])) - 1.0}
    if a.snapshot:
        res["snapshot"] = snapshot_cost(eng, tex, tey, bufs, done)
        eng.backend.check_error()
    gpu_timing.emit(res, a.out)


if __name__ == "__main__":
    main()
