#!/usr/bin/env python
"""Cost of checkpoints to the training step on one GPU, synthetic data.  Prints one JSON line.

The training loop is driven as ``train.py``'s pipelined loop drives it (see tools/eval_overhead.py): ``step_packed`` (native
runner, one CUDA graph per step), the host waiting for step i while step i+1 is queued.  Step time is device time: CUDA
events around a window of steps, divided by the steps.  A checkpoint is taken after every E-th step, E = off, 100 and 20,
in two ways that alternate over several rounds:

  capture  the device capture of the sm_90a engine (``enqueue_checkpoint``, K = N: a copy of the live arena), polled with an
           event query at every later step, as ``train._AsyncCheckpointer`` does;
  drain    the drain-and-copy it replaced: ``torch.cuda.synchronize()`` and ``spec.to_state_dict(params)`` (device -> host
           copy) on the training thread.

Neither writes a file: that happens on the saver thread in both.  The capture alone is also timed with CUDA events between
two steps, for the live capture and for the snapshot capture of K != N runs (quiescent weights: the first attempt is
accepted, the other three exit at once).

    python tools/ckpt_overhead.py [--steps 2000] [--rounds 3] [--batch 256] [--out results/ckpt_overhead.json]
"""
import argparse
import sys

import gpu_timing
import numpy as np
import torch
from distributedmnist_b200.data import make_synthetic_mnist
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
from distributedmnist_b200.schedule import LearningRateSchedule


class _Capture:
    """The checkpointer's device mode without the file IO: at most one capture in flight, polled at every step."""

    def __init__(self, eng):
        self.eng, self.pending, self.buf, self.landed = eng, False, 0, 0

    def poll(self):
        if self.pending and self.eng.checkpoint_poll() is not None:
            self.pending = False
            self.landed += 1

    def save(self):
        if not self.pending:
            self.eng.enqueue_checkpoint(self.buf)
            self.buf ^= 1
            self.pending = True

    def finish(self):
        if self.pending and self.eng.checkpoint_wait() is not None:
            self.pending = False
            self.landed += 1


def window(eng, bufs, steps, every, first, how):
    """Device time per step over `steps` steps with a checkpoint after every `every`-th (0: none)."""
    cap = _Capture(eng)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    pending = None
    e0.record()
    for i in range(steps):
        tok = eng.step_packed(bufs[(first + i) % len(bufs)])
        if pending is not None:
            pending[0].synchronize()
        pending = tok
        if how == "capture":
            cap.poll()
        if every and (first + i + 1) % every == 0:
            if how == "capture":
                cap.save()
            else:
                torch.cuda.synchronize()
                eng.spec.to_state_dict(eng.params)
    e1.record()
    torch.cuda.synchronize()
    cap.finish()
    return e0.elapsed_time(e1) * 1e-3 / steps, cap.landed


def capture_alone(eng, bufs, done, snapshot, reps=20):
    """Median device time of one capture enqueued between two training steps: what it puts on the training stream (CUDA
    events on that stream) and until its arena has landed in host memory (the second event on the capture's copy stream)."""
    eng.arm_checkpoint(snapshot=snapshot)
    on_stream, landed = [], []
    for _ in range(reps):
        tok = eng.step_packed(bufs[done % len(bufs)])
        done += 1
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        eng.enqueue_checkpoint(0)
        e1.record()
        e2.record(eng._ck_stream)
        tok[0].synchronize()
        eng.checkpoint_wait()
        torch.cuda.synchronize()
        on_stream.append(e0.elapsed_time(e1) * 1e-3)
        landed.append(e0.elapsed_time(e2) * 1e-3)
    return {"on_training_stream_us": float(np.median(on_stream)) * 1e6, "until_landed_us": float(np.median(landed)) * 1e6}, done


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ckpt_overhead.py measures on a GPU; none found")
    B = a.batch
    eng = gpu_timing.one_replica_engine(
        "lenet", B, 0, lambda be: SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 10 ** 6, 1.0), 1, 1))
    eng.arm_checkpoint(snapshot=False)
    trx, try_, _tex, _tey = make_synthetic_mnist(B * 16, 16, seed=5)
    bufs = [eng.pack_batch(trx[i * B:(i + 1) * B], try_[i * B:(i + 1) * B]) for i in range(16)]
    done = 0
    for how in ("capture", "drain"):                    # warm-up: graphs, native runner, both checkpoint paths
        window(eng, bufs, 200, 20, done, how)
        done += 200
    configs = [(0, "capture"), (100, "capture"), (100, "drain"), (20, "capture"), (20, "drain")]
    t_step = {c: [] for c in configs}
    landed = 0
    for _ in range(a.rounds):
        for every, how in configs:
            done += (-done) % 100                       # every window starts on a multiple of 100 steps
            t, n = window(eng, bufs, a.steps, every, done, how)
            done += a.steps
            t_step[(every, how)].append(t)
            landed += n
    live, done = capture_alone(eng, bufs, done, snapshot=False)
    snap, done = capture_alone(eng, bufs, done, snapshot=True)
    snap["stats"] = eng.checkpoint_stats()
    eng._leave_native_runner()
    eng.backend.check_error()
    base = float(np.mean(t_step[(0, "capture")]))

    def name(c):
        return "off" if c[0] == 0 else "E=%d_%s" % c
    res = dict(gpu_timing.card(), batch=B, steps_per_window=a.steps, rounds=a.rounds, arena_bytes=4 * eng.spec.arena_numel,
               captures_landed=landed,
               step_us={name(c): {"mean": float(np.mean(v)) * 1e6, "min": float(np.min(v)) * 1e6,
                                  "max": float(np.max(v)) * 1e6} for c, v in t_step.items()},
               overhead={name(c): float(np.mean(v)) / base - 1.0 for c, v in t_step.items() if c[0]},
               capture_live=live, capture_snapshot=snap)
    gpu_timing.emit(res, a.out)


if __name__ == "__main__":
    main()
