#!/usr/bin/env python
"""Cost of the learning-rate warmup and cosine decay (``--lr_warmup_steps``, ``--lr_cosine_decay_steps``) on one GPU,
lenet, synthetic data.  Prints one JSON line.

Blocks of graph-replayed training steps (the pipelined loop's native runner) are bracketed by CUDA events, the three
configurations alternating block by block in the same call so that they share the same conditions:

  off       no schedule in the control block: the staircase decay, as before;
  warmup    a warmup longer than the run, so every step's aggregation kernels evaluate the warmup factor;
  cosine    warmup and cosine decay both longer than the run: every step evaluates the double sin and the warmup.

The step graph is the same in all three; only the control block's schedule words change between blocks.

    python tools/lr_schedule.py [--blocks 40] [--block-steps 50] [--batch 256] [--out results/lr_schedule.json]
"""
import argparse
import sys

import gpu_timing
import numpy as np
import torch
from distributedmnist_b200.data import make_synthetic_mnist
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
from distributedmnist_b200.schedule import LearningRateSchedule

LONG = 2 ** 31                     # steps: longer than any run of this tool
CONFIGS = {"off": (0, 1.0 / 3, 0, 0.0), "warmup": (LONG, 0.1, 0, 0.0), "cosine": (LONG, 0.1, LONG, 0.01)}


def _stats(v):
    return {"median": float(np.median(v)) * 1e6, "min": float(np.min(v)) * 1e6, "max": float(np.max(v)) * 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=40, help="timed step blocks per configuration")
    ap.add_argument("--block-steps", type=int, default=50, help="training steps per block")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("lr_schedule.py measures on a GPU; none found")
    B = a.batch
    eng = gpu_timing.one_replica_engine(
        "lenet", B, 0, lambda be: SyncReplicasOptimizer(be, LearningRateSchedule(0.01, 10 ** 6, 1.0), 1, 1))
    be = eng.backend
    trx, try_, _tex, _tey = make_synthetic_mnist(B * 16, 100, seed=5)
    bufs = [eng.pack_batch(trx[i * B:(i + 1) * B], try_[i * B:(i + 1) * B]) for i in range(16)]
    names = list(CONFIGS)
    step_s = {k: [] for k in names}
    done = 0
    for i in range(len(names) * (a.blocks + 2)):            # the first 2 blocks of each configuration warm up
        name = names[i % len(names)]
        torch.cuda.synchronize()
        be.set_lr_schedule(*CONFIGS[name])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.block_steps):
            tok = eng.step_packed(bufs[done % len(bufs)])
            done += 1
        e1.record()
        tok[0].synchronize()
        torch.cuda.synchronize()
        if i >= 2 * len(names):
            step_s[name].append(e0.elapsed_time(e1) * 1e-3 / a.block_steps)
    eng._leave_native_runner()
    be.check_error()
    be.set_lr_schedule(*CONFIGS["off"])

    ms = {k: float(np.median(v)) for k, v in step_s.items()}
    res = dict(gpu_timing.card(), batch=B, step_blocks_per_config=a.blocks, steps_per_block=a.block_steps,
               step_us={k: _stats(v) for k, v in step_s.items()},
               images_per_s={k: B / v for k, v in ms.items()},
               step_added_us={k: (ms[k] - ms["off"]) * 1e6 for k in names if k != "off"},
               step_added_share={k: ms[k] / ms["off"] - 1.0 for k in names if k != "off"})
    gpu_timing.emit(res, a.out)


if __name__ == "__main__":
    main()
