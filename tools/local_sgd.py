#!/usr/bin/env python
"""Device time of a local-SGD step (--local_sgd_steps) against the default K = N path, LeNet at B = 256, on the GPUs of
this machine.  The card's name, power limit and max SM clock are recorded next to the numbers.

For each H in {1, 4, 16}, and for K = N, blocks of graph-replayed steps are timed with CUDA events after a warm-up; the
modes alternate block by block, so a drift of the clocks spreads over all of them.  The local step and the averaging step
are timed apart: a block of steps that never average (the averaging period set past the block) and a block of averaging
steps only (H = 1).  With several GPUs every replica runs in its own process and the numbers are rank 0's.

    python tools/local_sgd.py [--gpus 1] [--steps 2000] [--warmup 300] [--repeats 5] [--out results/local_sgd.json]
"""
import gpu_timing
from distributedmnist_b200.parallel.aggregators import LocalSGDOptimizer, SyncReplicasOptimizer

MODES = {
    "k_eq_n": lambda be, sched, n: SyncReplicasOptimizer(be, sched, n, n),
    "local_step": lambda be, sched, n: LocalSGDOptimizer(be, sched, n, period=1 << 30),
    "average_step": lambda be, sched, n: LocalSGDOptimizer(be, sched, n, period=1),
    "H4": lambda be, sched, n: LocalSGDOptimizer(be, sched, n, period=4),
    "H16": lambda be, sched, n: LocalSGDOptimizer(be, sched, n, period=16),
}

if __name__ == "__main__":
    gpu_timing.compare_modes(MODES)
