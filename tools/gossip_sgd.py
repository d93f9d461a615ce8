#!/usr/bin/env python
"""Device time of a gossip-SGD step (--gossip_method) against the default K = N path and --local_sgd_steps=1, LeNet at
B = 256, on the GPUs of this machine.  The card's name, power limit and max SM clock are recorded next to the numbers.

For each mode blocks of graph-replayed steps are timed with CUDA events after a warm-up; the modes alternate block by
block, so a drift of the clocks spreads over all of them.  With several GPUs every replica runs in its own process and the
numbers are rank 0's.

    python tools/gossip_sgd.py [--gpus 1] [--steps 2000] [--warmup 300] [--repeats 5] [--out results/gossip_sgd.json]
"""
import gpu_timing
from distributedmnist_b200.parallel.aggregators import GossipSGDOptimizer, LocalSGDOptimizer, SyncReplicasOptimizer

MODES = {
    "k_eq_n": lambda be, sched, n: SyncReplicasOptimizer(be, sched, n, n),
    "local_H1": lambda be, sched, n: LocalSGDOptimizer(be, sched, n, period=1),
    "gossip": lambda be, sched, n: GossipSGDOptimizer(be, sched, n),
}

if __name__ == "__main__":
    gpu_timing.compare_modes(MODES)
