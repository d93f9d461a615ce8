#!/usr/bin/env python
"""Step-time cost of the staleness bound (--ssp_staleness): plain asynchronous SGD against s = 0, LeNet at B = 256 on one
replica, in one process, the two engines' blocks of graph-replayed steps alternated (CUDA events around each block).  One
replica never waits, so the difference is the cost of the two 1-warp kernels the bound adds to every step.  The card's
name, power limit and max SM clock are printed next to the numbers.

    python tools/ssp.py [--steps 3000] [--warmup 300] [--blocks 5] [--out results/ssp.json]
"""
import argparse
import statistics

import gpu_timing
from distributedmnist_b200.parallel.aggregators import AsyncSGDOptimizer
from distributedmnist_b200.schedule import LearningRateSchedule


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3000)
    ap.add_argument("--warmup", type=int, default=300)
    ap.add_argument("--blocks", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    configs = {}
    for mode, s in (("async", -1), ("ssp_0", 0)):
        eng = gpu_timing.one_replica_engine(
            "lenet", 256, 0, lambda be: AsyncSGDOptimizer(be, LearningRateSchedule(0.01, 1000, 0.95), 1, ssp_staleness=s))
        configs[mode] = (eng, gpu_timing.packed_batches(eng, 4, 1, on_device=False))
    us = gpu_timing.alternate(configs, a.steps, a.warmup, a.blocks)
    rows = []
    for mode, (eng, _bufs) in configs.items():
        eng.backend.check_error()
        rows.append(dict(mode=mode, us_per_step=us[mode], median_us=statistics.median(us[mode]),
                         launches_per_step=eng.launches_per_step))
    st = configs["ssp_0"][0].ssp_stats()
    out = dict(gpu_timing.card(), model="lenet", batch=256, replicas=1, steps_per_block=a.steps, results=rows,
               ssp_waits=st["waits"], cost_us=statistics.median(us["ssp_0"]) - statistics.median(us["async"]))
    gpu_timing.emit(out, a.out)


if __name__ == "__main__":
    main()
