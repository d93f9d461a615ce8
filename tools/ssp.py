#!/usr/bin/env python
"""Step-time cost of the staleness bound (--ssp_staleness): plain asynchronous SGD against s = 0, LeNet at B = 256 on one
replica, in one process, the two engines' blocks of graph-replayed steps alternated (CUDA events around each block).  One
replica never waits, so the difference is the cost of the two 1-warp kernels the bound adds to every step.  The card's
name and power limit are printed next to the numbers.

    python tools/ssp.py [--steps 3000] [--warmup 300] [--blocks 5] [--out results/ssp.json]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3000)
    ap.add_argument("--warmup", type=int, default=300)
    ap.add_argument("--blocks", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    import torch
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.aggregators import AsyncSGDOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    torch.cuda.set_device(0)
    engines = {}
    gen = torch.Generator().manual_seed(1)
    batches = [(torch.rand(256, 784, generator=gen) - 0.5, torch.randint(0, 10, (256,), generator=gen)) for _ in range(4)]
    for mode, s in (("async", -1), ("ssp_0", 0)):
        be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
        eng = CudaLeNetEngine(256, be, use_graph=True)
        eng.attach_optimizer(AsyncSGDOptimizer(be, LearningRateSchedule(0.01, 1000, 0.95), 1, ssp_staleness=s))
        bufs = [eng.pack_batch(x, y) for x, y in batches]
        for i in range(a.warmup):
            eng.step_packed(bufs[i % 4])
        torch.cuda.synchronize()
        engines[mode] = (eng, be, bufs)
    us = {m: [] for m in engines}
    for _ in range(a.blocks):
        for mode, (eng, be, bufs) in engines.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for i in range(a.steps):
                eng.step_packed(bufs[i % 4])
            t1.record()
            t1.synchronize()
            us[mode].append(t0.elapsed_time(t1) * 1e3 / a.steps)
    rows = []
    for mode, (eng, be, bufs) in engines.items():
        be.check_error()
        rows.append(dict(mode=mode, us_per_step=us[mode], median_us=statistics.median(us[mode]),
                         launches_per_step=eng.launches_per_step))
    st = engines["ssp_0"][0].ssp_stats()
    out = dict(gpu=q[0] if q else "unknown", model="lenet", batch=256, replicas=1, steps_per_block=a.steps,
               results=rows, ssp_waits=st["waits"],
               cost_us=statistics.median(us["ssp_0"]) - statistics.median(us["async"]))
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
