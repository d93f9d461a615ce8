#!/usr/bin/env python
"""Device time of a gossip-SGD step (--gossip_method) against the default K = N path and --local_sgd_steps=1, LeNet at
B = 256, on the GPUs of this machine.  The card's name and power limit are recorded next to the numbers.

For each mode blocks of graph-replayed steps are timed with CUDA events after a warm-up; the modes alternate block by
block, so a drift of the clocks spreads over all of them.  With several GPUs every replica runs in its own process and the
numbers are rank 0's.

    python tools/gossip_sgd.py [--gpus 1] [--steps 2000] [--warmup 300] [--repeats 5] [--out results/gossip_sgd.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def worker(steps: int, warmup: int, repeats: int) -> dict:
    sys.path.insert(0, ROOT)
    import torch
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.aggregators import GossipSGDOptimizer, LocalSGDOptimizer, SyncReplicasOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext, init_context
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.schedule import LearningRateSchedule
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        FLAGS.parse([])
        ctx = init_context(FLAGS, want_gpu=True)
    else:
        torch.cuda.set_device(0)
        ctx = ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none")
    n = ctx.world_size
    engines = {}
    sched = LearningRateSchedule(0.01, 1000, 0.95)
    # one engine per mode, each with its own arenas and control block, so the modes can alternate without re-capturing
    for mode in ("k_eq_n", "local_H1", "gossip"):
        be = FusedBackend(ctx)
        eng = CudaLeNetEngine(256, be, use_graph=True)
        if mode == "k_eq_n":
            opt = SyncReplicasOptimizer(be, sched, n, n)
        elif mode == "local_H1":
            opt = LocalSGDOptimizer(be, sched, n, period=1)
        else:
            opt = GossipSGDOptimizer(be, sched, n)
        eng.attach_optimizer(opt)
        engines[mode] = (be, eng)
    gen = torch.Generator().manual_seed(1 + ctx.rank)
    bufs = {m: [e.pack_batch(torch.rand(256, 784, generator=gen) - 0.5, torch.randint(0, 10, (256,), generator=gen))
                for _ in range(4)] for m, (_, e) in engines.items()}

    def block(mode, k):
        be, eng = engines[mode]
        be.device_barrier()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(k):
            eng.step_packed(bufs[mode][i % 4])
        b.record()
        b.synchronize()
        return a.elapsed_time(b) * 1e3 / k

    for mode in engines:
        block(mode, warmup)
    us = {m: [] for m in engines}
    for _ in range(repeats):
        for mode in engines:
            us[mode].append(block(mode, steps))
    for be, eng in engines.values():
        torch.cuda.synchronize()
        be.check_error()
    return dict(replicas=n, us_per_step=us, launches_per_step={m: e.launches_per_step for m, (_, e) in engines.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=300)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default="")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        res = worker(a.steps, a.warmup, a.repeats)
        if int(os.environ.get("RANK", "0")) == 0:
            print(json.dumps(res), flush=True)
        return
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    cmd = [os.path.abspath(__file__), "--worker", "--steps", str(a.steps), "--warmup", str(a.warmup), "--repeats",
           str(a.repeats)]
    if a.gpus > 1:
        sys.path.insert(0, ROOT)
        import tempfile
        from distributedmnist_b200.parallel.launcher import run_replicas
        with tempfile.TemporaryDirectory() as d:
            codes = run_replicas(cmd, a.gpus, timeout=1800, out_dir=d)
            text = open(os.path.join(d, sorted(os.listdir(d))[0])).read()
        if codes != [0] * a.gpus:
            raise SystemExit("a replica failed: %s" % codes)
    else:
        text = subprocess.run([sys.executable] + cmd, capture_output=True, text=True, check=True).stdout
    res = json.loads([l for l in text.splitlines() if l.startswith("{")][-1])
    out = dict(gpu=q[0] if q else "unknown", model="lenet", batch=256, **res)
    med = {m: sorted(v)[len(v) // 2] for m, v in res["us_per_step"].items()}
    out["median_us_per_step"] = med
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
