#!/usr/bin/env python
"""Cost of random affine augmentation (``--augment_max_*``) on one GPU.  Prints one JSON line.

1. Device-timed step time with augmentation off and on, for lenet at B = 256 and mlp3 at B = 8192, H = 4096 (K = N = 1).
   Both engines of a configuration live in one process; after ``--warmup`` steps of each, ``--rounds`` windows of
   ``--steps`` back-to-back graph-replayed steps alternate between them, each window timed with CUDA events around it.
2. augment_affine alone (CUDA events over ``--iters`` eager launches, after a warm-up) at B = 256 and B = 8192, with the
   bytes one launch moves (the B x 784 fp32 images read and written) and the resulting rate.
3. The card's name and power limit, read in the same call.

    python tools/augment.py [--rounds 5] [--out results/augment.json]
"""
import argparse
import os

import gpu_timing
import torch
from distributedmnist_b200 import augment
from distributedmnist_b200.ops.lib import load, stream_ptr
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
from distributedmnist_b200.schedule import LearningRateSchedule

RANGES = (2.0, 15.0, 0.1)                  # shift px, rotation degrees, zoom


def _engine(model, B, hidden, on):
    eng = gpu_timing.one_replica_engine(
        model, B, hidden, lambda be: SyncReplicasOptimizer(be, LearningRateSchedule(0.01, 10 ** 6, 1.0), 1, 1))
    if on:
        eng.arm_augment(*RANGES)
    return eng, gpu_timing.packed_batches(eng, 2, 1, on_device=True)


def step_times(model, B, hidden, rounds, steps, warmup):
    engines = {k: _engine(model, B, hidden, k == "on") for k in ("off", "on")}
    us = gpu_timing.alternate(engines, steps, warmup, rounds)
    out = dict(model=model, batch=B, hidden=hidden if model != "lenet" else None)
    for k, (eng, _p) in engines.items():
        eng.backend.check_error()
        eng._leave_native_runner()
        out["launches_per_step_" + k] = eng.launches_per_step
        out["us_per_step_" + k] = us[k]
    out["median_off_us"] = sorted(us["off"])[len(us["off"]) // 2]
    out["median_on_us"] = sorted(us["on"])[len(us["on"]) // 2]
    out["cost_pct"] = 100.0 * (out["median_on_us"] / out["median_off_us"] - 1.0)
    return out


def kernel_time(B, iters):
    lib = load()
    src = torch.rand(B, 784, device="cuda") - 0.5
    dst = torch.empty_like(src)
    ctr = torch.zeros(2, dtype=torch.int32, device="cuda")
    mix, sp = augment.seed_mix(66478, 0), stream_ptr()

    def launch():
        lib.dm_augment_affine(src, dst, B, ctr, mix, *RANGES, None, sp)

    us = gpu_timing.timed_launches(launch, iters, 50)
    nbytes = 2 * B * 784 * 4
    return dict(batch=B, us=us, bytes_per_launch=nbytes, gb_per_s=nbytes / us * 1e-3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--mlp_steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    torch.cuda.set_device(0)
    out = dict(tool="augment", ranges=dict(zip(("max_shift", "max_rotation", "max_scale"), RANGES)), **gpu_timing.card())
    out["kernel"] = [kernel_time(B, args.iters) for B in (256, 8192)]
    out["step_time"] = [step_times("lenet", 256, 0, args.rounds, args.steps, args.warmup),
                        step_times("mlp3", 8192, 4096, args.rounds, args.mlp_steps, args.warmup // 10)]
    gpu_timing.emit(out, args.out)


if __name__ == "__main__":
    main()
