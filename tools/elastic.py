#!/usr/bin/env python
"""Cost of elastic distortion (``--augment_elastic_alpha`` / ``_sigma``) on one GPU, beside random affine augmentation.
Prints one JSON line.

1. Device-timed step time of three engines per configuration: augmentation off, affine only (2 px, 15 degrees, 0.1) and
   affine + elastic (alpha 34, sigma 4), for lenet at B = 256 and mlp3 at B = 8192, H = 4096 (K = N = 1).  The three
   engines live in one process; after ``--warmup`` steps of each, ``--rounds`` windows of ``--steps`` back-to-back
   graph-replayed steps alternate between them, each window timed with CUDA events around it.
2. augment_elastic and augment_affine alone (CUDA events over ``--iters`` eager launches, after a warm-up) at B = 256
   and B = 8192, with the double FMAs of the two field passes per launch.
3. The card's name and power limit, read in the same call.

    python tools/elastic.py [--rounds 5] [--out results/elastic.json]
"""
import argparse
import ctypes
import os

import gpu_timing
import torch
from distributedmnist_b200 import augment
from distributedmnist_b200.ops.lib import load, stream_ptr
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
from distributedmnist_b200.schedule import LearningRateSchedule

RANGES = (2.0, 15.0, 0.1)                  # shift px, rotation degrees, zoom
ALPHA, SIGMA = 34.0, 4.0
CONFIGS = ("off", "affine", "elastic")


def _engine(model, B, hidden, config):
    eng = gpu_timing.one_replica_engine(
        model, B, hidden, lambda be: SyncReplicasOptimizer(be, LearningRateSchedule(0.01, 10 ** 6, 1.0), 1, 1))
    if config != "off":
        eng.arm_augment(*RANGES, elastic=augment.Elastic(ALPHA, SIGMA) if config == "elastic" else None)
    return eng, gpu_timing.packed_batches(eng, 2, 1, on_device=True)


def _median(v):
    return sorted(v)[len(v) // 2]


def step_times(model, B, hidden, rounds, steps, warmup):
    engines = {k: _engine(model, B, hidden, k) for k in CONFIGS}
    us = gpu_timing.alternate(engines, steps, warmup, rounds)
    out = dict(model=model, batch=B, hidden=hidden if model != "lenet" else None)
    for k, (eng, _p) in engines.items():
        eng.backend.check_error()
        eng._leave_native_runner()
        out["launches_per_step_" + k] = eng.launches_per_step
        out["us_per_step_" + k] = us[k]
        out["median_%s_us" % k] = _median(us[k])
    for k in ("affine", "elastic"):
        out["cost_%s_pct" % k] = 100.0 * (out["median_%s_us" % k] / out["median_off_us"] - 1.0)
    return out


def kernel_time(B, iters):
    lib = load()
    src = torch.rand(B, 784, device="cuda") - 0.5
    dst = torch.empty_like(src)
    ctr = torch.zeros(2, dtype=torch.int32, device="cuda")
    mix, sp = augment.seed_mix(66478, 0), stream_ptr()
    w = augment.gaussian_weights(SIGMA)
    taps = (ctypes.c_double * len(w))(*w)
    R = len(w) - 1

    def elastic():
        lib.dm_augment_elastic(src, dst, B, ctr, mix, *RANGES, ALPHA, taps, R, None, None, sp)

    def affine():
        lib.dm_augment_affine(src, dst, B, ctr, mix, *RANGES, None, sp)

    out = dict(batch=B)
    for name, launch in (("elastic", elastic), ("affine", affine)):
        out[name + "_us"] = gpu_timing.timed_launches(launch, iters, 50)
    # taps inside the image per output, summed over the 28 positions of a line: both passes, both components
    taps_per_line = sum(min(R, 27 - p) + min(R, p) + 1 for p in range(28))
    out["dfma_per_launch"] = B * 2 * 2 * 28 * taps_per_line
    out["dfma_per_s"] = out["dfma_per_launch"] / out["elastic_us"] * 1e6
    return out


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
    out = dict(tool="elastic", ranges=dict(zip(("max_shift", "max_rotation", "max_scale"), RANGES)),
               elastic=dict(alpha=ALPHA, sigma=SIGMA), **gpu_timing.card())
    out["kernel"] = [kernel_time(B, args.iters) for B in (256, 8192)]
    out["step_time"] = [step_times("lenet", 256, 0, args.rounds, args.steps, args.warmup),
                        step_times("mlp3", 8192, 4096, args.rounds, args.mlp_steps, args.warmup // 10)]
    gpu_timing.emit(out, args.out)


if __name__ == "__main__":
    main()
