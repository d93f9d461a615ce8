#!/usr/bin/env python
"""Cost of ``--weight_decay`` on one GPU (lenet, batch 256, K = N = 1).  Prints one JSON line.

1. Step time with lambda = 0 and lambda = 5e-4: each in a process of its own, alternated for ``--rounds`` rounds.  A process
   builds the engine, replays ``--warmup`` steps, then times ``--steps`` back-to-back steps from a device-resident packed
   batch with CUDA events around the whole window.
2. The fc1 weight-gradient GEMM alone, plain and decayed, fp32 and bf16 stores (CUDA events over ``--iters`` launches,
   the variants alternated in blocks), and the fc2_wgrad kernel plain and decayed.  These are eager launches: for kernels
   of about 10 us the host's launch rate bounds them as much as the kernel does.
3. The card's name and power limit, read in the same call.

    python tools/weight_decay.py [--rounds 3] [--lam 5e-4] [--out results/weight_decay.json]
"""
import argparse
import json
import os

import gpu_timing
import torch
from distributedmnist_b200.ops import gemm as G
from distributedmnist_b200.ops.lib import load, stream_ptr
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
from distributedmnist_b200.schedule import LearningRateSchedule

B = 256


def child_step_time(lam, steps, warmup):
    eng = gpu_timing.one_replica_engine(
        "lenet", B, 0, lambda be: SyncReplicasOptimizer(be, LearningRateSchedule(0.01, 10 ** 6, 1.0), 1, 1))
    if lam:
        eng.arm_weight_decay(lam)
    packed = gpu_timing.packed_batches(eng, 2, 1, on_device=True)
    gpu_timing.timed_steps(eng, packed, warmup)
    us = gpu_timing.timed_steps(eng, packed, steps)
    eng.backend.check_error()
    eng._leave_native_runner()
    return dict(lam=lam, launches_per_step=eng.launches_per_step, us_per_step=us)


def kernel_times(lam, iters, blocks=5):
    lib = load()
    g = torch.Generator().manual_seed(2)
    a2 = torch.rand(B, 3136, generator=g).to(torch.bfloat16).cuda()
    dh = (torch.randn(B, 512, generator=g) * 0.01).to(torch.bfloat16).cuda()
    w = (torch.randn(3136, 512, generator=g) * 0.1).cuda()
    o32 = torch.empty(3136, 512, device="cuda")
    o16 = torch.empty(3136, 512, dtype=torch.bfloat16, device="cuda")
    ws = torch.zeros(int(lib.dm_gemm_decay_ctas(3136, 512)) + 64, dtype=torch.float64, device="cuda")
    h = torch.relu(torch.randn(B, 512, generator=g)).cuda()
    dl = (torch.randn(B, 12, generator=g) * 0.01).cuda()
    w2, b2, b1 = torch.randn(512, 10, device="cuda"), torch.randn(10, device="cuda"), torch.randn(512, device="cuda")
    gw2, gb2, gb1 = torch.empty_like(w2), torch.empty_like(b2), torch.empty_like(b1)
    sp = stream_ptr()
    variants = {
        "fc1_wgrad_f32": lambda: G.gemm_bf16_raw(a2, dh, o32, 3136, 512, B, 3136, 512, 512, True, True, G.EPI_STORE_F32),
        "fc1_wgrad_f32_decay": lambda: lib.dm_gemm_bf16_decay(a2, dh, o32, 3136, 512, B, 3136, 512, 512, 0, w, lam, ws, sp),
        "fc1_wgrad_bf16": lambda: G.gemm_bf16_raw(a2, dh, o16, 3136, 512, B, 3136, 512, 512, True, True, G.EPI_STORE_BF16),
        "fc1_wgrad_bf16_decay": lambda: lib.dm_gemm_bf16_decay(a2, dh, o16, 3136, 512, B, 3136, 512, 512, 1, w, lam, ws, sp),
        "fc2_wgrad": lambda: lib.dm_fc2_wgrad(h, dl, dh, gw2, gb2, gb1, B, sp),
        "fc2_wgrad_decay": lambda: lib.dm_fc2_wgrad_decay(h, dl, dh, gw2, gb2, gb1, B, w2, b2, b1, lam, ws, sp),
    }
    tot = {k: 0.0 for k in variants}
    for fn in variants.values():
        for _ in range(20):
            fn()
    torch.cuda.synchronize()
    for _ in range(blocks):
        for name, fn in variants.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(iters):
                fn()
            t1.record()
            torch.cuda.synchronize()
            tot[name] += t0.elapsed_time(t1) * 1e3 / iters / blocks
    return {k + "_us": v for k, v in tot.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3000)
    ap.add_argument("--warmup", type=int, default=300)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--lam", type=float, default=5e-4)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    if args.child is not None:
        print(json.dumps(child_step_time(float(args.child), args.steps, args.warmup)))
        return
    steps = [gpu_timing.child_json([__file__, "--steps=%d" % args.steps, "--warmup=%d" % args.warmup, "--child=%r" % lam])
             for _ in range(args.rounds) for lam in (0.0, args.lam)]
    out = dict(tool="weight_decay", model="lenet", batch=B, lam=args.lam, step_time=steps,
               kernel=kernel_times(args.lam, args.iters), **gpu_timing.card())
    gpu_timing.emit(out, args.out)


if __name__ == "__main__":
    main()
