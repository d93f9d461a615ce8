#!/usr/bin/env python
"""Cost and benefit of ``--moving_average_decay`` on one GPU.  Prints one JSON line.

1. Step time with and without the average: each configuration in a process of its own, alternated for ``--rounds`` rounds.
   A process builds the engine (K = N = 1), replays ``--warmup`` steps, then times ``--steps`` back-to-back steps from a
   device-resident packed batch with CUDA events around the whole window.  Configurations: lenet at batch 256, and mlp3 at
   batch 8192 / hidden 4096 (an arena of about 20 M floats).
2. The update kernel alone on each arena (CUDA events over 200 launches): the update, the update plus the bf16 copy of
   lenet's conv2 / fc1 ranges, and that copy alone (what an averaged evaluation pass runs first).
3. Time to accuracy at K = N on one GPU, scoring the live weights versus the averaged ones: ``train()`` with the data, the
   target and the evaluation period of ``tools/time_to_accuracy.py``, alternated for ``--rounds`` rounds.

    python tools/moving_average.py [--rounds 3] [--decay 0.999] [--target 0.95] [--out results/moving_average.json]
"""
import argparse
import json
import os
import tempfile

import gpu_timing
import torch
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
from distributedmnist_b200.schedule import LearningRateSchedule

STEP_CONFIGS = [("lenet", 256, 1024), ("mlp3", 8192, 4096)]


def child_step_time(model, batch, hidden, decay, steps, warmup):
    eng = gpu_timing.one_replica_engine(
        model, batch, hidden, lambda be: SyncReplicasOptimizer(be, LearningRateSchedule(0.01, 10 ** 6, 1.0), 1, 1))
    if decay:
        eng.arm_moving_average(decay)
    packed = gpu_timing.packed_batches(eng, 2, 1, on_device=True)
    gpu_timing.timed_steps(eng, packed, warmup)
    us = gpu_timing.timed_steps(eng, packed, steps)
    eng.backend.check_error()
    eng._leave_native_runner()
    return dict(model=model, batch=batch, hidden=hidden if model != "lenet" else None, average=bool(decay),
                arena_floats=eng.spec.arena_numel, launches_per_step=eng.launches_per_step, us_per_step=us)


def kernel_times(iters=200):
    from distributedmnist_b200.models import get_model
    from distributedmnist_b200.ops.lib import load, stream_ptr
    lib = load()
    out = []
    for model, hidden in (("lenet", 1024), ("mlp3", 4096)):
        spec = get_model(model, hidden)[0]
        n = spec.arena_numel
        s, w = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
        bf = torch.zeros(n, dtype=torch.bfloat16, device="cuda")
        epoch = torch.full((1,), 1000, dtype=torch.int32, device="cuda")
        rg = [0, 0, 0, 0]
        if model == "lenet":
            rg = []
            for name in ("conv2_weights", "fc1_weights"):
                q = spec.param(name)
                rg += [q.offset, q.offset + q.numel]
        variants = {"update": (w, None, [0, 0, 0, 0]), "update_bf16": (w, bf, rg), "bf16_only": (None, bf, rg)}
        row = dict(model=model, arena_floats=n)
        for name, (wp, bp, r) in variants.items():
            if model != "lenet" and name != "update":
                continue

            def launch():
                lib.dm_moving_average(s, wp, n, epoch, 0.999, None, bp, *r, stream_ptr())
            for _ in range(10):
                launch()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(iters):
                launch()
            t1.record()
            torch.cuda.synchronize()
            us = t0.elapsed_time(t1) * 1e3 / iters
            nbytes = n * 12 if name == "update" else (n * 12 + (rg[1] - rg[0] + rg[3] - rg[2]) * 2 if name == "update_bf16"
                                                      else n * 4 + (rg[1] - rg[0] + rg[3] - rg[2]) * 2)
            row[name + "_us"] = us
            row[name + "_gbps"] = nbytes / us * 1e-3
        out.append(row)
    return out


def tta_run(ds, args, average: bool) -> dict:
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import train
    FLAGS.reset()
    with tempfile.TemporaryDirectory() as d:
        FLAGS.parse(["--train_dir=%s" % d, "--batch_size=128", "--max_steps=%d" % args.max_steps, "--model=lenet",
                     "--device_data=true", "--eval_every_steps=%d" % args.eval_every, "--target_accuracy=%r" % args.target,
                     "--initial_learning_rate=0.05", "--log_every=100000", "--save_results_period=100000000",
                     "--save_interval_secs=1e9", "--moving_average_decay=%r" % args.decay]
                    + (["--eval_moving_average=true"] if average else []))
        ctx = init_context(FLAGS)
        res = train(ctx, ds.train, ds.validation, FLAGS)
    rep = res["time_to_accuracy"]
    return dict(weights="moving_average" if average else "live", reached=rep["reached"], global_step=rep["global_step"],
                accuracy=rep["accuracy"], train_time_s=rep["train_time_s"], wall_time_s=rep["wall_time_s"],
                final_step=res["final_step"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--decay", type=float, default=0.999)
    ap.add_argument("--target", type=float, default=0.95)
    ap.add_argument("--eval-every", type=int, default=20)
    ap.add_argument("--max-steps", type=int, default=5000)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    if args.child:
        model, batch, hidden, decay = args.child.split(":")
        print(json.dumps(child_step_time(model, int(batch), int(hidden), float(decay), args.steps, args.warmup)))
        return
    steps = [gpu_timing.child_json([__file__, "--steps=%d" % args.steps, "--warmup=%d" % args.warmup,
                                    "--child=%s:%d:%d:%r" % (model, batch, hidden, decay)])
             for _ in range(args.rounds) for model, batch, hidden in STEP_CONFIGS for decay in (0.0, args.decay)]
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.flags import FLAGS
    kern = kernel_times()
    FLAGS.reset()
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True)
    tta = []
    for _ in range(args.rounds):
        for average in (False, True):
            tta.append(tta_run(ds, args, average))
    out = dict(tool="moving_average", decay=args.decay, step_time=steps, kernel=kern,
               time_to_accuracy=dict(data="synthetic MNIST-shaped (not MNIST)", target=args.target, batch_size=128,
                                     eval_every_steps=args.eval_every, runs=tta), **gpu_timing.card())
    gpu_timing.emit(out, args.out)


if __name__ == "__main__":
    main()
