#!/usr/bin/env python
"""Step time and time to a target accuracy of asynchronous SGD (--async_method) against the default K = N path and the
single aggregation kernel (DMNIST_BUCKET=0), LeNet at B = 256 on one GPU.  The card's name and power limit are recorded
next to the numbers.

* step time: the device time of blocks of graph-replayed steps, with CUDA events;
* time to accuracy: ``train()`` with ``--device_data``, ``--eval_every_steps`` and ``--target_accuracy`` (what
  ``worker0_time_to_accuracy.json`` reports: the training time on the device clock up to the evaluation that reached the
  target, the passes before it taken out).  The data is the synthetic MNIST-shaped set, so these are not MNIST numbers.

Every measurement runs in a fresh process.

    python tools/async_sgd.py [--steps 3000] [--warmup 300] [--blocks 3] [--target 0.95] [--max-steps 5000]
                              [--eval-every 20] [--out results/async_sgd.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def one(mode: str, steps: int, warmup: int, blocks: int) -> dict:
    sys.path.insert(0, ROOT)
    import torch
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.aggregators import AsyncSGDOptimizer, SyncReplicasOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    torch.cuda.set_device(0)
    be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
    eng = CudaLeNetEngine(256, be, use_graph=True)
    sched = LearningRateSchedule(0.01, 1000, 0.95)
    eng.attach_optimizer(AsyncSGDOptimizer(be, sched, 1) if mode == "async" else SyncReplicasOptimizer(be, sched, 1, 1))
    gen = torch.Generator().manual_seed(1)
    bufs = [eng.pack_batch(torch.rand(256, 784, generator=gen) - 0.5, torch.randint(0, 10, (256,), generator=gen))
            for _ in range(4)]
    for i in range(warmup):
        eng.step_packed(bufs[i % 4])
    torch.cuda.synchronize()
    us = []
    for _ in range(blocks):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(steps):
            eng.step_packed(bufs[i % 4])
        b.record()
        b.synchronize()
        us.append(a.elapsed_time(b) * 1e3 / steps)
    be.check_error()
    return dict(mode=mode, us_per_step=us, launches_per_step=eng.launches_per_step)


def time_to_accuracy(mode: str, target: float, max_steps: int, eval_every: int) -> dict:
    sys.path.insert(0, ROOT)
    import tempfile
    from distributedmnist_b200 import data as mnist_data
    from distributedmnist_b200.flags import FLAGS
    from distributedmnist_b200.parallel.context import init_context
    from distributedmnist_b200.train import train
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True)
    with tempfile.TemporaryDirectory() as d:
        FLAGS.parse(["--train_dir=%s" % d, "--batch_size=256", "--max_steps=%d" % max_steps, "--model=lenet",
                     "--device_data=true", "--eval_every_steps=%d" % eval_every, "--target_accuracy=%r" % target,
                     "--initial_learning_rate=0.05", "--log_every=100000", "--save_results_period=100000000",
                     "--save_interval_secs=1e9"] + (["--async_method=true"] if mode == "async" else []))
        res = train(init_context(FLAGS), ds.train, ds.validation, FLAGS)
        with open(os.path.join(d, "worker0_time_to_accuracy.json")) as f:
            rep = json.load(f)
    return dict(reached=rep["reached"], global_step=rep["global_step"], accuracy=rep["accuracy"],
                train_time_s=rep["train_time_s"], wall_time_s=rep["wall_time_s"], final_step=res["final_step"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3000)
    ap.add_argument("--warmup", type=int, default=300)
    ap.add_argument("--blocks", type=int, default=3)
    ap.add_argument("--target", type=float, default=0.95)
    ap.add_argument("--max-steps", type=int, default=5000)
    ap.add_argument("--eval-every", type=int, default=20)
    ap.add_argument("--out", default="")
    ap.add_argument("--one", default="", help=argparse.SUPPRESS)
    ap.add_argument("--tta", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.one:
        print(json.dumps(time_to_accuracy(a.one, a.target, a.max_steps, a.eval_every) if a.tta
                         else one(a.one, a.steps, a.warmup, a.blocks)))
        return
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    rows = []
    for mode, env in (("k_eq_n", {}), ("single_kernel", {"DMNIST_BUCKET": "0"}), ("async", {})):
        cmd = [sys.executable, os.path.abspath(__file__), "--one", "async" if mode == "async" else "sync",
               "--steps", str(a.steps), "--warmup", str(a.warmup), "--blocks", str(a.blocks), "--target", str(a.target),
               "--max-steps", str(a.max_steps), "--eval-every", str(a.eval_every)]
        r = subprocess.run(cmd, capture_output=True, text=True, env=dict(os.environ, **env), check=True)
        row = json.loads(r.stdout.strip().splitlines()[-1])
        row["mode"] = mode
        r = subprocess.run(cmd + ["--tta"], capture_output=True, text=True, env=dict(os.environ, **env), check=True)
        row["time_to_accuracy"] = json.loads(r.stdout.strip().splitlines()[-1])
        rows.append(row)
        print(json.dumps(row), flush=True)
    out = dict(gpu=q[0] if q else "unknown", model="lenet", batch=256, replicas=1, target=a.target, results=rows)
    print(json.dumps(out))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
