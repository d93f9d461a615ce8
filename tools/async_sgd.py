#!/usr/bin/env python
"""Step time and time to a target accuracy of asynchronous SGD (--async_method) against the default K = N path and the
single aggregation kernel (DMNIST_BUCKET=0), LeNet at B = 256 on one GPU.  The card's name, power limit and max SM clock
are recorded next to the numbers.

* step time: the device time of blocks of graph-replayed steps, with CUDA events;
* time to accuracy: ``train()`` with ``--device_data``, ``--eval_every_steps`` and ``--target_accuracy`` (what
  ``worker0_time_to_accuracy.json`` reports: the training time on the device clock up to the evaluation that reached the
  target, the passes before it taken out).  The data is the synthetic MNIST-shaped set, so these are not MNIST numbers.

Every measurement runs in a fresh process.

    python tools/async_sgd.py [--steps 3000] [--warmup 300] [--blocks 3] [--target 0.95] [--max-steps 5000]
                              [--eval-every 20] [--out results/async_sgd.json]
"""
import argparse
import json
import os
import tempfile

import gpu_timing
from distributedmnist_b200.parallel.aggregators import AsyncSGDOptimizer, SyncReplicasOptimizer
from distributedmnist_b200.schedule import LearningRateSchedule


def one(mode: str, steps: int, warmup: int, blocks: int) -> dict:
    sched = LearningRateSchedule(0.01, 1000, 0.95)
    eng = gpu_timing.one_replica_engine("lenet", 256, 0, lambda be: (AsyncSGDOptimizer(be, sched, 1) if mode == "async"
                                                                     else SyncReplicasOptimizer(be, sched, 1, 1)))
    us = gpu_timing.alternate({mode: (eng, gpu_timing.packed_batches(eng, 4, 1, on_device=False))}, steps, warmup, blocks)
    eng.backend.check_error()
    return dict(mode=mode, us_per_step=us[mode], launches_per_step=eng.launches_per_step)


def time_to_accuracy(mode: str, target: float, max_steps: int, eval_every: int) -> dict:
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
    rows = []
    for mode, env in (("k_eq_n", {}), ("single_kernel", {"DMNIST_BUCKET": "0"}), ("async", {})):
        argv = [__file__, "--one", "async" if mode == "async" else "sync", "--steps", str(a.steps), "--warmup",
                str(a.warmup), "--blocks", str(a.blocks), "--target", str(a.target), "--max-steps", str(a.max_steps),
                "--eval-every", str(a.eval_every)]
        row = gpu_timing.child_json(argv, env)
        row["mode"] = mode
        row["time_to_accuracy"] = gpu_timing.child_json(argv + ["--tta"], env)
        rows.append(row)
        print(json.dumps(row), flush=True)
    gpu_timing.emit(dict(gpu_timing.card(), model="lenet", batch=256, replicas=1, target=a.target, results=rows), a.out)


if __name__ == "__main__":
    main()
