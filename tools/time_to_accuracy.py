#!/usr/bin/env python
"""Time to accuracy on one GPU: ``train.train()`` with ``--device_data``, ``--eval_every_steps`` and ``--target_accuracy``,
K = N = 1 and K > N (``--k``, default 4, on the one replica) alternating for ``--rounds`` rounds.  Prints one JSON line.

Per run: the global step of the evaluation that reached the target, the stop step, the training time to it on the chief's
device clock with the evaluation passes before it taken out (``worker0_time_to_accuracy.json``), the host wall time to it,
and the steps the run made.  The data is the synthetic MNIST-shaped set (``data.make_synthetic_mnist``: ten blurred glyph
prototypes, shifted, scaled and noised), so the numbers are not MNIST numbers.

    python tools/time_to_accuracy.py [--target 0.95] [--rounds 3] [--k 4] [--max-steps 5000] [--eval-every 20]
                                     [--out results/time_to_accuracy.json]
"""
import argparse
import os
import tempfile

import gpu_timing
from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.flags import FLAGS
from distributedmnist_b200.parallel.context import init_context
from distributedmnist_b200.train import train


def run(ds, args, k: int) -> dict:
    FLAGS.reset()
    with tempfile.TemporaryDirectory() as d:
        FLAGS.parse(["--train_dir=%s" % d, "--batch_size=%d" % args.batch_size, "--max_steps=%d" % args.max_steps,
                     "--model=lenet", "--device_data=true", "--eval_every_steps=%d" % args.eval_every,
                     "--target_accuracy=%r" % args.target, "--num_replicas_to_aggregate=%d" % k,
                     "--initial_learning_rate=%r" % args.lr, "--log_every=100000", "--save_results_period=100000000",
                     "--save_interval_secs=1e9"] + (["--eval_snapshot=true"] if k != 1 else []))
        ctx = init_context(FLAGS)
        res = train(ctx, ds.train, ds.validation, FLAGS)
    rep = res["time_to_accuracy"]
    return dict(k=k, reached=rep["reached"], global_step=rep["global_step"], accuracy=rep["accuracy"],
                train_time_s=rep["train_time_s"], wall_time_s=rep["wall_time_s"], final_step=res["final_step"],
                evals=len(res["evals"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--target", type=float, default=0.95)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--k", type=int, default=4)
    ap.add_argument("--max-steps", type=int, default=5000)
    ap.add_argument("--eval-every", type=int, default=20)
    ap.add_argument("--batch-size", type=int, default=128)
    ap.add_argument("--lr", type=float, default=0.05)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        os.environ.pop(k, None)
    FLAGS.reset()
    ds = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=True)
    runs = []
    for _ in range(args.rounds):
        for k in (1, args.k):
            runs.append(run(ds, args, k))
    out = dict(tool="time_to_accuracy", data="synthetic MNIST-shaped (not MNIST)", target=args.target,
               batch_size=args.batch_size, eval_every_steps=args.eval_every, max_steps=args.max_steps,
               validation_examples=ds.validation.num_examples, runs=runs, **gpu_timing.card())
    gpu_timing.emit(out, args.out)


if __name__ == "__main__":
    main()
