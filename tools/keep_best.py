#!/usr/bin/env python
"""Cost of keeping the best weights (``--keep_best_checkpoint``) in the lenet evaluation pass on one GPU, synthetic data.
Prints one JSON line.

One 10k pass enqueued between two training steps and bracketed by CUDA events on the training stream, three ways, pass by
pass in turn so that the three share the same conditions:

  off          the pass's graph without the best-keeping nodes;
  no_improve   with eval_best_decide and eval_best_copy, the best count set to the whole set: the copy exits at once;
  improve      the same graph, the best count reset to 0 in front of every pass: every pass copies the 6.65 MB arena.

    python tools/keep_best.py [--passes 60] [--batch 256] [--out results/keep_best.json]
"""
import argparse
import sys

import gpu_timing
import numpy as np
import torch
from distributedmnist_b200.best import BEST_CORRECT_WORD, BEST_VALID_WORD
from distributedmnist_b200.data import make_synthetic_mnist
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
from distributedmnist_b200.schedule import LearningRateSchedule


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=60, help="timed passes per configuration")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("keep_best.py measures on a GPU; none found")
    B = a.batch
    eng = gpu_timing.one_replica_engine(
        "lenet", B, 0, lambda be: SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 10 ** 6, 1.0), 1, 1))
    n = 10000
    trx, try_, tex, tey = make_synthetic_mnist(B * 16, n, seed=5)
    bufs = [eng.pack_batch(trx[i * B:(i + 1) * B], try_[i * B:(i + 1) * B]) for i in range(16)]
    eng.arm_eval(tex, tey)
    graph_off = eng._ev_graph
    eng.arm_best()
    graph_on = eng._ev_graph
    state = eng._best[0]
    seeds = {"off": None, "no_improve": n, "improve": 0}
    times = {k: [] for k in seeds}
    copies = {k: 0 for k in seeds}
    done = 0
    for i in range(3 * (a.passes + 10)):                     # the first 10 rounds warm up
        name = list(seeds)[i % 3]
        eng._ev_graph = graph_off if seeds[name] is None else graph_on
        if seeds[name] is not None:
            state[BEST_CORRECT_WORD] = seeds[name]
            state[BEST_VALID_WORD] = 0
        tok = eng.step_packed(bufs[done % len(bufs)])
        done += 1
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.enqueue_eval()
        e1.record()
        tok[0].synchronize()
        torch.cuda.synchronize()
        if i >= 30:
            times[name].append(e0.elapsed_time(e1) * 1e-3)
            if seeds[name] is not None:
                copies[name] += int(state[BEST_VALID_WORD].item())
        eng.eval_records()
    eng._leave_native_runner()
    eng.backend.check_error()
    assert copies["improve"] == a.passes and copies["no_improve"] == 0, copies
    med = {k: float(np.median(v)) for k, v in times.items()}
    res = dict(gpu_timing.card(), batch=B, eval_examples=n, passes_per_config=a.passes, arena_bytes=4 * eng.spec.arena_numel,
               pass_us={k: {"median": med[k] * 1e6, "min": float(np.min(v)) * 1e6, "max": float(np.max(v)) * 1e6}
                        for k, v in times.items()},
               added_us={k: (med[k] - med["off"]) * 1e6 for k in ("no_improve", "improve")},
               added_share={k: med[k] / med["off"] - 1.0 for k in ("no_improve", "improve")})
    gpu_timing.emit(res, a.out)


if __name__ == "__main__":
    main()
