#!/usr/bin/env python
"""Cost of early stopping (``--early_stopping_patience``) in the lenet evaluation pass on one GPU, synthetic data.  Prints
one JSON line.

One 10k pass enqueued between two training steps, replayed from its CUDA graph as the training loop replays it and
bracketed by CUDA events on the training stream, two ways, pass by pass in turn so that both share the same conditions:

  off      the pass's graph without eval_patience;
  armed    the same pass with eval_patience as its last node.  The patience is never exhausted (P is larger than the
           number of passes), so every pass runs the whole rule and none sets the stop word.

    python tools/early_stopping.py [--passes 200] [--batch 256] [--out results/early_stopping.json]
"""
import argparse
import sys

import gpu_timing
import numpy as np
import torch
from distributedmnist_b200.data import make_synthetic_mnist
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
from distributedmnist_b200.schedule import LearningRateSchedule
from distributedmnist_b200.train import STOP_MARGIN


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=200, help="timed passes per configuration")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("early_stopping.py measures on a GPU; none found")
    B = a.batch
    eng = gpu_timing.one_replica_engine(
        "lenet", B, 0, lambda be: SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 10 ** 6, 1.0), 1, 1))
    n = 10000
    trx, try_, tex, tey = make_synthetic_mnist(B * 16, n, seed=5)
    bufs = [eng.pack_batch(trx[i * B:(i + 1) * B], try_[i * B:(i + 1) * B]) for i in range(16)]
    eng.arm_eval(tex, tey)
    eng.arm_stop()                                           # both configurations run the same step graph
    graph_off = eng._ev_graph
    rounds = a.passes + 10                                   # the first 10 rounds warm up
    eng.arm_patience(2 * rounds, 0, STOP_MARGIN)
    graph_on = eng._ev_graph
    graphs = {"off": graph_off, "armed": graph_on}
    times = {k: [] for k in graphs}
    done = 0
    for i in range(2 * rounds):
        name = list(graphs)[i % 2]
        eng._ev_graph = graphs[name]
        tok = eng.step_packed(bufs[done % len(bufs)])
        done += 1
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        eng.enqueue_eval()
        e1.record()
        tok[0].synchronize()
        torch.cuda.synchronize()
        if i >= 20:
            times[name].append(e0.elapsed_time(e1) * 1e-3)
        eng.eval_records()
    eng._leave_native_runner()
    eng.backend.check_error()
    st = eng.patience_state()
    assert st.baseline and st.since < 2 * rounds and eng.stop_step() == 0, st
    med = {k: float(np.median(v)) for k, v in times.items()}
    res = dict(gpu_timing.card(), batch=B, eval_examples=n, passes_per_config=a.passes,
               pass_us={k: {"median": med[k] * 1e6, "min": float(np.min(v)) * 1e6, "max": float(np.max(v)) * 1e6}
                        for k, v in times.items()},
               added_us=(med["armed"] - med["off"]) * 1e6, added_share=med["armed"] / med["off"] - 1.0)
    gpu_timing.emit(res, a.out)


if __name__ == "__main__":
    main()
