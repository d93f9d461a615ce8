#!/usr/bin/env python
"""Cost of learning-rate cuts at a plateau (``--lr_plateau_patience``) on one GPU, lenet, synthetic data.  Prints one JSON
line with two measurements, each alternating its two configurations in the same call so that both share the same
conditions:

  pass     One 10k evaluation pass enqueued between two training steps, replayed from its CUDA graph and bracketed by
           CUDA events on the training stream: ``off`` without eval_plateau, ``armed`` with eval_plateau as its last
           node.  The patience is never exhausted, so every pass runs the whole rule and stores no cut.
  step     Blocks of graph-replayed training steps (the pipelined loop's native runner) bracketed by CUDA events:
           ``off`` with no cut table in the control block, ``armed`` with a table whose entries are all 0xFFFFFFFF (no
           cut), which every aggregation kernel's CTAs then read in cta_scale.  The step graph is the same in both.

    python tools/lr_plateau.py [--passes 200] [--blocks 40] [--block-steps 50] [--batch 256] [--out results/lr_plateau.json]
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


def _stats(v):
    return {"median": float(np.median(v)) * 1e6, "min": float(np.min(v)) * 1e6, "max": float(np.max(v)) * 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=200, help="timed passes per configuration")
    ap.add_argument("--blocks", type=int, default=40, help="timed step blocks per configuration")
    ap.add_argument("--block-steps", type=int, default=50, help="training steps per block")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("lr_plateau.py measures on a GPU; none found")
    B = a.batch
    eng = gpu_timing.one_replica_engine(
        "lenet", B, 0, lambda be: SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 10 ** 6, 1.0), 1, 1))
    be = eng.backend
    n = 10000
    trx, try_, tex, tey = make_synthetic_mnist(B * 16, n, seed=5)
    bufs = [eng.pack_batch(trx[i * B:(i + 1) * B], try_[i * B:(i + 1) * B]) for i in range(16)]
    eng.arm_eval(tex, tey)
    eng.arm_lr_cuts(0.1)                                     # every configuration runs the same step graph
    graph_off = eng._ev_graph
    rounds = a.passes + 10                                   # the first 10 rounds warm up
    eng.arm_lr_plateau(2 * rounds, 0, STOP_MARGIN)
    graphs = {"off": graph_off, "armed": eng._ev_graph}
    done = 0

    # ---- the pass, with and without eval_plateau ----------------------------------------------------------------------
    pass_s = {k: [] for k in graphs}
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
            pass_s[name].append(e0.elapsed_time(e1) * 1e-3)
        eng.eval_records()
    st = eng.lr_plateau_state()
    assert st.baseline and st.cuts == 0, st

    # ---- training steps, with and without a cut table -----------------------------------------------------------------
    table = eng._lr_table.local_ptr
    ctrl = be.ctrl.local_ptr
    step_s = {"off": [], "armed": []}
    for i in range(2 * (a.blocks + 2)):                      # the first 2 blocks of each warm up
        name = ("off", "armed")[i % 2]
        torch.cuda.synchronize()
        be.lib.dm_sync_set_lr_cuts(ctrl, table if name == "armed" else None, 0.1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.block_steps):
            tok = eng.step_packed(bufs[done % len(bufs)])
            done += 1
        e1.record()
        tok[0].synchronize()
        torch.cuda.synchronize()
        if i >= 4:
            step_s[name].append(e0.elapsed_time(e1) * 1e-3 / a.block_steps)
    eng._leave_native_runner()
    be.check_error()
    assert eng.lr_cut_table() == [0xFFFFFFFF] * 32

    mp = {k: float(np.median(v)) for k, v in pass_s.items()}
    ms = {k: float(np.median(v)) for k, v in step_s.items()}
    res = dict(gpu_timing.card(), batch=B, eval_examples=n, passes_per_config=a.passes, step_blocks_per_config=a.blocks,
               steps_per_block=a.block_steps,
               pass_us={k: _stats(v) for k, v in pass_s.items()},
               pass_added_us=(mp["armed"] - mp["off"]) * 1e6,
               step_us={k: _stats(v) for k, v in step_s.items()},
               step_added_us=(ms["armed"] - ms["off"]) * 1e6, step_added_share=ms["armed"] / ms["off"] - 1.0)
    gpu_timing.emit(res, a.out)


if __name__ == "__main__":
    main()
