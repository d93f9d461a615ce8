"""Time the fully connected block of the LeNet training step on the GPU: its four kernels (fc1_fwd, fc2_fwd_bwd,
fc1_dgrad + un-pool, fc1_wgrad) alone and launched back to back, and the fc1 data- and weight-gradient GEMMs side by
side on two streams as the step graph runs them.

Each figure is CUDA events around N graph-replayed iterations, divided by N (a graph, so that the host's launch cost
does not hide the kernels' time).  The card's name, power limit and max SM clock are read in the same call and printed
with the numbers.  Prints one JSON line.

    python tools/fc_kernels.py [--iters 2000] [--batches 256,1024]
"""
import argparse
import json
import sys

import gpu_timing
import torch


def graph_us(fn, iters: int, reps: int = 5) -> float:
    """Median over ``reps`` replays of a graph holding ``iters`` calls of ``fn``: microseconds per call."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t = []
    for _ in range(reps):
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        t.append(e0.elapsed_time(e1) * 1e3 / iters)
    return sorted(t)[len(t) // 2]


def engine(B: int):
    from distributedmnist_b200.engine_cuda import CudaLeNetEngine
    from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer
    from distributedmnist_b200.parallel.context import ReplicaContext
    from distributedmnist_b200.parallel.fused import FusedBackend
    from distributedmnist_b200.schedule import LearningRateSchedule
    ctx = ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none")
    be = FusedBackend(ctx)
    eng = CudaLeNetEngine(B, be, use_graph=False)
    eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.01, 100, 1.0), 1, 1))
    g = torch.Generator().manual_seed(B)
    eng.load_batch((torch.rand(B, 28, 28, 1, generator=g) - 0.5).numpy(), torch.randint(0, 10, (B,), generator=g).numpy())
    eng.train_step()                      # fills a2, code2 and the rest of the fc block's inputs
    torch.cuda.synchronize()
    return eng, be


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=2000)
    ap.add_argument("--batches", default="256,1024")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fc_kernels.py needs a CUDA device")
    from distributedmnist_b200.ops.lib import stream_ptr
    torch.cuda.set_device(0)
    res = gpu_timing.card()
    for B in [int(b) for b in args.batches.split(",")]:
        eng, be = engine(B)
        lbl = eng.labels[eng._slot]
        side = torch.cuda.Stream()

        def fwd():
            eng._fc1_fwd(B)

        def head():
            eng._fc2_fwd_bwd(lbl, B, True, stream_ptr())

        def dgrad():
            eng._fc1_dgrad(B, stream_ptr())

        def wgrad():
            eng._fc1_wgrad(eng.g["fc1_weights"], B)

        def four():
            fwd()
            head()
            dgrad()
            wgrad()

        def grads_side_by_side():
            # the step graph's shape: dgrad on the calling stream, wgrad forked beside it
            cur = torch.cuda.current_stream()
            side.wait_stream(cur)
            dgrad()
            with torch.cuda.stream(side):
                wgrad()
            cur.wait_stream(side)

        for name, fn in [("fc1_fwd", fwd), ("fc2_fwd_bwd", head), ("fc1_dgrad", dgrad), ("fc1_wgrad", wgrad),
                         ("four_back_to_back", four), ("dgrad_beside_wgrad", grads_side_by_side)]:
            res["%s_us_B%d" % (name, B)] = graph_us(fn, args.iters)
        torch.cuda.synchronize()
        be.check_error()
        be.close()
    res["iters"] = args.iters
    print(json.dumps({k: (round(v, 2) if isinstance(v, float) else v) for k, v in res.items()}), flush=True)


if __name__ == "__main__":
    main()
