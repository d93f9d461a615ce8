"""Time the conv1 kernels on the GPU: conv1_fwd at the training batch and at the evaluation chunk, conv1_wgrad alone,
and conv1_wgrad on a second stream beside conv2_wgrad + its reduction, as the training step runs them.

Each figure is CUDA events around N warmed back-to-back launches, divided by N.  The card's name, power limit and max
SM clock are read in the same call and printed with the numbers.  Prints one JSON line.

    python tools/conv1_kernels.py [--launches 2000] [--batch 256] [--eval-batch 2048]
"""
import argparse
import json
import sys

import gpu_timing
import torch
from distributedmnist_b200.ops.lib import load, stream_ptr

BF = torch.bfloat16


def inputs(B: int, seed: int):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.rand(B, 28, 28, generator=g) - 0.5
    w = torch.randn(25, 32, generator=g) * 0.1
    b = torch.randn(32, generator=g) * 0.1
    dpool = (torch.randn(B, 14, 14, 32, generator=g) * 0.1).to(BF)
    code = (torch.randint(0, 4, (B, 14, 14, 32), generator=g) | (torch.randint(0, 2, (B, 14, 14, 32), generator=g) * 4)).to(torch.uint8)
    a1 = torch.rand(B, 14, 14, 32, generator=g).to(BF)
    dy = (torch.randn(B, 14, 14, 64, generator=g) * 0.1).to(BF)
    return [t.cuda() for t in (x, w, b, dpool, code, a1, dy)]


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--eval-batch", type=int, default=2048)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("conv1_kernels.py needs a CUDA device")
    lib = load()
    res = gpu_timing.card()
    n, wu = args.launches, args.warmup

    def fwd(B):
        x, w, b = inputs(B, 1)[:3]
        out = torch.empty(B, 14, 14, 32, dtype=BF, device="cuda")
        code = torch.empty(B, 14, 14, 32, dtype=torch.uint8, device="cuda")
        return lambda: lib.dm_conv1_fwd_tc(x, w, b, out, code, B, None, 0, None, 0, None, 0, stream_ptr())

    res["conv1_fwd_us_B%d" % args.batch] = gpu_timing.timed_launches(fwd(args.batch), n, wu)
    res["conv1_fwd_us_B%d" % args.eval_batch] = gpu_timing.timed_launches(fwd(args.eval_batch), n, wu)

    B = args.batch
    x, _, _, dpool, code, a1, dy = inputs(B, 2)
    gw1, gb1 = torch.zeros(25, 32, device="cuda"), torch.zeros(32, device="cuda")
    gw2 = torch.zeros(5, 5, 32, 64, device="cuda")
    main_s = torch.cuda.current_stream()
    side = torch.cuda.Stream()

    def c1(stream=None):
        lib.dm_conv1_wgrad_tc(x, dpool, code, gw1, gb1, B, stream_ptr(stream))

    def c2():
        lib.dm_conv2_wgrad(a1, dy, gw2, B, stream_ptr())

    def both():                                    # fork / join as in the step graph
        fork = torch.cuda.Event()
        fork.record(main_s)
        side.wait_event(fork)
        c2()
        c1(side)
        join = torch.cuda.Event()
        join.record(side)
        main_s.wait_event(join)

    res["conv1_wgrad_us_B%d" % B] = gpu_timing.timed_launches(c1, n, wu)
    res["conv2_wgrad_reduce_us_B%d" % B] = gpu_timing.timed_launches(c2, n, wu)
    res["conv2_wgrad_reduce_plus_conv1_wgrad_beside_us_B%d" % B] = gpu_timing.timed_launches(both, n, wu)
    res["launches"] = n
    print(json.dumps({k: (round(v, 2) if isinstance(v, float) else v) for k, v in res.items()}), flush=True)


if __name__ == "__main__":
    main()
