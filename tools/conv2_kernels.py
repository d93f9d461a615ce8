"""Time the conv2 forward and data-gradient kernels alone on the GPU, at the training batch and at the evaluation chunk.

Each figure is CUDA events around N warmed back-to-back launches, divided by N.  The card's name, power limit and max
SM clock are read in the same call and printed with the numbers.  Prints one JSON line.

    python tools/conv2_kernels.py [--launches 2000] [--batches 256,1000]
"""
import argparse
import json
import sys

import gpu_timing
import torch
from distributedmnist_b200.ops.lib import load, stream_ptr

BF = torch.bfloat16


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--batches", default="256,1000")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("conv2_kernels.py needs a CUDA device")
    lib = load()
    res = gpu_timing.card()
    for B in [int(b) for b in args.batches.split(",")]:
        g = torch.Generator(device="cpu").manual_seed(B)
        a1 = torch.rand(B, 14, 14, 32, generator=g).to(BF).cuda()
        w = (torch.randn(5, 5, 32, 64, generator=g) * 0.05).to(BF).cuda()
        b = (torch.randn(64, generator=g) * 0.1).cuda()
        dy = (torch.randn(B, 14, 14, 64, generator=g) * 0.1).to(BF).cuda()
        out = torch.empty(B, 7, 7, 64, dtype=BF, device="cuda")
        code = torch.empty(B, 7, 7, 64, dtype=torch.uint8, device="cuda")
        dx = torch.empty(B, 14, 14, 32, dtype=BF, device="cuda")
        res["conv2_fwd_us_B%d" % B] = gpu_timing.timed_launches(
            lambda: lib.dm_conv2_fwd(a1, w, b, out, code, B, stream_ptr()), args.launches, args.warmup)
        res["conv2_dgrad_us_B%d" % B] = gpu_timing.timed_launches(
            lambda: lib.dm_conv2_dgrad(dy, w, dx, B, stream_ptr()), args.launches, args.warmup)
    res["launches"] = args.launches
    print(json.dumps({k: (round(v, 2) if isinstance(v, float) else v) for k, v in res.items()}), flush=True)


if __name__ == "__main__":
    main()
