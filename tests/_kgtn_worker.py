"""Helper process: the K > N count-triggered kernels (csrc/fused_interval.cu) driven directly, no model.

Every replica free-runs `iters` iterations of [adopt -> (delay) -> gate -> accumulate -> close -> apply] with the same constant
gradient, so the mean of any set of accumulated gradients is that gradient and after T commits the weights must be
w0 - T * lr * g up to fp32 rounding, whoever contributed.  The last rank is delayed on the device.

argv: <out json with RANK placeholder> <k> <iters> <delay_us of the last rank>"""
import hashlib
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.parallel.fused import FusedBackend  # noqa: E402


def main():
    out_json = sys.argv[1].replace("RANK", os.environ.get("RANK", "0"))
    k, iters, delay_us = int(sys.argv[2]), int(sys.argv[3]), float(sys.argv[4])
    ctx = init_context(None, want_gpu=True)
    n, r = ctx.world_size, ctx.rank
    be = FusedBackend(ctx, timeout_ms=10000.0)
    numel = 1 << 18
    params, grads, acc = be.allocate(numel), be.allocate(numel), be.allocate(numel)
    be.attach_shadow(params)
    gen = torch.Generator(device="cpu").manual_seed(99)
    w0 = torch.randn(numel, generator=gen).to(ctx.device)
    g = torch.randn(numel, generator=gen).to(ctx.device)
    params.copy_(w0)
    grads.copy_(g)
    be.refresh_shadow(params)
    lr = 0.01
    be.kgtn_arm()
    slow = n > 1 and r == n - 1
    if slow:
        iters = max(4, int(iters * 200.0 / max(delay_us, 200.0)))      # about the same wall time as the fast replicas
    t0 = time.monotonic()
    rows = []
    for it in range(iters):
        be.enqueue_kgtn_begin(params)
        be.enqueue_straggler_delay(1.0, delay_us if slow else 200.0)
        be.enqueue_kgtn_end(params, grads, acc, k, lr)
        st = be.read_status()
        rows.append([st["epoch"], st["last_late"], st["last_mask"], st["last_count"]])
    torch.cuda.synchronize()
    wall = time.monotonic() - t0
    be.check_error()
    # quiesce, then adopt whatever was pushed last
    be.barrier()
    time.sleep(0.05)
    be.enqueue_kgtn_begin(params)
    torch.cuda.synchronize()
    be.barrier()
    st = be.read_status()
    steps = st["epoch"]
    err = (params - (w0 - steps * lr * g)).abs().max().item()
    state = int(be._ctrl_bytes[be._off["iv_state"]:be._off["iv_state"] + 8].view(torch.int64).item())
    pending = (state & 0xFFFFFFFF) if (state >> 32) == steps + 1 else 0      # accumulated for the step not yet committed
    json.dump({"rank": r, "steps": steps, "err": err, "pmax": params.abs().max().item(),
               "shadow_err": (be.shadow.float() - params).abs().max().item(),
               "fp": hashlib.sha1(params.cpu().numpy().tobytes()).hexdigest(), "rows": rows, "wall_s": wall,
               "iters": iters, "accepted": st["accepted_steps"], "dropped": st["dropped_steps"], "last_count": st["last_count"],
               "ticks_committed": be._read_u32("iv_ticks_committed"), "nvls": be.nvls_active, "pending": pending}, open(out_json, "w"))
    be.close()
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
