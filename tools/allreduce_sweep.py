#!/usr/bin/env python
"""Gradient-aggregation bandwidth sweep: fused allreduce+scale+SGD kernel vs NCCL allreduce + scale + SGD.

BASELINE.json config 5 ("gradient-allreduce bandwidth sweep 4 KB-256 MB at 2/4/8 GPUs vs NCCL").  Run under
torchrun (one rank per GPU).  Device-timed with CUDA events, max over ranks.  Bus bandwidth uses the standard
allreduce convention 2*(N-1)/N * bytes / time so both arms are comparable with the nominal per-direction NVLink
bandwidth of the box (H100 SXM, NVLink 4: 450 GB/s).
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.parallel.fused import FusedBackend  # noqa: E402


def timed(fn, iters, n, device):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    if n > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1) / iters], device=device)
    if n > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    return float(ms.item())


def main():
    ctx = init_context(None, want_gpu=True)
    n, dev = ctx.world_size, ctx.device
    be = FusedBackend(ctx)
    max_bytes = int(os.environ.get("DM_SWEEP_MAX", str(256 << 20)))
    numel = max_bytes // 4
    params, grads = be.allocate(numel), be.allocate(numel)
    nccl_buf = torch.zeros(numel, device=dev)
    nccl_w = torch.zeros(numel, device=dev)
    rows = []
    size = 4096
    while size <= max_bytes:
        ne = size // 4
        p2, g2 = params[:ne], grads[:ne]
        be._by_ptr[p2.data_ptr()] = be._by_ptr[params.data_ptr()]
        be._by_ptr[g2.data_ptr()] = be._by_ptr[grads.data_ptr()]
        iters = 50 if size <= (8 << 20) else 10
        ms_f = timed(lambda: be.enqueue(p2, g2, n, lr0=0.01), iters, n, dev)

        def nccl_step():
            b = nccl_buf[:ne]
            if n > 1:
                dist.all_reduce(b)
            b.mul_(1.0 / n)                      # separate scale kernel
            nccl_w[:ne].add_(b, alpha=-0.01)     # separate SGD kernel
        ms_n = timed(nccl_step, iters, n, dev)
        bus = 2.0 * (n - 1) / n * size if n > 1 else size
        rows.append({"bytes": size, "fused_ms": ms_f, "nccl_ms": ms_n, "fused_bus_gbs": bus / ms_f / 1e6,
                     "nccl_bus_gbs": bus / ms_n / 1e6})
        size *= 4
    be.check_error()
    if ctx.rank == 0:
        print(json.dumps({"n_gpus": n, "rows": rows}))
        os.makedirs("results", exist_ok=True)
        with open("results/allreduce_sweep_n%d_nvls%s.json" % (n, os.environ.get("DMNIST_NVLS", "auto")), "w") as f:
            json.dump({"n_gpus": n, "rows": rows}, f, indent=1)
    be.close()
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
