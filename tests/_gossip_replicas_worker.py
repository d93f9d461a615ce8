"""Helper process: N replicas of gossip SGD, all on one GPU, each on its own stream (csrc/fused_gossip.cu).

The replicas' control blocks, send buffers, arenas, shadows and statistics are plain device allocations, reached through
8-entry pointer tables.  Every replica's gradients are drawn up front; replica q's iteration s reads grads[q][s].  After
every iteration a copy of the replica's arena is recorded on its own stream.  The host enqueues every iteration of every
replica without synchronising between rounds; the replica ``slow`` sleeps before each iteration's apply, as a slow
gradient would.  The run ends with the local-SGD round every gossip run ends with (dm_local_average, period 1, no step
closed), on every stream.  For N <= 3 the same gradients are also run through the local-SGD kernels with H = 1.

gs_barrier polls words that other streams' kernels write, so two replicas' streams must never share a hardware queue:
the process runs with CUDA_DEVICE_MAX_CONNECTIONS=32 (set by the test that starts it).  Every kernel is loaded by a lone
replica (N = 1, which waits on nobody) before the replicas launch them together: a lazy module load on the host could
otherwise wait behind a barrier that waits for a replica the host has not launched yet.

argv: <out npz> -- per case n: the initial arena, the gradients, the records, the final arenas and shadows, every
replica's t_arrive and t_pass stamps, statistics and error word, and for n <= 3 the local-SGD records."""
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributedmnist_b200.ops.lib import load  # noqa: E402
from distributedmnist_b200.parallel.fused import FusedBackend  # noqa: E402

NUMEL = 16384 + 12           # a ragged tail for the grid-stride loops
ITERS = 12
LR = 0.03125
WATCHDOG_MS = 5000.0
SLEEP_CYCLES = 2000000       # about 1 ms: longer than the host takes to enqueue a round of every replica
CTAS = 16                    # every replica's grids fit on the GPU at once


def _table(ptrs):
    return (ctypes.c_void_p * 8)(*([int(p) for p in ptrs] + [int(ptrs[0])] * (8 - len(ptrs))))


def _ctrl(lib):
    return torch.zeros(int(lib.dm_sync_ctrl_bytes()), dtype=torch.uint8, device="cuda")


def run_gossip(lib, n, w0, grads, slow):
    ctrl = [_ctrl(lib) for _ in range(n)]
    send = [torch.zeros(2 * NUMEL, device="cuda") for _ in range(n)]
    params = [w0.clone() for _ in range(n)]
    shadow = [torch.zeros(NUMEL, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
    stats = [torch.zeros(int(lib.dm_gossip_stats_bytes()), dtype=torch.uint8, device="cuda") for _ in range(n)]
    ls_stats = [torch.zeros(int(lib.dm_local_stats_bytes()), dtype=torch.uint8, device="cuda") for _ in range(n)]
    rec = [torch.zeros(ITERS, NUMEL, device="cuda") for _ in range(n)]
    streams = [torch.cuda.Stream() for _ in range(n)]
    sp = [ctypes.c_void_p(st.cuda_stream) for st in streams]
    ct, st_tab, pt = _table([c.data_ptr() for c in ctrl]), _table([s.data_ptr() for s in send]), \
        _table([p.data_ptr() for p in params])
    torch.cuda.synchronize()
    for s in range(ITERS):
        for q in range(n):
            with torch.cuda.stream(streams[q]):
                if q == slow:
                    torch.cuda._sleep(SLEEP_CYCLES)
                lib.dm_gossip_apply(ct, q, params[q], grads[q][s], send[q], NUMEL, LR, 1.0, 1, CTAS, sp[q])
                lib.dm_gossip_exchange(ct, st_tab, params[q], shadow[q], stats[q], q, n, NUMEL, WATCHDOG_MS, CTAS, sp[q])
                rec[q][s].copy_(params[q])
    torch.cuda.synchronize()
    err = int(lib.dm_sync_ctrl_offset(b"error"))
    errors = [int(c[err:err + 4].view(torch.int32).item()) for c in ctrl]
    mixed = [p.clone() for p in params]
    for q in range(n):
        lib.dm_local_average(ct, pt, shadow[q], ls_stats[q], q, n, NUMEL, 1, 0, WATCHDOG_MS, CTAS, sp[q], None)
    torch.cuda.synchronize()
    ep, ta = int(lib.dm_sync_ctrl_offset(b"epoch")), int(lib.dm_sync_ctrl_offset(b"t_arrive"))
    out = dict(errors=np.array(errors + [int(c[err:err + 4].view(torch.int32).item()) for c in ctrl]),
               epochs=np.array([int(c[ep:ep + 4].view(torch.int32).item()) for c in ctrl]),
               rec=torch.stack(rec).cpu().numpy(), mixed=torch.stack(mixed).cpu().numpy(),
               final=torch.stack(params).cpu().numpy(),
               shadow=torch.stack(shadow).view(torch.int16).cpu().numpy().view(np.uint16),
               t_arrive=np.stack([c[ta:ta + 8 * ITERS].cpu().numpy().view("<u8") for c in ctrl]))
    gs = [FusedBackend.gossip_stats(x) for x in stats]
    out["t_pass"] = np.stack([g["t_pass"][:ITERS] for g in gs])
    out["stats"] = np.array(json.dumps([{k: v for k, v in g.items() if k != "t_pass"} for g in gs]))
    return out


def run_local(lib, n, w0, grads):
    """The same gradients through dm_local_apply + dm_local_average with H = 1 on the peer path."""
    ctrl = [_ctrl(lib) for _ in range(n)]
    params = [w0.clone() for _ in range(n)]
    shadow = [torch.zeros(NUMEL, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
    stats = [torch.zeros(int(lib.dm_local_stats_bytes()), dtype=torch.uint8, device="cuda") for _ in range(n)]
    rec = [torch.zeros(ITERS, NUMEL, device="cuda") for _ in range(n)]
    streams = [torch.cuda.Stream() for _ in range(n)]
    sp = [ctypes.c_void_p(st.cuda_stream) for st in streams]
    ct, pt = _table([c.data_ptr() for c in ctrl]), _table([p.data_ptr() for p in params])
    torch.cuda.synchronize()
    for s in range(ITERS):
        for q in range(n):
            with torch.cuda.stream(streams[q]):
                lib.dm_local_apply(ct, q, params[q], grads[q][s], shadow[q], NUMEL, 1, LR, 1.0, 1, CTAS, sp[q], None)
                lib.dm_local_average(ct, pt, shadow[q], stats[q], q, n, NUMEL, 1, 1, WATCHDOG_MS, CTAS, sp[q], None)
                rec[q][s].copy_(params[q])
    torch.cuda.synchronize()
    return torch.stack(rec).cpu().numpy()


def main():
    lib = load()
    torch.cuda.set_device(0)
    gen = torch.Generator(device="cuda").manual_seed(11)
    w0 = torch.randn(NUMEL, generator=gen, device="cuda")
    grads = [[torch.randn(NUMEL, generator=gen, device="cuda") for _ in range(ITERS)] for _ in range(8)]
    torch.cuda._sleep(1)
    run_gossip(lib, 1, w0, grads, -1)          # loads every kernel while nothing waits on another replica
    run_local(lib, 1, w0, grads)
    out = dict(w0=w0.cpu().numpy(), grads=torch.stack([torch.stack(g) for g in grads]).cpu().numpy())
    for n in range(2, 9):
        res = run_gossip(lib, n, w0, grads, n - 1)
        out.update({"n%d_%s" % (n, k): v for k, v in res.items()})
        if n <= 3:
            out["n%d_local" % n] = run_local(lib, n, w0, grads)
    np.savez(sys.argv[1], **out)


if __name__ == "__main__":
    main()
