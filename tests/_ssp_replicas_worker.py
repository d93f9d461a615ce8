"""Helper process: N replicas of asynchronous SGD under the staleness bound, all on one GPU, each on its own stream.

The replicas' control blocks, clock boards, master copies, working arenas and statistics are plain device allocations
and the peer path of the apply is used.  Replica p's gradient is 1 in slot p and 0 elsewhere and the rate is 1, so every
update subtracts exactly 1 from slot p of every master copy, and slots 0..N-1 of a pulled arena count the updates of each
replica it holds.  A copy of those slots is recorded on the replica's stream after every pull.  The last replica sleeps
before each iteration.

Unlike the unbounded async kernels, ssp_wait polls words that other streams' kernels write, so two replicas' streams must
never share a hardware queue: a wait queued in front of the publication it waits for would stall until the watchdog
fires.  The process therefore runs with CUDA_DEVICE_MAX_CONNECTIONS=32 (set by the test that starts it), one queue per
stream.

argv: <out json> -- a list of one record per case (n, s, iterations per replica): the recorded pulls, the final
copies and boards, the error words and every replica's statistics."""
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributedmnist_b200.ops.lib import load  # noqa: E402
from distributedmnist_b200.parallel.fused import FusedBackend  # noqa: E402

NUMEL = 64
WATCHDOG_MS = 2000.0
SLEEP_CYCLES = 2000000      # about 1 ms: longer than the host takes to enqueue a round of every replica


def _table(ptrs):
    return (ctypes.c_void_p * 8)(*([int(p) for p in ptrs] + [int(ptrs[0])] * (8 - len(ptrs))))


def run_case(lib, n, s, iters):
    """``iters[q]`` iterations of replica q, enqueued round robin; a replica retires once its last one is enqueued."""
    U = max(iters)
    ctrl = [torch.zeros(int(lib.dm_sync_ctrl_bytes()), dtype=torch.uint8, device="cuda") for _ in range(n)]
    board = [torch.zeros(256, dtype=torch.int32, device="cuda") for _ in range(n)]
    master = [torch.zeros(NUMEL, device="cuda") for _ in range(n)]
    params = [torch.zeros(NUMEL, device="cuda") for _ in range(n)]
    grads = [torch.zeros(NUMEL, device="cuda") for _ in range(n)]
    for q in range(n):
        grads[q][q] = 1.0
    as_stats = [torch.zeros(int(lib.dm_async_stats_bytes()), dtype=torch.uint8, device="cuda") for _ in range(n)]
    ssp_stats = [torch.zeros(int(lib.dm_ssp_stats_bytes()), dtype=torch.uint8, device="cuda") for _ in range(n)]
    rec = [torch.full((U, n), float("nan"), device="cuda") for _ in range(n)]
    streams = [torch.cuda.Stream() for _ in range(n)]
    sp = [ctypes.c_void_p(st.cuda_stream) for st in streams]
    ct, mt, bt = _table([c.data_ptr() for c in ctrl]), _table([m.data_ptr() for m in master]), \
        _table([b.data_ptr() for b in board])
    torch.cuda.synchronize()
    for j in range(U + 1):
        for q in range(n):
            if j == iters[q]:
                assert lib.dm_ssp_publish(bt, ssp_stats[q], q, n, 1, sp[q]) == 0      # retire
            if j >= iters[q]:
                continue
            with torch.cuda.stream(streams[q]):
                if q == n - 1:
                    torch.cuda._sleep(SLEEP_CYCLES)
                assert lib.dm_ssp_wait(board[q], ctrl[q], ssp_stats[q], q, n, s, WATCHDOG_MS, sp[q]) == 0
                assert lib.dm_async_begin(ct, q, master[q], params[q], None, NUMEL, 4, sp[q]) == 0
                rec[q][j].copy_(params[q][:n])
                assert lib.dm_async_end(ct, mt, grads[q], as_stats[q], q, n, NUMEL, 1.0, 1.0, 1, 4, sp[q], None) == 0
                assert lib.dm_ssp_publish(bt, ssp_stats[q], q, n, 0, sp[q]) == 0
    torch.cuda.synchronize()
    err = int(lib.dm_sync_ctrl_offset(b"error"))
    out = dict(n=n, s=s, iters=list(iters), errors=[int(c[err:err + 4].view(torch.int32).item()) for c in ctrl],
               pulled=[(-r.cpu().numpy()).tolist() for r in rec], master=[(-m[:n].cpu().numpy()).tolist() for m in master],
               boards=[b.view(-1, 32)[:n, 0].cpu().numpy().view(np.uint32).tolist() for b in board])
    out["async"] = []
    out["ssp"] = []
    for q in range(n):
        a = FusedBackend.async_stats(as_stats[q])
        out["async"].append(dict(updates=a["updates"], pairs=a["pairs"].tolist()))
        b = FusedBackend.ssp_stats(ssp_stats[q])
        b["pairs"] = b["pairs"].tolist()
        out["ssp"].append(b)
    return out


def main():
    lib = load()
    torch.cuda.set_device(0)
    cases = []
    for n in (2, 4, 8):
        for s in (0, 1, 4):
            cases.append(run_case(lib, n, s, [24] * n))
    cases.append(run_case(lib, 4, 0, [12, 24, 24, 24]))       # replica 0 retires half way
    cases.append(run_case(lib, 4, 1, [24, 24, 24, 12]))       # so does the slow one
    with open(sys.argv[1], "w") as f:
        json.dump(cases, f)


if __name__ == "__main__":
    main()
