"""Helper process: message-passing litmus (csrc/litmus.cu) between rank 0 (writer) and rank 1 (reader)."""
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from distributedmnist_b200.ops.lib import load, stream_ptr  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.parallel.symm_mem import SymmetricBuffer, allocate_symmetric  # noqa: E402


def main():
    out_json = sys.argv[1].replace("RANK", os.environ["RANK"])
    rounds = int(sys.argv[2])
    ctx = init_context(None, want_gpu=True)
    n, r = ctx.world_size, ctx.rank
    lib = load()
    lib.dm_set_device(ctx.device.index or 0)
    numel = 4096
    data = allocate_symmetric(numel * 4, r, n, ctx.device, want_multicast=True)     # VMM + NVLS multicast when available
    flags = SymmetricBuffer(4096, r, n, ctx.device)                                # like the control block: cudaMalloc + IPC
    result = torch.zeros(4, dtype=torch.int64, device=ctx.device)
    torch.cuda.synchronize()
    import torch.distributed as dist
    dist.barrier()
    if r < 2:
        peer = 1 - r
        lib.dm_litmus_mp(r, ctypes.c_void_p(data.local_ptr), ctypes.c_void_p(data.peer_ptrs[0]),
                         ctypes.c_void_p(data.multicast_ptr if n == 2 else 0), ctypes.c_void_p(flags.local_ptr),
                         ctypes.c_void_p(flags.peer_ptrs[peer]), ctypes.c_void_p(result.data_ptr()), numel, rounds,
                         ctypes.c_double(10000.0), stream_ptr())
    torch.cuda.synchronize()
    dist.barrier()
    res = result.cpu().tolist()
    json.dump({"rank": r, "bad_p2p": res[0], "bad_mc": res[1], "rounds": res[2], "aborted": res[3],
               "multicast": bool(data.multicast_ptr), "alloc": type(data).__name__}, open(out_json, "w"))
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
