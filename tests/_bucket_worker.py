"""Helper process: a few LeNet training steps on the sm_90a engine, aggregation = bucketed (overlapped) or single kernel.

argv: <out json with RANK placeholder> <steps>.  DMNIST_BUCKET / DMNIST_NVLS select the path."""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from distributedmnist_b200.engine_cuda import CudaLeNetEngine  # noqa: E402
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.parallel.fused import FusedBackend  # noqa: E402
from distributedmnist_b200.schedule import LearningRateSchedule  # noqa: E402


def fp(t):
    return hashlib.sha1(t.detach().cpu().numpy().tobytes()).hexdigest()


def main():
    out_json = sys.argv[1].replace("RANK", os.environ["RANK"])
    steps = int(sys.argv[2])
    ctx = init_context(None, want_gpu=True)
    n, r = ctx.world_size, ctx.rank
    be = FusedBackend(ctx, timeout_ms=10000.0)
    B = 64
    eng = CudaLeNetEngine(B, be, seed=77, rank=r, use_graph=True)
    opt = SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 3, 0.5), n, n)
    eng.attach_optimizer(opt)
    g = torch.Generator().manual_seed(100 + r)          # every replica trains on its own batches
    xs = torch.rand(steps, B, 28, 28, generator=g) - 0.5
    ys = torch.randint(0, 10, (steps, B), generator=g)
    rows = []
    for s in range(steps):
        eng.load_batch(xs[s], ys[s])
        eng.train_step()
        loss, acc = eng.loss_acc()
        info = eng.step_info()
        torch.cuda.synchronize()
        rows.append({"step": info.global_step, "mask": info.mask, "count": info.count, "loss": loss,
                     "fp": fp(eng.params), "shadow_err": (eng.shadow.float() - eng.params).abs().max().item(),
                     "pmax": eng.params.abs().max().item(), "sample": eng.params[::40009].cpu().tolist()})
    be.check_error()
    json.dump({"rank": r, "bucketed": bool(eng._bucketed), "v2": bool(eng._bucket_v2), "nvls": bool(be.nvls_active), "rows": rows,
               "params_sum": eng.params.double().sum().item(), "sample": eng.params[::40009].cpu().tolist()},
              open(out_json, "w"))
    be.close()
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
