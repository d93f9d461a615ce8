"""Helper process for the two-replica learning-rate schedule test (one rank per GPU): lenet steps through the warmup and
the cosine (W = 2, T = 4) at K of 2, then a probe of the single aggregation kernel with weights 0 and gradients 1 at
steps across the schedule, whose committed updates must be fp32(lr(step) / count) * count."""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributedmnist_b200.engine_cuda import CudaLeNetEngine  # noqa: E402
from distributedmnist_b200.ops import aggrefs as A  # noqa: E402
from distributedmnist_b200.parallel.aggregators import SyncReplicasOptimizer  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.parallel.fused import FusedBackend  # noqa: E402
from distributedmnist_b200.schedule import LearningRateSchedule  # noqa: E402


def main():
    out = sys.argv[1].replace("RANK", os.environ["RANK"])
    k = int(sys.argv[2])
    ctx = init_context(None, want_gpu=True)
    n, r = ctx.world_size, ctx.rank
    be = FusedBackend(ctx, timeout_ms=10000.0)
    eng = CudaLeNetEngine(128, be, seed=3, rank=r, use_graph=True)
    sched = LearningRateSchedule(0.05, 2, 0.999, warmup_steps=2, warmup_start=0.25, cosine_steps=4, cosine_alpha=0.1)
    eng.attach_optimizer(SyncReplicasOptimizer(be, sched, k, n))
    assert be.lr_schedule_armed
    gen = torch.Generator().manual_seed(9 + r)
    for _ in range(8):
        eng.load_batch(torch.rand(128, 28, 28, generator=gen) - 0.5, torch.randint(0, 10, (128,), generator=gen))
        eng.train_step()
    torch.cuda.synchronize()
    be.barrier()
    be.check_error()
    res = {"rank": r, "params_fp": hashlib.sha1(eng.params.detach().cpu().numpy().tobytes()).hexdigest(),
           "epoch": be.device_epoch}

    params, grads = be.allocate(1024), be.allocate(1024)
    checked, wrong = 0, []
    for s in (0, 1, 2, 3, 4, 5, 9, 1000):
        params.zero_()
        grads.fill_(1.0)
        torch.cuda.synchronize()
        be.set_global_step(s)                      # synchronises and holds a barrier
        be.enqueue(params, grads, k, sched.initial_learning_rate, sched.decay_rate, sched.decay_steps)
        torch.cuda.synchronize()
        be.barrier()                               # every push of the step has landed in my arena
        st = be.read_status()
        count = st["last_count"]
        got = -params[0].item() / count
        host = sched(s) / count
        if host < A.FLT_MIN:
            ok = got == 0.0
        else:
            assert A.midpoint_distance_ulps(host) > 16, (s, host)
            ok = np.float32(got) == np.float32(host)
        checked += 1
        if not ok:
            wrong.append([s, count, got, float(np.float32(host))])
    be.check_error()
    res.update(probe_checked=checked, probe_wrong=wrong)
    with open(out, "w") as f:
        json.dump(res, f)
    be.close()
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
