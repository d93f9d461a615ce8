"""Helper process for the multi-GPU snapshot-evaluation tests (one rank per GPU): trains through ``train.train`` with the
flags given on the command line, keeping the chief's last accepted weight snapshot (``CudaLeNetEngine.SNAP_KEEP``).  Once
every replica has finished (a barrier after the device drained, so no push is in flight) it saves the replica's parameter
arena to ``argv[1]`` (RANK replaced) and, on the chief, scores the kept snapshot with a standalone live pass."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributedmnist_b200 import data as mnist_data  # noqa: E402
from distributedmnist_b200.engine_cuda import CudaLeNetEngine  # noqa: E402
from distributedmnist_b200.flags import FLAGS  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.train import train  # noqa: E402


def main():
    out = sys.argv[1].replace("RANK", os.environ["RANK"])
    FLAGS.parse(sys.argv[2:])
    CudaLeNetEngine.SNAP_KEEP = True
    ctx = init_context(FLAGS)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=ctx.rank, n_workers=ctx.world_size, seed=FLAGS.seed,
                               synthetic=FLAGS.synthetic_data, fake_data=FLAGS.fake_data)
    res = train(ctx, ds.train, ds.validation, FLAGS)
    eng = res["engine"]
    torch.cuda.synchronize()
    eng.backend.barrier()                   # every replica's last push has landed everywhere
    np.save(out + ".npy", res["params"].detach().cpu().numpy())
    meta = {"rank": ctx.rank, "final_step": res["final_step"], "dropped_steps": res["dropped"],
            "accepted_steps": res["accepted"], "evals": [list(r) for r in res.get("evals", [])]}
    kept = eng.eval_snapshot() if getattr(eng, "_snapshot", False) else None
    if kept is not None:
        snap, step = kept
        meta["eval_dropped"] = eng.eval_dropped
        meta["snapshot_stats"] = eng.eval_snapshot_stats()
        eng.params.copy_(snap)                # local arena only; the peers are past their last step
        eng.params_updated()
        eng.arm_eval(ds.validation.images, ds.validation.labels)
        meta["kept_step"] = step
        meta["standalone"] = list(eng.run_eval())
    eng.backend.barrier()
    with open(out + ".json", "w") as f:
        json.dump(meta, f)
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
