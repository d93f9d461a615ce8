"""Helper process for the multi-GPU moving-average test (one rank per GPU): trains through ``train.train`` with the flags
given on the command line, then saves the replica's parameter arena to ``argv[1]`` (RANK replaced) with its launches per
step and whether its engine keeps an average."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributedmnist_b200 import data as mnist_data  # noqa: E402
from distributedmnist_b200.flags import FLAGS  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.train import train  # noqa: E402


def main():
    out = sys.argv[1].replace("RANK", os.environ["RANK"])
    FLAGS.parse(sys.argv[2:])
    ctx = init_context(FLAGS)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=ctx.rank, n_workers=ctx.world_size, seed=FLAGS.seed,
                               synthetic=FLAGS.synthetic_data, fake_data=FLAGS.fake_data)
    res = train(ctx, ds.train, ds.validation, FLAGS)
    eng = res["engine"]
    torch.cuda.synchronize()
    eng.backend.barrier()
    np.save(out + ".npy", res["params"].detach().cpu().numpy())
    meta = {"rank": ctx.rank, "final_step": res["final_step"], "launches_per_step": eng.launches_per_step,
            "average": eng._ema is not None}
    if eng._ema is not None:
        avg, step = eng.moving_average()
        np.save(out + "_average.npy", avg.cpu().numpy())
        meta["average_step"] = step
    eng.backend.barrier()
    with open(out + ".json", "w") as f:
        json.dump(meta, f)
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
