"""Helper process for the sampled-straggler GPU tests (one rank per GPU): trains through ``train.train`` with the flags given
on the command line, then saves the replica's parameter arena to ``argv[1]``.npy (RANK replaced) and, to ``argv[1]``.json,
its accepted / dropped step counts, its straggler stream key and the (iteration, drawn, spun) entries of the device ring."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributedmnist_b200 import data as mnist_data  # noqa: E402
from distributedmnist_b200.flags import FLAGS  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.parallel.straggler import seed_mix  # noqa: E402
from distributedmnist_b200.train import train  # noqa: E402


def main():
    out = sys.argv[1].replace("RANK", os.environ["RANK"])
    FLAGS.parse(sys.argv[2:])
    ctx = init_context(FLAGS)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=ctx.rank, n_workers=ctx.world_size, seed=FLAGS.seed,
                               synthetic=FLAGS.synthetic_data, fake_data=FLAGS.fake_data)
    res = train(ctx, ds.train, ds.validation, FLAGS)
    be = res["engine"].backend
    torch.cuda.synchronize()
    be.barrier()                            # every replica's last push has landed everywhere
    np.save(out + ".npy", res["params"].detach().cpu().numpy())
    j, drawn, spun = be.straggler_samples()
    with open(out + ".json", "w") as f:
        json.dump({"rank": ctx.rank, "final_step": res["final_step"], "accepted_steps": res["accepted"],
                   "dropped_steps": res["dropped"], "seed_mix": seed_mix(FLAGS.seed, ctx.rank),
                   "j": j.tolist(), "drawn": drawn.tolist(), "spun": spun.tolist()}, f)
    be.barrier()
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
