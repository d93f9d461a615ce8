"""Helper process for the --device_data training tests (one rank per GPU): trains through ``train.train`` on a synthetic set
of ``argv[2]`` rows with the flags that follow, and saves the replica's final parameter arena plus its per-step
(loss, train accuracy) rows to ``argv[1]`` (RANK replaced).

The host-fed pipelined loop packs batches with ONE packer thread here: with two, batches are handed to the engine in the
order their threads finish, so which batch a step trains on is not reproducible and no run could be compared bit for bit."""
import functools
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributedmnist_b200 import data as mnist_data  # noqa: E402
from distributedmnist_b200 import train as train_mod  # noqa: E402
from distributedmnist_b200.flags import FLAGS  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402


def main():
    out = sys.argv[1].replace("RANK", os.environ["RANK"])
    rows = int(sys.argv[2])
    FLAGS.parse(sys.argv[3:])
    train_mod._BatchPacker = functools.partial(train_mod._BatchPacker, workers=1)
    ctx = init_context(FLAGS)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=ctx.rank, n_workers=ctx.world_size, seed=FLAGS.seed,
                               synthetic=True, synthetic_sizes=(rows, 1000))
    res = train_mod.train(ctx, ds.train, ds.validation, FLAGS)
    torch.cuda.synchronize()
    np.save(out + ".npy", res["params"].detach().cpu().numpy())
    acc = np.load(os.path.join(FLAGS.train_dir, "worker%d_time_acc.npy" % ctx.rank))
    with open(out + ".json", "w") as f:
        json.dump({"final_step": res["final_step"], "steps": res["steps"], "losses": res["losses"],
                   "rows": acc[:, 1:].tolist()}, f)                # (train_acc, test_acc, loss); column 0 is wall time
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
