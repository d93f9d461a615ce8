"""Helper process: one replica of a gossip-SGD training run (``train()`` with ``--gossip_method``) on its own GPU, lenet
on the synthetic set.  Saves the final weights (after the run's closing average), the final global step and the report.

argv: <train_dir> <out npz with RANK placeholder> <extra flags...>"""
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
    train_dir, out = sys.argv[1], sys.argv[2]
    rank = int(os.environ.get("RANK", "0"))
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=128", "--save_interval_secs=1000", "--log_every=100",
                 "--initial_learning_rate=0.05", "--gossip_method"] + sys.argv[3:])
    ctx = init_context(FLAGS, want_gpu=True)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=ctx.rank, n_workers=ctx.world_size, seed=FLAGS.seed,
                               synthetic=True, synthetic_sizes=(8192, 1024))
    res = train(ctx, ds.train, ds.validation, FLAGS)
    eng = res["engine"]
    torch.cuda.synchronize()
    np.savez(out.replace("RANK", str(rank)), final=eng.params.detach().cpu().numpy(), final_step=res["final_step"],
             report=json.dumps(res["gossip"]))
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
