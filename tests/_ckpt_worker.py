"""Helper process for tests/test_ckpt_capture_gpu.py: trains one replica through ``train.train`` with the flags given on the
command line, then saves the chief's live parameter arena (after the device has drained) to ``argv[1]``."""
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
    FLAGS.parse(sys.argv[2:])
    ctx = init_context(FLAGS)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=ctx.rank, n_workers=ctx.world_size, seed=FLAGS.seed,
                               synthetic=FLAGS.synthetic_data, fake_data=FLAGS.fake_data)
    res = train(ctx, ds.train, ds.validation, FLAGS)
    torch.cuda.synchronize()
    np.save(sys.argv[1], res["params"].detach().cpu().numpy())
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
