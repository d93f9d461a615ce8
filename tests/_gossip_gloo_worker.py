"""Helper process for the gossip-SGD gloo tests: runs the training driver with ``--gossip_method`` and records, after
every step, the replica's global step, its half step and its weights after the mix."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributedmnist_b200 import data as mnist_data  # noqa: E402
from distributedmnist_b200.flags import FLAGS  # noqa: E402
from distributedmnist_b200.parallel import aggregators as G  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.train import train  # noqa: E402


def main():
    out_npz = sys.argv[1]
    FLAGS.parse(sys.argv[2:])
    torch.set_num_threads(1)
    ctx = init_context(FLAGS, want_gpu=False)
    after, half, steps = [], [], []
    cls = G.GossipSGDOptimizer if FLAGS.gossip_method else G.LocalSGDOptimizer
    orig_apply = cls.apply_gradients

    def apply(self, params, grads):
        info = orig_apply(self, params, grads)
        after.append(params.detach().clone().numpy())
        if FLAGS.gossip_method:
            half.append(self.half_step.detach().clone().numpy())
        steps.append(info.global_step)
        return info
    cls.apply_gradients = apply
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=ctx.rank, n_workers=ctx.world_size, seed=FLAGS.seed,
                               synthetic=True, synthetic_sizes=(512, 128))
    res = train(ctx, ds.train, ds.validation, FLAGS)
    stack = lambda xs: np.stack(xs) if xs else np.zeros((0, res["params"].numel()), np.float32)   # noqa: E731
    np.savez(out_npz, after=stack(after), half=stack(half), steps=np.array(steps, dtype=np.int64),
             final=res["params"].numpy(), final_step=res["final_step"],
             report=json.dumps(res.get("gossip", res.get("local_sgd"))))
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
