"""Helper process for the CPU/gloo K > N test: runs the real training driver and records every committed update of the
replica (fingerprint of the parameters after it, divisor, own contribution)."""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from distributedmnist_b200 import data as mnist_data  # noqa: E402
from distributedmnist_b200.flags import FLAGS  # noqa: E402
from distributedmnist_b200.parallel import backends as B  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.train import train  # noqa: E402


def main():
    out_json = sys.argv[1].replace("RANK", os.environ.get("RANK", "0"))
    FLAGS.parse(sys.argv[2:])
    torch.set_num_threads(1)
    ctx = init_context(FLAGS, want_gpu=False)
    commits, calls = [], [0]
    orig = B._CollectiveBackend.accumulate_step

    def spy(self, params, grads, lr, local_step, k, delay_s=0.0):
        calls[0] += 1
        info = orig(self, params, grads, lr, local_step, k, delay_s)
        if info.applied:
            commits.append([info.global_step, info.count, info.contributed,
                            hashlib.sha1(params.numpy().tobytes()).hexdigest()])
        return info
    B._CollectiveBackend.accumulate_step = spy
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=ctx.rank, n_workers=ctx.world_size, seed=FLAGS.seed,
                               synthetic=True, synthetic_sizes=(512, 128))
    res = train(ctx, ds.train, ds.validation, FLAGS)
    with open(out_json, "w") as f:
        json.dump({"rank": ctx.rank, "commits": commits, "calls": calls[0], "final_step": res["final_step"],
                   "accepted": res["accepted"], "dropped": res["dropped"], "losses": res["losses"],
                   "final_fp": hashlib.sha1(res["params"].numpy().tobytes()).hexdigest()}, f)
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
