"""Helper process: one replica of a local-SGD training run (``train()`` with ``--local_sgd_steps``) on its own GPU, lenet
on the synthetic set, without the step pipeline and without CUDA graphs so that the weights can be recorded after every
step.  Records, after every step, the global step and the replica's weights, and the weights the step's update produced
before any average (the copy that entered the average on an averaging step).

argv: <train_dir> <out npz with RANK placeholder> <extra flags...>"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributedmnist_b200 import data as mnist_data  # noqa: E402
from distributedmnist_b200.engine_cuda import _CudaEngine  # noqa: E402
from distributedmnist_b200.flags import FLAGS  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.parallel.fused import FusedBackend  # noqa: E402
from distributedmnist_b200.train import train  # noqa: E402


def main():
    train_dir, out = sys.argv[1], sys.argv[2]
    rank = int(os.environ.get("RANK", "0"))
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=128", "--save_interval_secs=1000", "--log_every=100",
                 "--initial_learning_rate=0.05", "--pipeline_steps=false", "--use_cuda_graph=false"] + sys.argv[3:])
    ctx = init_context(FLAGS, want_gpu=True)
    after, before, steps = [], [], []
    orig_step, orig_train = FusedBackend.enqueue_local_step, _CudaEngine.train_step

    def local_step(self, params, *a, **k):
        orig_step(self, params, *a, **k)
        torch.cuda.synchronize()
        before.append(params.detach().cpu().numpy().copy())

    def train_step(self):
        orig_train(self)
        torch.cuda.synchronize()
        after.append(self.params.detach().cpu().numpy().copy())
        steps.append(self.backend.device_epoch)
    FusedBackend.enqueue_local_step, _CudaEngine.train_step = local_step, train_step
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=ctx.rank, n_workers=ctx.world_size, seed=FLAGS.seed,
                               synthetic=True, synthetic_sizes=(8192, 1024))
    res = train(ctx, ds.train, ds.validation, FLAGS)
    eng = res["engine"]
    torch.cuda.synchronize()
    np.savez(out.replace("RANK", str(rank)), after=np.stack(after), before=np.stack(before), steps=np.array(steps),
             final=eng.params.detach().cpu().numpy(), final_step=res["final_step"], report=json.dumps(res["local_sgd"]),
             nvls=bool(eng.backend._local_mc(eng.params)))
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
