"""Helper process: one replica of a stale-synchronous training run (``train()`` with ``--async_method`` and
``--ssp_staleness``) on its own GPU, lenet on the synthetic set, with a fixed device-side delay on the replica the
straggler spec names.

argv: <train_dir> <out json with RANK placeholder> <max_steps> <--inject_straggler spec> <s>"""
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from distributedmnist_b200 import data as mnist_data  # noqa: E402
from distributedmnist_b200.flags import FLAGS  # noqa: E402
from distributedmnist_b200.parallel.context import init_context, shutdown_context  # noqa: E402
from distributedmnist_b200.train import train  # noqa: E402


def _sha(t):
    return hashlib.sha1(t.detach().cpu().numpy().tobytes()).hexdigest()


def main():
    train_dir, out_json, max_steps, straggler, s = sys.argv[1], sys.argv[2], int(sys.argv[3]), sys.argv[4], int(sys.argv[5])
    rank = int(os.environ.get("RANK", "0"))
    FLAGS.parse(["--train_dir=%s" % train_dir, "--batch_size=128", "--max_steps=%d" % max_steps, "--async_method",
                 "--ssp_staleness=%d" % s, "--inject_straggler=%s" % straggler, "--save_interval_secs=1000",
                 "--log_every=100", "--initial_learning_rate=0.01"])
    ctx = init_context(FLAGS, want_gpu=True)
    ds = mnist_data.load_mnist(FLAGS.data_dir, worker_id=ctx.rank, n_workers=ctx.world_size, seed=FLAGS.seed,
                               synthetic=True, synthetic_sizes=(8192, 1024))
    res = train(ctx, ds.train, ds.validation, FLAGS)
    eng = res["engine"]
    torch.cuda.synchronize()
    st, b = res["staleness"], res["ssp"]
    json.dump({"rank": rank, "final_step": res["final_step"], "updates": st["updates"], "max_tau": st["max"],
               "lead_max": b["lead_max"], "waits": b["waits"], "params": _sha(eng.params), "master": _sha(eng._master),
               "nvls": bool(eng.backend.use_nvls and eng._master is not None
                            and eng.backend._by_ptr[eng._master.data_ptr()].multicast_ptr)},
              open(out_json.replace("RANK", str(rank)), "w"))
    shutdown_context(ctx)


if __name__ == "__main__":
    main()
