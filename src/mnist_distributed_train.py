"""Train distributed MNIST -- worker / ps entrypoint.

Command-line compatible with the reference's src/mnist_distributed_train.py:15-45
(``--job_name --task_id --ps_hosts --worker_hosts --train_dir ...``).  Under
``torchrun`` the rank/world come from the environment; with the reference's own
flags the replica count is ``len(worker_hosts)`` and the rank is ``--task_id``.
A ``--job_name=ps`` process has nothing to serve (the H100 engine keeps weights
replicated in HBM and aggregates over NVLink), so it logs that and exits 0.
"""
import _bootstrap  # noqa: F401

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200.flags import FLAGS, app_run
from distributedmnist_b200.parallel.context import init_context, shutdown_context
from distributedmnist_b200.train import train
from distributedmnist_b200.utils.logging import get_logger

log = get_logger()


def main(unused_args):
    assert FLAGS.job_name in ("ps", "worker", ""), "job_name must be ps or worker"
    log.info("PS hosts are: %s" % FLAGS.ps_hosts.split(","))
    log.info("Worker hosts are: %s" % FLAGS.worker_hosts.split(","))
    if FLAGS.job_name == "ps":
        log.info("ps task %d: no parameter server in this engine (weights are replicated in HBM, "
                 "gradients aggregate over NVLink); nothing to serve, exiting." % FLAGS.task_id)
        return 0
    ctx = init_context(FLAGS)
    dataset = mnist_data.load_mnist(FLAGS.data_dir, worker_id=ctx.rank, n_workers=ctx.world_size,
                                    seed=FLAGS.seed, synthetic=FLAGS.synthetic_data, fake_data=FLAGS.fake_data)
    train(ctx, dataset.train, dataset.validation, FLAGS)
    shutdown_context(ctx)
    return 0


if __name__ == "__main__":
    app_run(main)
