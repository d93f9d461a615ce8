"""Evaluator binary: wipe eval_dir, then score checkpoints as they appear.

Command-line compatible with the reference's src/mnist_eval.py:30-35
(``--eval_dir --checkpoint_dir --eval_interval_secs --run_once``).  ``--eval_moving_average`` scores each checkpoint's
``<variable>/ExponentialMovingAverage`` tensors instead of its weights, and skips a checkpoint that has none.
"""
import _bootstrap  # noqa: F401

import os
import shutil

from distributedmnist_b200 import data as mnist_data
from distributedmnist_b200 import evaluator as nn_eval
from distributedmnist_b200.flags import FLAGS, app_run


def main(unused_argv=None):
    dataset = mnist_data.load_mnist(FLAGS.data_dir, seed=FLAGS.seed, synthetic=FLAGS.synthetic_data,
                                    fake_data=FLAGS.fake_data)
    if os.path.exists(FLAGS.eval_dir):
        shutil.rmtree(FLAGS.eval_dir)
    os.makedirs(FLAGS.eval_dir)
    nn_eval.evaluate(dataset.validation, FLAGS)
    return 0


if __name__ == "__main__":
    app_run(main)
