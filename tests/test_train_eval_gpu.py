"""End-to-end on one GPU: reference-compatible entrypoints train the convnet with the sm_90a engine,
checkpoint in the reference's layout, and the evaluator scores it (SURVEY §4 item 5)."""
import os
import re
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_train_checkpoint_evaluate(tmp_path):
    train_dir, eval_dir = str(tmp_path / "train_dir"), str(tmp_path / "eval_dir")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="0")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(k, None)
    tr = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_distributed_train.py"), "--job_name=worker",
                         "--task_id=0", "--worker_hosts=localhost:1234", "--ps_hosts=localhost:1235",
                         "--batch_size=128", "--max_steps=300", "--initial_learning_rate=0.05",
                         "--learning_rate_decay_factor=1", "--train_dir=" + train_dir, "--log_every=50",
                         "--timeline_logging=false"], env=env, capture_output=True, text=True, timeout=600)
    log = tr.stdout + tr.stderr
    assert tr.returncode == 0, log[-3000:]
    steps = [int(x) for x in re.findall(r"Worker 0: .*: step ([0-9]+), loss = ", log)]
    assert steps and max(steps) >= 250, log[-2000:]
    losses = [float(x) for x in re.findall(r"loss = ([0-9.]+),", log)]
    assert losses[-1] < 0.5 * losses[0], losses
    assert os.path.exists(os.path.join(train_dir, "checkpoint"))
    assert os.path.exists(os.path.join(train_dir, "model.ckpt-301.index"))
    ev = subprocess.run([sys.executable, os.path.join(ROOT, "src", "mnist_eval.py"), "--run_once=true",
                         "--checkpoint_dir=" + train_dir, "--eval_dir=" + eval_dir], env=env, capture_output=True,
                        text=True, timeout=600)
    out = ev.stdout + ev.stderr
    assert ev.returncode == 0, out[-3000:]
    m = re.search(r"Num examples: 10000  Precision @ 1: ([0-9.]+) Loss: ([0-9.]+) Time: ([0-9.]+)", out)
    assert m and "Succesfully loaded model from model.ckpt-301 at step=301." in out, out[-2000:]
    assert float(m.group(1)) > 0.9, out[-500:]       # synthetic MNIST-shaped data is learnable

