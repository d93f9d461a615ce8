"""Continuous evaluator: polls a checkpoint directory, scores the 10k validation set.

reference: src/nn_eval.py -- ``evaluate(dataset)`` (:117-140) loops ``do_eval``
(:49-115): read the ``checkpoint`` state, restore, skip when the step equals the
previous one (:84-88), one forward over the whole set, print
``Num examples: %d  Precision @ 1: %f Loss: %f Time: %f`` (:102-103, scraped by
tools/benchmark.py:151), write the two scalar summaries (:107-110), sleep
``--eval_interval_secs`` unless ``--run_once`` (:136-140).  The time axis is
seconds since the evaluator process started (:47).

Precision is the plain top-1 fraction; the reference divides an already-mean
accuracy by the batch size a second time (:124; SURVEY §5.9 item 4), which is a
bug we do not reproduce.
"""
from __future__ import annotations

import sys
import time
from typing import Optional

import torch

from . import moving_average
from .checkpoint import Saver, get_checkpoint_state, resolve_checkpoint_path
from .engine import TorchEngine
from .flags import FLAGS
from .utils.summary import SummaryWriter

start_time = time.time()


def _make_eval_engine(flags, device: torch.device):
    if device.type == "cuda" and flags.backend in ("auto", "fused"):
        from .engine_cuda import make_cuda_eval_engine
        return make_cuda_eval_engine(flags, device)
    return TorchEngine(flags.model, 1, device, lambda n: torch.zeros(n, dtype=torch.float32, device=device),
                       seed=flags.seed, keep_prob=flags.dropout_keep_prob, mlp_hidden=flags.mlp_hidden)


def do_eval(engine, writer: Optional[SummaryWriter], data_set, flags=FLAGS, prev_global_step=-1):
    """One evaluation against the full validation set.  Returns the step evaluated
    (as the string taken from the file name, like the reference), the previous
    step when nothing new exists, or -1 when there is no checkpoint."""
    ckpt = get_checkpoint_state(flags.checkpoint_dir)
    if not (ckpt and ckpt.model_checkpoint_path):
        print("No checkpoint file found")
        sys.stdout.flush()
        return -1
    path = resolve_checkpoint_path(flags.checkpoint_dir, ckpt)
    global_step = ckpt.model_checkpoint_path.split("/")[-1].split("-")[-1]
    if prev_global_step == global_step:   # don't evaluate the same checkpoint twice
        return prev_global_step
    try:
        state, _ = Saver.restore(path)
    except (OSError, ValueError, KeyError) as e:   # checkpoint being rotated under us
        print("Could not restore %s: %s" % (path, e))
        sys.stdout.flush()
        return prev_global_step
    if getattr(flags, "eval_moving_average", False):
        # TF's variables_to_restore(): every variable is loaded from its moving average
        flat = moving_average.from_state_dict(engine.spec, state)
        if flat is None:
            print("Could not restore %s: the checkpoint holds no moving averages (<variable>%s); it was written without "
                  "--moving_average_decay" % (path, moving_average.SUFFIX))
            sys.stdout.flush()
            return prev_global_step
        engine.params.copy_(flat.to(engine.params.device))
    else:
        engine.params.copy_(engine.spec.from_state_dict(state).to(engine.params.device))
    if hasattr(engine, "params_updated"):
        engine.params_updated()
    print("Succesfully loaded model from %s at step=%s." % (ckpt.model_checkpoint_path, global_step))
    sys.stdout.flush()

    num_examples = data_set.num_examples
    loss, acc = engine.evaluate(data_set.images, data_set.labels)
    print("Num examples: %d  Precision @ 1: %f Loss: %f Time: %f"
          % (num_examples, acc, loss, time.time() - start_time))
    sys.stdout.flush()
    if writer is not None:
        writer.add_scalars({"Validation Accuracy": float(acc), "Validation Loss": float(loss)}, int(global_step))
    return global_step


def evaluate(dataset, flags=FLAGS, device: Optional[torch.device] = None, max_evals: Optional[int] = None):
    """Evaluate checkpoints as they appear (reference nn_eval.py:117-140)."""
    if device is None:
        device = torch.device("cuda", 0) if torch.cuda.is_available() else torch.device("cpu")
    engine = _make_eval_engine(flags, device)
    writer = SummaryWriter(flags.eval_dir)
    step = -1
    n = 0
    while True:
        step = do_eval(engine, writer, dataset, flags, prev_global_step=step)
        n += 1
        if flags.run_once or (max_evals is not None and n >= max_evals):
            break
        time.sleep(flags.eval_interval_secs)
    writer.close()
    return step
