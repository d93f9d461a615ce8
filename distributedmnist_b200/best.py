"""Best-scoring weights of the in-training evaluation (``--keep_best_checkpoint``).

The selection rule lives in :func:`improves`: the torch engine applies it on the host after each ``evaluate``, and
:func:`emulate_decide` applies it to the device words ``eval_best_decide`` (csrc/eval_best.cu) reads and writes, which the
kernel tests compare against.
"""
from __future__ import annotations

from typing import Optional, Tuple

# BestState (csrc/eval_best.cu) as 32-bit words: loss_sum (double) in words 0-1, then step, correct, examples, valid
BEST_STEP_WORD, BEST_CORRECT_WORD, BEST_EXAMPLES_WORD, BEST_VALID_WORD = 2, 3, 4, 5

# file names under train_dir: the checkpoint directory of the best weights and the chief's summary of them
BEST_DIR = "best"
BEST_JSON = "worker%d_best.json"


def counts(examples: int, n: int, status: Optional[int] = None) -> bool:
    """True if a pass over ``examples`` rows may be compared with others at all: it scored the whole validation set of
    ``n`` rows, and ``status`` -- None for a pass over the live arena or the moving average; for a snapshot pass its
    SnapState.status -- says the snapshot was accepted (> 0).  The test eval_target and eval_patience apply too."""
    return (status is None or status > 0) and examples == n


def improves(correct: int, examples: int, n: int, best_correct: int, status: Optional[int] = None) -> bool:
    """True if a pass with ``correct`` of ``examples`` rows becomes the new best over ``best_correct``: it counts (see
    :func:`counts`) and beats the best strictly (on ties the earlier pass stays)."""
    return counts(examples, n, status) and correct > best_correct


def emulate_decide(correct: int, examples: int, loss_sum: float, step: int, n: int, best: Tuple,
                   status: Optional[int] = None) -> Tuple[Tuple, int]:
    """``eval_best_decide`` on the host: ``best`` = BestState as ``(step, correct, examples, loss_sum, valid)``; returns
    the new BestState and the decision word."""
    if not improves(correct, examples, n, best[1], status):
        return tuple(best), 0
    return (step, correct, examples, loss_sum, 1), 1
