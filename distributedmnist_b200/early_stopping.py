"""Early stopping with a patience (``--early_stopping_patience``, ``--early_stopping_min_delta``).

The rule lives in :func:`advance`.  ``eval_patience`` (csrc/eval_patience.cu) applies it on the device as the last node of
the chief's evaluation pass and sets the stop step; the torch engine applies it on the host after ``evaluate``; the
training loop replays it over the pass records for its report; the kernel tests compare the device words against it.

A pass *counts* when :func:`best.counts` says so (the whole validation set, and for a snapshot pass an accepted snapshot).
The first counting pass of the run sets the baseline; after it, a counting pass with ``correct > best + min_delta_rows``
becomes the best and resets the count of passes since the best, and any other counting pass adds one to it.  When that
count reaches the patience P, the pass's global step g exhausts it, the run stops at S = g + STOP_MARGIN, and the state
no longer changes.  A pass that does not count changes nothing.
"""
from __future__ import annotations

import math
from fractions import Fraction
from typing import NamedTuple, Optional, Tuple

from . import best

# PatienceState (csrc/eval_patience.cu) as 32-bit words
PAT_BEST_WORD, PAT_SINCE_WORD, PAT_BEST_STEP_WORD, PAT_TRIGGER_WORD, PAT_BASELINE_WORD = 0, 1, 2, 3, 4

EARLY_STOPPING_JSON = "worker%d_early_stopping.json"


class State(NamedTuple):
    """PatienceState: the correct count to beat, counting passes since the best, the best pass's step, the step of the
    pass that exhausted the patience (0 until then), and whether a counting pass has set the baseline."""
    best: int = 0
    since: int = 0
    best_step: int = 0
    trigger_step: int = 0
    baseline: bool = False


def min_delta_rows(min_delta: float, examples: int) -> int:
    """``--early_stopping_min_delta`` as a row count, exactly (the decimal value of ``min_delta``, rounded down)."""
    return math.floor(Fraction(str(min_delta)) * examples)


def exhausted(state: State, patience: int) -> bool:
    return state.baseline and state.since >= patience


def advance(state: State, step: int, correct: int, examples: int, n: int, patience: int, delta_rows: int,
            status: Optional[int] = None) -> Tuple[State, bool]:
    """One evaluation pass of global ``step`` with ``correct`` of ``examples`` rows over a validation set of ``n`` rows
    (``status`` as :func:`best.counts` takes it).  Returns the new state and True if this pass exhausted the patience."""
    if exhausted(state, patience) or not best.counts(examples, n, status):
        return state, False
    if not state.baseline or correct > state.best + delta_rows:
        return State(correct, 0, step, state.trigger_step, True), False
    since = state.since + 1
    if since < patience:
        return state._replace(since=since), False
    return state._replace(since=since, trigger_step=step), True
