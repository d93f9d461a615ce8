"""Learning-rate cuts at a plateau (``--lr_plateau_patience``, ``--lr_plateau_factor``, ``--lr_plateau_min_delta``).

The rule lives in :func:`advance`.  ``eval_plateau`` (csrc/eval_plateau.cu) applies it on the device as the last node of
the chief's evaluation pass and stores each cut's step into every replica's cut table; the torch engine applies it on the
host after ``evaluate``; the training loop replays it over the pass records for its log, summary, file and restarts; the
kernel tests compare the device words against it.

A pass *counts* when :func:`best.counts` says so.  The first counting pass sets the baseline; after it, a counting pass
with ``correct > best + min_delta_rows`` becomes the best and resets the count of passes since the best, and any other
counting pass adds one to it.  When that count reaches the patience P, the pass's global step g triggers a *cut*: the
count restarts from 0, the best is kept (as Keras's ReduceLROnPlateau keeps it), and the cut takes effect from global step
S = g + STOP_MARGIN.  At most :data:`MAX_CUTS` cuts are made per run; a later trigger restarts the count but cuts nothing.
A pass that does not count changes nothing.

With c(s) cuts whose S <= s, the update of the weights of global step s uses
``lr0 * decay^floor(s / decay_steps) * F^c(s) / count`` (:class:`~distributedmnist_b200.schedule.LearningRateSchedule`).
"""
from __future__ import annotations

from typing import NamedTuple, Optional, Tuple

from . import best

# csrc/fused_sync.cuh SYNC_MAX_CUTS: the entries of a replica's cut table
MAX_CUTS = 32
NO_CUT = 0xFFFFFFFF            # a table entry no cut has been stored into

# PlateauState (csrc/eval_plateau.cu) as 32-bit words
PL_BEST_WORD, PL_SINCE_WORD, PL_BASELINE_WORD, PL_CUTS_WORD, PL_TRIGGER_WORD = 0, 1, 2, 3, 4

LR_PLATEAU_JSON = "worker%d_lr_plateau.json"


class State(NamedTuple):
    """PlateauState: the correct count to beat, counting passes since the best or the last trigger, whether a counting
    pass has set the baseline, the cuts made so far, and the step of the last pass that triggered (0 until one did)."""
    best: int = 0
    since: int = 0
    baseline: bool = False
    cuts: int = 0
    trigger_step: int = 0


def advance(state: State, step: int, correct: int, examples: int, n: int, patience: int, delta_rows: int,
            status: Optional[int] = None) -> Tuple[State, bool]:
    """One evaluation pass of global ``step`` with ``correct`` of ``examples`` rows over a validation set of ``n`` rows
    (``status`` as :func:`best.counts` takes it).  Returns the new state and True if the pass triggered, whether or not
    the trigger made a cut (it did when the new state's ``cuts`` is larger)."""
    if not best.counts(examples, n, status):
        return state, False
    if not state.baseline or correct > state.best + delta_rows:
        return state._replace(best=correct, since=0, baseline=True), False
    since = state.since + 1
    if since < patience:
        return state._replace(since=since), False
    return state._replace(since=0, trigger_step=step, cuts=min(state.cuts + 1, MAX_CUTS)), True
