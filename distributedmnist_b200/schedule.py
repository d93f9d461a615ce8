"""Learning-rate schedule: staircase exponential decay with the /K rule, or a cosine decay, with an optional linear warmup.

reference: src/distributed_train.py:143-156 --
``decay_steps = int(num_batches_per_epoch * num_epochs_per_decay / num_replicas_to_aggregate)``
and ``tf.train.exponential_decay(lr0, global_step, decay_steps, factor, staircase=True)``.
The value is a host scalar handed to the fused allreduce+SGD kernel each step
(SURVEY §2.4 K12) -- it never needs a device op.
"""
from __future__ import annotations

import math


def decay_steps_for(num_examples: int, batch_size: int, num_epochs_per_decay: float,
                    num_replicas_to_aggregate: int) -> int:
    num_batches_per_epoch = num_examples / float(batch_size)
    steps = int(num_batches_per_epoch * num_epochs_per_decay / num_replicas_to_aggregate)
    # The reference lets this reach 0 only for absurd settings; TF would then
    # divide by zero. Clamp to 1 so the schedule stays defined.
    return max(steps, 1)


def exponential_decay(initial_learning_rate: float, global_step: int, decay_steps: int,
                      decay_rate: float, staircase: bool = True) -> float:
    p = global_step / float(decay_steps)
    if staircase:
        p = float(global_step // decay_steps)
    return float(initial_learning_rate) * (float(decay_rate) ** p)


def cosine_decay(global_step: int, decay_steps: int, alpha: float) -> float:
    """TF's ``tf.train.cosine_decay`` factor ``(1 - alpha) * c + alpha``, c = (1 + cos(pi * min(s, T) / T)) / 2, written
    as ``c = sin(pi * q)^2``, q = (T - min(s, T)) / (2T): the same value without the cancellation of 1 + cos near T, and
    exactly ``alpha`` from T on.  The operations are those of ``cta_scale`` (csrc/fused_sync.cuh), in the same order."""
    t = int(decay_steps)
    q = (t - min(int(global_step), t)) / (2 * t)
    v = math.sin(math.pi * q)
    return (1.0 - alpha) * (v * v) + alpha


def warmup_factor(global_step: int, warmup_steps: int, warmup_start: float) -> float:
    """Linear warmup ``f0 + ((1 - f0) * s) / W`` for s < W, else 1.0 (``torch.optim.lr_scheduler.LinearLR``)."""
    s = int(global_step)
    if s >= warmup_steps:
        return 1.0
    return warmup_start + ((1.0 - warmup_start) * s) / warmup_steps


class LearningRateSchedule:
    """Callable ``step -> lr`` built from the reference's flags.

    ``cuts`` (``--lr_plateau_patience``, lr_plateau.py): the global steps S_k from which a cut of the rate by ``factor``
    takes effect.  With c(s) of them <= s the rate is ``lr0 * decay^p * factor^c(s)``, the product in that order in double
    (``cta_scale`` in csrc/fused_sync.cuh computes the same); with no cut in effect it is the staircase decay alone.  The
    training loop appends to ``cuts`` as the cuts are decided.

    ``warmup_steps`` W > 0 (``--lr_warmup_steps``) multiplies the rate by :func:`warmup_factor` from ``warmup_start``;
    ``cosine_steps`` T > 0 (``--lr_cosine_decay_steps``) replaces ``decay^p`` by :func:`cosine_decay` with the floor
    ``cosine_alpha``.  The rate is then ``lr0 * D(s) * Wf(s) * factor^c(s)``, left to right in double.  Both count global
    steps from 0, so the warmup multiplies the cosine's first W steps."""

    def __init__(self, initial_learning_rate: float, decay_steps: int, decay_rate: float,
                 staircase: bool = True, factor: float = 1.0, cuts=(), warmup_steps: int = 0,
                 warmup_start: float = 1.0 / 3, cosine_steps: int = 0, cosine_alpha: float = 0.0):
        self.initial_learning_rate = float(initial_learning_rate)
        self.decay_steps = int(decay_steps)
        self.decay_rate = float(decay_rate)
        self.staircase = staircase
        self.factor = float(factor)
        self.cuts = [int(s) for s in cuts]
        self.warmup_steps = int(warmup_steps)
        self.warmup_start = float(warmup_start)
        self.cosine_steps = int(cosine_steps)
        self.cosine_alpha = float(cosine_alpha)

    @classmethod
    def from_flags(cls, flags, num_examples: int, num_replicas_to_aggregate: int) -> "LearningRateSchedule":
        return cls(flags.initial_learning_rate,
                   decay_steps_for(num_examples, flags.batch_size, flags.num_epochs_per_decay,
                                   num_replicas_to_aggregate),
                   flags.learning_rate_decay_factor,
                   warmup_steps=getattr(flags, "lr_warmup_steps", 0),
                   warmup_start=getattr(flags, "lr_warmup_start_factor", 1.0 / 3),
                   cosine_steps=getattr(flags, "lr_cosine_decay_steps", 0),
                   cosine_alpha=getattr(flags, "lr_cosine_alpha", 0.0))

    @property
    def shaped(self) -> bool:
        """A warmup or a cosine decay is on (the aggregation kernels then need it armed in their control block)."""
        return self.warmup_steps > 0 or self.cosine_steps > 0

    def describe(self) -> dict:
        """The schedule's shape: W, f0, T, alpha."""
        return dict(warmup_steps=self.warmup_steps, warmup_start_factor=self.warmup_start,
                    cosine_decay_steps=self.cosine_steps, cosine_alpha=self.cosine_alpha)

    def __call__(self, global_step: int) -> float:
        s = int(global_step)
        if self.cosine_steps > 0:
            lr = self.initial_learning_rate * cosine_decay(s, self.cosine_steps, self.cosine_alpha)
        else:
            lr = exponential_decay(self.initial_learning_rate, s, self.decay_steps, self.decay_rate, self.staircase)
        if s < self.warmup_steps:
            lr = lr * warmup_factor(s, self.warmup_steps, self.warmup_start)
        c = sum(1 for x in self.cuts if x <= s)
        return lr * self.factor ** c if c else lr
