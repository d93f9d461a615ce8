"""Learning-rate schedule: staircase exponential decay with the /K rule.

reference: src/distributed_train.py:143-156 --
``decay_steps = int(num_batches_per_epoch * num_epochs_per_decay / num_replicas_to_aggregate)``
and ``tf.train.exponential_decay(lr0, global_step, decay_steps, factor, staircase=True)``.
The value is a host scalar handed to the fused allreduce+SGD kernel each step
(SURVEY §2.4 K12) -- it never needs a device op.
"""
from __future__ import annotations


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


class LearningRateSchedule:
    """Callable ``step -> lr`` built from the reference's flags.

    ``cuts`` (``--lr_plateau_patience``, lr_plateau.py): the global steps S_k from which a cut of the rate by ``factor``
    takes effect.  With c(s) of them <= s the rate is ``lr0 * decay^p * factor^c(s)``, the product in that order in double
    (``cta_scale`` in csrc/fused_sync.cuh computes the same); with no cut in effect it is the staircase decay alone.  The
    training loop appends to ``cuts`` as the cuts are decided."""

    def __init__(self, initial_learning_rate: float, decay_steps: int, decay_rate: float,
                 staircase: bool = True, factor: float = 1.0, cuts=()):
        self.initial_learning_rate = float(initial_learning_rate)
        self.decay_steps = int(decay_steps)
        self.decay_rate = float(decay_rate)
        self.staircase = staircase
        self.factor = float(factor)
        self.cuts = [int(s) for s in cuts]

    @classmethod
    def from_flags(cls, flags, num_examples: int, num_replicas_to_aggregate: int) -> "LearningRateSchedule":
        return cls(flags.initial_learning_rate,
                   decay_steps_for(num_examples, flags.batch_size, flags.num_epochs_per_decay,
                                   num_replicas_to_aggregate),
                   flags.learning_rate_decay_factor)

    def __call__(self, global_step: int) -> float:
        lr = exponential_decay(self.initial_learning_rate, int(global_step), self.decay_steps,
                               self.decay_rate, self.staircase)
        c = sum(1 for s in self.cuts if s <= int(global_step))
        return lr * self.factor ** c if c else lr
