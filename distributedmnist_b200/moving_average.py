"""Exponential moving average of the weights (``--moving_average_decay``): the formula, its float32 emulation and the
checkpoint names.

TF's ``ExponentialMovingAverage(decay, num_updates=global_step)``, which the reference's optimizers take as
``variable_averages`` / ``variables_to_average`` (sync_replicas_optimizer_modified.py:150-185): after the update that
produces global step g the chief moves every average towards the weights of step g,

    d = min(D, (1 + g) / (10 + g))       (double)
    m = float32(1 - d)
    s = s - (s - w) * m                  (float32, each operation rounded on its own)

The sm_90a kernel (csrc/moving_average.cu) and the torch engine compute exactly this, so :func:`emulate` reproduces both
bit for bit.  A checkpoint holds the average of variable ``v`` as ``v/ExponentialMovingAverage`` (TF's name).
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

SUFFIX = "/ExponentialMovingAverage"


def multiplier(decay: float, global_step: int) -> np.float32:
    """``m = float32(1 - min(D, (1 + g) / (10 + g)))``."""
    g = float(int(global_step))
    return np.float32(1.0 - min(float(decay), (1.0 + g) / (10.0 + g)))


def emulate(shadow: np.ndarray, weights: np.ndarray, decay: float, global_step: int) -> np.ndarray:
    """One update in float32 numpy: the new shadow (the inputs are not modified)."""
    s = np.asarray(shadow, dtype=np.float32)
    w = np.asarray(weights, dtype=np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        return (s - (s - w) * multiplier(decay, global_step)).astype(np.float32)


def names(spec):
    """Checkpoint names of the averages, in the order of ``spec.ckpt_names()``."""
    return [n + SUFFIX for n in spec.ckpt_names()]


def to_state_dict(spec, flat: torch.Tensor) -> Dict[str, torch.Tensor]:
    """``<ckpt_name>/ExponentialMovingAverage`` -> contiguous CPU fp32 tensor, from an average arena."""
    return {n + SUFFIX: t for n, t in spec.to_state_dict(flat).items()}


def from_state_dict(spec, state: Dict[str, torch.Tensor]) -> Optional[torch.Tensor]:
    """The average arena of a restored state dict, or None unless it holds the average of every variable."""
    if not all(n in state for n in names(spec)):
        return None
    return spec.from_state_dict({n: state[n + SUFFIX] for n in spec.ckpt_names()})
