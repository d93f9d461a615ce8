"""L2 weight decay of the fully connected layers (``--weight_decay``).

The reference model carries the TF MNIST tutorial's regulariser, commented out (src/mnist.py:142-143):
``l2_loss(fc1_weights) + l2_loss(fc1_biases) + l2_loss(fc2_weights) + l2_loss(fc2_biases)``, with ``l2_loss(v) =
sum(v^2) / 2``.  With ``--weight_decay=lambda`` the objective each replica differentiates is ``CE + lambda * R``, R the
sum of ``l2_loss`` over the decayed variables, so the gradient of a decayed variable gains ``lambda * v`` -- inside each
replica's own gradient, at the weights its forward read, as in TF's graph.  Nothing is stateful: the aggregation, the
checkpoints and the learning-rate schedule do not change.

The decayed variables are the fully connected layers: lenet's four (the conv layers are not decayed), and every variable
of mlp2 / mlp3.  The logged training loss becomes ``CE + lambda * R``; the in-training evaluation and the evaluator
score CE only, as the reference's evaluator scores ``mnist.loss``.

Where it runs: the torch engine adds ``lambda * R`` to its loss (every model); the sm_90a engine adds ``lambda * v`` in
the epilogues of the lenet fc weight-gradient kernels and ``(float)(lambda * R)`` to the step's loss word
(``CudaLeNetEngine.arm_weight_decay``).  The sm_90a MLP engine does not implement it and refuses the flag.
"""
from __future__ import annotations

import math
from typing import List

import numpy as np

from .models.spec import ModelSpec, ParamSpec

# lenet's decayed variables, the four of the reference's regulariser
LENET_DECAYED = ("fc1_weights", "fc1_biases", "fc2_weights", "fc2_biases")


def decayed(spec: ModelSpec) -> List[ParamSpec]:
    """The parameters of ``spec`` whose gradients gain ``lambda * v``, in arena order."""
    if spec.name == "lenet":
        return [p for p in spec.params if p.name in LENET_DECAYED]
    return [p for p in spec.params if p.name.startswith("fc")]      # mlp2 / mlp3: every layer is fully connected


def value(flags) -> float:
    """``--weight_decay`` as the one fp32 value the engines use (0.0: off).  Raises ValueError unless 0 <= lambda < 1
    and finite."""
    lam = float(getattr(flags, "weight_decay", 0.0) or 0.0)
    if not math.isfinite(lam) or not 0.0 <= lam < 1.0:
        raise ValueError("--weight_decay must be finite and lie in [0, 1) (0 = off), got %r" % lam)
    f = float(np.float32(lam))
    if f >= 1.0 or (lam > 0.0 and f == 0.0):
        raise ValueError("--weight_decay=%r rounds to %r in float32, outside (0, 1)" % (lam, f))
    return f


def check_flags(flags, ctx) -> None:
    """``--weight_decay`` values and combinations that cannot work, rejected before any device work starts."""
    lam = value(flags)
    if lam == 0.0:
        return
    if ctx.on_gpu and flags.backend in ("auto", "fused") and flags.model != "lenet":
        raise ValueError("--weight_decay on the GPU path is implemented for lenet, not --model=%s: the MLP bias gradients "
                         "are accumulated with atomics, which the decay term would need to follow (the torch engine, "
                         "--backend=nccl or gloo, decays every model)" % flags.model)
