"""Model specification: parameter inventory + flat parameter/gradient arena.

Every model is a list of :class:`ParamSpec` in *creation order*.  The order
matters twice:

* it reproduces the reference's checkpoint names -- none of its variables is
  named, so TF auto-names them ``Variable, Variable_1, ... Variable_7`` in
  creation order (reference src/mnist.py:81-101; SURVEY §2.4 table), and
* it defines the layout of the single flat fp32 arena that holds all weights
  (and, mirrored, all gradients).  The fused allreduce+SGD kernel works on that
  arena as one message, so the contributor set of a K-of-N step is uniform
  across variables (the reference's per-variable accumulators allow it to
  differ, sync_replicas_optimizer_modified.py:289-306).

Tensor layouts inside the arena are exactly the TF layouts (conv HWIO, fc
``[in, out]``): the wgmma kernels consume them natively through K-major /
MN-major shared-memory descriptors, so checkpoints need no transposition.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Tuple

import torch

# Tensor starts are aligned to 64 elements (256 B fp32 / 128 B bf16 shadow) so a
# TMA tensor map can be built on any tensor of the arena; the arena length is a
# multiple of 2048 elements so it shards evenly over 1/2/4/8 ranks in 16-byte
# vectors for any rank count used by the fused kernel.
TENSOR_ALIGN = 64
ARENA_ALIGN = 2048


@dataclass
class ParamSpec:
    name: str                 # human name, e.g. "conv1_weights"
    shape: Tuple[int, ...]
    init: str                 # "truncated_normal" | "zeros" | "constant"
    init_arg: float = 0.0     # stddev or constant
    offset: int = 0           # element offset inside the flat arena (filled by ModelSpec)
    ckpt_name: str = ""       # "Variable", "Variable_1", ... (filled by ModelSpec)

    @property
    def numel(self) -> int:
        return int(math.prod(self.shape))


@dataclass
class ModelSpec:
    name: str
    params: List[ParamSpec]
    input_shape: Tuple[int, ...] = (28, 28, 1)
    num_classes: int = 10
    arena_numel: int = field(init=False, default=0)

    def __post_init__(self) -> None:
        off = 0
        for i, p in enumerate(self.params):
            off = (off + TENSOR_ALIGN - 1) // TENSOR_ALIGN * TENSOR_ALIGN
            p.offset = off
            p.ckpt_name = "Variable" if i == 0 else "Variable_%d" % i
            off += p.numel
        self.arena_numel = (off + ARENA_ALIGN - 1) // ARENA_ALIGN * ARENA_ALIGN

    # ---- inventory ------------------------------------------------------
    @property
    def num_trainable(self) -> int:
        return sum(p.numel for p in self.params)

    def param(self, name: str) -> ParamSpec:
        for p in self.params:
            if p.name == name or p.ckpt_name == name:
                return p
        raise KeyError(name)

    def ckpt_names(self) -> List[str]:
        return [p.ckpt_name for p in self.params]

    # ---- arena views ----------------------------------------------------
    def views(self, flat: torch.Tensor) -> Dict[str, torch.Tensor]:
        """Name -> view (no copy) into a flat arena tensor of ``arena_numel`` elements."""
        assert flat.dim() == 1 and flat.numel() >= self.arena_numel, (flat.shape, self.arena_numel)
        return {p.name: flat[p.offset:p.offset + p.numel].view(p.shape) for p in self.params}

    def valid_mask(self) -> torch.Tensor:
        """Boolean mask of arena elements that belong to a tensor (not padding)."""
        m = torch.zeros(self.arena_numel, dtype=torch.bool)
        for p in self.params:
            m[p.offset:p.offset + p.numel] = True
        return m

    # ---- init -------------------------------------------------------------
    def init_flat(self, seed: int = 66478, device: str = "cpu") -> torch.Tensor:
        """Random-init arena.  Same distributions as the reference (mnist.py:81-101):
        truncated normal (resampled beyond 2 sigma) with stddev 0.1, zeros, or
        constant 0.1.  The generator is seeded explicitly so every replica can
        build bit-identical initial weights without a broadcast (SURVEY §2.5 X10).
        """
        g = torch.Generator(device="cpu")
        g.manual_seed(int(seed))
        flat = torch.zeros(self.arena_numel, dtype=torch.float32)
        for p in self.params:
            dst = flat[p.offset:p.offset + p.numel]
            if p.init == "zeros":
                dst.zero_()
            elif p.init == "constant":
                dst.fill_(p.init_arg)
            elif p.init == "truncated_normal":
                dst.copy_(truncated_normal(p.numel, p.init_arg, g))
            else:
                raise ValueError(p.init)
        return flat.to(device)

    def to_state_dict(self, flat: torch.Tensor) -> Dict[str, torch.Tensor]:
        """Checkpoint-name -> contiguous CPU fp32 tensor (TF variable layout)."""
        flat = flat.detach().to("cpu", torch.float32)
        return {p.ckpt_name: flat[p.offset:p.offset + p.numel].view(p.shape).clone() for p in self.params}

    def from_state_dict(self, state: Dict[str, torch.Tensor]) -> torch.Tensor:
        flat = torch.zeros(self.arena_numel, dtype=torch.float32)
        for p in self.params:
            t = state[p.ckpt_name]
            if tuple(t.shape) != tuple(p.shape):
                raise ValueError("checkpoint tensor %s has shape %s, model wants %s"
                                 % (p.ckpt_name, tuple(t.shape), p.shape))
            flat[p.offset:p.offset + p.numel] = t.reshape(-1).to(torch.float32)
        return flat


def truncated_normal(n: int, stddev: float, gen: torch.Generator) -> torch.Tensor:
    """N(0, stddev^2) truncated to +-2 stddev by resampling (TF semantics)."""
    out = torch.randn(n, generator=gen)
    bad = out.abs() > 2.0
    while bool(bad.any()):
        k = int(bad.sum())
        out[bad] = torch.randn(k, generator=gen)
        bad = out.abs() > 2.0
    return out * stddev
