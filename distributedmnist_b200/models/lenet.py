"""The reference's MNIST convnet ("LeNet-like", 1,663,370 parameters).

reference: src/mnist.py:76-147 --
``conv5x5(1->32,SAME)+bias+ReLU -> maxpool2x2/2 -> conv5x5(32->64,SAME)+bias+ReLU
-> maxpool2x2/2 -> flatten 3136 -> FC 3136->512 + ReLU -> dropout(0.5, train only)
-> FC 512->10``; loss = mean sparse softmax cross entropy (:149-159); accuracy =
mean top-1 hit (:161-164).

This module holds (a) the parameter inventory and (b) a plain-PyTorch fp32
forward used as the CPU execution path and as the numerics reference for the
sm_90a kernels (``emulate_bf16=True`` rounds weights/activations to bf16 at the
points where the CUDA pipeline does, so comparisons can be tight).
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from .spec import ModelSpec, ParamSpec

NUM_LABELS = 10
IMAGE_SIZE = 28
NUM_CHANNELS = 1
SEED = 66478  # reference mnist.py:32
FC1_IN = (IMAGE_SIZE // 4) * (IMAGE_SIZE // 4) * 64  # 3136
FC1_OUT = 512


def lenet_spec() -> ModelSpec:
    # Creation order == reference mnist.py:81-101 (-> Variable .. Variable_7).
    return ModelSpec(
        name="lenet",
        params=[
            ParamSpec("conv1_weights", (5, 5, NUM_CHANNELS, 32), "truncated_normal", 0.1),
            ParamSpec("conv1_biases", (32,), "zeros"),
            ParamSpec("conv2_weights", (5, 5, 32, 64), "truncated_normal", 0.1),
            ParamSpec("conv2_biases", (64,), "constant", 0.1),
            ParamSpec("fc1_weights", (FC1_IN, FC1_OUT), "truncated_normal", 0.1),
            ParamSpec("fc1_biases", (FC1_OUT,), "constant", 0.1),
            ParamSpec("fc2_weights", (FC1_OUT, NUM_LABELS), "truncated_normal", 0.1),
            ParamSpec("fc2_biases", (NUM_LABELS,), "constant", 0.1),
        ],
    )


# ----------------------------------------------------------------------------
# Counter-based dropout mask shared by the torch reference and the CUDA kernels.
# ----------------------------------------------------------------------------
_M32 = 0xFFFFFFFF


def dropout_seed_mix(seed: int, step: int, rank: int = 0) -> int:
    return (seed * 0x632BE5AB + step * 0x9E3779B9 + rank * 0x85EBCA77 + 0x7F4A7C15) & _M32


def dropout_threshold(keep_prob: float) -> int:
    """The 24-bit keep threshold as the kernels compute it: ``(uint32_t)(keep_prob * 16777216.f)`` with ``keep_prob``
    an fp32.  The product is exact (a power of two), so this is floor(fp32(keep_prob) * 2^24).  It differs from
    floor(keep_prob * 2^24) wherever fp32 rounds ``keep_prob`` up (0.3, 0.8, 0.99, ...)."""
    return int(float(np.float32(keep_prob)) * (1 << 24))


def dropout_keep_mask(seed_mix: int, rows: int, cols: int, keep_prob: float,
                      device: str = "cpu") -> torch.Tensor:
    """Deterministic Bernoulli(keep_prob) mask ``[rows, cols]`` (bool).

    A murmur3-style finaliser over the element index; the CUDA epilogue
    (csrc/common.cuh ``dropout_keep``) computes the identical function, with the
    threshold of :func:`dropout_threshold`, so the backward pass regenerates the
    mask instead of storing it (SURVEY §2.4 K7).
    """
    idx = torch.arange(rows * cols, dtype=torch.int64, device=device)
    x = (idx * 0x9E3779B1 + seed_mix) & _M32
    x = x ^ (x >> 16)
    x = (x * 0x85EBCA6B) & _M32
    x = x ^ (x >> 13)
    x = (x * 0xC2B2AE35) & _M32
    x = x ^ (x >> 16)
    return ((x >> 8) < dropout_threshold(keep_prob)).view(rows, cols)


def _q(t: torch.Tensor, on: bool) -> torch.Tensor:
    return t.to(torch.bfloat16).to(torch.float32) if on else t


def lenet_forward(p: Dict[str, torch.Tensor], images: torch.Tensor, train: bool = True,
                  keep_mask: Optional[torch.Tensor] = None, keep_prob: float = 0.5,
                  emulate_bf16: bool = False, conv1_bf16: Optional[bool] = None) -> torch.Tensor:
    """Logits ``[B, 10]`` from NHWC fp32 images ``[B, 28, 28, 1]``.

    ``p`` maps parameter names to tensors in TF layout (HWIO / [in, out]).  ``conv1_bf16`` (default: same as
    ``emulate_bf16``) rounds the conv1 operands too -- the wgmma conv1 (csrc/conv1_tc.cu) does, the SIMT one does not.
    """
    q = emulate_bf16
    q1 = q if conv1_bf16 is None else conv1_bf16
    x = _q(images.permute(0, 3, 1, 2), q1)  # NHWC -> NCHW
    w1 = _q(p["conv1_weights"], q1).permute(3, 2, 0, 1)  # HWIO -> OIHW
    y = F.conv2d(x, w1, p["conv1_biases"], padding=2)
    y = _q(F.max_pool2d(F.relu(y), 2, 2), q)
    w2 = _q(p["conv2_weights"], q).permute(3, 2, 0, 1)
    y = F.conv2d(y, w2, p["conv2_biases"], padding=2)
    y = _q(F.max_pool2d(F.relu(y), 2, 2), q)
    # Flatten in NHWC order, as tf.reshape of an NHWC tensor does (mnist.py:130-133).
    flat = y.permute(0, 2, 3, 1).reshape(y.shape[0], -1)
    h = F.relu(flat @ _q(p["fc1_weights"], q) + p["fc1_biases"])
    if train:
        if keep_mask is None:
            raise ValueError("train=True needs an explicit keep_mask (counter-based dropout)")
        h = h * keep_mask.to(h.dtype) * (1.0 / keep_prob)
    h = _q(h, q)
    return h @ p["fc2_weights"] + p["fc2_biases"]


def loss_and_accuracy(logits: torch.Tensor, labels: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Mean sparse softmax CE and top-1 accuracy (reference mnist.py:149-164)."""
    loss = F.cross_entropy(logits, labels.long(), reduction="mean")
    acc = (logits.argmax(dim=1) == labels.long()).to(torch.float32).mean()
    return loss, acc
