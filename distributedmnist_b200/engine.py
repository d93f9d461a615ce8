"""Compute engines: forward + backward of one replica on one batch.

An engine owns the flat fp32 parameter arena and the flat gradient arena of its
replica (allocated through the aggregation backend so that, on the GPU path,
both live in NVLink-symmetric memory) and exposes four calls:

* ``load_batch(images, labels)``  -- host (pinned) -> device copy of the step's inputs
  (``pack_batch`` / ``load_packed``: the same with one contiguous buffer and one copy per step)
* ``forward_backward(step)``      -- loss, train accuracy and all gradients
* ``loss_acc()``                  -- device -> host read of the step's scalars
* ``evaluate(images, labels)``    -- inference-only loss/accuracy (evaluator)

:class:`TorchEngine` is the plain-PyTorch implementation: the execution path on
CPU (gloo plumbing config) and the cuDNN/cuBLAS *baseline* on GPU.  The product
path on H100 is ``CudaLeNetEngine`` / ``CudaMlpEngine`` in ``engine_cuda.py``
(hand-written sm_90a kernels).  Unlike the reference, loss and accuracy come
from the training forward itself -- the reference runs a second forward per
iteration only for logging (src/distributed_train.py:334; SURVEY §5.9 item 6).
"""
from __future__ import annotations

from typing import Callable, Optional, Tuple

import numpy as np
import torch

from . import augment, best
from . import moving_average as ema
from . import weight_decay
from .models import ModelSpec, dropout_keep_mask, dropout_seed_mix, get_model, loss_and_accuracy
from .models.lenet import FC1_OUT


class ComputeEngine:
    spec: ModelSpec
    params: torch.Tensor
    grads: torch.Tensor
    batch_size: int

    def load_batch(self, images, labels) -> None:
        raise NotImplementedError

    def forward_backward(self, step: int) -> None:
        raise NotImplementedError

    def loss_acc(self) -> Tuple[float, float]:
        raise NotImplementedError

    def evaluate(self, images, labels) -> Tuple[float, float]:
        raise NotImplementedError

    def h2d_bytes_per_step(self) -> int:
        raise NotImplementedError

    # ---- packed batches: one contiguous buffer per step (fp32 images [B,784] then int64 labels [B]) -----------------
    def pack_batch(self, images, labels, pin: bool = True) -> torch.Tensor:
        """Input pipelines fill one (page-locked) buffer per batch; ``load_packed`` then moves it with a single copy
        (the sm_90a engines keep images and labels of a slot in one device allocation for exactly this)."""
        B = self.batch_size
        buf = torch.empty(B * 784 * 4 + B * 8, dtype=torch.uint8)
        if pin and torch.cuda.is_available():
            buf = buf.pin_memory()
        buf[:B * 784 * 4].view(torch.float32).copy_(torch.as_tensor(images, dtype=torch.float32).reshape(B * 784))
        buf[B * 784 * 4:].view(torch.int64).copy_(torch.as_tensor(labels, dtype=torch.int64).reshape(B))
        return buf

    def load_packed(self, packed: torch.Tensor) -> None:
        B = self.batch_size
        self.load_batch(packed[:B * 784 * 4].view(torch.float32).view(B, 28, 28, 1), packed[B * 784 * 4:].view(torch.int64))


class TorchEngine(ComputeEngine):
    def __init__(self, model: str, batch_size: int, device: torch.device, allocate: Callable[[int], torch.Tensor],
                 seed: int = 66478, rank: int = 0, keep_prob: float = 0.5, mlp_hidden: int = 1024,
                 autocast_bf16: bool = False):
        self.spec, self._fwd = get_model(model, mlp_hidden)
        self.model = model
        self.batch_size = batch_size
        self.device = device
        self.seed, self.rank, self.keep_prob = seed, rank, keep_prob
        self.autocast_bf16 = autocast_bf16 and device.type == "cuda"
        self.params = allocate(self.spec.arena_numel)
        self.params.copy_(self.spec.init_flat(seed))
        self.grads = allocate(self.spec.arena_numel)
        self._images: Optional[torch.Tensor] = None
        self._labels: Optional[torch.Tensor] = None
        self._loss = torch.zeros((), device=device)
        self._acc = torch.zeros((), device=device)
        self._h2d = 0

    def load_batch(self, images, labels) -> None:
        if isinstance(images, np.ndarray):
            images = torch.from_numpy(np.ascontiguousarray(images))
            labels = torch.from_numpy(np.ascontiguousarray(labels))
        self._h2d = images.numel() * images.element_size() + labels.numel() * labels.element_size()
        nb = self.device.type == "cuda"
        self._images = images.to(self.device, non_blocking=nb)
        self._labels = labels.to(self.device, non_blocking=nb)

    def _logits(self, flat: torch.Tensor, images: torch.Tensor, train: bool, step: int) -> torch.Tensor:
        views = self.spec.views(flat)
        mask = None
        if train and self.model == "lenet":
            mix = dropout_seed_mix(self.seed, step, self.rank)
            mask = dropout_keep_mask(mix, images.shape[0], FC1_OUT, self.keep_prob, device=str(flat.device))
        if self.autocast_bf16:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return self._fwd(views, images, train=train, keep_mask=mask, keep_prob=self.keep_prob).float()
        return self._fwd(views, images, train=train, keep_mask=mask, keep_prob=self.keep_prob)

    # ---- L2 weight decay (see weight_decay.py) ----------------------------------------------------------------------------
    _decay = 0.0

    def arm_weight_decay(self, lam: float) -> None:
        """From the next step on, differentiate CE + ``lam`` * R (R = sum of v^2 / 2 over the decayed variables); the loss
        :meth:`loss_acc` reports includes the term."""
        self._decay = float(lam)

    # ---- random affine augmentation and elastic distortion (see augment.py) ---------------------------------------------
    _aug = None                    # (augment.Ranges, seed mix)
    _aug_elastic = None            # augment.Elastic while elastic distortion is armed
    _aug_images: Optional[torch.Tensor] = None

    def arm_augment(self, max_shift: float, max_rotation: float, max_scale: float, start_iteration: int = 0,
                    elastic: Optional[augment.Elastic] = None) -> None:
        """Augment every training batch from the next :meth:`forward_backward` on, its first draws those of iteration
        ``start_iteration``; all three ranges 0 and no ``elastic`` (or alpha 0) turns it off.  ``elastic``: the elastic
        distortion composed in front of the affine map.  The same transform and draws as the sm_90a kernels, by the
        float64 warp rounded to fp32."""
        r = augment.Ranges(float(max_shift), float(max_rotation), float(max_scale))
        augment.check_ranges(r)
        if elastic is not None:
            elastic = augment.Elastic(float(elastic.alpha), float(elastic.sigma))
            augment.check_elastic(elastic)
        self._aug_elastic = elastic if elastic is not None and elastic.alpha != 0.0 else None
        on = any(r) or self._aug_elastic is not None
        self._aug = (r, augment.seed_mix(self.seed, self.rank)) if on else None
        self._aug_iteration = int(start_iteration) & 0xFFFFFFFF

    def augment_iteration(self) -> int:
        return self._aug_iteration

    def augmented_batch(self) -> Optional[torch.Tensor]:
        """The images the last augmented step read (None when augmentation is off)."""
        return None if self._aug is None else self._aug_images

    def forward_backward(self, step: int) -> None:
        images = self._images
        if self._aug is not None:
            r, mix = self._aug
            out = augment.augment_batch(images.detach().cpu().numpy(), mix, self._aug_iteration, r, self._aug_elastic)
            images = self._aug_images = torch.from_numpy(out).to(self.device)
            self._aug_iteration = (self._aug_iteration + 1) & 0xFFFFFFFF
        p = self.params.detach().requires_grad_(True)
        logits = self._logits(p, images, True, step)
        loss, acc = loss_and_accuracy(logits, self._labels)
        if self._decay:
            views = self.spec.views(p)
            reg = sum((views[q.name] * views[q.name]).sum() for q in weight_decay.decayed(self.spec)) * 0.5
            loss = loss + self._decay * reg
        (g,) = torch.autograd.grad(loss, p)
        self.grads.copy_(g)
        self._loss, self._acc = loss.detach(), acc.detach()

    def loss_acc(self) -> Tuple[float, float]:
        return float(self._loss.item()), float(self._acc.item())

    # ---- moving average of the weights (see moving_average.py) ------------------------------------------------------------
    _ema: Optional[torch.Tensor] = None

    def arm_moving_average(self, decay: float, global_step: int = 0) -> None:
        """Keep an fp32 average arena, starting from the current weights, which :meth:`update_moving_average` moves
        towards the weights after every global step."""
        if not 0.0 < float(decay) < 1.0:
            raise ValueError("moving average decay must lie in (0, 1), got %r" % decay)
        self._ema_decay = float(decay)
        self._ema = self.params.detach().clone()
        self._ema_step = int(global_step)

    def update_moving_average(self, global_step: int) -> None:
        """The update after the step that produced ``global_step``, from the current weights."""
        m = torch.tensor(float(ema.multiplier(self._ema_decay, global_step)), dtype=torch.float32, device=self._ema.device)
        self._ema.sub_((self._ema - self.params.detach()) * m)      # three float32 operations, each rounded on its own
        self._ema_step = int(global_step)

    def moving_average(self) -> Tuple[torch.Tensor, int]:
        """(copy of the average arena, global step of the weights it was last updated from)."""
        return self._ema.clone(), self._ema_step

    def load_moving_average(self, flat: torch.Tensor) -> None:
        self._ema.copy_(flat.to(self._ema.device, torch.float32))

    @torch.no_grad()
    def evaluate(self, images, labels, moving_average: bool = False) -> Tuple[float, float]:
        """``moving_average``: score the average arena instead of the weights."""
        if isinstance(images, np.ndarray):
            images, labels = torch.from_numpy(np.ascontiguousarray(images)), torch.from_numpy(np.ascontiguousarray(labels))
        images, labels = images.to(self.device), labels.to(self.device)
        flat = self._ema if moving_average else self.params
        tot_loss, tot_hit, n = 0.0, 0.0, images.shape[0]
        for s in range(0, n, 2048):
            lg = self._logits(flat, images[s:s + 2048], False, 0)
            loss, acc = loss_and_accuracy(lg, labels[s:s + 2048])
            m = lg.shape[0]
            tot_loss += float(loss) * m
            tot_hit += float(acc) * m
        return tot_loss / n, tot_hit / n

    def h2d_bytes_per_step(self) -> int:
        return self._h2d

    # ---- best-scoring weights (see best.py) -------------------------------------------------------------------------------
    _best_correct = 0
    _best: Optional[Tuple] = None

    def arm_best(self, initial_correct: int = 0) -> None:
        """Keep the weights of the best evaluation from here on; ``initial_correct``: an earlier run's best count."""
        self._best_correct, self._best = int(initial_correct), None

    def note_eval(self, step: int, n: int, examples: int, correct: int, loss_sum: float,
                  moving_average: bool = False) -> bool:
        """After an ``evaluate`` of global step ``step`` (``moving_average``: of the average arena): keep a copy of the
        scored arena if the pass is the new best.  True if it is."""
        if not best.improves(correct, examples, n, self._best_correct):
            return False
        flat = self._ema if moving_average else self.params
        self._best_correct = int(correct)
        self._best = (flat.detach().clone(), int(step), int(correct), int(examples), float(loss_sum))
        return True

    def best_weights(self) -> Optional[Tuple]:
        """``(fp32 arena, global step, correct, examples, loss_sum)`` of the best pass since :meth:`arm_best`, or None."""
        return self._best


def make_engine(flags, ctx, backend, force_torch: bool = False) -> ComputeEngine:
    """GPU -> hand-written sm_90a engine (fails loudly if the extension is absent);
    CPU -> torch engine."""
    if ctx.on_gpu and not force_torch and flags.backend in ("auto", "fused"):
        from .engine_cuda import make_cuda_engine
        return make_cuda_engine(flags, ctx, backend)
    return TorchEngine(flags.model, flags.batch_size, ctx.device, backend.allocate, seed=flags.seed,
                       rank=ctx.rank, keep_prob=flags.dropout_keep_prob, mlp_hidden=flags.mlp_hidden,
                       autocast_bf16=(flags.compute_dtype == "bf16"))
