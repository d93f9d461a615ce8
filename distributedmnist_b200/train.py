"""Training driver: the per-replica hot loop.

reference: ``distributed_train.train(target, dataset, dataset_test, cluster_spec)``
(src/distributed_train.py:109-408).  Behaviour kept: K defaults to the number of
workers (:118-121); replica 0 is the chief (:130); staircase LR decay with the /K
rule (:143-156); mode selection from ``--interval_method`` /
``--worker_times_cdf_method`` (:176-188); optional drop-connect in the default mode
only (:194-203); chief restores the latest checkpoint at start (Supervisor,
:244-262) and saves every ``--save_interval_secs`` plus once at the end (:252,
405-408); start-up barrier (:277); the log-line formats (:296,325,341-342,367-371,
398-399); ``worker<id>_time_acc.npy`` every ``--save_results_period`` global steps
(:373-379); per-step chrome timelines (:354-358); loop exit when
``step > max_steps`` checked after the work (:360).

Dropped on purpose (SURVEY §5.9): the second forward pass per iteration that the
reference runs only to log loss/accuracy (:334), ``sess.kill()/reset_kill()``
(:391-396, not in stock TF), ``np.set_printoptions(threshold=np.nan)`` (:31).
"""
from __future__ import annotations

import json
import math
import os
import queue
import threading
import time
from datetime import datetime
from fractions import Fraction
from typing import Dict, Optional

import numpy as np
import torch

from . import augment, best, early_stopping, lr_plateau, moving_average, weight_decay
from .best import BEST_DIR, BEST_JSON
from .checkpoint import Saver
from .early_stopping import EARLY_STOPPING_JSON
from .engine import make_engine
from .lr_plateau import LR_PLATEAU_JSON
from .flags import FLAGS
from .parallel.aggregators import (AsyncSGDOptimizer, LocalSGDOptimizer, SyncReplicasOptimizer, TimeoutReplicasOptimizer,
                                   local_sgd_report, parse_straggler_spec, ssp_report, staleness_report)
from .parallel.backends import make_backend
from .parallel.context import ReplicaContext
from .parallel.timeout_manager import launch_manager
from .schedule import LearningRateSchedule
from .utils.logging import get_logger
from .utils.summary import SummaryWriter
from .utils.timeline import Timeline, cupti_device_spans, timeline_path

log = get_logger()

STALENESS_JSON = "worker%d_staleness.json"
SSP_JSON = "worker%d_ssp.json"
LOCAL_SGD_JSON = "worker%d_local_sgd.json"

LOG_FORMAT = ("Worker %d: %s: step %d, loss = %f, train_acc = %f, test_acc = %f"
              "(%.1f examples/sec; %.3f  sec/batch)")


class _AsyncCheckpointer:
    """Chief-side saver; file IO runs on a helper thread.

    Without ``engine`` (torch engine, CPU path) the weights are copied to the host on the training thread.  With the sm_90a
    engine (``engine`` armed by ``arm_checkpoint``) a checkpoint is a device capture: ``maybe_save`` enqueues it on the
    training stream after the launched step and returns; later calls poll its event (never a wait) and, once it has landed
    in one of the engine's page-locked host arenas, hand that arena and the step the capture names to the saver thread,
    which slices it into the state dict and writes the files.  An arena goes back into use only after the saver thread is
    done with it, and at most one capture is in flight.  A capture that found no consistent snapshot writes no file; it is
    counted in ``failed`` and retried at the next call instead of after another ``interval_s``."""

    def __init__(self, train_dir: str, spec, interval_s: float, engine=None, timeout_s: float = 30.0, average=None):
        self.train_dir, self.spec, self.interval_s = train_dir, spec, interval_s
        # --moving_average_decay: every file also holds <variable>/ExponentialMovingAverage.  ``average`` is the torch
        # engine's average arena (saved with the weights, on the training thread); a device capture carries its own copy
        # of the average, taken after the same step as the weights
        self.average = average
        self._device_average = engine is not None and getattr(engine, "_ck_ema_dev", None) is not None
        self.saver = Saver()
        self._next = time.time() + interval_s
        self._thread: Optional[threading.Thread] = None
        self.engine, self.timeout_s = engine, timeout_s
        self.failed = 0                          # captures without a consistent snapshot (each retried)
        self._retry = False
        self._pending = False                    # a capture is in flight
        if engine is not None:
            self._lock = threading.Lock()
            self._free = [True] * len(engine.ckpt_host)
            self._queue: "queue.Queue" = queue.Queue()
            self._error: Optional[BaseException] = None
            self._thread = threading.Thread(target=self._write_loop, daemon=True)
            self._thread.start()

    def maybe_save(self, params: torch.Tensor, global_step: int, capture: bool = True) -> None:
        """``capture=False``: the weights after the step are not to be saved (local SGD between two averages); a capture
        in flight is still collected, and a due one waits for a call that allows it."""
        if self.engine is not None:
            self._collect(self.engine.checkpoint_poll() if self._pending else None)
            if self._pending or not capture or not (self._retry or time.time() >= self._next):
                return
            with self._lock:
                buf = next((b for b, free in enumerate(self._free) if free), None)
            if buf is None:
                return                           # both arenas are still being written: try again at the next step
            self._next = time.time() + self.interval_s
            self._enqueue(buf)
            return
        if capture and time.time() >= self._next:
            self._next = time.time() + self.interval_s
            self.save(params, global_step, blocking=False)

    def save(self, params: torch.Tensor, global_step: int, blocking: bool = True) -> None:
        if self.engine is not None:
            assert blocking, "device captures are saved without blocking through maybe_save"
            self._save_final()
            return
        state = self.spec.to_state_dict(params)  # consistent snapshot (device -> host copy)
        if self.average is not None:
            state.update(moving_average.to_state_dict(self.spec, self.average))
        if self._thread is not None:
            self._thread.join()
        self._thread = threading.Thread(target=self.saver.save, args=(self.train_dir, state, global_step))
        self._thread.start()
        if blocking:
            self._thread.join()

    def close(self) -> None:
        if self.engine is not None:
            self._queue.put(None)
        if self._thread is not None:
            self._thread.join()
        if self.engine is not None and self._error is not None:
            raise RuntimeError("writing a checkpoint failed") from self._error

    # ---- device captures -----------------------------------------------------------------------------------------------
    def _enqueue(self, buf: int) -> None:
        with self._lock:
            self._free[buf] = False
        self.engine.enqueue_checkpoint(buf)
        self._pending = True
        self._retry = False

    def _collect(self, landed) -> bool:
        """Hand a landed capture ``(seq, buffer, step)`` to the saver thread, or count it as failed.  True if it was accepted."""
        if landed is None:
            return False
        self._pending = False
        _seq, buf, step = landed
        if step < 0:
            self.failed += 1
            self._retry = True
            with self._lock:
                self._free[buf] = True
            return False
        self._queue.put((buf, step))
        return True

    def _save_final(self) -> None:
        """Blocking capture after the last step, retried until one is accepted or ``timeout_s`` has passed.  The file's step
        is the step the captured weights hold."""
        self._collect(self.engine.checkpoint_wait())      # a periodic capture still in flight is a checkpoint too
        deadline = time.time() + self.timeout_s
        while True:
            self._queue.join()                   # every arena is free again
            self._enqueue(0)
            if self._collect(self.engine.checkpoint_wait()):
                break
            if time.time() >= deadline:
                raise RuntimeError("final checkpoint: no consistent snapshot of the weights within %.0f ms (%d capture(s) "
                                   "failed)" % (self.timeout_s * 1e3, self.failed))
        self._queue.join()

    def _write_loop(self) -> None:
        while True:
            item = self._queue.get()
            try:
                if item is None:
                    return
                buf, step = item
                try:
                    state = self.spec.to_state_dict(self.engine.ckpt_host[buf])
                    if self._device_average:
                        state.update(moving_average.to_state_dict(self.spec, self.engine.ckpt_ema_host[buf]))
                    self.saver.save(self.train_dir, state, step)
                except BaseException as e:  # noqa: BLE001  (re-raised by close())
                    self._error = e
                finally:
                    with self._lock:
                        self._free[buf] = True
            finally:
                self._queue.task_done()


class _BatchPacker:
    """Input pipeline of the GPU path: a helper thread draws batches from the DataSet and packs each into one page-locked
    buffer (fp32 images then int64 labels, the device slot's layout), a few batches ahead of the training loop, so a step's
    input is ONE host->device DMA and the hot loop never touches numpy.  Buffers rotate through a ring deep enough that a
    buffer is not rewritten before the copy that reads it has run (the engine double-buffers its device slots)."""

    def __init__(self, engine, dataset, batch_size: int, depth: int = 8, workers: int = 2):
        import queue
        self.engine, self.dataset, self.batch_size = engine, dataset, batch_size
        B = batch_size
        self._nimg = B * 784 * 4
        self.workers = max(1, workers)
        # every worker owns a private ring segment deep enough that a buffer is never rewritten while the DMA that reads it
        # may still be pending (the queue bounds how far ahead of the training loop the workers can run)
        self.rings = [[torch.empty(B * 784 * 4 + B * 8, dtype=torch.uint8).pin_memory() for _ in range(depth + 4)]
                      for _ in range(self.workers)]
        self.ready: "queue.Queue" = queue.Queue(maxsize=depth)
        self._draw = threading.Lock()          # batches are drawn from the DataSet one at a time; the gathers run in parallel
        self._stop = False
        # fast path: gather the batch's rows straight from the dataset arrays into the page-locked buffer with torch
        # (multi-threaded, releases the GIL -- the training loop's interpreter is not held up by the packer)
        self._src = None
        if hasattr(dataset, "next_batch_indices") and not getattr(dataset, "fake_data", False):
            imgs = np.ascontiguousarray(dataset.images, dtype=np.float32).reshape(dataset.num_examples, -1)
            if imgs.shape[1] == 784:
                self._src = (torch.from_numpy(imgs), torch.from_numpy(np.ascontiguousarray(dataset.labels)).to(torch.int64))
        self._threads = [threading.Thread(target=self._run, args=(w,), daemon=True) for w in range(self.workers)]
        for t in self._threads:
            t.start()

    def _run(self, w: int) -> None:
        i = 0
        ring = self.rings[w]
        while not self._stop:
            buf = ring[i % len(ring)]
            if self._src is not None:
                with self._draw:
                    idx = torch.from_numpy(self.dataset.next_batch_indices(self.batch_size).copy())
                torch.index_select(self._src[0], 0, idx, out=buf[:self._nimg].view(torch.float32).view(self.batch_size, 784))
                torch.index_select(self._src[1], 0, idx, out=buf[self._nimg:].view(torch.int64))
            else:
                with self._draw:
                    images, labels = self.dataset.next_batch(self.batch_size)
                buf[:self._nimg].view(torch.float32).copy_(torch.from_numpy(np.ascontiguousarray(images, dtype=np.float32)).reshape(-1))
                buf[self._nimg:].view(torch.int64).copy_(torch.from_numpy(np.ascontiguousarray(labels)).to(torch.int64).reshape(-1))
            while not self._stop:
                try:
                    self.ready.put(buf, timeout=0.1)
                    break
                except Exception:  # noqa: BLE001  (queue.Full)
                    continue
            i += 1

    def next(self) -> torch.Tensor:
        return self.ready.get()

    def close(self) -> None:
        self._stop = True
        try:
            while True:
                self.ready.get_nowait()
        except Exception:  # noqa: BLE001  (queue.Empty)
            pass
        for t in self._threads:
            t.join(timeout=2.0)


class _IndexFeed:
    """Input pipeline of ``--device_data``: each step's B row indices (``dataset.next_batch_indices``, cast to int32) in a
    small ring of page-locked buffers, drawn on the training thread -- one numpy slice per step.  The engine's index DMA
    reads a buffer asynchronously, so a buffer is rewritten only after the step after the next one has been enqueued: the
    ring holds ``depth`` >= 3 buffers and the loop enqueues one buffer per step."""

    def __init__(self, dataset, batch_size: int, depth: int = 4):
        assert depth >= 3
        self.dataset, self.batch_size = dataset, batch_size
        self.ring = [torch.empty(batch_size, dtype=torch.int32).pin_memory() for _ in range(depth)]
        self._i = 0

    def next(self) -> torch.Tensor:
        buf = self.ring[self._i % len(self.ring)]
        self._i += 1
        np.copyto(buf.numpy(), self.dataset.next_batch_indices(self.batch_size), casting="unsafe")
        return buf

    def close(self) -> None:
        pass                       # no helper thread to stop (same interface as _BatchPacker)


def check_async_flags(flags, ctx: ReplicaContext) -> None:
    """``--async_method`` (and ``--ssp_staleness``) combinations that cannot work, rejected before any device work
    starts."""
    s = getattr(flags, "ssp_staleness", -1)
    if isinstance(s, bool) or not isinstance(s, int):
        raise ValueError("--ssp_staleness must be an integer, got %r" % (s,))
    if not -1 <= s < 2 ** 31:
        raise ValueError("--ssp_staleness is the number of its own updates a replica may run ahead of the slowest one: "
                         "0 <= s < 2^31, or -1 for off; got %d" % s)
    if not getattr(flags, "async_method", False):
        if s != -1:
            raise ValueError("--ssp_staleness bounds asynchronous SGD and needs --async_method")
        return
    if flags.interval_method:
        raise ValueError("--async_method cannot be combined with --interval_method: both are aggregation modes, and "
                         "asynchronous SGD applies every gradient on its own instead of a tick's mean")
    if getattr(flags, "worker_times_cdf_method", False):
        raise ValueError("--async_method cannot be combined with --worker_times_cdf_method: the cdf mode waits for all "
                         "replicas behind a full barrier, and asynchronous SGD never waits")
    k = flags.num_replicas_to_aggregate
    if k != -1 and k != ctx.world_size:
        raise ValueError("--async_method applies every gradient on its own, so --num_replicas_to_aggregate must be left "
                         "unset or equal the number of replicas (%d), got %d" % (ctx.world_size, k))
    if flags.drop_connect:
        raise ValueError("--async_method cannot be combined with --drop_connect: the gradient mask is implemented in the "
                         "synchronous aggregation kernels only")
    if int(getattr(flags, "lr_plateau_patience", 0) or 0):
        raise ValueError("--async_method cannot be combined with --lr_plateau_patience: its replicas are not in lock "
                         "step, so no global step can be named from which every replica applies a cut")
    if float(getattr(flags, "moving_average_decay", 0.0) or 0.0):
        raise ValueError("--async_method cannot be combined with --moving_average_decay: the chief's average follows its "
                         "own arena once per global step, and asynchronous updates land in it at any time")
    if not (ctx.on_gpu and flags.backend in ("auto", "fused")) and ctx.world_size > 1:
        raise ValueError("--async_method with the torch engine (--backend=%s%s) is implemented for one replica, not %d: "
                         "the replicas would need shared weights that every one of them updates"
                         % (flags.backend, "" if ctx.on_gpu else ", no GPU", ctx.world_size))


def check_local_sgd_flags(flags, ctx: ReplicaContext) -> None:
    """``--local_sgd_steps`` combinations that cannot work, rejected before any device work starts."""
    h = getattr(flags, "local_sgd_steps", 0)
    if isinstance(h, bool) or not isinstance(h, int):
        raise ValueError("--local_sgd_steps must be an integer, got %r" % (h,))
    if h == 0:
        return
    if not 1 <= h < 2 ** 31:
        raise ValueError("--local_sgd_steps is the number of local steps between two averages: 1 <= H < 2^31, or 0 for "
                         "off; got %d" % h)
    if flags.interval_method:
        raise ValueError("--local_sgd_steps cannot be combined with --interval_method: both are aggregation modes, and "
                         "local SGD averages weights every H steps instead of a tick's gradients")
    if getattr(flags, "worker_times_cdf_method", False):
        raise ValueError("--local_sgd_steps cannot be combined with --worker_times_cdf_method: the cdf mode times a full "
                         "barrier on every step, and local SGD has one only every H steps")
    if getattr(flags, "async_method", False):
        raise ValueError("--local_sgd_steps cannot be combined with --async_method: asynchronous SGD shares one set of "
                         "weights, and local SGD keeps one per replica")
    k = flags.num_replicas_to_aggregate
    if k != -1 and k != ctx.world_size:
        raise ValueError("--local_sgd_steps averages every replica's weights, so --num_replicas_to_aggregate must be left "
                         "unset or equal the number of replicas (%d), got %d" % (ctx.world_size, k))
    if flags.drop_connect:
        raise ValueError("--local_sgd_steps cannot be combined with --drop_connect: the gradient mask is implemented in "
                         "the synchronous aggregation kernels only")
    if float(getattr(flags, "moving_average_decay", 0.0) or 0.0):
        raise ValueError("--local_sgd_steps cannot be combined with --moving_average_decay: between two averages the "
                         "chief's weights are its own, not the model's")
    if int(getattr(flags, "lr_plateau_patience", 0) or 0):
        raise ValueError("--local_sgd_steps cannot be combined with --lr_plateau_patience: a cut must take effect on "
                         "the same global step on every replica, and the plateau rule does not place it on an "
                         "averaging step")
    every = int(getattr(flags, "eval_every_steps", 0) or 0)
    if every % h:
        raise ValueError("--eval_every_steps (%d) must be a multiple of --local_sgd_steps (%d): the in-training "
                         "evaluation scores the averaged model, which exists only after an averaging step" % (every, h))


def stop_margin(flags) -> int:
    """S - g: the stop step S of an evaluation pass of global step g that stops the run.  STOP_MARGIN steps, or
    STOP_MARGIN averaging periods with local SGD (DESIGN §4.4)."""
    return STOP_MARGIN * max(1, int(getattr(flags, "local_sgd_steps", 0) or 0))


def check_device_data_flags(flags, ctx: ReplicaContext, dataset) -> None:
    """``--device_data`` combinations that cannot work, rejected before any device work starts."""
    if not getattr(flags, "device_data", False):
        return
    if flags.fake_data or getattr(dataset, "fake_data", False):
        raise ValueError("--device_data cannot be combined with --fake_data: there is no training set to keep on the GPU")
    if not (ctx.on_gpu and flags.backend in ("auto", "fused")):
        raise ValueError("--device_data needs the sm_90a engine (a GPU and --backend=auto or fused); the torch engine "
                         "(--backend=%s%s) feeds its batches from the host" % (flags.backend, "" if ctx.on_gpu else ", no GPU"))


def check_batch_flags(flags, ctx: ReplicaContext) -> None:
    """A ``--batch_size`` the GPU path's LeNet kernels cannot run, rejected before any device work starts."""
    if ctx.on_gpu and flags.backend in ("auto", "fused") and flags.model == "lenet":
        from .engine_cuda import check_lenet_batch
        check_lenet_batch(flags.batch_size)


def check_eval_flags(flags, ctx: ReplicaContext, num_replicas_to_aggregate: int, dataset_test) -> None:
    """``--eval_every_steps`` combinations that cannot work, rejected before any device work starts."""
    if getattr(flags, "eval_every_steps", 0) < 0:
        raise ValueError("--eval_every_steps must be >= 0 (0 = off)")
    if not getattr(flags, "eval_every_steps", 0):
        return
    if dataset_test is None:
        raise ValueError("--eval_every_steps needs the validation set, but no dataset_test was given")
    if not (ctx.on_gpu and flags.backend in ("auto", "fused")):
        return                     # torch engine: evaluated synchronously with engine.evaluate, every mode and model
    if flags.model != "lenet":
        raise ValueError("--eval_every_steps on the GPU path is implemented for lenet, not --model=%s" % flags.model)
    # the live pass reads the chief's parameter arena between two of its steps: sound only when no peer can write that
    # arena then, i.e. when every step waits for all N replicas.  --eval_snapshot scores a validated copy instead.
    if getattr(flags, "eval_snapshot", False):
        return
    hint = " (--eval_snapshot=true scores a validated snapshot of the weights instead)"
    if flags.interval_method:
        raise ValueError("--eval_every_steps cannot be combined with --interval_method: interval commits push weights into "
                         "the chief's arena at any time, so the pass would not see one step's weights" + hint)
    # --worker_times_cdf_method (without --interval_method, which wins when both are set) always aggregates all N
    # gradients behind a full barrier and ignores --num_replicas_to_aggregate
    cdf = getattr(flags, "worker_times_cdf_method", False)
    if not cdf and num_replicas_to_aggregate != ctx.world_size:
        raise ValueError("--eval_every_steps needs --num_replicas_to_aggregate = number of replicas (%d): with K < N or "
                         "K > N peers push weights into the chief's arena while it is between steps or late"
                         % ctx.world_size + hint)


def check_target_flags(flags, ctx: ReplicaContext) -> None:
    """``--target_accuracy`` combinations that cannot work, rejected before any device work starts."""
    a = float(getattr(flags, "target_accuracy", 0.0) or 0.0)
    if a == 0.0:
        return
    if not 0.0 < a <= 1.0:
        raise ValueError("--target_accuracy must lie in (0, 1] (0 = off), got %r" % a)
    if getattr(flags, "eval_every_steps", 0) <= 0:
        raise ValueError("--target_accuracy needs --eval_every_steps > 0: the run stops after the first in-training "
                         "evaluation that reaches the target")
    if not (ctx.on_gpu and flags.backend in ("auto", "fused")) and ctx.world_size > 1:
        raise ValueError("--target_accuracy with the torch engine (--backend=%s%s) is implemented for one replica, not %d: "
                         "only the chief evaluates and nothing tells the other replicas to stop"
                         % (flags.backend, "" if ctx.on_gpu else ", no GPU", ctx.world_size))


def check_early_stopping_flags(flags, ctx: ReplicaContext) -> None:
    """``--early_stopping_patience`` / ``--early_stopping_min_delta`` combinations that cannot work, rejected before any
    device work starts.  Where the in-training evaluation itself is refused (check_eval_flags), so is early stopping."""
    p = int(getattr(flags, "early_stopping_patience", 0) or 0)
    d = float(getattr(flags, "early_stopping_min_delta", 0.0) or 0.0)
    if p < 0:
        raise ValueError("--early_stopping_patience must be >= 1 (0 = off), got %d" % p)
    if not 0.0 <= d < 1.0:
        raise ValueError("--early_stopping_min_delta must lie in [0, 1), got %r" % d)
    if p == 0:
        if d != 0.0:
            raise ValueError("--early_stopping_min_delta needs --early_stopping_patience >= 1: without a patience there "
                             "is nothing for it to change")
        return
    if getattr(flags, "eval_every_steps", 0) <= 0:
        raise ValueError("--early_stopping_patience needs --eval_every_steps > 0: the patience counts in-training "
                         "evaluations")
    if not (ctx.on_gpu and flags.backend in ("auto", "fused")) and ctx.world_size > 1:
        raise ValueError("--early_stopping_patience with the torch engine (--backend=%s%s) is implemented for one "
                         "replica, not %d: only the chief evaluates and nothing tells the other replicas to stop"
                         % (flags.backend, "" if ctx.on_gpu else ", no GPU", ctx.world_size))


def check_lr_plateau_flags(flags, ctx: ReplicaContext, num_replicas_to_aggregate: int) -> None:
    """``--lr_plateau_patience`` / ``--lr_plateau_factor`` / ``--lr_plateau_min_delta`` combinations that cannot work,
    rejected before any device work starts.  Where the in-training evaluation itself is refused (check_eval_flags), so
    are learning-rate cuts."""
    p = int(getattr(flags, "lr_plateau_patience", 0) or 0)
    f = float(getattr(flags, "lr_plateau_factor", 0.1))
    d = float(getattr(flags, "lr_plateau_min_delta", 0.0) or 0.0)
    if p < 0:
        raise ValueError("--lr_plateau_patience must be >= 1 (0 = off), got %d" % p)
    if not 0.0 < f < 1.0:
        raise ValueError("--lr_plateau_factor must lie in (0, 1), got %r" % f)
    if not 0.0 <= d < 1.0:
        raise ValueError("--lr_plateau_min_delta must lie in [0, 1), got %r" % d)
    if p == 0:
        if d != 0.0 or f != 0.1:
            raise ValueError("--lr_plateau_factor and --lr_plateau_min_delta need --lr_plateau_patience >= 1: without a "
                             "patience there is nothing for them to change")
        return
    if getattr(flags, "eval_every_steps", 0) <= 0:
        raise ValueError("--lr_plateau_patience needs --eval_every_steps > 0: the patience counts in-training evaluations")
    if not (ctx.on_gpu and flags.backend in ("auto", "fused")):
        if ctx.world_size > 1:
            raise ValueError("--lr_plateau_patience with the torch engine (--backend=%s%s) is implemented for one replica, "
                             "not %d: only the chief evaluates and nothing tells the other replicas to cut their rate"
                             % (flags.backend, "" if ctx.on_gpu else ", no GPU", ctx.world_size))
        return
    # every replica must apply a cut from the same global step S: the chief's table stores reach a peer before it finishes
    # the chief's next step only when every step waits for all N replicas (DESIGN §4, learning-rate cuts)
    why = ": its replicas are not in lock step, so no global step can be named from which every replica applies a cut " \
          "(supported: K = N, or --worker_times_cdf_method without --interval_method)"
    if flags.interval_method:
        raise ValueError("--lr_plateau_patience cannot be combined with --interval_method" + why)
    if not getattr(flags, "worker_times_cdf_method", False) and num_replicas_to_aggregate != ctx.world_size:
        raise ValueError("--lr_plateau_patience needs --num_replicas_to_aggregate = number of replicas (%d), got %d (K %s N)"
                         % (ctx.world_size, num_replicas_to_aggregate,
                            "<" if num_replicas_to_aggregate < ctx.world_size else ">") + why)


def check_lr_schedule_flags(flags) -> None:
    """``--lr_warmup_steps`` / ``--lr_warmup_start_factor`` / ``--lr_cosine_decay_steps`` / ``--lr_cosine_alpha``
    values and combinations that cannot work, rejected before any device work starts.  The schedule itself works in every
    aggregation mode: it is a function of the global step alone."""
    w = int(getattr(flags, "lr_warmup_steps", 0) or 0)
    f0 = float(getattr(flags, "lr_warmup_start_factor", 1.0 / 3))
    t = int(getattr(flags, "lr_cosine_decay_steps", 0) or 0)
    alpha = float(getattr(flags, "lr_cosine_alpha", 0.0))
    limit = 2 ** 32 - 1
    if not 0 <= w < limit:
        raise ValueError("--lr_warmup_steps must lie in [0, 2^32 - 1) (0 = off), got %d" % w)
    if not 0 <= t < limit:
        raise ValueError("--lr_cosine_decay_steps must lie in [0, 2^32 - 1) (0 = off), got %d" % t)
    if not 0.0 <= f0 < 1.0:           # also refuses nan and inf
        raise ValueError("--lr_warmup_start_factor must lie in [0, 1), got %r" % f0)
    if not 0.0 <= alpha < 1.0:
        raise ValueError("--lr_cosine_alpha must lie in [0, 1), got %r" % alpha)
    if w == 0 and f0 != 1.0 / 3:
        raise ValueError("--lr_warmup_start_factor needs --lr_warmup_steps >= 1: without a warmup there is nothing for "
                         "it to change")
    if t == 0 and alpha != 0.0:
        raise ValueError("--lr_cosine_alpha needs --lr_cosine_decay_steps >= 1: without a cosine decay there is nothing "
                         "for it to change")
    if t > 0:
        present = getattr(flags, "is_present", lambda name: False)
        given = [n for n in ("learning_rate_decay_factor", "num_epochs_per_decay") if present(n)]
        if given:
            raise ValueError("--lr_cosine_decay_steps replaces the staircase decay, so %s would do nothing"
                             % " and ".join("--" + n for n in given))


def describe_lr_schedule(sched: LearningRateSchedule) -> str:
    """The start-up log's account of the schedule (without the plateau cuts, which are logged as they are made)."""
    if sched.cosine_steps:
        text = "%g with cosine decay over %d global steps to %g" % (
            sched.initial_learning_rate, sched.cosine_steps, sched.initial_learning_rate * sched.cosine_alpha)
    else:
        text = "%g decayed by %g every %d global steps" % (sched.initial_learning_rate, sched.decay_rate,
                                                           sched.decay_steps)
    if sched.warmup_steps:
        text += ", linear warmup from %g of it over global steps 0 to %d" % (sched.warmup_start, sched.warmup_steps - 1)
    return text


def restart_lr_cuts(train_dir: str, rank: int, restored_step: int, factor: float):
    """The cuts an earlier run's ``worker<rank>_lr_plateau.json`` lists that a run restarted from the checkpoint of
    ``restored_step`` keeps -- those with ``from_step <= restored_step`` -- as ``(kept, None)``, or ``([], reason)`` when
    the restart must be refused: cuts are kept but the file's factor differs from ``factor``."""
    try:
        with open(os.path.join(train_dir, LR_PLATEAU_JSON % rank)) as f:
            earlier = json.load(f)
    except FileNotFoundError:
        return [], None
    kept = [dict(trigger_step=int(c["trigger_step"]), from_step=int(c["from_step"])) for c in earlier["cuts"]
            if int(c["from_step"]) <= restored_step]
    if kept and float(earlier["factor"]) != factor:
        return [], ("--lr_plateau_factor=%r differs from the factor %r of the %d learning-rate cut(s) the restored "
                    "checkpoint of global step #%d was trained with (%s)"
                    % (factor, float(earlier["factor"]), len(kept), restored_step, LR_PLATEAU_JSON % rank))
    return kept, None


def check_best_flags(flags) -> None:
    """``--keep_best_checkpoint`` combinations that cannot work, rejected before any device work starts.  Where the
    in-training evaluation itself is refused (check_eval_flags), so is keeping its best weights."""
    if getattr(flags, "keep_best_checkpoint", False) and getattr(flags, "eval_every_steps", 0) <= 0:
        raise ValueError("--keep_best_checkpoint needs --eval_every_steps > 0: the best weights are those of the "
                         "best-scoring in-training evaluation")


def read_best(train_dir: str, rank: int) -> Optional[Dict]:
    """The best-weights summary an earlier run left in ``train_dir``, or None."""
    try:
        with open(os.path.join(train_dir, BEST_JSON % rank)) as f:
            return json.load(f)
    except FileNotFoundError:
        return None


def save_best(engine, spec, train_dir: str, rank: int, weights: str) -> Optional[Dict]:
    """Write the best weights the engine kept, if any pass of this run qualified: ``train_dir/best/model.ckpt-<step>``
    under the plain variable names (the evaluator scores it as it is), then ``worker<rank>_best.json``.  Returns the
    summary, or None when nothing was written."""
    b = engine.best_weights()
    if b is None:
        return None
    arena, step, correct, examples, loss_sum = b
    d = os.path.join(train_dir, BEST_DIR)
    saver = Saver(max_to_keep=1)
    saver.adopt(d)                 # a restarted run's better best replaces the earlier one
    saver.save(d, spec.to_state_dict(arena), step)
    report = dict(global_step=step, correct=correct, examples=examples, accuracy=correct / float(examples),
                  mean_loss=loss_sum / examples, weights=weights)
    with open(os.path.join(train_dir, BEST_JSON % rank), "w") as f:
        json.dump(report, f, indent=1)
        f.write("\n")
    return report


def check_moving_average_flags(flags, ctx: ReplicaContext, num_replicas_to_aggregate: int) -> None:
    """``--moving_average_decay`` / ``--eval_moving_average`` combinations that cannot work, rejected before any device
    work starts.  The same rule holds on every engine, so a flag set means the same thing everywhere."""
    d = float(getattr(flags, "moving_average_decay", 0.0) or 0.0)
    on_eval = bool(getattr(flags, "eval_moving_average", False))
    if d == 0.0:
        if on_eval:
            raise ValueError("--eval_moving_average needs --moving_average_decay: there is no moving average to score")
        return
    if not 0.0 < d < 1.0:
        raise ValueError("--moving_average_decay must lie in (0, 1) (0 = off), got %r" % d)
    # the chief updates the average from its arena after each of its steps: that arena must hold exactly one global step
    # then, and name it -- true only when every step waits for all N replicas and no peer pushes weights in between
    why = ": peers push weights into the chief's arena at any time, so the chief cannot name the global steps it would " \
          "average (supported: K = N, or --worker_times_cdf_method without --interval_method)"
    if flags.interval_method:
        raise ValueError("--moving_average_decay cannot be combined with --interval_method" + why)
    if not getattr(flags, "worker_times_cdf_method", False) and num_replicas_to_aggregate != ctx.world_size:
        raise ValueError("--moving_average_decay needs --num_replicas_to_aggregate = number of replicas (%d), got %d (K %s N)"
                         % (ctx.world_size, num_replicas_to_aggregate,
                            "<" if num_replicas_to_aggregate < ctx.world_size else ">") + why)
    if on_eval and getattr(flags, "eval_every_steps", 0) <= 0:
        raise ValueError("--eval_moving_average needs --eval_every_steps > 0: it selects the weights the in-training "
                         "evaluation scores")


def need_count(target: float, examples: int) -> int:
    """Smallest correct count ``need`` with ``need / examples >= target``, exactly (the decimal value of ``target``)."""
    return math.ceil(Fraction(str(target)) * examples)


# Stop step S = g + STOP_MARGIN for the first evaluation of global step g that reaches the target.  With K = N or cdf mode
# (replicas in lock step) this is the smallest margin with which every replica's host knows S before it launches step
# S + 1, so each one ends exactly as a run with --max_steps=S does (DESIGN §4.4 has the ordering argument):
#   the pass of g and its target test run on the chief's stream after step g, so step g + 1's last kernel, on every
#   replica, reads S -- and each host reads that word after waiting for step g + 1, which the pipelined loop does right
#   after launching step g + 2 and the non-pipelined loop right after running it.  Launching step S + 1 = g + 3 is then
#   decided with S known; with a margin of 1 step S + 1 = g + 2 would already be launched (and its final evaluation pass
#   decided) before S is known.
STOP_MARGIN = 2


class _TimeToAccuracy:
    """``--target_accuracy`` on the chief: the first evaluation that reaches ``need`` correct rows, and the training time up
    to it.  Clock values are in one unit per run (%globaltimer ns on the sm_90a path, host seconds with the torch engine);
    ``scale`` converts them to seconds."""

    def __init__(self, target: float, need: int, examples: int, scale: float, clock: str):
        self.target, self.need, self.examples, self.scale, self.clock = target, need, examples, scale, clock
        self.reached = None          # (global step, t_begin, correct, wall seconds) of the reaching pass
        self._eval_time = 0          # sum of (t_end - t_begin) over the passes before it

    def add(self, step: int, t_begin, t_end, examples: int, correct: int, counts: bool, wall_s: float) -> bool:
        """One completed pass (``counts``: its record is valid, i.e. not a dropped snapshot pass).  True if it is the first
        one to reach the target."""
        if self.reached is not None:
            return False
        if counts and examples == self.examples and correct >= self.need:
            self.reached = (step, t_begin, correct, wall_s)
            return True
        self._eval_time += t_end - t_begin
        return False

    def report(self, t0) -> Dict:
        out = dict(target=self.target, need=self.need, examples=self.examples, reached=self.reached is not None,
                   global_step=None, correct=None, accuracy=None, train_time_s=None, wall_time_s=None, clock=self.clock)
        if self.reached is not None:
            step, t_begin, correct, wall_s = self.reached
            out.update(global_step=step, correct=correct, accuracy=correct / float(self.examples),
                       train_time_s=(t_begin - t0 - self._eval_time) * self.scale, wall_time_s=wall_s)
        return out


class _EarlyStopping:
    """``--early_stopping_patience`` on the chief: :func:`early_stopping.advance` over the evaluation passes, in order.  On
    the sm_90a path eval_patience has made the same decisions on the device, which set the stop; this replays them from
    the pass records for the report.  With the torch engine this is where the stop is decided."""

    def __init__(self, patience: int, min_delta: float, examples: int, weights: str, margin: int = None):
        self.patience, self.min_delta, self.examples, self.weights = patience, min_delta, examples, weights
        self.margin = STOP_MARGIN if margin is None else int(margin)
        self.delta_rows = early_stopping.min_delta_rows(min_delta, examples)
        self.state = early_stopping.State()
        self.counted = 0             # counting passes up to the one that exhausted the patience

    def add(self, step: int, examples: int, correct: int, status: Optional[int] = None) -> bool:
        """One completed pass (``status`` as best.counts takes it).  True if it exhausted the patience."""
        if not early_stopping.exhausted(self.state, self.patience) and best.counts(examples, self.examples, status):
            self.counted += 1
        self.state, fired = early_stopping.advance(self.state, step, correct, examples, self.examples, self.patience,
                                                   self.delta_rows, status)
        return fired

    def report(self) -> Dict:
        s = self.state
        fired = early_stopping.exhausted(s, self.patience)
        return dict(patience=self.patience, min_delta=self.min_delta, min_delta_rows=self.delta_rows,
                    examples=self.examples, triggered=fired, trigger_step=s.trigger_step if fired else None,
                    stop_step=s.trigger_step + self.margin if fired else None,
                    best_step=s.best_step if s.baseline else None, best_correct=s.best if s.baseline else None,
                    counted_passes=self.counted, weights=self.weights)


class _LrPlateau:
    """``--lr_plateau_patience`` on the chief: :func:`lr_plateau.advance` over the evaluation passes, in order.  On the
    sm_90a path eval_plateau has made the same decisions on the device and stored the cuts into every replica's table;
    this replays them from the pass records for the log, the summary rate (``schedule``), the file and restarts.  With the
    torch engine this is where the cuts are decided.  The file is rewritten as soon as a cut is known, before any
    checkpoint of its ``from_step`` or later can be written."""

    def __init__(self, patience: int, factor: float, min_delta: float, examples: int, weights: str, schedule,
                 path: str, kept):
        self.patience, self.factor, self.min_delta, self.examples, self.weights = patience, factor, min_delta, examples, weights
        self.delta_rows = early_stopping.min_delta_rows(min_delta, examples)
        self.schedule, self.path = schedule, path
        self.cuts = list(kept)       # [{trigger_step, from_step}], the restored ones first
        self.state = lr_plateau.State(cuts=len(self.cuts))
        self.capped = False

    def add(self, step: int, examples: int, correct: int, status: Optional[int] = None) -> None:
        """One completed pass (``status`` as best.counts takes it)."""
        cuts = self.state.cuts
        self.state, fired = lr_plateau.advance(self.state, step, correct, examples, self.examples, self.patience,
                                               self.delta_rows, status)
        if not fired:
            return
        if self.state.cuts == cuts:
            if not self.capped:
                log.warning("Learning rate plateau: the evaluation of global step #%d exhausted the patience again, but "
                            "%d cuts have been made, the most a run makes; this and every later trigger are ignored"
                            % (step, lr_plateau.MAX_CUTS))
                self.capped = True
            return
        s = step + STOP_MARGIN
        self.cuts.append(dict(trigger_step=step, from_step=s))
        self.schedule.cuts.append(s)
        self.write()
        log.info("Learning rate plateau: cut %d after the evaluation of global step #%d (%d of %d correct, best %d, "
                 "patience %d, min_delta %d rows); from global step #%d the learning rate is %g"
                 % (len(self.cuts), step, correct, examples, self.state.best, self.patience, self.delta_rows, s,
                    self.schedule(s)))

    def report(self) -> Dict:
        return dict(patience=self.patience, factor=self.factor, min_delta=self.min_delta, min_delta_rows=self.delta_rows,
                    examples=self.examples, weights=self.weights, cuts=list(self.cuts))

    def write(self) -> None:
        tmp = self.path + ".tmp"
        with open(tmp, "w") as f:
            json.dump(self.report(), f, indent=1)
            f.write("\n")
        os.replace(tmp, self.path)


def eval_due(global_step: int, last_mark: int, every: int) -> bool:
    """Snapshot passes (K < N, interval): the host learns the global step only after a step completes, and it may jump by
    more than one.  A pass is due once the newest consumed global step has crossed a multiple of ``every`` since
    ``last_mark``, the global step consumed when the previous pass was enqueued (the restored step before the first)."""
    return every > 0 and global_step // every > last_mark // every


def train(ctx: ReplicaContext, dataset, dataset_test=None, flags=FLAGS) -> Dict:
    num_workers = ctx.world_size
    # reference distributed_train.py:118-121
    if flags.num_replicas_to_aggregate == -1:
        num_replicas_to_aggregate = num_workers
    else:
        num_replicas_to_aggregate = flags.num_replicas_to_aggregate
    assert num_workers > 0
    is_chief = ctx.is_chief
    check_async_flags(flags, ctx)
    check_local_sgd_flags(flags, ctx)
    check_batch_flags(flags, ctx)
    check_eval_flags(flags, ctx, num_replicas_to_aggregate, dataset_test)
    check_target_flags(flags, ctx)
    check_early_stopping_flags(flags, ctx)
    check_lr_plateau_flags(flags, ctx, num_replicas_to_aggregate)
    check_lr_schedule_flags(flags)
    check_best_flags(flags)
    check_moving_average_flags(flags, ctx, num_replicas_to_aggregate)
    check_device_data_flags(flags, ctx, dataset)
    weight_decay.check_flags(flags, ctx)
    aug_ranges = augment.from_flags(flags)
    aug_elastic = augment.elastic_from_flags(flags)
    if aug_elastic is not None and aug_ranges is None:
        aug_ranges = augment.Ranges(0.0, 0.0, 0.0)          # elastic distortion alone
    device_data = bool(getattr(flags, "device_data", False))
    target = float(getattr(flags, "target_accuracy", 0.0) or 0.0)
    patience = int(getattr(flags, "early_stopping_patience", 0) or 0)
    stop_armed = bool(target or patience)      # something may set a stop step S before --max_steps
    plateau = int(getattr(flags, "lr_plateau_patience", 0) or 0)
    ema_decay = float(getattr(flags, "moving_average_decay", 0.0) or 0.0) if is_chief else 0.0
    eval_average = bool(ema_decay and getattr(flags, "eval_moving_average", False))

    backend = make_backend(ctx, flags.backend, flags)
    engine = make_engine(flags, ctx, backend)
    spec = engine.spec
    lr_schedule = LearningRateSchedule.from_flags(flags, dataset.num_examples, num_replicas_to_aggregate)
    straggler = parse_straggler_spec(flags.inject_straggler, flags.sync_timeout_ms)

    async_mode = bool(getattr(flags, "async_method", False))
    local_h = int(getattr(flags, "local_sgd_steps", 0) or 0)
    margin = stop_margin(flags)
    if async_mode:
        opt = AsyncSGDOptimizer(backend, lr_schedule, total_num_replicas=num_workers, straggler=straggler, seed=flags.seed,
                                ssp_staleness=int(getattr(flags, "ssp_staleness", -1)))
    elif local_h:
        opt = LocalSGDOptimizer(backend, lr_schedule, total_num_replicas=num_workers, period=local_h, straggler=straggler,
                                seed=flags.seed)
    elif flags.interval_method or flags.worker_times_cdf_method:
        # reference :179-183 -- interval wins when both are set, as there.
        mode = "interval" if flags.interval_method else "cdf"
        opt = TimeoutReplicasOptimizer(backend, lr_schedule, total_num_replicas=num_workers, mode=mode,
                                       interval_ms=flags.interval_ms, straggler=straggler, seed=flags.seed)
    else:
        opt = SyncReplicasOptimizer(
            backend, lr_schedule, replicas_to_aggregate=num_replicas_to_aggregate,
            total_num_replicas=num_workers,
            drop_connect_probability=flags.drop_connect_probability if flags.drop_connect else None,
            straggler=straggler, seed=flags.seed)
    # GPU path: every mode runs as one CUDA graph per step -- K-of-N / full barrier through the fused aggregation kernels,
    # interval through the device-side deadline protocol (csrc/fused_interval.cu)
    fused_step = hasattr(engine, "attach_optimizer")
    if fused_step:
        engine.attach_optimizer(opt)   # GPU path: compute + fused allreduce/SGD replay as one CUDA graph
    decay = weight_decay.value(flags)
    if decay:
        engine.arm_weight_decay(decay)  # GPU path: after attach_optimizer, whose mode it checks
        log.info("L2 weight decay %g of %s; the logged training loss includes it"
                 % (decay, ", ".join(q.name for q in weight_decay.decayed(spec))))

    # Supervisor semantics: chief restores the newest checkpoint, everyone gets it.
    restored_step = 0
    restored_average = None        # --moving_average_decay: the averages of the restored checkpoint, if it holds all
    restored = False
    if is_chief:
        os.makedirs(flags.train_dir, exist_ok=True)
        latest = Saver.latest(flags.train_dir)
        if latest is not None:
            state, restored_step = Saver.restore(latest)
            engine.params.copy_(spec.from_state_dict(state).to(engine.params.device))
            log.info("Restored model from %s at step=%d" % (latest, restored_step))
            restored = True
            if ema_decay:
                restored_average = moving_average.from_state_dict(spec, state)
    if num_workers > 1:
        restored_step = backend.all_gather_object(restored_step)[0]
        if restored_step > 0:
            backend.broadcast_(engine.params, 0)
    if restored_step > 0:
        opt.local_step = restored_step
        if hasattr(backend, "set_global_step"):
            backend.set_global_step(restored_step)
    if hasattr(engine, "params_updated"):
        engine.params_updated()
    if aug_ranges is not None:
        # every replica, after attach_optimizer: each training iteration draws from its own counter, which starts past the
        # iterations that went into the restored global step, so that a restarted one-replica run does not replay their
        # draws (multi-replica K > N and interval runs can: see augment.start_iteration)
        aug_start = augment.start_iteration(restored_step, isinstance(opt, SyncReplicasOptimizer),
                                            num_replicas_to_aggregate, num_workers)
        if aug_elastic is None:
            engine.arm_augment(*aug_ranges, start_iteration=aug_start)
            log.info("Random affine augmentation of the training images: %s, draws from iteration %d; evaluation is "
                     "not augmented" % (augment.describe(aug_ranges), aug_start))
        else:
            engine.arm_augment(*aug_ranges, start_iteration=aug_start, elastic=aug_elastic)
            log.info("Random affine augmentation and elastic distortion of the training images: %s, draws from "
                     "iteration %d; evaluation is not augmented" % (augment.describe(aug_ranges, aug_elastic), aug_start))
    if ema_decay:
        # the chief's average starts from the restored averages, else from the (initial or restored) weights; from here on
        # every global step ends with its update (GPU path: a node at the end of the chief's step graph)
        if fused_step:
            engine.arm_moving_average(ema_decay)
        else:
            engine.arm_moving_average(ema_decay, restored_step)
        if restored_average is not None:
            engine.load_moving_average(restored_average)
        elif restored:
            log.info("Moving average: the restored checkpoint holds no complete set of averages; they start from the "
                     "restored weights")
        log.info("Moving average of the weights: decay %g; the in-training evaluation scores the %s weights"
                 % (ema_decay, "averaged" if eval_average else "live"))
    log.info("Learning rate schedule: %s; the update of global step #%d is made at %g"
             % (describe_lr_schedule(lr_schedule), restored_step, lr_schedule(restored_step)))
    log.info("%s Supervisor" % datetime.now())

    # --eval_every_steps: the chief scores the validation set after every E-th global step and after the last one.  GPU path:
    # a forward-only pass on the training stream right after the step (engine.enqueue_eval), read back from page-locked
    # host memory once the following step has been consumed; torch engine: engine.evaluate, synchronously.
    eval_every = int(getattr(flags, "eval_every_steps", 0) or 0) if is_chief else 0
    device_eval = bool(eval_every and fused_step)
    # local SGD is in lock step too: every replica makes one iteration per global step, and no peer writes the chief's
    # arena outside the averaging rounds the chief takes part in
    exact = isinstance(opt, SyncReplicasOptimizer) and num_replicas_to_aggregate == num_workers \
        or bool(flags.worker_times_cdf_method and not flags.interval_method) or bool(local_h)
    # K < N / interval: peers push into the chief's arena at any time -> score a validated snapshot (--eval_snapshot);
    # the host cannot name the step a pass scores in advance, so passes follow the consumed global step (eval_due)
    snapshot_eval = device_eval and bool(getattr(flags, "eval_snapshot", False)) and not exact and not async_mode
    # asynchronous SGD: the working arena is private to its replica between iterations, so the pass scores it live, labelled
    # with the global step r it was pulled at; like snapshot passes, passes follow the consumed global step
    follow_eval = snapshot_eval or (device_eval and async_mode)
    if device_eval:
        if eval_average:
            engine.arm_eval(dataset_test.images, dataset_test.labels, snapshot=snapshot_eval, moving_average=True)
        else:
            engine.arm_eval(dataset_test.images, dataset_test.labels, snapshot=snapshot_eval)
    if device_data:
        # every replica keeps its own copy, in its own shuffled order: a step's input is then B row indices
        engine.arm_train_data(dataset.images, dataset.labels)
    # --target_accuracy: the run ends as --max_steps = min(--max_steps, S) would end it, S = the stop step of the first
    # evaluation that reaches the target.  GPU path: the chief's pass sets S in every replica's stop word on the device and
    # every step's last kernel copies it to the host; torch engine (one replica): decided on the host after `evaluate`.
    max_steps = flags.max_steps
    tta = None
    if stop_armed and fused_step:
        engine.arm_stop()                  # every replica (a symmetric allocation), for a target or a patience
    if target and is_chief:
        n_val = dataset_test.num_examples
        tta = _TimeToAccuracy(target, need_count(target, n_val), n_val, 1e-9 if device_eval else 1.0,
                              "device %globaltimer" if device_eval else "host")
        if device_eval:
            engine.arm_target(tta.need, margin)
    eval_weights = "snapshot" if snapshot_eval else ("moving_average" if eval_average else "live")
    # --early_stopping_patience: the run ends as --max_steps = min(--max_steps, S) would end it, S = g + STOP_MARGIN for the
    # pass of global step g that exhausts the patience -- decided like the target (GPU path: eval_patience on the device,
    # after eval_target, so whichever fires first sets S; torch engine: on the host after `evaluate`).
    es = None
    if patience and is_chief:
        es = _EarlyStopping(patience, float(getattr(flags, "early_stopping_min_delta", 0.0) or 0.0),
                            dataset_test.num_examples, eval_weights, margin)
        if device_eval:
            engine.arm_patience(patience, es.delta_rows, margin)
    # --lr_plateau_patience: from S = g + STOP_MARGIN on, for the pass of global step g that exhausts the patience, every
    # update is made at the rate times --lr_plateau_factor once more (GPU path: eval_plateau stores S into every replica's
    # cut table, which the aggregation kernels read; torch engine: decided on the host after `evaluate`, into the shared
    # schedule).  A restarted run keeps the cuts of the restored checkpoint's past, from its file.
    lp = None
    if plateau:
        factor = float(flags.lr_plateau_factor)
        kept, refusal = restart_lr_cuts(flags.train_dir, ctx.rank, restored_step, factor) if is_chief else ([], None)
        if num_workers > 1:
            kept, refusal = backend.all_gather_object((kept, refusal))[0]
        if refusal:
            raise ValueError(refusal)
        lr_schedule.factor = factor
        lr_schedule.cuts = [c["from_step"] for c in kept]
        if fused_step:
            engine.arm_lr_cuts(factor, lr_schedule.cuts)          # every replica (a symmetric allocation)
        if is_chief:
            lp = _LrPlateau(plateau, factor, float(getattr(flags, "lr_plateau_min_delta", 0.0) or 0.0),
                            dataset_test.num_examples, eval_weights, lr_schedule,
                            os.path.join(flags.train_dir, LR_PLATEAU_JSON % ctx.rank), kept)
            lp.write()
            if kept:
                log.info("Learning rate plateau: %d cut(s) up to the restored global step #%d kept; from there the "
                         "learning rate is %g" % (len(kept), restored_step, lr_schedule(restored_step)))
            if device_eval:
                engine.arm_lr_plateau(plateau, lp.delta_rows, STOP_MARGIN, len(kept))
    # --keep_best_checkpoint: the chief keeps the weights of its best-scoring evaluation (GPU path: decided and copied on the
    # device inside the pass's graph; torch engine: after `evaluate`) and writes them once, after the final pass.  A best
    # file of an earlier run sets the count to beat.
    keep_best = bool(eval_every and getattr(flags, "keep_best_checkpoint", False))
    if keep_best:
        earlier = read_best(flags.train_dir, ctx.rank)
        best_seed = int(earlier["correct"]) if earlier else 0
        engine.arm_best(best_seed)
        if earlier:
            log.info("Best weights: an earlier run kept the evaluation of global step #%d (%d of %d correct); only a "
                     "better one replaces it" % (earlier["global_step"], earlier["correct"], earlier["examples"]))
    eval_rows = []                 # (global_step, t_begin_unix_s, eval_seconds, examples, correct, mean_loss)
    last_eval_step = -1
    eval_mark = restored_step      # snapshot passes: global step consumed when the last one was enqueued
    test_acc_value = 0.0           # newest complete evaluation; hard-wired to 0 in the reference (:363) and when off

    ckpt = None
    if is_chief:
        # GPU path: checkpoints are device captures of the chief's arena after a launched step -- a copy of the live arena
        # when no peer writes it between steps (the same `exact` test as the evaluation pass), else a validated snapshot
        device_ckpt = fused_step and hasattr(engine, "arm_checkpoint")
        if device_ckpt:
            engine.arm_checkpoint(snapshot=not (exact or async_mode))
        ckpt = _AsyncCheckpointer(flags.train_dir, spec, flags.save_interval_secs, engine=engine if device_ckpt else None,
                                  timeout_s=flags.sync_timeout_ms * 1e-3,
                                  average=engine._ema if ema_decay and not device_ckpt else None)
    summary = SummaryWriter(flags.train_dir) if (is_chief and flags.should_summarize) else None

    # Even if not using timeout, we want to wait until all machines are ready (reference :275-277).
    timeout_client, timeout_server = launch_manager(backend, flags)

    next_summary_time = time.time() + flags.save_summaries_secs
    begin_time = time.time()
    cur_iteration = -1
    if flags.interval_method:
        if fused_step and hasattr(backend, "interval_arm"):
            backend.interval_arm(float(flags.interval_ms))   # reference :287-288 (chief timer) -> %globaltimer deadline on the device
        else:
            opt.start_interval_updates()   # CPU plumbing path: shared absolute host-clock deadlines
    elif getattr(engine, "_kgtn_k", 0):
        backend.kgtn_arm()                 # K > N on the device: a restore moved the step counter, accumulate from there
    elif async_mode and fused_step:
        engine.async_arm()                 # every master copy holds the (restored) weights before the first pull

    time_acc_list = []
    step = restored_step
    loss_value = train_acc_value = float("nan")
    results = {"steps": [], "losses": [], "accepted": 0, "dropped": 0, "lr_schedule": lr_schedule.describe()}
    # cdf telemetry (reference timeout_manager.py:55-61): compute time = gradient done - token dequeued, the barrier wait
    # NOT included.  interval wins when both flags are set (as in the reference) and its replicas are not in lock step, so
    # the collective flush of the cdf tables must not run then.
    cdf = bool(flags.worker_times_cdf_method and not flags.interval_method)
    device_times = cdf and fused_step and hasattr(backend, "read_timing")   # %globaltimer stamps written by the step's kernels
    cdf_pushed = 0                 # first iteration whose device stamps have not been handed to the timeout client yet
    # GPU path: the host runs ONE step ahead of the device -- step i+1 is enqueued before step i's (loss, status words) are
    # read from the page-locked buffers the step's graph copied them to, so no iteration ever waits for a device sync, and
    # batches are packed into page-locked buffers by a helper thread (`_BatchPacker`).
    pipelined = bool(fused_step and getattr(flags, "pipeline_steps", True) and hasattr(engine, "read_result_async")
                     and not flags.timeline_logging)
    # --device_data: the batch is gathered on the device from B row indices (_IndexFeed) instead of packed on the host
    packer = (_IndexFeed(dataset, flags.batch_size) if device_data else _BatchPacker(engine, dataset, flags.batch_size)) \
        if pipelined else None
    every = max(flags.log_every, 1)
    pending = None                 # (iteration, start_time, result token) of the step in flight
    launched = 0
    stop = False

    def finish_iteration(it: int, start_time: float, info, loss_acc) -> None:
        nonlocal step, loss_value, train_acc_value, next_summary_time, stop
        step = info.global_step
        do_log = (it % every == 0)
        if loss_acc is not None:
            loss_value, train_acc_value = loss_acc
        if do_log:
            log.info("Global step attained: %d" % step)
            log.info("DONE RUNNING SESSION...")
        finish_time = time.time()
        if step > max_steps:
            stop = True
            return
        duration = finish_time - start_time
        examples_per_sec = flags.batch_size / float(max(duration, 1e-9))
        if do_log:
            log.info(LOG_FORMAT % (ctx.rank, datetime.now(), step, loss_value, train_acc_value,
                                   test_acc_value, examples_per_sec, duration))
        time_acc_list.append((finish_time, train_acc_value, test_acc_value, loss_value))
        results["steps"].append(step)
        results["losses"].append(loss_value)
        if step % flags.save_results_period == 0:
            np.save(os.path.join(flags.train_dir, "worker%d_time_acc.npy" % ctx.rank), np.array(time_acc_list))
            if eval_every:
                save_evals()
        if is_chief:
            # local SGD: only the weights after an averaging step are the model; the capture follows the newest launched
            # step (one past `step` in the pipelined loop)
            ckpt.maybe_save(engine.params, step, capture=not local_h or (restored_step + launched if pipelined else step)
                            % local_h == 0)
            if summary is not None and next_summary_time < time.time():
                log.info("Running Summary operation on the chief.")
                summary.add_scalars({"loss": loss_value, "train_acc": train_acc_value,
                                     "learning_rate": lr_schedule(step)}, step)
                log.info("Finished running Summary operation.")
                next_summary_time += flags.save_summaries_secs

    def collect_evals() -> None:
        """Device records completed so far (%globaltimer ns -> seconds, as push_device_times converts them)."""
        nonlocal test_acc_value
        if tta is None and es is None and lp is None:
            recs = [(r, 0) for r in engine.eval_records()]
        else:                      # dropped snapshot passes took training-stream time too, and count for neither rule
            recs = engine.eval_records_with_status()
            engine.eval_dropped += sum(1 for _r, status in recs if status < 0)
        for (gs, t0, t1, n_ex, correct, loss_sum), status in recs:
            if tta is not None:
                tta.add(gs, t0, t1, n_ex, correct, status >= 0, time.time() - tta_wall0)
            if es is not None:
                es.add(gs, n_ex, correct, status if snapshot_eval else None)
            if lp is not None:
                lp.add(gs, n_ex, correct, status if snapshot_eval else None)
            if status < 0:
                continue
            eval_rows.append((gs, t0 * 1e-9, (t1 - t0) * 1e-9, n_ex, correct, loss_sum / max(n_ex, 1)))
            test_acc_value = correct / float(max(n_ex, 1))

    def note_stop() -> None:
        """GPU path: the stop step S the chief's target test set, as the step just waited for read it."""
        nonlocal max_steps
        s = engine.stop_step()
        if s:
            max_steps = min(max_steps, s)

    def eval_after_step(global_step: int) -> None:
        """Non-pipelined loops: called once the step's outcome has been read back."""
        nonlocal test_acc_value, last_eval_step, eval_mark, max_steps
        if device_eval:
            collect_evals()        # the step read-back above waited for the pass enqueued after the previous step
        if follow_eval:
            if global_step <= max_steps and eval_due(global_step, eval_mark, eval_every):
                eval_mark = global_step
                engine.enqueue_eval()          # the final pass follows the loop
            return
        if global_step == last_eval_step or not (global_step % eval_every == 0 or global_step > max_steps):
            return
        if local_h and global_step > max_steps and not local_done:
            return                 # the final pass follows the run's final average
        last_eval_step = global_step
        if device_eval:
            engine.enqueue_eval()
            return
        t0 = time.time()
        if eval_average:
            loss, acc = engine.evaluate(dataset_test.images, dataset_test.labels, moving_average=True)
        else:
            loss, acc = engine.evaluate(dataset_test.images, dataset_test.labels)
        t1 = time.time()
        n_ex = dataset_test.num_examples
        correct = int(round(acc * n_ex))
        eval_rows.append((global_step, t0, t1 - t0, n_ex, correct, loss))
        test_acc_value = correct / float(n_ex)
        if keep_best:
            engine.note_eval(global_step, n_ex, n_ex, correct, loss * n_ex, moving_average=eval_average)
        if tta is not None and tta.add(global_step, t0, t1, n_ex, correct, True, t1 - tta_wall0):
            max_steps = min(max_steps, global_step + margin)
        if es is not None and es.add(global_step, n_ex, correct):
            max_steps = min(max_steps, global_step + margin)
        if lp is not None:
            lp.add(global_step, n_ex, correct)

    def save_evals() -> None:
        np.save(os.path.join(flags.train_dir, "worker%d_eval.npy" % ctx.rank),
                np.array(eval_rows, dtype=np.float64).reshape(-1, 6))

    def push_device_times(upto: int) -> None:
        """Hand the %globaltimer stamps of iterations [cdf_pushed, upto] to the timeout client: 'dequeued' = the step's first
        kernel started, 'finished' = the aggregation kernel was entered (gradient complete, barrier not yet waited for)."""
        nonlocal cdf_pushed
        if upto < cdf_pushed:
            return
        pairs = backend.read_timing(restored_step + cdf_pushed, restored_step + upto)
        for it, (ts, ta) in zip(range(cdf_pushed, upto + 1), pairs):
            timeout_client.broadcast_worker_dequeued_token(it, ts * 1e-9)
            timeout_client.broadcast_worker_finished_computing_gradients(it, ta * 1e-9)
        cdf_pushed = upto + 1

    local_done = False
    last_consume = time.time()
    tta_wall0 = time.time()        # --target_accuracy: the run's first step starts now (host clock) ...
    if tta is not None and device_eval:
        engine.enqueue_start_stamp()   # ... and on the chief's device clock, in stream order before that step
    while not stop:
        cur_iteration += 1
        do_log = (cur_iteration % every == 0)
        if do_log:
            log.info("A new iteration...")

        if cdf and not device_times:
            t_deq = opt.wait_op()
            timeout_client.broadcast_worker_dequeued_token(cur_iteration, t_deq)

        if pipelined:
            if do_log:
                log.info("RUNNING SESSION... %f" % time.time())
            # input DMA (+ gather) + step graph: one native call
            token = (cur_iteration, engine.step_indices(packer.next()) if device_data else engine.step_packed(packer.next()))
            launched += 1
            if device_eval and not follow_eval and \
                    ((restored_step + launched) % eval_every == 0 or restored_step + launched > max_steps) and \
                    not (local_h and restored_step + launched > max_steps):
                engine.enqueue_eval()          # K == N: restored_step + launched is the global step of the weights it scores
            prev, pending = pending, token
            if prev is not None:
                it, (ev, lbuf, seq) = prev
                ev.synchronize()
                info = opt._account(backend.mirror_info(seq, check=True))
                if device_eval:
                    collect_evals()            # passes enqueued before the step just waited for are complete
                if stop_armed:
                    note_stop()
                now = time.time()
                finish_iteration(it, last_consume, info, (float(lbuf[0]), float(lbuf[1])))
                last_consume = now
                if follow_eval and not stop and eval_due(step, eval_mark, eval_every):
                    eval_mark = step
                    engine.enqueue_eval()      # after the step just launched: scores the newest committed weights then
                if device_times and it > 10 and (it % 50 == 0 or it == 500):
                    push_device_times(it)
            # K == N: the global step after `launched` steps is known without reading anything -> stop launching exactly there
            if exact and restored_step + launched > max_steps:
                break
            continue

        tl = Timeline(pid=ctx.rank) if flags.timeline_logging else None
        start_time = time.time()
        if device_data:
            rows = dataset.next_batch_indices(flags.batch_size)
        else:
            images, labels = dataset.next_batch(flags.batch_size)
        if tl:
            tl.add_span("next_batch", 0.0, (time.time() - start_time) * 1e6)
        if do_log:
            log.info("RUNNING SESSION... %f" % time.time())

        t0 = time.perf_counter()
        if device_data:
            engine.load_indices(rows)
        else:
            engine.load_batch(images, labels)
        t1 = time.perf_counter()
        t_fin = None
        dev_spans = None
        if fused_step:
            if tl and ctx.on_gpu:
                # reference: RunOptions(trace_level=FULL_TRACE) per step (src/distributed_train.py:317-319) -> here CUPTI around
                # the graph replay: every kernel / copy of the step with its stream, start and duration
                dev_spans = cupti_device_spans(engine.train_step)
            else:
                engine.train_step()
            t2 = time.perf_counter()
            info = opt._account(engine.step_info())   # device -> host read of the step's outcome (one packed copy)
            if stop_armed:
                note_stop()                           # (the read above waited for the whole step)
        else:
            engine.forward_backward(opt.local_step)
            t2 = time.perf_counter()
            t_fin = time.time()                       # gradient complete; the barrier / reduction comes after this stamp
            info = opt.apply_gradients(engine.params, engine.grads) if not isinstance(opt, TimeoutReplicasOptimizer) \
                else opt.apply_gradients(engine.params, engine.grads, ctx.rank, cdf)
            if info.applied and hasattr(engine, "params_updated") and not hasattr(engine, "train_step"):
                engine.params_updated()
            if ema_decay and info.applied:
                engine.update_moving_average(info.global_step)
        la = engine.loss_acc() if (do_log or flags.timeline_logging) else None
        t3 = time.perf_counter()
        if eval_every:
            eval_after_step(info.global_step)

        if cdf:
            if device_times:
                if cur_iteration > 10 and (cur_iteration % 50 == 0 or cur_iteration == 500):
                    push_device_times(cur_iteration)
            else:
                opt.finish_times.append(t_fin if t_fin is not None else time.time())
                timeout_client.broadcast_worker_finished_computing_gradients(cur_iteration, opt.finish_times[-1])

        if tl:
            base = (t0 - tl._t0) * 1e6
            tl.add_span("load_batch(H2D)", base, (t1 - t0) * 1e6)
            tl.add_span("forward_backward", base + (t1 - t0) * 1e6, (t2 - t1) * 1e6)
            tl.add_span("aggregate+apply", base + (t2 - t0) * 1e6, (t3 - t2) * 1e6)
            if dev_spans:
                tl.add_device_spans(dev_spans, base + (t1 - t0) * 1e6)
            with open(timeline_path(flags.train_dir, ctx.rank, info.global_step), "w") as f:
                f.write(tl.generate_chrome_trace_format())
        finish_iteration(cur_iteration, start_time, info, la)

    if pending is not None:          # drain the step still in flight
        it, (ev, lbuf, seq) = pending
        ev.synchronize()
        info = opt._account(backend.mirror_info(seq, check=True))
        finish_iteration(it, last_consume, info, (float(lbuf[0]), float(lbuf[1])))
        pending = None
    if packer is not None:
        packer.close()
    if async_mode and fused_step:
        # every replica's last update applied, the device barrier, one more pull: the chief's arena, the final pass and
        # the final checkpoint hold every update of the run, and their global step is the number of updates
        step = engine.async_finish()
    local_done = True              # local SGD: eval_after_step may score the step past --max_steps from here on
    if local_h:
        # the last step was not an averaging step: one more average, so the final pass, the final checkpoint and the
        # returned weights are the model every replica holds (collective: every replica ends on the same step)
        if fused_step:
            step = engine.local_finish()
        elif step % local_h:
            opt.average(engine.params)
            if hasattr(engine, "params_updated"):
                engine.params_updated()
        if eval_every:
            if device_eval:
                engine.enqueue_eval()
            else:
                eval_after_step(step)
    if follow_eval:
        engine.enqueue_eval()          # once after the last step
    if device_eval:
        torch.cuda.synchronize()       # the pass after the final step
        collect_evals()
        if snapshot_eval and engine.eval_dropped:
            log.info("in-training evaluation: %d pass(es) found no consistent weight snapshot and were dropped"
                     % engine.eval_dropped)
    if eval_every:
        save_evals()
    if tta is not None:
        report = tta.report(engine.start_stamp_ns() if device_eval else tta_wall0)
        if eval_average:
            report["weights"] = "moving_average"       # the evaluations scored the averaged weights
        results["time_to_accuracy"] = report
        with open(os.path.join(flags.train_dir, "worker%d_time_to_accuracy.json" % ctx.rank), "w") as f:
            json.dump(report, f, indent=1)
            f.write("\n")
        if report["reached"]:
            log.info("Time to accuracy: target %g reached by the evaluation of global step #%d (accuracy %f, %d of %d "
                     "correct); training time %.6f s without the evaluations (%s clock); wall time %.6f s"
                     % (target, report["global_step"], report["accuracy"], report["correct"], report["examples"],
                        report["train_time_s"], tta.clock, report["wall_time_s"]))
        else:
            log.info("Time to accuracy: target %g not reached" % target)
    if es is not None:
        rep = results["early_stopping"] = es.report()
        with open(os.path.join(flags.train_dir, EARLY_STOPPING_JSON % ctx.rank), "w") as f:
            json.dump(rep, f, indent=1)
            f.write("\n")
        device_state = engine.patience_state() if device_eval else None
        if device_state is not None and device_state != es.state:
            log.warning("Early stopping: the device state %s differs from the replay of the evaluation records %s"
                        % (device_state, es.state))
        if rep["triggered"]:
            log.info("Early stopping: patience %d exhausted by the evaluation of global step #%d, the best being that of "
                     "global step #%d (%d of %d correct, min_delta %d rows); the run ends as --max_steps=%d would end it"
                     % (patience, rep["trigger_step"], rep["best_step"], rep["best_correct"], rep["examples"],
                        rep["min_delta_rows"], rep["stop_step"]))
        else:
            log.info("Early stopping: patience %d not exhausted after %d counted evaluation(s)"
                     % (patience, rep["counted_passes"]))
    if lp is not None:
        results["lr_plateau"] = lp.report()
        lp.write()
        device_state = engine.lr_plateau_state() if device_eval else None
        if device_state is not None and device_state != lp.state:
            log.warning("Learning rate plateau: the device state %s differs from the replay of the evaluation records %s"
                        % (device_state, lp.state))
    if keep_best:
        rep = results["best"] = save_best(engine, spec, flags.train_dir, ctx.rank, eval_weights)
        if rep is not None:
            log.info("Best weights: the evaluation of global step #%d (accuracy %f, %d of %d correct, mean loss %f, %s "
                     "weights) saved under %s" % (rep["global_step"], rep["accuracy"], rep["correct"], rep["examples"],
                                                  rep["mean_loss"], eval_weights, os.path.join(flags.train_dir, BEST_DIR)))
        else:
            log.info("Best weights: no complete evaluation of this run scored more than %d correct; nothing written"
                     % best_seed)
    if device_times:
        push_device_times(cur_iteration)

    if is_chief:
        log.info("Elapsed Time: %f" % (time.time() - begin_time))
    if cdf:
        timeout_client.flush()
        if ctx.rank == 0 and device_times:
            timeout_server.report()

    # Save after the training ends (reference :405-408).
    if is_chief:
        ckpt.save(engine.params, step, blocking=True)
        ckpt.close()
        if ckpt.failed:
            log.info("checkpoints: %d capture(s) found no consistent weight snapshot; each was retried at the next step"
                     % ckpt.failed)
    if summary is not None:
        summary.close()
    if eval_every:
        results["evals"] = eval_rows
    if getattr(engine, "_kgtn_k", 0):
        # K > N on the device: the control block counts exactly the gradients that entered a committed update (credited
        # by the committers) and the dropped ones; the per-iteration status words the loop consumed cannot tell them apart
        torch.cuda.synchronize()
        st = backend.read_status()
        opt.accepted_steps, opt.dropped_steps = st["accepted_steps"], st["dropped_steps"]
    if async_mode:
        st = engine.async_staleness() if fused_step else None
        rep = staleness_report(st["hist"], st["tau_sum"], st["tau_max"]) if st is not None else opt.staleness()
        opt.accepted_steps, opt.dropped_steps = rep["updates"], 0
        results["staleness"] = rep
        with open(os.path.join(flags.train_dir, STALENESS_JSON % ctx.rank), "w") as f:
            json.dump(rep, f, indent=1)
            f.write("\n")
        log.info("Staleness: worker %d applied %d update(s); staleness of its updates (global steps between pull and "
                 "update) mean %.3f, p50 %d, p99 %d, max %d; final global step %d"
                 % (ctx.rank, rep["updates"], rep["mean"], rep["p50"], rep["p99"], rep["max"], step))
        ssp = int(getattr(flags, "ssp_staleness", -1))
        if ssp >= 0:
            # the torch engine runs one replica, which never waits
            b = engine.ssp_stats() if fused_step else dict(waits=0, wait_total_ns=0, wait_max_ns=0, lead_max=0)
            rep = ssp_report(ssp, b["waits"], b["wait_total_ns"], b["wait_max_ns"], b["lead_max"], rep["updates"])
            results["ssp"] = rep
            with open(os.path.join(flags.train_dir, SSP_JSON % ctx.rank), "w") as f:
                json.dump(rep, f, indent=1)
                f.write("\n")
            log.info("Stale synchronous: worker %d ran at most %d update(s) ahead of the slowest running replica; %d of "
                     "its %d update(s) waited, %.6f s in total, longest %.6f s; largest lead seen %d; final global step %d"
                     % (ctx.rank, ssp, rep["waits"], rep["updates"], rep["wait_total_ns"] * 1e-9,
                        rep["wait_max_ns"] * 1e-9, rep["lead_max"], step))
    if local_h:
        st = engine.local_stats() if fused_step else None
        rep = local_sgd_report(local_h, st["rounds"], st["wait_total_ns"], st["wait_max_ns"]) if st is not None \
            else opt.report()
        results["local_sgd"] = rep
        with open(os.path.join(flags.train_dir, LOCAL_SGD_JSON % ctx.rank), "w") as f:
            json.dump(rep, f, indent=1)
            f.write("\n")
        log.info("Local SGD: worker %d averaged every %d step(s); %d averaging round(s), %.6f s in their barriers "
                 "(mean %.6f s, max %.6f s); final global step %d"
                 % (ctx.rank, local_h, rep["rounds"], rep["wait_total_s"], rep["wait_mean_s"], rep["wait_max_s"], step))
    results.update(final_step=step, accepted=opt.accepted_steps, dropped=opt.dropped_steps,
                   params=engine.params, elapsed=time.time() - begin_time,
                   timeout_server=timeout_server, engine=engine, optimizer=opt)
    return results
