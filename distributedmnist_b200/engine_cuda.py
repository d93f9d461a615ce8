"""sm_90a compute engine: the reference convnet's training step as 11 hand-written kernels
replayed from one CUDA graph.

Step = (reference src/distributed_train.py:332 ``sess.run(apply_gradients_op)``)::

    memset(small grads, loss)                              folded into conv1_fwd
    conv1_fwd        wgmma, software im2col + bias/ReLU/pool  csrc/conv1_tc.cu
    conv2_fwd        wgmma implicit GEMM + bias/ReLU/pool csrc/conv2_tc.cu
    fc1_fwd          wgmma GEMM, split-K into fp32        csrc/gemm_tc.cu
    fc2_fwd_bwd      bias+ReLU+dropout, fc2, softmax-CE,
                     accuracy, dlogits, d(fc1)              csrc/lenet_simt.cu
    fc2_wgrad        fc2 weight/bias + fc1 bias gradients   (side branch)
    fc1_wgrad        wgmma GEMM (MN-major x MN-major) -> gradient arena
    fc1_dgrad        wgmma GEMM, maxpool2/ReLU2 backward + conv2 bias grad in the epilogue
    conv2_wgrad      wgmma, K = whole images, per-CTA partials -> workspace
    conv2_wgrad_reduce  the partials summed in fixed order -> gradient arena
    conv2_dgrad      wgmma
    conv1_wgrad      wgmma, maxpool1/ReLU1 backward fused into the operand build
    fused_sync_sgd   arrival -> mask -> NVLink reduce -> 1/count -> SGD -> push -> bf16 shadow

Weights live in TF layouts in one flat fp32 arena (symmetric memory); the tensor-core
kernels read the bf16 shadow arena the fused kernel refreshes.  Nothing on this path
calls cuDNN, cuBLAS or NCCL.
"""
from __future__ import annotations

import contextlib
import ctypes
import gc
import os
from typing import Optional, Tuple

import numpy as np
import torch

from . import augment, early_stopping, lr_plateau, weight_decay
from .best import BEST_CORRECT_WORD, BEST_EXAMPLES_WORD, BEST_STEP_WORD, BEST_VALID_WORD
from .early_stopping import PAT_BASELINE_WORD, PAT_BEST_STEP_WORD, PAT_BEST_WORD, PAT_SINCE_WORD, PAT_TRIGGER_WORD
from .lr_plateau import PL_BASELINE_WORD, PL_BEST_WORD, PL_CUTS_WORD, PL_SINCE_WORD, PL_TRIGGER_WORD
from .engine import ComputeEngine
from .models import get_model
from .models.lenet import dropout_seed_mix
from .ops import gemm as G
from .ops.lib import load, stream_ptr
from .parallel.backends import StepInfo
from .parallel.fused import FusedBackend


@contextlib.contextmanager
def _capture(graph: torch.cuda.CUDAGraph, stream: torch.cuda.Stream):
    """Capture into ``graph`` on ``stream`` with the cyclic garbage collector paused.  Engines sit in reference cycles (an
    engine and its _Snapshot), so only the collector frees an old one, and its graphs' destructors would then run inside
    this capture, where destroying a graph is not permitted: the capture would be invalidated.  thread_local: other threads
    (NCCL watchdog, pin-memory) may call CUDA while we capture."""
    enabled = gc.isenabled()
    gc.disable()
    try:
        with torch.cuda.graph(graph, stream=stream, capture_error_mode="thread_local"):
            yield
    finally:
        if enabled:
            gc.enable()


class _RunnerEvent:
    """Completion of a step launched through the native runner: ``synchronize()`` like a ``torch.cuda.Event``."""

    def __init__(self, lib, runner, slot: int):
        self.lib, self.runner, self.slot = lib, runner, slot

    def synchronize(self) -> None:
        self.lib.dm_runner_wait(self.runner, self.slot)

    def query(self) -> bool:
        return self.lib.dm_runner_query(self.runner, self.slot) == 1


class _Snapshot:
    """Validated copy of the newest committed weights of an engine's arena (csrc/eval_snapshot.cu) into its owner's buffers:
    a SnapState of its own, an fp32 arena ``snap`` and, for the ``bf_ranges`` ([begin, end) pairs, multiples of 4), their
    bf16 shadow in ``snap16``.  Each owner (the evaluation pass, the checkpoint capture) instantiates one, so their statistics
    and accepted steps stay apart."""

    def __init__(self, engine: "_CudaEngine", snap: torch.Tensor, snap16: Optional[torch.Tensor] = None, bf_ranges=(),
                 keep: Optional[torch.Tensor] = None):
        assert len(bf_ranges) in (0, 4) and (snap16 is not None or not bf_ranges)
        self.eng, self.snap, self.snap16, self.keep = engine, snap, snap16, keep
        self.bf_ranges = list(bf_ranges)
        self.state = torch.zeros(int(engine.lib.dm_snap_state_bytes()), dtype=torch.uint8, device=engine.device)
        self.reset()

    def reset(self) -> None:
        """Statistics and the kept step start over (enqueued on the current stream)."""
        self.state.zero_()
        self.state[40:44].fill_(255)             # SnapState.keep_step: nothing kept yet

    def launch(self, attempts: int) -> None:
        """``attempts`` select / copy / validate rounds on the current stream; an attempt after an accepted one exits at
        once.  ``SnapState.step`` / ``.status`` (the first 8 bytes of ``state``) then hold the outcome."""
        eng = self.eng
        lib, sp = eng.lib, stream_ptr()
        ctrl = eng.backend.ctrl.local_ptr
        st = self.state
        interval = int(bool(getattr(eng, "_interval", False)))      # K > N runs the interval commit ordering too
        r = self.bf_ranges or (0, 0, 0, 0)
        for a in range(attempts):
            lib.dm_snap_select(ctrl, st, a, interval, eng.SNAP_WATCHDOG_MS, sp)
            lib.dm_snap_copy(st, eng.params, self.snap, self.snap16, eng.spec.arena_numel, *r, sp)
            lib.dm_snap_validate(ctrl, st, a, attempts, sp)
        if self.keep is not None:
            lib.dm_snap_keep(st, self.snap, self.keep, eng.spec.arena_numel, sp)

    def stats(self) -> dict:
        """Attempts made, rejected by validate, ended by the watchdog, ended a ring lap behind; passes accepted / failed
        (synchronises the current stream)."""
        torch.cuda.current_stream().synchronize()
        w = self.state[:40].cpu().view(torch.int32).tolist()
        return dict(attempts=w[4], rejected=w[5], timeouts=w[6], accepted_passes=w[7], failed_passes=w[8], laps=w[9])


class _CudaEngine(ComputeEngine):
    """What the sm_90a engines share: parameter / gradient arenas, two input slots fed on a copy stream, the native step
    runner, the optimizer binding and the graph-replayed step.  A subclass builds its kernel sequence in ``_launch_step``,
    clears its gradients in ``_launch_zero`` and names its early bucket (``_bucket_early``, ``_g16_shape``)."""
    _kgtn_k = 0                  # K > N: gradients per update (count trigger); 0 = the K <= N / interval paths
    _async = False               # asynchronous SGD (csrc/fused_async.cu), see attach_optimizer
    _master = None               # asynchronous SGD: this replica's master copy of the weights (symmetric memory)
    _ssp = -1                    # asynchronous SGD: the staleness bound s (--ssp_staleness); -1 = unbounded
    _ssp_stats = None            # its statistics and clock (FusedBackend.ssp_arm)
    _local = 0                   # local SGD (csrc/fused_local.cu): H, the averaging period; 0 = off
    _gossip = False              # gossip SGD (csrc/fused_gossip.cu), see attach_optimizer
    _gs_stats = None             # its statistics (FusedBackend.gossip_arm)
    _table = None                # device-resident training set (images, labels), see arm_train_data
    _runner = None               # native step runner (csrc/step_runner.cu), see _make_runner
    _stamp = False               # cdf telemetry stamps in the step
    _main_priority = 0           # priority of the stream the step graph is captured on

    def __init__(self, spec, batch_size: int, backend: FusedBackend, seed: int, use_graph: bool, image_shape):
        self.lib = load()
        self.backend = backend
        self.device = dev = backend.ctx.device
        self.spec = spec
        self.batch_size = B = batch_size
        self.seed = seed
        self.use_graph = use_graph
        self.params = backend.allocate(spec.arena_numel)
        self.params.copy_(spec.init_flat(seed).to(dev))
        self.grads = backend.allocate(spec.arena_numel)
        self.shadow = backend.attach_shadow(self.params)
        self.p, self.g, self.pb = (spec.views(t) for t in (self.params, self.grads, self.shadow))
        f32 = torch.float32
        # two input slots so the H2D copy of step i+1 overlaps the compute of step i
        # (images and labels of a slot share one allocation so a packed host batch moves with ONE host->device copy)
        self._in_bytes = B * 784 * 4 + B * 8
        self.in_dev = [torch.zeros(self._in_bytes, dtype=torch.uint8, device=dev) for _ in range(2)]
        self.images = [t[:B * 784 * 4].view(f32).view(B, *image_shape) for t in self.in_dev]
        self.labels = [t[B * 784 * 4:].view(torch.int64) for t in self.in_dev]
        self.h_images = [torch.zeros(B, *image_shape, dtype=f32).pin_memory() for _ in range(2)]
        self.h_labels = [torch.zeros(B, dtype=torch.int64).pin_memory() for _ in range(2)]
        self.d_loss_acc = torch.zeros(2, dtype=f32, device=dev)
        self.h_loss_bufs = [torch.zeros(2, dtype=f32).pin_memory() for _ in range(2)]
        self._slot = 0            # input slot the next step computes from
        self._loaded = 0
        self.copy_stream = torch.cuda.Stream(device=dev)
        self._copy_done = [torch.cuda.Event() for _ in range(2)]
        self._slot_free = [torch.cuda.Event() for _ in range(2)]
        self._graphs = [None, None]
        self._opt_args: Optional[dict] = None
        self._straggler = None
        self._bucketed = False
        self._bucket_v2 = False       # bf16-wire early bucket + pushed late bucket (csrc/fused_bucket.cu)
        self._g16 = self._g16_view = self._inbox = None
        self.launches_per_step = 0

    # ---- inputs ------------------------------------------------------------------------------
    def _leave_native_runner(self) -> None:
        """The torch-dispatched path takes over again: its events know nothing about steps the native runner launched."""
        if self._runner is not None:
            torch.cuda.synchronize()
            self.lib.dm_runner_destroy(self._runner)
            self._runner = None

    @contextlib.contextmanager
    def _filling(self, s: int):
        """Input slot ``s`` is filled by what the body enqueues on the copy stream: after the step that last read the slot,
        and before the step that reads it next."""
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self._slot_free[s])   # the step that last read this slot is done
            yield
            self._copy_done[s].record(self.copy_stream)
        self._slot = s
        self._loaded += 1

    def load_batch(self, images, labels) -> None:
        """Pinned host staging -> device slot, on the copy stream (overlaps the previous step)."""
        self._leave_native_runner()
        s = self._loaded & 1
        if isinstance(images, torch.Tensor) and images.dtype == torch.float32 and labels.dtype == torch.int64 \
                and ((images.is_pinned() and labels.is_pinned()) or (images.is_cuda and labels.is_cuda)):
            # already page-locked (or device-resident): DMA straight from the caller's buffers (they must stay untouched
            # until the copy has run, i.e. until the step that consumes them has been enqueued twice)
            hi, hl = images.view(self.images[0].shape), labels
        else:
            hi, hl = self.h_images[s], self.h_labels[s]
            # the DMA of this buffer's previous fill waits for the step two loads back: it must have run before the host
            # overwrites the buffer (returns at once unless the caller enqueues steps without ever waiting for one)
            self._copy_done[s].synchronize()
            if isinstance(images, np.ndarray):
                hi.copy_(torch.from_numpy(images).view(hi.shape))
                hl.copy_(torch.from_numpy(labels))
            else:
                hi.copy_(images.reshape(hi.shape))
                hl.copy_(labels)
        with self._filling(s):
            self.images[s].copy_(hi, non_blocking=True)
            self.labels[s].copy_(hl, non_blocking=True)

    def pack_batch(self, images, labels, pin: bool = True) -> torch.Tensor:
        """One contiguous (page-locked) host buffer holding a batch in the device slot's layout: fp32 images
        ``[B,784]`` followed by int64 labels ``[B]``.  Input pipelines that fill such buffers hand each batch to
        :meth:`load_packed`, which is a single DMA."""
        B = self.batch_size
        buf = torch.empty(self._in_bytes, dtype=torch.uint8)
        if pin:
            buf = buf.pin_memory()
        img = torch.as_tensor(images, dtype=torch.float32).reshape(B * 784)
        buf[:B * 784 * 4].view(torch.float32).copy_(img)
        buf[B * 784 * 4:].view(torch.int64).copy_(torch.as_tensor(labels, dtype=torch.int64).reshape(B))
        return buf

    def load_packed(self, packed: torch.Tensor) -> None:
        """Packed batch (see :meth:`pack_batch`; pinned host or device memory) -> device slot with one copy on the copy
        stream.  The buffer must stay untouched until the step after the next one has been enqueued."""
        self._leave_native_runner()
        s = self._loaded & 1
        with self._filling(s):
            self.in_dev[s].copy_(packed, non_blocking=True)

    def h2d_bytes_per_step(self) -> int:
        return self._in_bytes

    # ---- device-resident training set (csrc/batch_gather.cu) ------------------------------------------------------------
    def arm_train_data(self, images, labels) -> None:
        """Upload the training set once (fp32 images ``[N,784]``, int64 labels ``[N]``, in the order given) and allocate two
        device index slots of B int32.  From then on :meth:`step_indices` / :meth:`load_indices` fill an input slot from B
        row indices: the gather kernel writes the rows in :meth:`pack_batch`'s layout, so the step reads the same bytes."""
        self._leave_native_runner()
        x = torch.as_tensor(np.ascontiguousarray(images) if isinstance(images, np.ndarray) else images, dtype=torch.float32)
        y = torch.as_tensor(np.ascontiguousarray(labels) if isinstance(labels, np.ndarray) else labels).to(torch.int64)
        n = int(x.shape[0])
        if n < 1 or x.numel() != n * 784 or y.numel() != n:
            raise ValueError("arm_train_data: %s images, %d labels (need [N, 784] values and N labels)" % (tuple(x.shape), y.numel()))
        dev = self.device
        self._table = (x.reshape(n, 784).to(dev).contiguous(), y.reshape(n).to(dev).contiguous())
        self._idx_dev = [torch.zeros(self.batch_size, dtype=torch.int32, device=dev) for _ in range(2)]
        self._h_idx = [torch.zeros(self.batch_size, dtype=torch.int32).pin_memory() for _ in range(2)]

    def _as_indices(self, idx) -> torch.Tensor:
        """``idx`` as a contiguous int32 host tensor of B rows, each checked to lie in ``[0, N)``."""
        if self._table is None:
            raise RuntimeError("arm_train_data() first")
        t = idx if isinstance(idx, torch.Tensor) else torch.from_numpy(np.asarray(idx))
        if t.device.type != "cpu" or t.dtype.is_floating_point or t.dtype == torch.bool or t.dtype.is_complex:
            raise ValueError("row indices must be an integer host array, got %s on %s" % (t.dtype, t.device))
        if t.numel() != self.batch_size:
            raise ValueError("%d row indices for a batch of %d" % (t.numel(), self.batch_size))
        n = self._table[1].numel()
        lo, hi = int(t.min()), int(t.max())
        if lo < 0 or hi >= n:
            raise ValueError("row index %d outside the training set [0, %d)" % (lo if lo < 0 else hi, n))
        if t.dtype != torch.int32 or not t.is_contiguous():
            t = t.reshape(-1).to(torch.int32).contiguous()
        return t.reshape(-1)

    def _gather(self, s: int) -> None:
        img, lbl = self._table
        self.lib.dm_gather_batch(self._idx_dev[s], img, lbl, self.batch_size, self.in_dev[s], stream_ptr(self.copy_stream))

    def load_indices(self, idx) -> None:
        """Counterpart of :meth:`load_batch` for the armed training set: B row indices -> pinned staging -> device index
        slot, then the gather into the input slot, on the copy stream (overlaps the previous step)."""
        self._leave_native_runner()
        t = self._as_indices(idx)
        s = self._loaded & 1
        h = self._h_idx[s]
        self._copy_done[s].synchronize()                 # the previous fill's DMA has read h (see load_batch)
        h.copy_(t)
        with self._filling(s):
            self._idx_dev[s].copy_(h, non_blocking=True)
            self._gather(s)

    def step_indices(self, idx):
        """Counterpart of :meth:`step_packed` for the armed training set: one whole step from B row indices (index DMA,
        gather, event chaining and the graph launch in ONE native call once both slot graphs exist; before that, or with
        ``DMNIST_NATIVE_RUNNER=0``, the torch-dispatched path).  A page-locked ``idx`` is read by an asynchronous DMA: it must
        stay untouched until the step after the next one has been enqueued.  Returns ``(waitable, loss buffer, seq)``."""
        t = self._as_indices(idx)
        r = self._runner
        if r is None:
            r = self._make_runner()
            if r is None:
                self.load_indices(t)
                self.train_step()
                return self.read_result_async()
        if not t.is_pinned():
            # into the slot's page-locked staging buffer, once the DMA of its previous fill has read it (a fresh pinned copy
            # per call would go back to torch's host allocator, and be handed out again, while its DMA may still wait)
            s = self._loaded & 1
            self.lib.dm_runner_wait_copy(r, s)
            self._h_idx[s].copy_(t)
            t = self._h_idx[s]
        s = int(self.lib.dm_runner_step_indices(r, t))
        if s < 0:
            raise RuntimeError("dm_runner_step_indices failed: CUDA error %d" % -s)
        self._keep_alive[s] = t                          # the DMA reads it asynchronously
        self._slot = s
        self._loaded += 1
        self._steps_launched += 1
        return _RunnerEvent(self.lib, r, s), self.h_loss_bufs[s], self._seq0 + self._steps_launched

    # ---- native step executor (csrc/step_runner.cu) ----------------------------------------------------------------------
    def step_packed(self, packed: torch.Tensor):
        """One whole training step from a packed batch (see :meth:`pack_batch`; pinned host or device memory): input DMA,
        event chaining and the graph launch happen in ONE native call once both slot graphs exist (``DMNIST_NATIVE_RUNNER=0``
        keeps the torch-dispatched path).  Returns ``(waitable, loss buffer, seq)`` like :meth:`read_result_async`."""
        r = self._runner
        if r is None:
            r = self._make_runner()
            if r is None:
                self.load_packed(packed)
                self.train_step()
                return self.read_result_async()
        s = int(self.lib.dm_runner_step(r, packed))
        if s < 0:
            raise RuntimeError("dm_runner_step failed: CUDA error %d" % -s)
        self._keep_alive[s] = packed                     # the DMA reads it asynchronously
        self._slot = s
        self._loaded += 1
        self._steps_launched += 1
        return _RunnerEvent(self.lib, r, s), self.h_loss_bufs[s], self._seq0 + self._steps_launched

    def _make_runner(self):
        """The native runner, once both slot graphs exist (with an optimizer attached, unless ``DMNIST_NATIVE_RUNNER=0``);
        None until then: the caller takes the torch-dispatched path."""
        if not (self.use_graph and self._opt_args is not None and os.environ.get("DMNIST_NATIVE_RUNNER", "1") != "0"
                and all(g is not None and g[1] for g in self._graphs)):
            return None
        torch.cuda.synchronize()                         # hand-over point: nothing of the torch-dispatched path is in flight
        lib = self.lib
        cur = torch.cuda.current_stream()
        r = lib.dm_runner_create(cur.cuda_stream, self.copy_stream.cuda_stream, self._graphs[0][0].raw_cuda_graph_exec(),
                                 self._graphs[1][0].raw_cuda_graph_exec(), self.in_dev[0], self.in_dev[1], self._in_bytes,
                                 int(self._loaded & 1))
        if not r:
            return None
        if self._table is not None:
            lib.dm_runner_arm_gather(r, self._idx_dev[0], self._idx_dev[1], self._table[0], self._table[1], self.batch_size)
        self._runner = r
        self._keep_alive = [None, None]
        return self._runner

    # ---- optimizer binding ------------------------------------------------------------------------
    def attach_optimizer(self, opt) -> None:
        """Bind the aggregation policy so the whole step (compute + fused sync) is one graph."""
        sched = opt.lr_schedule
        k = getattr(opt, "replicas_to_aggregate", opt.total_num_replicas)
        n = self.backend.ctx.world_size
        # K > N (mode A): replicas free-run and accumulate; a step commits once K of its gradients are in (count trigger)
        self._kgtn_k = int(k) if int(k) > n else 0
        if self._kgtn_k and getattr(opt, "drop_connect_probability", None) is not None:
            raise ValueError("--drop_connect is not implemented on the GPU path with --num_replicas_to_aggregate (%d) > "
                             "the number of replicas (%d)" % (int(k), n))
        self._opt_args = dict(k=int(k), lr0=float(sched.initial_learning_rate), decay_rate=float(sched.decay_rate),
                              decay_steps=int(sched.decay_steps))
        # warmup / cosine decay: evaluated by the aggregation kernels at the step they update, from this replica's own
        # control block (every replica arms its own; nothing to agree on beyond the step)
        self.backend.set_lr_schedule(getattr(sched, "warmup_steps", 0), getattr(sched, "warmup_start", 1.0 / 3),
                                     getattr(sched, "cosine_steps", 0), getattr(sched, "cosine_alpha", 0.0))
        if getattr(opt, "drop_connect_probability", None) is not None:
            self.backend.drop_connect_(self.grads, opt.drop_connect_probability, 0)
        self._straggler = getattr(opt, "_straggler", None)
        if self._straggler is not None:
            self.backend.arm_straggler(self._straggler)      # sampled forms: table + iteration counter on the device
        self._stamp = getattr(opt, "mode", "") == "cdf"
        self._graphs = [None, None]
        self._runner = None                  # graphs are re-captured: the native runner is rebuilt on demand
        # mode C on the device (csrc/fused_interval.cu): every iteration adds its gradient to a symmetric accumulator; ticks
        # are committed by whichever replica first passes the %globaltimer deadline
        # K > N runs the same iteration with the count trigger (same accumulator, same snapshot ordering as interval mode)
        self._interval = getattr(opt, "mode", "") == "interval" or bool(self._kgtn_k)
        if self._interval and getattr(self, "_acc", None) is None:
            self._acc = self.backend.allocate(self.spec.arena_numel)
        if self._kgtn_k:
            self.backend.kgtn_arm()          # nothing else arms it (e.g. bench.py); train.py re-arms after a restore
        # asynchronous SGD (csrc/fused_async.cu): every iteration pulls this replica's master copy into the working arena
        # and adds its own update to every replica's master copy; the working arena stays private between iterations
        self._async = getattr(opt, "mode", "") == "async"
        if self._async:
            if getattr(opt, "drop_connect_probability", None) is not None:
                raise ValueError("--drop_connect cannot be combined with --async_method")
            if self._master is None:
                self._master = self.backend.allocate(self.spec.arena_numel)
                self._as_stats = torch.zeros(int(self.lib.dm_async_stats_bytes()), dtype=torch.uint8, device=self.device)
        # stale synchronous parallel: a wait before the pull and a clock publication after the apply
        self._ssp = int(getattr(opt, "ssp_staleness", -1)) if self._async else -1
        if self._async:
            if self._ssp >= 0 and self._ssp_stats is None:
                self._ssp_stats = self.backend.ssp_arm()
            self.async_arm()                 # train.py re-arms after a restore
        # local SGD (csrc/fused_local.cu): every iteration updates this replica's own arena; every H-th global step the
        # arenas are averaged between two device barriers.  Whether a step averages is decided on the device from the epoch
        # word, so the two slot graphs serve every step; a restore moves that word, and with it the next averaging step
        self._local = int(getattr(opt, "period", 0)) if getattr(opt, "mode", "") == "local" else 0
        if self._local:
            if getattr(opt, "drop_connect_probability", None) is not None:
                raise ValueError("--drop_connect cannot be combined with --local_sgd_steps")
            if getattr(self, "_ls_stats", None) is None:
                self._ls_stats = torch.zeros(int(self.lib.dm_local_stats_bytes()), dtype=torch.uint8, device=self.device)
            self._ls_stats.zero_()
        # gossip SGD (csrc/fused_gossip.cu): every iteration writes its half step into this replica's send buffer, takes the
        # barrier with its two ring neighbours and mixes the neighbourhood's half steps into its own arena; the run ends with
        # one local-SGD average of every arena (gossip_finish)
        self._gossip = getattr(opt, "mode", "") == "gossip"
        if self._gossip:
            if getattr(opt, "drop_connect_probability", None) is not None:
                raise ValueError("--drop_connect cannot be combined with --gossip_method")
            if self._gs_stats is None:
                self._gs_stats = self.backend.gossip_arm(self.spec.arena_numel)
                self._ls_stats = torch.zeros(int(self.lib.dm_local_stats_bytes()), dtype=torch.uint8, device=self.device)
            self._gs_stats.zero_()
        # Bucketed aggregation (csrc/fused_sync.cu): full participation on 2/4/8 replicas.  fc1's weight gradient (96.5 % of
        # the bytes) is exchanged by small co-resident CTAs NEXT TO conv2 dgrad/wgrad + conv1 wgrad; the rest goes one-shot.
        #   DMNIST_BUCKET=2 (default): csrc/fused_bucket.cu -- fc1's gradient leaves the GEMM epilogue as bf16, is reduced in
        #     place over NVLink (in-switch fp32 accumulation) and applied to the local fp32 master weights under the backward
        #     pass; the small bucket is pushed into every replica's inbox.  Also used on ONE replica (no exchange, the fc1
        #     update still leaves the critical path).   =1: round-1 fp32 two-shot / one-shot kernels.   =0: single kernel.
        mode = os.environ.get("DMNIST_BUCKET", "2")
        can = int(k) == n and self.backend.drop_keep <= 0.0 and \
            getattr(opt, "mode", "") not in ("interval", "async", "local", "gossip")
        self._bucket_v2 = can and mode == "2" and n in (1, 2, 4, 8)
        self._bucketed = can and ((mode == "1" and n in (2, 4, 8)) or self._bucket_v2)
        if self._bucket_v2 and self._g16 is None:
            e0, e1 = self._bucket_early
            assert e0 % 8 == 0 and (e1 - e0) % 8 == 0, "fc1 weights must start on a 32-byte boundary of the arena"
            self._g16 = self.backend.allocate_buffer((e1 - e0) * 2)
            self._g16_view = self._g16.view(torch.bfloat16, 0, e1 - e0).view(*self._g16_shape)
            n_late = self.spec.arena_numel - (e1 - e0)
            self._inbox = self.backend.allocate_buffer(2 * n * n_late * 8) if n > 1 else None   # LL lines: 8 bytes per float
        # early-bucket grid: the CTAs share SMs with the tensor-core kernels of the backward pass and every one of them fences
        # at system scope once, so with several replicas half the SMs carry the exchange
        sms = int(self.lib.dm_num_sms())
        self._early_ctas = int(os.environ.get("DMNIST_EARLY_CTAS", "0")) or (sms // 2 if n > 1 else sms)
        torch.cuda.synchronize()
        self._seq0 = self.backend.status_seq       # steps closed on this control block before the engine's first one
        self._steps_launched = 0
        self.lib.dm_set_max_ctas(int(os.environ.get("DMNIST_MAX_CTAS", "0")))

    def arm_weight_decay(self, lam: float) -> None:
        """L2 weight decay (see weight_decay.py): implemented for lenet only (:class:`CudaLeNetEngine`)."""
        if float(lam) != 0.0:
            raise ValueError("--weight_decay on the GPU path is implemented for lenet, not --model=%s" % self.spec.name)

    # ---- random affine augmentation (see augment.py, csrc/augment.cu) ---------------------------------------------------
    # With augmentation armed, every training step starts (after the cdf start stamp) with augment_affine, which warps the
    # input slot's images into _aug_images; every reader of the step's training images reads that buffer instead.  The
    # step graphs replay one after another on the training stream, so one buffer serves both slots.  The iteration word
    # _aug_counter[0] is advanced by the kernel itself; _aug_counter[1] is its ticket.  Evaluation never augments.
    # With elastic distortion armed, augment_elastic (csrc/augment_elastic.cu) takes augment_affine's place: the same
    # node, buffer and counter, the elastic field composed in front of the affine map.
    _aug = None                    # (augment.Ranges, seed mix), see arm_augment
    _aug_elastic = None            # augment.Elastic while elastic distortion is armed
    _aug_taps = None               # its Gaussian taps w_0 .. w_R as a ctypes double array, and R

    def arm_augment(self, max_shift: float, max_rotation: float, max_scale: float, start_iteration: int = 0,
                    elastic: Optional[augment.Elastic] = None) -> None:
        """Augment every training step from the next one on, its first draws those of iteration ``start_iteration`` (a
        restarted run: ``augment.start_iteration`` of the restored global step).  ``elastic``: elastic distortion
        composed in front of the affine map (None or alpha 0: none).  All three ranges 0 and no elastic distortion turns
        augmentation off.  Re-captures the step graphs."""
        r = augment.Ranges(float(max_shift), float(max_rotation), float(max_scale))
        augment.check_ranges(r)
        if elastic is not None:
            elastic = augment.Elastic(float(elastic.alpha), float(elastic.sigma))
            augment.check_elastic(elastic)
            if elastic.alpha == 0.0:
                elastic = None
            elif self.batch_size > augment.MAX_ELASTIC_BATCH:
                raise ValueError("elastic distortion takes at most %d rows per batch, got %d"
                                 % (augment.MAX_ELASTIC_BATCH, self.batch_size))
        self._leave_native_runner()
        torch.cuda.synchronize()
        if any(r) or elastic is not None:
            if getattr(self, "_aug_images", None) is None:
                self._aug_images = torch.zeros(self.batch_size, 784, dtype=torch.float32, device=self.device)
                self._aug_counter = torch.zeros(2, dtype=torch.int32, device=self.device)
            words = np.array([int(start_iteration) & 0xFFFFFFFF, 0], dtype=np.uint32).view(np.int32)
            self._aug_counter.copy_(torch.from_numpy(words))
            self._aug = (r, augment.seed_mix(self.seed, self.backend.ctx.rank))
        else:
            self._aug = None
        self._aug_elastic = elastic
        if elastic is not None:
            w = augment.gaussian_weights(elastic.sigma)
            self._aug_taps = ((ctypes.c_double * len(w))(*w), len(w) - 1)
        self._graphs = [None, None]
        torch.cuda.synchronize()

    def _launch_augment(self, slot: int) -> torch.Tensor:
        """augment_affine, or augment_elastic with elastic distortion armed, on the current stream: slot ``slot``'s
        images -> the augmented buffer, in the slot's shape."""
        r, mix = self._aug
        if self._aug_elastic is None:
            self.lib.dm_augment_affine(self.images[slot], self._aug_images, self.batch_size, self._aug_counter, mix,
                                       r.max_shift, r.max_rotation, r.max_scale, None, stream_ptr())
        else:
            w, radius = self._aug_taps
            self.lib.dm_augment_elastic(self.images[slot], self._aug_images, self.batch_size, self._aug_counter, mix,
                                        r.max_shift, r.max_rotation, r.max_scale, self._aug_elastic.alpha, w, radius,
                                        None, None, stream_ptr())
        return self._aug_images.view(self.images[slot].shape)

    def augment_iteration(self) -> int:
        """The iteration whose draws the next augmented step uses (synchronises the device)."""
        torch.cuda.synchronize()
        return int(self._aug_counter[0].item()) & 0xFFFFFFFF

    def augmented_batch(self) -> Optional[torch.Tensor]:
        """Copy of the images the last augmented step read, ``[B, 784]`` (None when augmentation is off)."""
        if self._aug is None:
            return None
        torch.cuda.synchronize()
        return self._aug_images.clone()

    def params_updated(self) -> None:
        """Parameters were written from the host (init / restore): refresh the bf16 shadow."""
        self.backend.refresh_shadow(self.params)

    # ---- step ---------------------------------------------------------------------------------------------------------
    def _launch_step(self, slot: int, with_sync: bool) -> None:
        raise NotImplementedError

    def _enqueue_iteration_begin(self) -> None:
        """Interval mode / K > N: adopt pushed weights (+ shadow refresh) at the start of an iteration.  Asynchronous SGD:
        read the update counter, pull the master copy (+ shadow), after the staleness bound's wait when one is armed."""
        if self._async:
            if self._ssp >= 0:
                self.backend.enqueue_ssp_wait(self._ssp_stats, self._ssp)
            self.backend.enqueue_async_begin(self._master, self.params)
        elif self._kgtn_k:
            self.backend.enqueue_kgtn_begin(self.params)
        else:
            self.backend.enqueue_interval_begin(self.params)

    def _enqueue_iteration_end(self) -> None:
        """Interval mode / K > N: gate, accumulate, close (+ commit attempt), apply.  Asynchronous SGD: ticket, apply.
        Local SGD: the local update, then the averaging round, which only an averaging step runs.  Gossip SGD: the half
        step, the neighbours' barrier, the mix."""
        oa = self._opt_args
        if self._gossip:
            self.backend.enqueue_gossip_step(self.params, self.grads, self._gs_stats, oa["lr0"], oa["decay_rate"],
                                             oa["decay_steps"])
        elif self._local:
            self.backend.enqueue_local_step(self.params, self.grads, self._local, oa["lr0"], oa["decay_rate"],
                                            oa["decay_steps"])
            self.backend.enqueue_local_average(self.params, self._ls_stats, self._local)
        elif self._async:
            self.backend.enqueue_async_end(self._master, self.grads, self._as_stats, oa["lr0"], oa["decay_rate"],
                                           oa["decay_steps"])
            if self._ssp >= 0:
                self.backend.enqueue_ssp_publish(self._ssp_stats)
        elif self._kgtn_k:
            self.backend.enqueue_kgtn_end(self.params, self.grads, self._acc, self._kgtn_k, oa["lr0"], oa["decay_rate"],
                                          oa["decay_steps"])
        else:
            self.backend.enqueue_interval_end(self.params, self.grads, self._acc, oa["lr0"], oa["decay_rate"], oa["decay_steps"])

    # ---- asynchronous SGD (csrc/fused_async.cu) ------------------------------------------------------------------------------
    def async_arm(self) -> None:
        """Every master copy := the working arena (the initial or restored weights), staleness statistics zeroed; the
        first pull reads them.  With the staleness bound armed, every clock board and the bound's statistics, with this
        replica's clock, are zeroed too.  Collective."""
        self._leave_native_runner()
        self.backend.async_arm(self._master, self.params, self._as_stats, self._ssp_stats if self._ssp >= 0 else None)

    def async_finish(self) -> int:
        """End of an asynchronous run, after the last step was enqueued: with the staleness bound armed, this replica
        retires (no peer waits for its clock again); every replica's last update has been applied, the device barrier
        (every replica's updates are in every master copy after it), then one more pull into the working arena.  Returns
        the global step of the pulled weights: the total number of updates.  Collective."""
        self._leave_native_runner()
        if self._ssp >= 0:
            # before anything waits for a peer: a peer still in its last iterations may be waiting for this clock
            self.backend.enqueue_ssp_retire(self._ssp_stats)
        torch.cuda.synchronize()
        self.backend.device_barrier()
        self.backend.enqueue_async_begin(self._master, self.params)
        torch.cuda.synchronize()
        self.backend.check_error()
        return self.backend.device_epoch

    def async_staleness(self) -> dict:
        """This replica's staleness statistics (see FusedBackend.async_stats); synchronises the device."""
        return self.backend.async_stats(self._as_stats)

    def ssp_stats(self) -> dict:
        """This replica's staleness-bound statistics (see FusedBackend.ssp_stats); synchronises the device."""
        return self.backend.ssp_stats(self._ssp_stats)

    # ---- local SGD (csrc/fused_local.cu) ---------------------------------------------------------------------------------
    def local_finish(self) -> int:
        """End of a local-SGD run, after the last step was enqueued: if that step was not an averaging step, one more
        average (without a step), so the weights every replica ends with are the mean.  Returns the global step.
        Collective: every replica ends on the same step, so all of them average here or none does."""
        self._leave_native_runner()
        torch.cuda.synchronize()
        step = self.backend.device_epoch
        if step % self._local:
            self.backend.enqueue_local_average(self.params, self._ls_stats, 1, close=False)
            torch.cuda.synchronize()
        self.backend.check_error()
        return step

    def local_stats(self) -> dict:
        """This replica's averaging statistics (see FusedBackend.local_stats); synchronises the device."""
        return self.backend.local_stats(self._ls_stats)

    # ---- gossip SGD (csrc/fused_gossip.cu) -------------------------------------------------------------------------------
    def gossip_finish(self) -> int:
        """End of a gossip run, after the last step was enqueued: one average of every replica's arena (the local-SGD
        round, unconditional, closing no step), so the weights every replica ends with are the consensus mean.  Returns the
        global step.  Collective: every replica ends on the same iteration."""
        self._leave_native_runner()
        torch.cuda.synchronize()
        self.backend.enqueue_local_average(self.params, self._ls_stats, 1, close=False)
        torch.cuda.synchronize()
        self.backend.check_error()
        return self.backend.device_epoch

    def gossip_stats(self) -> dict:
        """This replica's gossip statistics (see FusedBackend.gossip_stats); synchronises the device."""
        return self.backend.gossip_stats(self._gs_stats)

    def _run(self, with_sync: bool) -> None:
        s = self._slot
        cur = torch.cuda.current_stream()
        cur.wait_event(self._copy_done[s])
        if self.use_graph:
            key = s
            if self._graphs[key] is None or self._graphs[key][1] != with_sync:
                counter = self._aug_counter.clone() if self._aug is not None else None
                self._launch_step(s, False)           # warm-up (gradients only): sets func attributes outside capture
                torch.cuda.synchronize()
                if counter is not None:
                    self._aug_counter.copy_(counter)  # the warm-up is not an iteration: it must not consume draws
                gr = torch.cuda.CUDAGraph()
                cap = torch.cuda.Stream(device=self.device, priority=self._main_priority)
                with _capture(gr, cap):
                    self._launch_step(s, with_sync)
                self._graphs[key] = (gr, with_sync)
            self._graphs[key][0].replay()
        else:
            self._launch_step(s, with_sync)
        if with_sync:
            self._steps_launched = getattr(self, "_steps_launched", 0) + 1
        self._slot_free[s].record(cur)

    # ---- public step API ----------------------------------------------------------------------------------
    def forward_backward(self, step: int) -> None:
        """Gradients only (the aggregation is launched separately by the optimizer)."""
        self._run(with_sync=False)

    def train_step(self) -> None:
        """Whole step incl. the fused allreduce+SGD kernel, as one CUDA graph replay."""
        assert self._opt_args is not None, "attach_optimizer() first"
        self._run(with_sync=True)

    def read_loss_async(self):
        """``(event, buffer)`` of the step enqueued last: the step copies (loss, accuracy) into a pinned host buffer
        (two alternate, one per input slot) as its final node; wait on the event, then read ``buffer[0]`` / ``buffer[1]``."""
        s = self._slot                      # the step just enqueued copied its result into this slot's buffer itself
        return self._slot_free[s], self.h_loss_bufs[s]

    def read_result_async(self):
        """``(event, loss buffer, seq)`` of the step enqueued last: wait on the event, then ``loss[0]``/``loss[1]`` are (loss,
        accuracy) and ``backend.mirror_info(seq)`` is the step's StepInfo -- both were written into page-locked host memory
        by the step's own kernels, so the host never issues a device read."""
        s = self._slot
        return self._slot_free[s], self.h_loss_bufs[s], self._seq0 + self._steps_launched

    def loss_acc(self) -> Tuple[float, float]:
        ev, buf = self.read_loss_async()
        ev.synchronize()
        return float(buf[0]), float(buf[1])

    def step_info(self) -> StepInfo:
        return self.backend.last_step_info(check=True)     # one packed device->host read

    # ---- checkpoint capture ------------------------------------------------------------------------------------------------
    # A checkpoint is staged on the training stream right after the launched step, in a device buffer of its own, and copied
    # from there to one of CKPT_HOST_BUFFERS page-locked host arenas on a dedicated stream (not the copy stream: a multi-MB
    # DMA there would queue ahead of the next step's input).  The host learns that it landed from an event query.
    SNAP_ATTEMPTS = 4              # select / copy / validate attempts of one snapshot (evaluation pass, checkpoint capture)
    SNAP_WATCHDOG_MS = 2.0         # how long one attempt waits for the pushes of the newest committed step
    CKPT_HOST_BUFFERS = 2

    def arm_checkpoint(self, snapshot: bool) -> None:
        """Allocate the capture's buffers.  ``snapshot=False``: no peer writes this arena between two of its steps (K = N, cdf
        mode), so a capture is a device-to-device copy of the live arena plus the epoch word.  ``snapshot=True`` (K < N,
        K > N, interval): peers push weights into it at any time, so a capture is SNAP_ATTEMPTS select / copy / validate
        attempts (csrc/eval_snapshot.cu) into the staging buffer, and one whose attempts all fail reports step -1."""
        dev, n = self.device, self.spec.arena_numel
        self._ck_dev = torch.zeros(n, dtype=torch.float32, device=dev)
        self._ck_snap = _Snapshot(self, self._ck_dev) if snapshot else None      # no bf16 shadow: the file holds fp32 only
        # (step, status) of the capture: SnapState.step / .status; the live capture copies the epoch word into .step and
        # leaves .status at 0
        self._ck_state = self._ck_snap.state if snapshot else \
            torch.zeros(int(self.lib.dm_snap_state_bytes()), dtype=torch.uint8, device=dev)
        off = self.backend._off["epoch"]
        self._ck_epoch = self.backend._ctrl_bytes[off:off + 4]
        self.ckpt_host = [torch.zeros(n, dtype=torch.float32).pin_memory() for _ in range(self.CKPT_HOST_BUFFERS)]
        if self._ema is not None:
            self._arm_checkpoint_average()
        self._ck_rec = [torch.zeros(2, dtype=torch.int32).pin_memory() for _ in range(self.CKPT_HOST_BUFFERS)]  # step, status
        self._ck_stream = torch.cuda.Stream(device=dev)
        self._ck_staged, self._ck_landed = torch.cuda.Event(), torch.cuda.Event()
        self._ck_seq = 0
        self._ck_inflight: Optional[Tuple[int, int]] = None       # (seq, host buffer) of the capture not yet seen landed
        if snapshot:
            self._ck_snap.launch(self.SNAP_ATTEMPTS)   # loads the kernels now rather than at the first capture in training
            torch.cuda.synchronize()
            self._ck_snap.reset()                      # statistics count real captures only
        torch.cuda.synchronize()

    def enqueue_checkpoint(self, buf: int) -> int:
        """Capture the weights after the step enqueued last into page-locked host arena ``ckpt_host[buf]``, which the caller
        must not read or hand out again until :meth:`checkpoint_poll` / :meth:`checkpoint_wait` returned this capture.  One
        capture at a time.  No host synchronisation.  Returns the capture's sequence number."""
        if self._ck_inflight is not None:
            raise RuntimeError("enqueue_checkpoint: capture %d has not landed yet" % self._ck_inflight[0])
        cur = torch.cuda.current_stream()
        cur.wait_event(self._ck_landed)              # the staging buffer's previous device->host copy has completed
        if self._ck_snap is not None:
            self._ck_snap.launch(self.SNAP_ATTEMPTS)
        else:
            self._ck_dev.copy_(self.params)
            self._ck_state[0:4].copy_(self._ck_epoch)
            if self._ck_ema_dev is not None:
                self._ck_ema_dev.copy_(self._ema)        # the average after the same step as the weights
        self._ck_staged.record(cur)
        self._ck_seq += 1
        with torch.cuda.stream(self._ck_stream):
            self._ck_stream.wait_event(self._ck_staged)
            self.ckpt_host[buf].copy_(self._ck_dev, non_blocking=True)
            if self._ck_ema_dev is not None:
                self.ckpt_ema_host[buf].copy_(self._ck_ema_dev, non_blocking=True)
            self._ck_rec[buf].copy_(self._ck_state[0:8].view(torch.int32), non_blocking=True)
            self._ck_landed.record(self._ck_stream)
        self._ck_inflight = (self._ck_seq, buf)
        return self._ck_seq

    def _checkpoint_landed(self) -> Tuple[int, int, int]:
        seq, buf = self._ck_inflight
        self._ck_inflight = None
        step, status = (int(v) for v in self._ck_rec[buf].tolist())
        return seq, buf, (step & 0xFFFFFFFF) if status >= 0 else -1

    def checkpoint_poll(self) -> Optional[Tuple[int, int, int]]:
        """``(seq, host buffer, global step)`` once the capture in flight has landed in host memory (an event query, never
        a wait), else None.  Step -1: no consistent snapshot, the buffer holds nothing usable.  Landing is established by
        the event recorded after the device-to-host copies of the arena and of the (step, status) record; ``seq`` is the
        host's count of captures (the one :meth:`enqueue_checkpoint` returned), not read back from the device."""
        if self._ck_inflight is None or not self._ck_landed.query():
            return None
        return self._checkpoint_landed()

    def checkpoint_wait(self) -> Optional[Tuple[int, int, int]]:
        """Like :meth:`checkpoint_poll`, but waits for the capture in flight (None if there is none)."""
        if self._ck_inflight is None:
            return None
        self._ck_landed.synchronize()
        return self._checkpoint_landed()

    def checkpoint_stats(self) -> Optional[dict]:
        """Snapshot statistics of the capture (see :class:`_Snapshot`), None for the live capture."""
        return self._ck_snap.stats() if self._ck_snap is not None else None

    def _arm_checkpoint_average(self) -> None:
        """The capture's buffers for the moving average: a device staging arena and one page-locked host arena per host
        buffer of the weights."""
        n = self.spec.arena_numel
        self._ck_ema_dev = torch.zeros(n, dtype=torch.float32, device=self.device)
        self.ckpt_ema_host = [torch.zeros(n, dtype=torch.float32).pin_memory() for _ in range(self.CKPT_HOST_BUFFERS)]

    # ---- moving average of the weights (csrc/moving_average.cu) ---------------------------------------------------------
    # The chief keeps TF's ExponentialMovingAverage of its arena in a shadow arena of its own (plain device memory: no peer
    # reads it).  Each training step ends with one streaming kernel that moves the shadow towards the weights the step
    # committed; it reads the global step from the epoch word, so the captured graph holds no host value.  Only K = N and
    # cdf mode are supported: there no peer writes the chief's arena between two of its steps, so the arena holds exactly
    # one global step when the kernel runs.
    _ema = None                    # fp32 shadow arena of the average, see arm_moving_average
    _ck_ema_dev = None

    def arm_moving_average(self, decay: float) -> None:
        """Allocate the shadow arena, starting from the current weights, and re-capture the step graphs so that every
        training step ends with the average's update (before stop_publish when a stop is armed).  After
        :meth:`attach_optimizer`; K = N or cdf mode only."""
        if not 0.0 < float(decay) < 1.0:
            raise ValueError("moving average decay must lie in (0, 1), got %r" % decay)
        if self._opt_args is None:
            raise RuntimeError("arm_moving_average: attach_optimizer() first")
        if getattr(self, "_interval", False) or self._opt_args["k"] != self.backend.ctx.world_size:
            raise ValueError("the moving average is kept for K = N and cdf mode only: with K < N, K > N or interval "
                             "aggregation peers write the chief's arena at any time")
        if self._async:
            raise ValueError("the moving average is kept for K = N and cdf mode only, not for asynchronous SGD")
        if self._local:
            raise ValueError("the moving average is kept for K = N and cdf mode only, not for local SGD")
        if self._gossip:
            raise ValueError("the moving average is kept for K = N and cdf mode only, not for gossip SGD")
        self._leave_native_runner()
        torch.cuda.synchronize()
        off = self.backend._off["epoch"]
        self._ema_epoch = self.backend.ctrl.local_ptr + off
        self._ema_decay = float(decay)
        self._ema = self.params.detach().clone()
        self._ema_step = self.backend._ctrl_bytes[off:off + 4].view(torch.int32).clone()    # step the shadow holds
        if getattr(self, "_ck_dev", None) is not None and self._ck_ema_dev is None:
            self._arm_checkpoint_average()
        self._graphs = [None, None]
        torch.cuda.synchronize()

    def _launch_moving_average(self) -> None:
        self.lib.dm_moving_average(self._ema, self.params, self.spec.arena_numel, self._ema_epoch, self._ema_decay,
                                   self._ema_step, None, 0, 0, 0, 0, stream_ptr())

    def moving_average(self) -> Tuple[torch.Tensor, int]:
        """(copy of the shadow arena, global step of the weights it was last updated from); synchronises the device."""
        torch.cuda.synchronize()
        return self._ema.clone(), int(self._ema_step.item()) & 0xFFFFFFFF

    def load_moving_average(self, flat: torch.Tensor) -> None:
        """Restore: the shadow arena from a host or device arena (the step it holds stays the current global step)."""
        self._ema.copy_(flat.to(self.device, torch.float32))
        torch.cuda.synchronize()

    # ---- inference ------------------------------------------------------------------------------------------
    def _eval_forward(self, images: torch.Tensor, labels: torch.Tensor, B: int) -> None:
        """Inference forward of one batch: (mean loss, accuracy) of its B rows into ``d_loss_acc``."""
        raise NotImplementedError

    @torch.no_grad()
    def evaluate(self, images, labels) -> Tuple[float, float]:
        if isinstance(images, np.ndarray):
            images, labels = torch.from_numpy(np.ascontiguousarray(images)), torch.from_numpy(np.ascontiguousarray(labels))
        images = images.reshape(-1, *self.images[0].shape[1:]).to(self.device, torch.float32)
        labels = labels.to(self.device, torch.int64)
        n, B = images.shape[0], self.batch_size
        tot_loss = tot_hit = 0.0
        for s in range(0, n, B):
            m = min(B, n - s)
            self._eval_forward(images[s:s + m].contiguous(), labels[s:s + m].contiguous(), m)
            la = self.d_loss_acc.cpu()
            tot_loss += float(la[0]) * m      # kernel scales by 1/m
            tot_hit += float(la[1]) * m
        return tot_loss / n, tot_hit / n


def check_lenet_batch(batch_size: int) -> None:
    """Refuse a batch the LeNet kernels cannot run, before anything is allocated or launched.  The limit is
    ``dm_lenet_max_batch()``: fc1_dgrad_unpool keeps one conv2 bias-gradient slot per CTA in a workspace of 4096 slots,
    49 CTAs per 128-row tile (DESIGN.md §3, "Batch limit")."""
    limit = int(load().dm_lenet_max_batch())
    if not 1 <= batch_size <= limit:
        raise ValueError("--batch_size=%d is outside what the LeNet kernels on the GPU path can run: use 1 <= --batch_size "
                         "<= %d (fc1_dgrad_unpool keeps one conv2 bias-gradient slot per CTA, 4096 slots for 49 CTAs per "
                         "128 rows)" % (batch_size, limit))


class CudaLeNetEngine(_CudaEngine):
    _main_priority = -1           # see _side

    def __init__(self, batch_size: int, backend: FusedBackend, seed: int = 66478, rank: int = 0,
                 keep_prob: float = 0.5, use_graph: bool = True):
        check_lenet_batch(batch_size)
        super().__init__(get_model("lenet")[0], batch_size, backend, seed, use_graph, (28, 28))
        B, dev = batch_size, self.device
        self.seed, self.rank, self.keep_prob = seed, rank, keep_prob
        bf, u8, f32 = torch.bfloat16, torch.uint8, torch.float32
        self.a1 = torch.zeros(B, 14, 14, 32, dtype=bf, device=dev)
        self.code1 = torch.zeros(B, 14, 14, 32, dtype=u8, device=dev)
        self.a2 = torch.zeros(B, 3136, dtype=bf, device=dev)
        self.code2 = torch.zeros(B, 3136, dtype=u8, device=dev)
        self.fc1_splits = 7                                         # 49 k-blocks of 64 -> 7 per CTA
        self.h_part = torch.zeros(self.fc1_splits, B, 512, dtype=f32, device=dev)   # fc1 split-K partial sums
        self.dh = torch.zeros(B, 512, dtype=bf, device=dev)
        self.h_act = torch.zeros(B, 512, dtype=f32, device=dev)      # post ReLU/dropout fc1 activations (fc2_wgrad operand)
        self.dlogits = torch.zeros(B, 12, dtype=f32, device=dev)     # d loss / d logits, 48-byte rows
        self.dy2 = torch.zeros(B, 14, 14, 64, dtype=bf, device=dev)
        self.dx1 = torch.zeros(B, 14, 14, 32, dtype=bf, device=dev)
        # the data-gradient chain is the critical path: it is captured on a high-priority stream (_main_priority), the
        # weight-gradient side branches on low-priority ones, so the block scheduler serves the chain first whenever both
        # have CTAs pending
        self._side = [torch.cuda.Stream(device=dev, priority=0) for _ in range(4)]
        p_fc1 = self.spec.param("fc1_weights")
        self._zero_ranges = [(0, p_fc1.offset), (p_fc1.offset + p_fc1.numel, self.spec.arena_numel)]
        self._seed_mix0 = dropout_seed_mix(seed, 0, rank)
        # early bucket = fc1_weights (96.5 % of the bytes, final as soon as fc1_wgrad is done); everything else is late
        self._bucket_early = (p_fc1.offset, p_fc1.offset + p_fc1.numel)
        self._g16_shape = (3136, 512)
        self._epoch_ptr = backend.ctrl.local_ptr + backend._off["epoch"]

    # ---- kernels of the step, one launch each (the graph builder and time_kernels share them) ---------------------------
    # ``sp``: the stream to launch on (stream_ptr() of the caller's current stream, taken once per stream)
    def _conv1_fwd(self, images: torch.Tensor, B: int, train: bool, sp) -> None:
        p = self.p
        self.lib.dm_conv1_fwd_tc(images, p["conv1_weights"], p["conv1_biases"], self.a1, self.code1, B,
                                 *self._zero_args(train), sp)

    def _conv2_fwd(self, B: int, sp) -> None:
        self.lib.dm_conv2_fwd(self.a1, self.pb["conv2_weights"], self.p["conv2_biases"], self.a2, self.code2, B, sp)

    def _fc1_fwd(self, B: int) -> None:
        # a2[B,3136] (K-major) * W1[3136,512] (MN-major), split-K: 7 partial tiles stored side by side
        # (no atomics, nothing to zero); fc2_fwd_bwd sums them while applying bias + ReLU + dropout
        G.gemm_bf16_raw(self.a2, self.pb["fc1_weights"], self.h_part, B, 512, 3136, 3136, 512, 512, False, True,
                        G.EPI_STORE_F32, splits=self.fc1_splits, bn=64, split_stride=self.h_part.stride(0))

    def _fc2_fwd_bwd(self, labels: torch.Tensor, B: int, train: bool, sp, logits_out: Optional[torch.Tensor] = None) -> None:
        p = self.p
        self.lib.dm_fc2_fwd_bwd(self.h_part, self.h_part.stride(0), self.fc1_splits, p["fc1_biases"], p["fc2_weights"],
                                p["fc2_biases"], labels, self.dh, self.h_act, self.dlogits, self.d_loss_acc, logits_out, B,
                                int(train), self._seed_mix0, self._epoch_ptr if train else None, self.keep_prob, sp)

    def _fc1_wgrad(self, dst: torch.Tensor, B: int) -> None:
        # dW1[3136,512] = a2^T (A MN-major) * dh (B MN-major), K = batch: fp32 into the gradient arena, or bf16 (half the
        # epilogue stores, half the NVLink bytes) into the bucketed aggregation's symmetric wire buffer
        if self._decay:
            # + lambda * W1 in the epilogue, from the fp32 weights the step's forward read (DESIGN §4, weight decay)
            self.lib.dm_gemm_bf16_decay(self.a2, self.dh, dst, 3136, 512, B, 3136, 512, 512, int(dst.dtype == torch.bfloat16),
                                        self.p["fc1_weights"], self._decay, self._decay_ws, stream_ptr())
            return
        G.gemm_bf16_raw(self.a2, self.dh, dst, 3136, 512, B, 3136, 512, 512, True, True,
                        G.EPI_STORE_BF16 if dst.dtype == torch.bfloat16 else G.EPI_STORE_F32, bn=128)

    def _fc2_wgrad(self, B: int, sp) -> None:
        g = self.g
        if self._decay:
            p = self.p
            self.lib.dm_fc2_wgrad_decay(self.h_act, self.dlogits, self.dh, g["fc2_weights"], g["fc2_biases"], g["fc1_biases"],
                                        B, p["fc2_weights"], p["fc2_biases"], p["fc1_biases"], self._decay,
                                        self._decay_ws_fc2, sp)
            return
        self.lib.dm_fc2_wgrad(self.h_act, self.dlogits, self.dh, g["fc2_weights"], g["fc2_biases"], g["fc1_biases"], B, sp)

    # ---- L2 weight decay (see weight_decay.py) ---------------------------------------------------------------------------
    # The fc1 weight-gradient GEMM and fc2_wgrad add lambda * v to the four decayed variables' gradients in their epilogues
    # and store the sums of v^2 they read, one double per CTA, into a workspace; weight_decay_loss adds those partials in a
    # fixed order and (float)(lambda * R) to the step's loss word, on the loss read-back branch once both kernels are done.
    _decay = 0.0                   # lambda; 0: off (the plain kernels, the step graph of an engine without the flag)

    def arm_weight_decay(self, lam: float) -> None:
        """Train on CE + ``lam`` * R from the next step on (0 <= lam < 1; 0 turns it off): allocates the workspace, selects
        the decayed kernels and re-captures the step graphs.  The evaluation pass and :meth:`forward_logits` do not
        change."""
        lam = float(np.float32(lam))
        if not 0.0 <= lam < 1.0:
            raise ValueError("arm_weight_decay: lambda must lie in [0, 1), got %r" % lam)
        assert {q.name for q in weight_decay.decayed(self.spec)} == {"fc1_weights", "fc1_biases", "fc2_weights",
                                                                      "fc2_biases"}
        self._leave_native_runner()
        torch.cuda.synchronize()
        if lam and getattr(self, "_decay_ws", None) is None:
            n1 = int(self.lib.dm_gemm_decay_ctas(3136, 512))
            self._decay_parts = n1 + int(self.lib.dm_fc2_wgrad_decay_ctas())
            self._decay_ws = torch.zeros(self._decay_parts + 1, dtype=torch.float64, device=self.device)   # partials, R
            self._decay_ws_fc2 = self._decay_ws[n1:]
        self._decay = lam
        self._graphs = [None, None]

    def weight_decay_r(self) -> float:
        """R of the step completed last, as the device summed it (synchronises the device)."""
        torch.cuda.synchronize()
        return float(self._decay_ws[self._decay_parts].item())

    def _fc1_dgrad(self, B: int, sp) -> None:
        # d(pool2 out)[B,3136] = dh[B,512] (K-major) * W1[3136,512] (rows = in, K = out contiguous), with maxpool2/ReLU2
        # backward and the conv2 bias gradient in the GEMM epilogue (no [B,3136] intermediate)
        self.lib.dm_fc1_dgrad_unpool(self.dh, self.pb["fc1_weights"], self.code2, self.dy2, self.g["conv2_biases"], B, sp)

    def _conv2_wgrad(self, B: int, sp) -> None:
        self.lib.dm_conv2_wgrad(self.a1, self.dy2, self.g["conv2_weights"], B, sp)

    def _conv2_dgrad(self, B: int, sp) -> None:
        self.lib.dm_conv2_dgrad(self.dy2, self.pb["conv2_weights"], self.dx1, B, sp)

    def _conv1_wgrad(self, images: torch.Tensor, B: int, sp) -> None:
        g = self.g
        self.lib.dm_conv1_wgrad_tc(images, self.dx1, self.code1, g["conv1_weights"], g["conv1_biases"], B, sp)

    # ---- kernel sequence ------------------------------------------------------------------------------
    def _launch_forward(self, images: torch.Tensor, labels: torch.Tensor, B: int, train: bool,
                        logits_out: Optional[torch.Tensor] = None) -> int:
        sp = stream_ptr()
        self._conv1_fwd(images, B, train, sp)
        self._conv2_fwd(B, sp)
        self._fc1_fwd(B)
        self._fc2_fwd_bwd(labels, B, train, sp, logits_out)
        return 4

    def _launch_backward(self, images: torch.Tensor, B: int, early_sync: bool = False) -> int:
        """Backward as a small DAG: the weight-gradient kernels have no consumer before the aggregation, so they run
        on low-priority side streams (captured as parallel graph branches) next to the data-gradient chain
        fc1_dgrad(+unpool) -> conv2_dgrad -> conv1_wgrad.  ``early_sync``: bucketed aggregation -- the early-bucket
        kernel joins the fc1_wgrad branch and the small fc gradients get a branch of their own."""
        main = torch.cuda.current_stream()
        fork1 = torch.cuda.Event()
        fork1.record(main)
        self._side[0].wait_event(fork1)
        # (loss, accuracy) are final after fc2_fwd_bwd: their copy into the slot's page-locked host buffer is a branch of
        # the step (a memcpy node of the graph) that runs under the backward pass -- reading the result costs the host
        # no extra call, only a wait on the step's completion event
        # (its own branch, joined only at the very end of the step: a memcpy node in front of the aggregation kernel
        # would cost that kernel its programmatic launch edge)
        if not self._decay:
            self._launch_loss_readback(fork1)
        sp = stream_ptr()
        self._fc1_dgrad(B, sp)
        # (the side branch is issued AFTER the chain's kernel: both become ready together and the first one dispatched takes
        #  the SMs -- the data-gradient GEMM must be that one)
        with torch.cuda.stream(self._side[0]):
            self._fc1_wgrad(self._g16_view if early_sync and self._bucket_v2 else self.g["fc1_weights"], B)
            ev_w1 = torch.cuda.Event()
            ev_w1.record(self._side[0])
            if not early_sync:
                # fc2 weight/bias + fc1 bias gradients: only the aggregation kernel consumes them
                self._fc2_wgrad(B, stream_ptr())
                join1 = torch.cuda.Event()
                join1.record(self._side[0])
        if early_sync:
            # early bucket (fc1 weights): final once fc1_wgrad is done; the kernel also rewrites my shard of the fc1 bf16
            # shadow, which fc1_dgrad (launched above on the main stream) still reads -> ordered after it
            ev_du = torch.cuda.Event()
            ev_du.record(main)
            with torch.cuda.stream(self._side[0]):
                self._side[0].wait_event(ev_du)
                if self._straggler is not None and not getattr(self, "_delay_in_chain", False):
                    self.backend.enqueue_straggler(self._straggler, stream=self._side[0])
                oa = self._opt_args
                e0, e1 = self._bucket_early
                if self._bucket_v2:
                    self.backend.enqueue_bucket_v2(self.params, self.grads, self._g16, self._inbox, 1, e0, e1, oa["lr0"],
                                                   oa["decay_rate"], oa["decay_steps"], ctas=self._early_ctas,
                                                   stream=self._side[0])
                else:
                    self.backend.enqueue_bucket(self.params, self.grads, 1, e0, e1, e0, e1, oa["lr0"], oa["decay_rate"],
                                                oa["decay_steps"], ctas=self._early_ctas, stream=self._side[0])
                join1 = torch.cuda.Event()
                join1.record(self._side[0])
            # the small fc gradients (fc2 weights/biases, fc1 biases) belong to the late bucket: their own branch
            self._side[2].wait_event(fork1)
            with torch.cuda.stream(self._side[2]):
                self._fc2_wgrad(B, stream_ptr())
                join3 = torch.cuda.Event()
                join3.record(self._side[2])
        if self._decay:
            # the decay's loss term needs both weight-gradient kernels' partials (not the early bucket's exchange)
            self._launch_loss_readback(fork1, ev_w1, join3 if early_sync else join1)
        # conv2 dgrad and wgrad each fill the machine (1 CTA/SM, ~200 KB smem): side by side they only slow the chain
        # down.  wgrad is forked AFTER dgrad instead and shares the SMs with conv1_wgrad.
        self._conv2_dgrad(B, sp)
        fork2 = torch.cuda.Event()
        fork2.record(main)
        self._side[1].wait_event(fork2)
        with torch.cuda.stream(self._side[1]):
            self._conv2_wgrad(B, stream_ptr())
            join2 = torch.cuda.Event()
            join2.record(self._side[1])
        self._conv1_wgrad(images, B, sp)
        main.wait_event(join2)
        if self._stamp and early_sync:
            # every backward kernel of THIS replica is done (conv1_wgrad on the chain, conv2_wgrad joined): stamp it before
            # waiting for the exchange branch, which contains the all-to-all with the other replicas
            main.wait_event(join3)
            self.backend.enqueue_stamp_arrive()
        main.wait_event(join1)
        if early_sync:
            main.wait_event(join3)
        return 8 if self._decay else 7     # (conv2_wgrad is two launches: the kernel and its reduction)

    def _launch_loss_readback(self, *after: torch.cuda.Event) -> None:
        """The branch that copies (loss, accuracy) into the slot's page-locked host buffer, after the events ``after``;
        with weight decay it first adds the loss term."""
        for ev in after:
            self._side[3].wait_event(ev)
        with torch.cuda.stream(self._side[3]):
            if self._decay:
                self.lib.dm_weight_decay_loss(self._decay_ws, self._decay_parts, self._decay, self.d_loss_acc, stream_ptr())
            self.h_loss_bufs[self._slot].copy_(self.d_loss_acc, non_blocking=True)
            self._join_loss = torch.cuda.Event()
            self._join_loss.record(self._side[3])

    def _zero_args(self, train: bool):
        """Regions conv1_fwd clears at the start of a training step (atomically accumulated gradients + loss)."""
        if not train:
            return (None, 0, None, 0, self.d_loss_acc, 2)
        base = self.grads.data_ptr()
        (a0, b0), (a1, b1) = self._zero_ranges
        return (base + 4 * a0, b0 - a0, base + 4 * a1, b1 - a1, self.d_loss_acc, 2)

    def _launch_zero(self) -> int:
        return 0    # folded into conv1_fwd

    def time_kernels(self, iters: int = 20) -> dict:
        """Average device time of every kernel of the step, measured in place with CUDA events between
        eager launches (caches warm, as in the replayed graph; includes the launch gap).  ``unpool2`` is part of
        fc1_dgrad's epilogue and stays at 0."""
        names = ["memsets", "conv1_fwd", "conv2_fwd", "fc1_fwd", "fc2_fwd_bwd", "fc1_wgrad", "fc2_wgrad", "fc1_dgrad", "unpool2",
                 "conv2_wgrad", "conv2_dgrad", "conv1_wgrad"]
        # K > N: adopt + shadow refresh, and gate + accumulate + close + apply, in place of the fused sync kernel
        names = (["kgtn_begin"] + names + ["kgtn_end"]) if self._kgtn_k else \
            (["async_begin"] + names + ["async_end"]) if self._async else \
            names + ["local_end"] if self._local else names + ["gossip_end"] if self._gossip else names + ["fused_sync_sgd"]
        tot = {n: 0.0 for n in names}
        B, s = self.batch_size, self._slot
        img, lbl = self.images[s], self.labels[s]
        sp = stream_ptr()

        def seq():
            if self._kgtn_k:
                yield "kgtn_begin", lambda: self.backend.enqueue_kgtn_begin(self.params)
            elif self._async:
                yield "async_begin", lambda: self._enqueue_iteration_begin()
            yield "memsets", lambda: self._launch_zero()
            # forward / backward are issued kernel by kernel so an event can sit between any two
            yield "conv1_fwd", lambda: self._conv1_fwd(img, B, True, sp)
            yield "conv2_fwd", lambda: self._conv2_fwd(B, sp)
            yield "fc1_fwd", lambda: self._fc1_fwd(B)
            yield "fc2_fwd_bwd", lambda: self._fc2_fwd_bwd(lbl, B, True, sp)
            yield "fc1_wgrad", lambda: self._fc1_wgrad(self.g["fc1_weights"], B)
            yield "fc2_wgrad", lambda: self._fc2_wgrad(B, sp)
            yield "fc1_dgrad", lambda: self._fc1_dgrad(B, sp)
            yield "conv2_wgrad", lambda: self._conv2_wgrad(B, sp)
            yield "conv2_dgrad", lambda: self._conv2_dgrad(B, sp)
            yield "conv1_wgrad", lambda: self._conv1_wgrad(img, B, sp)
            if self._async:
                yield "async_end", lambda: self._enqueue_iteration_end()
            elif self._local:
                yield "local_end", lambda: self._enqueue_iteration_end()
            elif self._gossip:
                yield "gossip_end", lambda: self._enqueue_iteration_end()
            elif self._kgtn_k:
                oa = self._opt_args
                yield "kgtn_end", lambda: self.backend.enqueue_kgtn_end(self.params, self.grads, self._acc, self._kgtn_k, oa["lr0"],
                                                                        oa["decay_rate"], oa["decay_steps"])
            else:
                yield "fused_sync_sgd", lambda: self.backend.enqueue(self.params, self.grads, **self._opt_args)

        for it in range(iters + 3):
            evs = [torch.cuda.Event(enable_timing=True)]
            evs[0].record()
            order = []
            for name, fn in seq():
                fn()
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                evs.append(e)
                order.append(name)
            torch.cuda.synchronize()
            if self.backend.ctx.world_size > 1:
                self.backend.barrier()
            if it >= 3:
                for i, name in enumerate(order):
                    tot[name] += evs[i].elapsed_time(evs[i + 1]) * 1e3 / iters
        return tot

    def _launch_step(self, slot: int, with_sync: bool) -> None:
        n = 0
        own = bool(self._local) or self._gossip          # local / gossip SGD: an iteration end without an iteration begin
        interval = with_sync and (getattr(self, "_interval", False) or self._async or own)   # own iteration end
        bucketed = with_sync and self._bucketed and not interval
        self._delay_in_chain = False
        if self._stamp:
            self.backend.enqueue_stamp_start()
            n += 1
            if bucketed and self._straggler is not None:
                # cdf telemetry: the injected delay is part of THIS replica's compute (start stamp .. gradient-complete stamp)
                self.backend.enqueue_straggler(self._straggler)
                self._delay_in_chain = True
                n += 1
        images = self.images[slot]
        if self._aug is not None:
            images = self._launch_augment(slot)     # conv1_fwd and conv1_wgrad read the augmented batch
            n += 1
        if interval and not own:
            self._enqueue_iteration_begin()
            n += 3 if self._ssp >= 0 else 2       # the staleness bound's wait before the pull
        n += self._launch_zero()
        n += self._launch_forward(images, self.labels[slot], self.batch_size, True)
        n += self._launch_backward(images, self.batch_size, early_sync=bucketed)
        if bucketed:
            oa = self._opt_args
            e0, e1 = self._bucket_early
            if self._bucket_v2:
                self.backend.enqueue_bucket_v2(self.params, self.grads, self._g16, self._inbox, 2, e0, e1, oa["lr0"],
                                               oa["decay_rate"], oa["decay_steps"])
            else:
                self.backend.enqueue_bucket(self.params, self.grads, 2, 0, self.spec.arena_numel, e0, e1,
                                            oa["lr0"], oa["decay_rate"], oa["decay_steps"])
            n += 2 + (1 if self._straggler is not None else 0)
        elif with_sync:
            if self._straggler is not None:
                self.backend.enqueue_straggler(self._straggler)
                n += 1
            if interval:
                self._enqueue_iteration_end()
                # local SGD: the update, the round's four; gossip SGD: the half step, the barrier, the mix
                n += 5 if self._local else 3 if self._gossip else (2 + (self._ssp >= 0)) if self._async else 4
            else:
                self.backend.enqueue(self.params, self.grads, **self._opt_args)
                n += 1
        torch.cuda.current_stream().wait_event(self._join_loss)      # the loss read-back branch rejoins at the end of the step
        if with_sync and self._ema is not None:
            self._launch_moving_average()        # after the exchange has committed the step's weights and the epoch word
            n += 1
        if with_sync and self._stop is not None:
            self._launch_stop_publish()          # the step's last node: after its exchange, and after the loss read-back
            n += 1
        self.launches_per_step = n

    # ---- inference ------------------------------------------------------------------------------------------
    def _eval_forward(self, images: torch.Tensor, labels: torch.Tensor, B: int) -> None:
        self._launch_forward(images, labels, B, False)          # conv1_fwd clears the loss accumulator

    def forward_logits(self, images: torch.Tensor, labels: torch.Tensor, train: bool) -> torch.Tensor:
        """Debug/test helper: logits of one batch through the CUDA forward."""
        B = images.shape[0]
        out = torch.zeros(B, 10, dtype=torch.float32, device=self.device)
        self.d_loss_acc.zero_()
        self._launch_forward(images.reshape(B, 28, 28).contiguous(), labels, B, train, logits_out=out)
        return out

    # ---- in-training evaluation (csrc/eval_head.cu) ---------------------------------------------------------------------
    # The validation set is scored in chunks of EVAL_CHUNK rows by the forward kernels on buffers of its own, then by the
    # evaluation head, on the training stream right after the step whose weights it scores: nothing is shared with the step
    # (no activation buffer, no workspace, no ticket), so the next step computes exactly what it would have computed without
    # the pass.  The pass's record lands in page-locked host memory; the host reads it once an event that follows the pass
    # has fired (in the training loop: the next step's completion event).
    EVAL_CHUNK = 2048
    EVAL_RING = 16                 # host record slots
    SNAP_KEEP = False              # also keep the last accepted snapshot (one more 6.65 MB copy per accepted pass), see
                                   # eval_snapshot(); set before arm_eval
    _ev_average = False            # the pass scores the moving average, see arm_eval

    def arm_eval(self, images, labels, snapshot: bool = False, moving_average: bool = False) -> None:
        """Upload the validation set once (device-resident fp32 images, int64 labels) and allocate the pass's buffers and
        the host record ring.  With ``use_graph`` the whole pass is captured as one CUDA graph.

        ``snapshot``: peers may push weights into this (the chief's) arena at any time (K < N, interval mode).  The pass then
        scores a private copy of the newest committed weights that is checked to hold exactly one global step
        (csrc/eval_snapshot.cu): up to SNAP_ATTEMPTS select / copy / validate attempts run in front of the chunks, and a pass
        whose attempts all fail is dropped by :meth:`eval_records` (counted in ``eval_dropped``).

        ``moving_average``: score the moving average (after :meth:`arm_moving_average`) instead of the weights.  The pass
        first writes the bf16 copy of the average's conv2 / fc1 weights (its tensor-core operands), rounded as the training
        shadow is, and its record names the step of the averaged weights."""
        if moving_average and (self._ema is None or snapshot):
            raise ValueError("arm_eval(moving_average=True) needs arm_moving_average() first and no snapshot")
        self._leave_native_runner()
        lib, dev = self.lib, self.device
        x = torch.as_tensor(np.ascontiguousarray(images) if isinstance(images, np.ndarray) else images, dtype=torch.float32)
        y = torch.as_tensor(np.ascontiguousarray(labels) if isinstance(labels, np.ndarray) else labels).to(torch.int64)
        n = int(x.shape[0])
        if n < 1 or y.numel() != n:
            raise ValueError("arm_eval: %d images, %d labels" % (n, y.numel()))
        assert self.EVAL_CHUNK <= int(lib.dm_eval_max_rows())
        self._ev_x = x.reshape(n, 28, 28).to(dev).contiguous()
        self._ev_y = y.reshape(n).to(dev).contiguous()
        C = min(self.EVAL_CHUNK, n)
        bf, u8, f32 = torch.bfloat16, torch.uint8, torch.float32
        self._ev_a1 = torch.zeros(C, 14, 14, 32, dtype=bf, device=dev)
        self._ev_code1 = torch.zeros(C, 14, 14, 32, dtype=u8, device=dev)
        self._ev_a2 = torch.zeros(C, 3136, dtype=bf, device=dev)
        self._ev_code2 = torch.zeros(C, 3136, dtype=u8, device=dev)
        self._ev_hpart = torch.zeros(self.fc1_splits, C, 512, dtype=f32, device=dev)
        self._ev_ws = torch.zeros(2 * int(lib.dm_eval_max_rows()), dtype=f32, device=dev)
        self._ev_state = torch.zeros(int(lib.dm_eval_state_bytes()), dtype=u8, device=dev)
        self._ev_ring = torch.zeros(self.EVAL_RING, 8, dtype=torch.int64).pin_memory()
        self._ev_seen = 0
        self._ev_last = None
        self._ev_graph = None
        self.eval_dropped = 0
        self._snapshot = bool(snapshot)
        if self._snapshot:
            self._snap = torch.zeros(self.spec.arena_numel, dtype=f32, device=dev)
            # arena-sized so spec.views() applies, but only the conv2 / fc1 weight ranges (_snap_bf_ranges) are ever written
            # or read: the rest stays zero
            self._snap16 = torch.zeros(self.spec.arena_numel, dtype=bf, device=dev)
            self._snap_keep = torch.zeros(self.spec.arena_numel, dtype=f32, device=dev) if self.SNAP_KEEP else None
            # the bf16 operands of the pass: conv2 and fc1 weights (tensor-core kernels); everything else is read as fp32
            self._snap_bf_ranges = []
            for name in ("conv2_weights", "fc1_weights"):
                q = self.spec.param(name)
                assert q.offset % 4 == 0 and q.numel % 4 == 0, name
                self._snap_bf_ranges += [q.offset, q.offset + q.numel]
            self._ev_snap = _Snapshot(self, self._snap, self._snap16, self._snap_bf_ranges, self._snap_keep)
            self._snap_state = self._ev_snap.state
            self._ev_views = (self.spec.views(self._snap), self.spec.views(self._snap16))
        elif moving_average:
            # arena-sized like _snap16; only the conv2 / fc1 weight ranges are written
            self._ev_ema16 = torch.zeros(self.spec.arena_numel, dtype=bf, device=dev)
            self._ev_ema_ranges = []
            for name in ("conv2_weights", "fc1_weights"):
                q = self.spec.param(name)
                assert q.offset % 4 == 0 and q.numel % 4 == 0, name
                self._ev_ema_ranges += [q.offset, q.offset + q.numel]
            self._ev_views = (self.spec.views(self._ema), self.spec.views(self._ev_ema16))
        else:
            self._ev_views = (self.p, self.pb)
        self._ev_average = bool(moving_average)
        self._target = None
        self._best = None
        self._patience = None
        self._plateau = None
        self._launch_eval(publish=False)       # sets the kernels' function attributes outside a capture
        torch.cuda.synchronize()
        if self._snapshot:
            self._ev_snap.reset()                 # statistics count real passes only
        self._capture_eval()

    def _capture_eval(self) -> None:
        if self.use_graph:
            gr = torch.cuda.CUDAGraph()
            cap = torch.cuda.Stream(device=self.device)
            with _capture(gr, cap):
                self._launch_eval(publish=True)
            self._ev_graph = gr

    def _launch_snapshot(self, attempts: int) -> None:
        """The pass's ``attempts`` select / copy / validate rounds (see :meth:`_Snapshot.launch`)."""
        self._ev_snap.launch(attempts)

    def _launch_eval(self, publish: bool, logits_out: Optional[torch.Tensor] = None, p=None, pb=None) -> None:
        """One pass over the validation set with the weight views ``p`` (fp32) / ``pb`` (bf16): by default the armed ones --
        the live arena, or the snapshot, which the pass then takes first."""
        lib, sp = self.lib, stream_ptr()
        if p is None:
            if self._snapshot:
                self._launch_snapshot(self.SNAP_ATTEMPTS)
            elif self._ev_average:
                # the bf16 operands of the average (no weights: the kernel only converts)
                lib.dm_moving_average(self._ema, None, self.spec.arena_numel, None, 0.0, None, self._ev_ema16,
                                      *self._ev_ema_ranges, sp)
            p, pb = self._ev_views
        n, C = self._ev_x.shape[0], self._ev_a1.shape[0]
        stride = self._ev_hpart.stride(0)
        ring = self._ev_ring if publish else None
        armed = p is self._ev_views[0]
        if self._snapshot and armed:
            st = self._snap_state.data_ptr()
            step_ptr, status_ptr = st, st + 4                                        # SnapState.step, SnapState.status
            scored = self._snap
        elif self._ev_average and armed:
            step_ptr, status_ptr = self._ema_step, None                              # step of the averaged weights
            scored = self._ema
        else:
            step_ptr, status_ptr = self._epoch_ptr, None
            scored = self.params if armed else None                                  # fp32 arena the pass scores
        lib.dm_eval_stamp(self._ev_state, sp)
        for s in range(0, n, C):
            m = min(C, n - s)
            lib.dm_conv1_fwd_tc(self._ev_x[s:s + m], p["conv1_weights"], p["conv1_biases"], self._ev_a1, self._ev_code1, m,
                                None, 0, None, 0, None, 0, sp)
            lib.dm_conv2_fwd(self._ev_a1, pb["conv2_weights"], p["conv2_biases"], self._ev_a2, self._ev_code2, m, sp)
            G.gemm_bf16_raw(self._ev_a2, pb["fc1_weights"], self._ev_hpart, m, 512, 3136, 3136, 512, 512, False, True,
                            G.EPI_STORE_F32, splits=self.fc1_splits, bn=64, split_stride=stride)
            lg = None if logits_out is None else logits_out[s:s + m]
            lib.dm_eval_head(self._ev_hpart, stride, self.fc1_splits, p["fc1_biases"], p["fc2_weights"], p["fc2_biases"],
                             self._ev_y[s:s + m], self._ev_ws, self._ev_state, step_ptr, status_ptr, ring, self.EVAL_RING,
                             lg, m, int(s + m == n), sp)
        if publish and self._best is not None and scored is not None:
            state, decision, arena = self._best
            lib.dm_eval_best_decide(self._ev_state, step_ptr, status_ptr, n, state, decision, sp)
            lib.dm_eval_best_copy(decision, scored, arena, arena.numel(), sp)
        if publish and self._target is not None:
            need, margin = self._target
            lib.dm_eval_target(self._ev_state, step_ptr, status_ptr, need, n, margin, self._stop.ptr_table(),
                               self.backend.ctx.rank, self.backend.ctx.world_size, sp)
        if publish and self._patience is not None:
            state, patience, delta_rows, margin = self._patience
            lib.dm_eval_patience(self._ev_state, step_ptr, status_ptr, n, patience, delta_rows, margin, state,
                                 self._stop.ptr_table(), self.backend.ctx.rank, self.backend.ctx.world_size, sp)
        if publish and self._plateau is not None:
            state, patience, delta_rows, margin = self._plateau
            lib.dm_eval_plateau(self._ev_state, step_ptr, status_ptr, n, patience, delta_rows, margin, state,
                                self._lr_table.ptr_table(), self.backend.ctx.world_size, sp)

    def enqueue_eval(self) -> None:
        """Score the validation set with the current weights, on the current (training) stream, without a host
        synchronisation.  Enqueue it right after the step whose weights it scores; its record is complete once any event
        recorded after it -- e.g. the next step's completion event -- has fired (see :meth:`eval_record`)."""
        if self._ev_graph is not None:
            self._ev_graph.replay()
        else:
            self._launch_eval(publish=True)

    def eval_records(self):
        """Records completed since the previous call, oldest first: ``(global_step, t_begin_ns, t_end_ns, examples,
        correct, loss_sum)`` (``%globaltimer`` stamps; ``loss_sum`` is the sum of the per-row cross entropies).  With a
        snapshot pass, ``global_step`` is the step of the snapshot it scored; a pass that found no consistent snapshot is
        left out and counted in ``eval_dropped``.

        The ring holds the last EVAL_RING records: call this at least once per EVAL_RING enqueued passes.  A caller that
        falls further behind loses the overwritten records, and a slot the device is rewriting while it is read is skipped
        (the training loop reads after every step, with at most two passes outstanding)."""
        out = []
        for rec, status in self.eval_records_with_status():
            if status < 0:
                self.eval_dropped += 1
                continue
            out.append(rec)
        return out

    def eval_records_with_status(self):
        """Like :meth:`eval_records`, but every record of the ring, each with its snapshot outcome: 0 for a pass over the
        live arena, n > 0 when attempt n produced its snapshot, -1 when no attempt did (the record is then meaningless)."""
        raw = self._ev_ring.numpy()
        new = []
        for i in range(self.EVAL_RING):
            seq = int(raw[i, 0])
            if seq <= self._ev_seen:
                continue
            rec = raw[i].copy()
            if int(raw[i, 0]) != seq or int(rec[0]) != seq:
                continue                                 # slot rewritten while it was read: the pass is still running
            loss = float(rec[6:7].view(np.float64)[0])
            new.append((seq, (int(rec[1]), int(rec[2]), int(rec[3]), int(rec[4]), int(rec[5]), loss), int(rec[7])))
        new.sort()
        if new:
            self._ev_seen = new[-1][0]
            good = [r for _, r, st in new if st >= 0]
            if good:
                self._ev_last = good[-1]
        return [(r, st) for _, r, st in new]

    def eval_snapshot(self):
        """``(fp32 arena, global step)`` of a snapshot, or None (synchronises the current stream).  With ``SNAP_KEEP`` set
        when the pass was armed: the last ACCEPTED snapshot, kept aside by ``snap_keep``, whatever later passes found.
        Without it: the newest pass's snapshot if that pass found a consistent one, else None -- a failed attempt overwrites
        the snapshot buffer, so an older accepted snapshot is gone."""
        if not getattr(self, "_snapshot", False):
            return None
        torch.cuda.current_stream().synchronize()
        st = self._snap_state[:48].cpu().view(torch.int32).tolist()
        if self._snap_keep is not None:
            keep_step = st[10] & 0xFFFFFFFF
            return None if keep_step == 0xFFFFFFFF else (self._snap_keep.clone(), keep_step)
        if st[1] <= 0:
            return None
        return self._snap.clone(), st[0] & 0xFFFFFFFF

    def eval_snapshot_stats(self) -> dict:
        """Snapshot attempts since :meth:`arm_eval`: made, rejected by validate, ended by the watchdog, ended because the
        commit slot of the candidate step was already reused (a ring lap behind); passes accepted / failed (synchronises
        the current stream)."""
        return self._ev_snap.stats()

    def eval_record(self):
        """The newest complete record (see :meth:`eval_records`), or None."""
        self.eval_records()
        return self._ev_last

    def run_eval(self, logits_out: Optional[torch.Tensor] = None):
        """One pass, enqueued eagerly and waited for: its record.  ``logits_out`` [n,10] receives the logits."""
        self.eval_records()
        self._launch_eval(publish=True, logits_out=logits_out)
        torch.cuda.current_stream().synchronize()
        return self.eval_record()

    # ---- quality target (csrc/eval_target.cu) -----------------------------------------------------------------------------
    # With a target armed, the chief's evaluation pass ends with eval_target, which sets the stop step in every replica's
    # stop word, and every replica's step graph ends with stop_publish, which copies its own stop word into page-locked host
    # memory.  The host reads that word after the step's completion event, which the training loop waits for anyway.  Why a
    # K = N run then stops every replica after the same step: DESIGN §4.4.
    _stop = None                   # symmetric u32 stop word (0: no stop set), see arm_stop
    _target = None                 # (need, margin) of the chief's target test, see arm_target

    def arm_stop(self) -> None:
        """Allocate this replica's stop word (symmetric memory: collective, every rank calls it at the same point) and its
        page-locked host copy.  From then on every training step ends with stop_publish: the step graphs are re-captured."""
        self._leave_native_runner()
        self._stop = self.backend.allocate_buffer(4)
        self._stop.view(torch.int32, 0, 1).zero_()
        self._stop_host = torch.zeros(1, dtype=torch.int32).pin_memory()
        self._stop_host_np = self._stop_host.numpy().view(np.uint32)
        self._tta_t0 = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._graphs = [None, None]
        torch.cuda.synchronize()
        if self.backend.ctx.world_size > 1:
            self.backend.barrier()             # every stop word is zero before the chief can set one

    def arm_target(self, need: int, margin: int) -> None:
        """Chief, after :meth:`arm_eval` and :meth:`arm_stop`: every evaluation pass ends with eval_target.  The first pass
        over the whole validation set with at least ``need`` correct rows (a snapshot pass only if its snapshot was
        accepted) stores S = (global step it scored) + ``margin`` into every replica's stop word."""
        if self._stop is None or getattr(self, "_ev_x", None) is None:
            raise RuntimeError("arm_target: arm_eval() and arm_stop() first")
        n = int(self._ev_x.shape[0])
        if not 1 <= int(need) <= n or int(margin) < 1:
            raise ValueError("arm_target: need %d of %d examples, margin %d" % (need, n, margin))
        self._leave_native_runner()
        self._target = (int(need), int(margin))
        self._capture_eval()

    def _launch_stop_publish(self) -> None:
        self.lib.dm_stop_publish(self._stop.local_ptr, self._stop_host, stream_ptr())

    def stop_step(self) -> int:
        """Stop step S of this replica's stop word, 0 while none is set, as its newest completed step saw it (a host read:
        valid after waiting for a step's completion)."""
        return int(self._stop_host_np[0])

    def enqueue_start_stamp(self) -> None:
        """``%globaltimer`` into a device word, on the current stream: enqueue it right before the run's first step."""
        self.lib.dm_tta_stamp(self._tta_t0, stream_ptr())

    def start_stamp_ns(self) -> int:
        """The stamp of :meth:`enqueue_start_stamp` (a device read, ordered after the current stream's work)."""
        return int(self._tta_t0.cpu()[0])

    # ---- best-scoring weights (csrc/eval_best.cu) -------------------------------------------------------------------------
    # With best-keeping armed, every evaluation pass ends (before eval_target) with eval_best_decide, which applies the
    # selection rule of best.improves to the pass's record and BestState, and eval_best_copy, which copies the arena the pass
    # scored into the best arena when decide chose it.  Nothing is read back until best_weights().
    _best = None                   # (BestState bytes, decision word, best arena), see arm_best

    def arm_best(self, initial_correct: int = 0) -> None:
        """Chief, after :meth:`arm_eval`: every evaluation pass keeps its weights if it beats every earlier pass and
        ``initial_correct`` (an earlier run's best count).  Re-captures the evaluation graph."""
        if getattr(self, "_ev_x", None) is None:
            raise RuntimeError("arm_best: arm_eval() first")
        n = int(self._ev_x.shape[0])
        if not 0 <= int(initial_correct) <= n:
            raise ValueError("arm_best: initial count %d of %d examples" % (initial_correct, n))
        self._leave_native_runner()
        words = torch.zeros(int(self.lib.dm_best_state_bytes()) // 4, dtype=torch.int32)
        words[BEST_CORRECT_WORD] = int(initial_correct)
        self._best = (words.to(self.device), torch.zeros(1, dtype=torch.int32, device=self.device),
                      torch.zeros(self.spec.arena_numel, dtype=torch.float32, device=self.device))
        self._capture_eval()

    def best_weights(self):
        """``(fp32 arena, global step, correct, examples, loss_sum)`` of the best pass since :meth:`arm_best`, or None when
        no pass beat the initial count (synchronises the device)."""
        if self._best is None:
            return None
        torch.cuda.synchronize()
        state, _decision, arena = self._best
        w = state.cpu()
        if int(w[BEST_VALID_WORD]) == 0:
            return None
        u = w.numpy().view(np.uint32)
        return (arena.clone(), int(u[BEST_STEP_WORD]), int(u[BEST_CORRECT_WORD]), int(u[BEST_EXAMPLES_WORD]),
                float(w[:2].numpy().view(np.float64)[0]))

    # ---- early stopping (csrc/eval_patience.cu) ---------------------------------------------------------------------------
    # With a patience armed, every evaluation pass ends (after eval_best_* and eval_target) with eval_patience, which applies
    # the rule of early_stopping.advance to the pass's record and PatienceState and, once the patience is exhausted, sets
    # the stop step as eval_target does.  Nothing is read back until patience_state().
    _patience = None               # (PatienceState words, patience, min_delta rows, margin), see arm_patience

    def arm_patience(self, patience: int, min_delta_rows: int, margin: int) -> None:
        """Chief, after :meth:`arm_eval` and :meth:`arm_stop`: stop the run at S = g + ``margin`` once ``patience``
        counting passes in a row, the last of global step g, have not beaten the best count by more than
        ``min_delta_rows``.  Re-captures the evaluation graph."""
        if self._stop is None or getattr(self, "_ev_x", None) is None:
            raise RuntimeError("arm_patience: arm_eval() and arm_stop() first")
        n = int(self._ev_x.shape[0])
        if int(patience) < 1 or not 0 <= int(min_delta_rows) < n or int(margin) < 1:
            raise ValueError("arm_patience: patience %d, min_delta %d of %d rows, margin %d"
                             % (patience, min_delta_rows, n, margin))
        self._leave_native_runner()
        words = torch.zeros(int(self.lib.dm_patience_state_bytes()) // 4, dtype=torch.int32, device=self.device)
        self._patience = (words, int(patience), int(min_delta_rows), int(margin))
        self._capture_eval()

    def patience_state(self) -> Optional[early_stopping.State]:
        """The PatienceState as the passes so far left it, or None when no patience is armed (synchronises the device)."""
        if self._patience is None:
            return None
        torch.cuda.synchronize()
        u = self._patience[0].cpu().numpy().view(np.uint32)
        return early_stopping.State(int(u[PAT_BEST_WORD]), int(u[PAT_SINCE_WORD]), int(u[PAT_BEST_STEP_WORD]),
                                    int(u[PAT_TRIGGER_WORD]), bool(u[PAT_BASELINE_WORD]))

    # ---- learning-rate cuts at a plateau (csrc/eval_plateau.cu) -----------------------------------------------------------
    # Every replica owns a cut table (symmetric memory) that its control block points at: the aggregation kernels multiply
    # the rate by F^c, c = the table's entries <= the step they update (cta_scale, csrc/fused_sync.cuh).  With a plateau
    # armed, the chief's evaluation pass ends (after eval_patience) with eval_plateau, which applies the rule of
    # lr_plateau.advance and stores each cut's step S into every replica's table.  The step graphs are not re-captured: the
    # kernels read the table through the control block.  Nothing is read back until lr_plateau_state().
    _lr_table = None               # symmetric u32[lr_plateau.MAX_CUTS] cut table, see arm_lr_cuts
    _plateau = None                # (PlateauState words, patience, min_delta rows, margin), see arm_lr_plateau

    def arm_lr_cuts(self, factor: float, cuts=()) -> None:
        """Every replica (symmetric memory: collective, every rank calls it at the same point): allocate this replica's
        cut table, store the steps ``cuts`` (those a restarted run keeps) in its first entries and point the aggregation
        kernels at it, each cut multiplying the rate by ``factor``."""
        cuts = [int(s) for s in cuts]
        if not 0.0 < float(factor) < 1.0 or len(cuts) > lr_plateau.MAX_CUTS:
            raise ValueError("arm_lr_cuts: factor %r, %d cuts" % (factor, len(cuts)))
        self._lr_table = self.backend.allocate_buffer(4 * lr_plateau.MAX_CUTS)
        words = np.full(lr_plateau.MAX_CUTS, lr_plateau.NO_CUT, dtype=np.uint32)
        words[:len(cuts)] = cuts
        self._lr_table.view(torch.int32, 0, lr_plateau.MAX_CUTS).copy_(torch.from_numpy(words.view(np.int32)))
        torch.cuda.synchronize()
        self.lib.dm_sync_set_lr_cuts(self.backend.ctrl.local_ptr, self._lr_table.local_ptr, float(factor))
        if self.backend.ctx.world_size > 1:
            self.backend.barrier()             # every table is in place before the chief can store a cut

    def lr_cut_table(self):
        """This replica's cut table as the device holds it: ``lr_plateau.MAX_CUTS`` steps, ``lr_plateau.NO_CUT`` where no
        cut is stored (synchronises the device)."""
        torch.cuda.synchronize()
        return [int(x) for x in self._lr_table.view(torch.int32, 0, lr_plateau.MAX_CUTS).cpu().numpy().view(np.uint32)]

    def arm_lr_plateau(self, patience: int, min_delta_rows: int, margin: int, restored: int = 0) -> None:
        """Chief, after :meth:`arm_eval` and :meth:`arm_lr_cuts`: once ``patience`` counting passes in a row, the last of
        global step g, have not beaten the best count by more than ``min_delta_rows``, cut the rate from S = g +
        ``margin`` on every replica.  ``restored``: the cuts already in the tables (a restarted run's).  Re-captures the
        evaluation graph."""
        if self._lr_table is None or getattr(self, "_ev_x", None) is None:
            raise RuntimeError("arm_lr_plateau: arm_eval() and arm_lr_cuts() first")
        n = int(self._ev_x.shape[0])
        if int(patience) < 1 or not 0 <= int(min_delta_rows) < n or int(margin) < 1 or \
                not 0 <= int(restored) <= lr_plateau.MAX_CUTS:
            raise ValueError("arm_lr_plateau: patience %d, min_delta %d of %d rows, margin %d, %d restored cuts"
                             % (patience, min_delta_rows, n, margin, restored))
        self._leave_native_runner()
        words = torch.zeros(int(self.lib.dm_plateau_state_bytes()) // 4, dtype=torch.int32)
        words[PL_CUTS_WORD] = int(restored)
        self._plateau = (words.to(self.device), int(patience), int(min_delta_rows), int(margin))
        self._capture_eval()

    def lr_plateau_state(self) -> Optional[lr_plateau.State]:
        """The PlateauState as the passes so far left it, or None when no plateau is armed (synchronises the device)."""
        if self._plateau is None:
            return None
        torch.cuda.synchronize()
        u = self._plateau[0].cpu().numpy().view(np.uint32)
        return lr_plateau.State(int(u[PL_BEST_WORD]), int(u[PL_SINCE_WORD]), bool(u[PL_BASELINE_WORD]),
                                int(u[PL_CUTS_WORD]), int(u[PL_TRIGGER_WORD]))


# dm_dense10_xent (csrc/mlp_simt.cu) stages the output-layer weights as [H][11] floats and refuses more than 220 KiB
MLP_XENT_SMEM_PER_UNIT = 11 * 4
MLP_XENT_SMEM_LIMIT = 220 * 1024


class CudaMlpEngine(_CudaEngine):
    """2-/3-layer MLP on the sm_90a kernels: hidden layers = wgmma GEMM with bias+ReLU fused in the
    epilogue, output layer + softmax-CE = SIMT (csrc/mlp_simt.cu), every weight gradient = wgmma GEMM
    with MN-major operands writing straight into the gradient arena."""

    def __init__(self, model: str, batch_size: int, backend: FusedBackend, hidden: int = 1024, seed: int = 66478,
                 rank: int = 0, use_graph: bool = True):
        assert hidden % 64 == 0, "--mlp_hidden must be a multiple of 64 on the GPU path"
        if hidden * MLP_XENT_SMEM_PER_UNIT > MLP_XENT_SMEM_LIMIT:
            raise ValueError("--mlp_hidden=%d is too wide for the output-layer kernel (dense10_xent keeps the [H,10] weights "
                             "in %d bytes of shared memory per hidden unit, at most %d bytes): use --mlp_hidden <= %d"
                             % (hidden, MLP_XENT_SMEM_PER_UNIT, MLP_XENT_SMEM_LIMIT,
                                MLP_XENT_SMEM_LIMIT // MLP_XENT_SMEM_PER_UNIT // 64 * 64))
        super().__init__(get_model(model, hidden)[0], batch_size, backend, seed, use_graph, (784,))
        self.model, self.hidden = model, hidden
        self.n_layers = len(self.spec.params) // 2
        # 128 x 256 GEMM tiles when the hidden width allows: half the L2->SM operand traffic per FLOP of 128 x 128
        self._bn = 256 if hidden % 256 == 0 else 128
        B, dev, bf = batch_size, self.device, torch.bfloat16
        self.x16 = torch.zeros(B, 784, dtype=bf, device=dev)
        self.h = [torch.zeros(B, hidden, dtype=bf, device=dev) for _ in range(self.n_layers - 1)]
        self.dh = [torch.zeros(B, hidden, dtype=bf, device=dev) for _ in range(self.n_layers - 1)]
        self.dl_pad = torch.zeros(B, 64, dtype=bf, device=dev)
        # bucketed aggregation (csrc/fused_bucket.cu): the largest weight matrix is the early bucket (bf16 wire, exchanged next
        # to the remaining backward GEMMs), everything else the pushed late bucket
        big = max((q for q in self.spec.params if q.name.endswith("weights")), key=lambda q: q.numel)
        self._early_name = big.name
        self._bucket_early = (big.offset, big.offset + big.numel)
        self._g16_shape = (784 if big.name == "fc1_weights" else hidden, hidden if big.name != "fc%d_weights" % self.n_layers else 10)
        self._side = [torch.cuda.Stream(device=dev)]
        # everything except the weight matrices (written whole by GEMM stores) is accumulated with atomics
        stored = sorted((q.offset, q.offset + q.numel) for q in self.spec.params if q.name.endswith("weights"))
        self._zero_ranges, pos = [], 0
        for (a0, a1) in stored:
            if a0 > pos:
                self._zero_ranges.append((pos, a0))
            pos = a1
        if pos < self.spec.arena_numel:
            self._zero_ranges.append((pos, self.spec.arena_numel))

    def _forward(self, images: torch.Tensor, labels: torch.Tensor, B: int, train: bool,
                 logits_out: Optional[torch.Tensor] = None) -> int:
        lib, sp, p, pb, H = self.lib, stream_ptr(), self.p, self.pb, self.hidden
        n = 0
        lib.dm_f32_to_bf16(images, self.x16, B * 784, sp)
        src, K = self.x16, 784
        for i in range(1, self.n_layers):
            # h_i = relu(src @ W_i + b_i): A K-major, B = W_i [in,out] MN-major, bias+ReLU in the epilogue
            G.gemm_bf16_raw(src, pb["fc%d_weights" % i], self.h[i - 1], B, H, K, K, H, H, False, True,
                            G.EPI_BIAS_RELU_BF16, bn=self._bn, bias=p["fc%d_biases" % i])
            src, K = self.h[i - 1], H
            n += 1
        L = self.n_layers
        lib.dm_dense10_xent(src, p["fc%d_weights" % L], p["fc%d_biases" % L], labels, self.dh[-1], self.dl_pad,
                            self.g["fc%d_biases" % L], self.d_loss_acc, logits_out, B, H, int(train), sp)
        return n + 2

    def _backward(self, B: int, early_sync: bool = False) -> int:
        """``early_sync``: bucketed aggregation -- the big layer's weight gradient is stored as bf16 into the wire buffer and its
        exchange (phase 3) starts on a side stream at once, next to the data-gradient GEMM; the apply (phase 4) follows that
        GEMM, which is the last reader of the layer's bf16 shadow."""
        lib, sp, g, pb, H, L = self.lib, stream_ptr(), self.g, self.pb, self.hidden, self.n_layers
        n = 0
        main = torch.cuda.current_stream()
        oa, be = self._opt_args, self.backend
        self._join_early = None
        # output layer: dW_L[H,10] = h_last^T (MN-major) * dl (MN-major, 64-wide zero-padded rows, N = 10)
        G.gemm_bf16_raw(self.h[-1], self.dl_pad, g["fc%d_weights" % L], H, 10, B, H, 64, 10, True, True,
                        G.EPI_STORE_F32, bn=64)
        lib.dm_relu_bwd_colsum(self.dh[-1], None, None, g["fc%d_biases" % (L - 1)], B, H, sp)
        n += 2
        for i in range(L - 1, 0, -1):
            src, K = (self.h[i - 2], H) if i > 1 else (self.x16, 784)
            early = early_sync and self._early_name == "fc%d_weights" % i
            # dW_i[in,H] = src^T (MN-major) * dh_i (MN-major), K = batch
            if early:
                G.gemm_bf16_raw(src, self.dh[i - 1], self._g16_view, K, H, B, K, H, H, True, True, G.EPI_STORE_BF16, bn=self._bn)
                e0, e1 = self._bucket_early
                ev = torch.cuda.Event()
                ev.record(main)
                side = self._side[0]
                side.wait_event(ev)
                be.enqueue_bucket_v2(self.params, self.grads, self._g16, self._inbox, 3 if i > 1 else 1, e0, e1, oa["lr0"],
                                     oa["decay_rate"], oa["decay_steps"], stream=side)
                n += 1
                if i == 1:
                    self._join_early = torch.cuda.Event()
                    self._join_early.record(side)
            else:
                G.gemm_bf16_raw(src, self.dh[i - 1], g["fc%d_weights" % i], K, H, B, K, H, H, True, True,
                                G.EPI_STORE_F32, bn=self._bn)
            n += 1
            if i > 1:
                # dh_{i-1} = (dh_i @ W_i^T) * relu'(h_{i-1});  W_i [in,out]: rows = in (N), K = out contiguous
                G.gemm_bf16_raw(self.dh[i - 1], pb["fc%d_weights" % i], self.dh[i - 2], B, H, H, H, H, H, False, False,
                                G.EPI_STORE_BF16, bn=self._bn)
                if early:
                    # the data-gradient GEMM above was the last reader of this layer's bf16 shadow: the apply may rewrite it
                    ev2 = torch.cuda.Event()
                    ev2.record(main)
                    side = self._side[0]
                    side.wait_event(ev2)
                    be.enqueue_bucket_v2(self.params, self.grads, self._g16, self._inbox, 4, e0, e1, oa["lr0"],
                                         oa["decay_rate"], oa["decay_steps"], stream=side)
                    n += 1
                    self._join_early = torch.cuda.Event()
                    self._join_early.record(side)
                lib.dm_relu_bwd_colsum(self.dh[i - 2], self.h[i - 2], self.dh[i - 2], g["fc%d_biases" % (i - 1)], B, H, sp)
                n += 2
        if self._join_early is not None:
            main.wait_event(self._join_early)
        return n

    def _launch_zero(self) -> int:
        sp, base = stream_ptr(), self.grads.data_ptr()
        for (a, b) in self._zero_ranges:
            self.lib.dm_memset_async(base + 4 * a, 0, 4 * (b - a), sp)
        self.lib.dm_memset_async(self.d_loss_acc, 0, 8, sp)
        return 0

    def _launch_step(self, slot: int, with_sync: bool) -> None:
        B = self.batch_size
        n = 0
        if self._stamp:
            # cdf telemetry: the start of the step's compute (read_timing); the aggregation kernel stamps its arrival
            self.backend.enqueue_stamp_start()
            n += 1
        images = self.images[slot]
        if self._aug is not None:
            images = self._launch_augment(slot)     # dm_f32_to_bf16 reads the augmented batch
            n += 1
        own = bool(self._local) or self._gossip          # local / gossip SGD: an iteration end without an iteration begin
        interval = with_sync and (getattr(self, "_interval", False) or self._async or own)   # own iteration end
        if interval and not own:
            self._enqueue_iteration_begin()
            n += 3 if self._ssp >= 0 else 2       # the staleness bound's wait before the pull
        bucketed = with_sync and self._bucket_v2 and not interval
        n += self._launch_zero()
        n += self._forward(images, self.labels[slot], B, True)
        n += self._backward(B, early_sync=bucketed)
        if bucketed:
            if self._straggler is not None:
                self.backend.enqueue_straggler(self._straggler)
                n += 1
            oa = self._opt_args
            e0, e1 = self._bucket_early
            self.backend.enqueue_bucket_v2(self.params, self.grads, self._g16, self._inbox, 2, e0, e1, oa["lr0"],
                                           oa["decay_rate"], oa["decay_steps"])
            n += 1
        elif with_sync:
            if self._straggler is not None:
                self.backend.enqueue_straggler(self._straggler)
                n += 1
            if interval:
                self._enqueue_iteration_end()
                # local SGD: the update, the round's four; gossip SGD: the half step, the barrier, the mix
                n += 5 if self._local else 3 if self._gossip else (2 + (self._ssp >= 0)) if self._async else 4
            else:
                self.backend.enqueue(self.params, self.grads, **self._opt_args)
                n += 1
        self.h_loss_bufs[slot].copy_(self.d_loss_acc, non_blocking=True)     # result read-back is part of the step
        if with_sync and self._ema is not None:
            self._launch_moving_average()
            n += 1
        self.launches_per_step = n

    def _eval_forward(self, images: torch.Tensor, labels: torch.Tensor, B: int) -> None:
        self.d_loss_acc.zero_()
        self._forward(images, labels, B, False)


def make_cuda_engine(flags, ctx, backend) -> ComputeEngine:
    if not isinstance(backend, FusedBackend):
        raise RuntimeError("the sm_90a engine needs the fused backend")
    if flags.model == "lenet":
        return CudaLeNetEngine(flags.batch_size, backend, seed=flags.seed, rank=ctx.rank,
                               keep_prob=flags.dropout_keep_prob, use_graph=flags.use_cuda_graph)
    return CudaMlpEngine(flags.model, flags.batch_size, backend, hidden=flags.mlp_hidden, seed=flags.seed,
                         rank=ctx.rank, use_graph=flags.use_cuda_graph)


def make_cuda_eval_engine(flags, device: torch.device) -> ComputeEngine:
    from .parallel.context import ReplicaContext
    ctx = ReplicaContext(0, 1, device.index or 0, device, "none")
    backend = FusedBackend(ctx)
    if flags.model == "lenet":
        return CudaLeNetEngine(1000, backend, seed=flags.seed, keep_prob=flags.dropout_keep_prob, use_graph=False)
    return CudaMlpEngine(flags.model, 1000, backend, hidden=flags.mlp_hidden, seed=flags.seed, use_graph=False)
