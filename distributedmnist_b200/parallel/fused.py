"""FusedBackend: gradient aggregation by the single sm_90a kernel of ``csrc/fused_sync.cu``.

The product path for SURVEY §2.5 X1-X8: the parameter arena, the gradient arena and a
control block live in symmetric memory; one kernel per step publishes arrival, obtains
the commit mask (all-to-all flags for K == N, chief-owned bitmap + CAS for K < N), sums
the contributors' gradients straight out of peer HBM over NVLink, scales by
``lr / popcount(mask)``, applies SGD on its shard and pushes the new weights into every
rank's arena, then refreshes the local bf16 shadow used by the tensor-core kernels.
No NCCL collective and no separate elementwise kernel is launched.

Two ways to drive it:

* ``sync_step`` -- eager, host-visible result (tests, the reference-style training loop);
* ``enqueue`` -- stream-ordered launch with the LR schedule evaluated on the device from
  the device-resident step counter, so the whole training step replays as a CUDA graph
  with no per-step host input.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional

import numpy as np
import torch

from ..ops.lib import load, require_hopper, stream_ptr
from . import straggler
from .backends import Backend, StepInfo
from .context import ReplicaContext
from .symm_mem import SymmetricBuffer, allocate_symmetric

SSP_LINES = 8                  # clock-board lines, one per possible replica (SYNC_MAX_RANKS in csrc/fused_sync.cuh)


class FusedBackend(Backend):
    name = "fused"
    _STATUS = ("epoch", "error", "accepted_steps", "dropped_steps", "last_mask", "last_count", "last_late")

    def __init__(self, ctx: ReplicaContext, ctas: int = 0, timeout_ms: float = 30000.0, use_nvls: Optional[bool] = None,
                 debug_sync: bool = False):
        super().__init__(ctx)
        assert ctx.on_gpu, "FusedBackend needs a GPU"
        self.lib = load()
        require_hopper(ctx.device)
        self.lib.dm_set_device(ctx.device.index or 0)
        # programmatic dependent launch between the kernels of a step (DMNIST_PDL=0 disables)
        self.lib.dm_set_pdl(0 if os.environ.get("DMNIST_PDL", "1") == "0" else 1)
        self.ctas = ctas or int(os.environ.get("DMNIST_SYNC_CTAS", "0")) or int(self.lib.dm_num_sms())
        # NVLS (in-switch reduction + multicast store) for the arenas when the fabric offers it; DMNIST_NVLS=0 -> P2P only
        #   DMNIST_NVLS unset: allocate multicast-capable arenas, use multimem from 4 replicas up (at 2 the peer path
        #   moves fewer bytes per replica); =1 always; =0 never (CUDA-IPC arenas)
        #   (--use_nvls=false forces the P2P kernels and CUDA-IPC arenas, like DMNIST_NVLS=0)
        nv = os.environ.get("DMNIST_NVLS", "") if use_nvls is None else ("1" if use_nvls else "0")
        self.want_nvls = nv != "0"
        self.use_nvls = nv == "1" or (nv == "" and ctx.world_size >= 4)
        self.timeout_ms = timeout_ms
        self._buffers: List[SymmetricBuffer] = []
        self._by_ptr: Dict[int, SymmetricBuffer] = {}
        nbytes = int(self.lib.dm_sync_ctrl_bytes())
        self.ctrl = SymmetricBuffer(nbytes, ctx.rank, ctx.world_size, ctx.device)
        self._ctrl_bytes = self.ctrl.view(torch.uint8)
        self._off = {f: int(self.lib.dm_sync_ctrl_offset(f.encode())) for f in
                     ("epoch", "error", "accepted_steps", "dropped_steps", "last_mask", "last_count", "last_late",
                      "global_step", "t_arrive", "t_start", "cta_counter", "t_phase", "t_phase_e", "arrive", "done",
                      "arrive_e", "done_e", "commit_local", "bitmap", "commit", "last_in_mask", "decided_tag",
                      "decided_mask", "decided_late", "decided_target", "cta_counter_e", "cta_counter2", "status_seq",
                      "host_mirror", "iv_state", "iv_busy", "iv_deadline", "iv_ticks_committed", "decider_claim")}
        assert all(v >= 0 for v in self._off.values()), self._off
        # the host-readable status words (epoch .. last_late) sit next to each other: ONE device->host copy per query
        self._status_lo = min(self._off[f] for f in self._STATUS)
        self._status_hi = max(self._off[f] for f in self._STATUS) + 4
        self.debug_sync = debug_sync or os.environ.get("DMNIST_DEBUG_SYNC", "0") == "1"
        self.late_ll = os.environ.get("DMNIST_LATE_LL", "1") != "0"     # LL lines (data + tags in one store) for the late bucket
        self.late_bf16 = os.environ.get("DMNIST_LATE_BF16", "1") != "0"  # ... carrying bf16 gradients (half the bytes)
        # host mirror of the status words: the kernel that closes a step stores them into page-locked host memory itself
        self._mirror = torch.zeros(4 * 8, dtype=torch.int32).pin_memory()
        self.lib.dm_sync_set_host_mirror(self.ctrl.local_ptr, self._mirror)
        self._mirror_np = self._mirror.numpy().view("<u4")
        self.shadow: Optional[torch.Tensor] = None     # bf16 copy of the parameter arena
        self.drop_keep = 0.0
        self.drop_seed = 0
        self.interval_ns: Optional[int] = None     # the interval clock's period, once armed (interval_arm)
        self.lr_schedule_armed = False             # the control block evaluates a warmup / cosine (set_lr_schedule)
        self._ssp_board: Optional[SymmetricBuffer] = None   # stale synchronous parallel: this replica's clock board
        self._gossip_send: Optional[SymmetricBuffer] = None  # gossip SGD: this replica's two send buffers

    # ---- memory ---------------------------------------------------------------------------
    def allocate(self, numel: int) -> torch.Tensor:
        buf = allocate_symmetric(numel * 4, self.ctx.rank, self.ctx.world_size, self.ctx.device, self.want_nvls)
        self._buffers.append(buf)
        t = buf.view(torch.float32, 0, numel)
        self._by_ptr[t.data_ptr()] = buf
        return t

    def allocate_buffer(self, nbytes: int):
        """Raw symmetric allocation (peer-mapped, NVLS-multicast-mapped when available): the bf16 gradient buffer and the
        late-bucket inbox of the bucketed aggregation.  Collective: every rank calls it in the same order."""
        buf = allocate_symmetric(int(nbytes), self.ctx.rank, self.ctx.world_size, self.ctx.device, self.want_nvls)
        self._buffers.append(buf)
        return buf

    def attach_shadow(self, params: torch.Tensor) -> torch.Tensor:
        """Create the local bf16 shadow arena of ``params`` and fill it."""
        self.shadow = torch.empty(params.numel(), dtype=torch.bfloat16, device=params.device)
        self.refresh_shadow(params)
        return self.shadow

    def refresh_shadow(self, params: torch.Tensor) -> None:
        if self.shadow is not None:
            self.lib.dm_f32_to_bf16(params, self.shadow, params.numel(), stream_ptr())

    # ---- control-block access ---------------------------------------------------------------
    def _read_u32(self, field: str, index: int = 0) -> int:
        off = self._off[field] + 4 * index
        return int(self._ctrl_bytes[off:off + 4].view(torch.int32).item()) & 0xFFFFFFFF

    def _write_u32(self, field: str, value: int) -> None:
        off = self._off[field]
        self._ctrl_bytes[off:off + 4].view(torch.int32).fill_(value if value < 2 ** 31 else value - 2 ** 32)

    @property
    def device_epoch(self) -> int:
        return self._read_u32("epoch")

    def set_global_step(self, step: int) -> None:
        """Checkpoint restore: every rank starts from ``step`` (also the chief's commit counter)."""
        self._write_u32("epoch", step)
        self._write_u32("global_step", step)
        self._write_u32("decider_claim", step)
        torch.cuda.synchronize()
        self.barrier()

    def set_lr_schedule(self, warmup_steps: int, warmup_start: float, cosine_steps: int, alpha: float) -> None:
        """Arm this replica's control block with the learning-rate schedule's warmup and cosine decay (``cta_scale`` in
        csrc/fused_sync.cuh): every aggregation kernel then evaluates them at the step it updates.  Not collective: each
        replica arms its own block.  ``warmup_steps = cosine_steps = 0`` disarms it."""
        self.lib.dm_sync_set_lr_schedule(self.ctrl.local_ptr, int(warmup_steps), float(warmup_start), int(cosine_steps),
                                         float(alpha))
        self.lr_schedule_armed = int(warmup_steps) > 0 or int(cosine_steps) > 0

    def _refuse_host_rate(self, what: str) -> None:
        if self.lr_schedule_armed:
            raise RuntimeError("FusedBackend.%s passes a learning rate the host evaluated, but the control block has a "
                               "learning-rate schedule armed that the kernel would apply on top of it" % what)

    def read_status(self) -> Dict[str, int]:
        """epoch / error / accepted / dropped / last_mask / last_count / last_late with ONE device->host copy (synchronises
        the current stream)."""
        raw = self._ctrl_bytes[self._status_lo:self._status_hi].cpu().numpy().view("<u4")
        return {f: int(raw[(self._off[f] - self._status_lo) // 4]) for f in self._STATUS}

    @property
    def status_seq(self) -> int:
        """Number of steps closed on the device so far (device read)."""
        return self._read_u32("status_seq")

    def mirror_info(self, seq: int, check: bool = False) -> StepInfo:
        """StepInfo of the ``seq``-th closed step (1-based) from the host mirror -- valid once that step's completion event
        has been waited for; no device read.  Falls back to a device read if the slot was already overwritten (the host
        fell more than three steps behind) or the mirror is not in use."""
        m = self._mirror_np[8 * ((seq - 1) & 3):8 * ((seq - 1) & 3) + 8]
        if int(m[7]) != seq:
            return self.last_step_info(check=check)
        st = dict(zip(self._STATUS, (int(x) for x in m[:7])))
        if check:
            self.check_error(st)
        late = st["last_late"]
        return StepInfo(global_step=st["epoch"], accepted=not late, mask=st["last_mask"], count=st["last_count"],
                        stale=bool(late))

    def check_error(self, status: Optional[Dict[str, int]] = None) -> None:
        e = (status or self.read_status())["error"]
        if e:
            if self.debug_sync:
                import sys
                self.debug_dump(sys.stderr)
            raise RuntimeError("fused sync watchdog fired on rank %d: %s timeout (DMNIST_DEBUG_SYNC=1 / --debug_sync dumps "
                               "the control block)" % (self.ctx.rank, {1: "arrival", 2: "push-complete", 3: "staleness-bound"}.get(e, str(e))))

    def debug_dump(self, out=None) -> str:
        """The accumulator / token-queue state of the reference's debug Print ops (…modified.py:230-234,383-387), here: every
        handshake word of this rank's control block -- which peers have arrived / finished for which step, the chief's
        arrival bitmap and commit ring, the local decision.  Printed when a watchdog fires under ``--debug_sync``."""
        n = self.ctx.world_size
        raw = self._ctrl_bytes.cpu().numpy()
        u32 = lambda off: int(raw[off:off + 4].view("<u4")[0])           # noqa: E731
        u64 = lambda off: int(raw[off:off + 8].view("<u8")[0])           # noqa: E731
        lines = ["[sync-debug rank %d/%d] epoch=%d error=%d accepted=%d dropped=%d last(mask=%#x count=%d late=%d) global_step=%d"
                 % (self.ctx.rank, n, u32(self._off["epoch"]), u32(self._off["error"]), u32(self._off["accepted_steps"]),
                    u32(self._off["dropped_steps"]), u32(self._off["last_mask"]), u32(self._off["last_count"]),
                    u32(self._off["last_late"]), u32(self._off["global_step"]))]
        for f in ("arrive", "done", "arrive_e", "done_e"):
            lines.append("  %-9s per peer (value = step+1): %s" % (f, [u32(self._off[f] + 128 * q) for q in range(n)]))
        lines.append("  decided: tag=%d mask=%#x late=%d target=%d   cta counters: %d / %d / %d"
                     % (u32(self._off["decided_tag"]), u32(self._off["decided_mask"]), u32(self._off["decided_late"]),
                        u32(self._off["decided_target"]), u32(self._off["cta_counter"]), u32(self._off["cta_counter_e"]),
                        u32(self._off["cta_counter2"])))
        ep = u32(self._off["epoch"])
        slots = sorted({(ep + d) % 64 for d in (-2, -1, 0, 1)})
        lines.append("  commit_local[slot]=(step+1, mask): %s"
                     % {sl: (u64(self._off["commit_local"] + 8 * sl) >> 32, hex(u64(self._off["commit_local"] + 8 * sl) & 0xffffffff))
                        for sl in slots})
        if self.ctx.rank == 0:
            lines.append("  chief bitmap[slot]: %s   commit[slot]: %s   last_in_mask: %s"
                         % ({sl: hex(u32(self._off["bitmap"] + 4 * sl)) for sl in slots},
                            {sl: (u64(self._off["commit"] + 8 * sl) >> 32, hex(u64(self._off["commit"] + 8 * sl) & 0xffffffff)) for sl in slots},
                            [u32(self._off["last_in_mask"] + 4 * q) for q in range(n)]))
        txt = "\n".join(lines)
        if out is not None:
            print(txt, file=out, flush=True)
        return txt

    def read_phases(self):
        """%globaltimer stamps of the last launch: start, decided, reduced, pushed, landed, end (ns, relative)."""
        t = self._ctrl_bytes[self._off["t_phase"]:self._off["t_phase"] + 48].view(torch.int64).cpu().tolist()
        return [x - t[0] for x in t]

    def read_phases_early(self):
        """Early-bucket kernel of the last step: start, arrived, reduced (CTA 0), all pushes out, all shards landed,
        applied (CTA 0) (ns, relative)."""
        t = self._ctrl_bytes[self._off["t_phase_e"]:self._off["t_phase_e"] + 48].view(torch.int64).cpu().tolist()
        return [x - t[0] for x in t]

    def read_timing(self, first_step: int, last_step: int):
        """(start_ns, arrive_ns) %globaltimer stamps of local steps [first, last] (cdf telemetry)."""
        ring = 1024
        ta = self._ctrl_bytes[self._off["t_arrive"]:self._off["t_arrive"] + 8 * ring].view(torch.int64).cpu()
        ts = self._ctrl_bytes[self._off["t_start"]:self._off["t_start"] + 8 * ring].view(torch.int64).cpu()
        return [(int(ts[s % ring]), int(ta[s % ring])) for s in range(first_step, last_step + 1)]

    # ---- launches -------------------------------------------------------------------------------
    def enqueue(self, params: torch.Tensor, grads: torch.Tensor, k: int, lr0: float, decay_rate: float = 1.0,
                decay_steps: int = 1, stream: Optional[torch.cuda.Stream] = None) -> None:
        pb, gb = self._by_ptr[params.data_ptr()], self._by_ptr[grads.data_ptr()]
        self.lib.dm_fused_sync_sgd(
            self.ctrl.ptr_table(), pb.ptr_table(), gb.ptr_table(), self.ctx.rank, self.ctx.world_size, int(k), params.numel(),
            lr0, decay_rate, int(decay_steps), self.drop_keep, self.drop_seed, self.timeout_ms, self.shadow, int(self.ctas),
            stream_ptr(stream), *self._mc_ptrs(pb, gb))

    def _mc_ptrs(self, pb, gb):
        on = self.use_nvls and pb.multicast_ptr and gb.multicast_ptr
        return gb.multicast_ptr if on else 0, pb.multicast_ptr if on else 0

    def enqueue_bucket(self, params: torch.Tensor, grads: torch.Tensor, phase: int, begin: int, end: int,
                       early_begin: int, early_end: int, lr0: float, decay_rate: float = 1.0, decay_steps: int = 1,
                       ctas: int = 0, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Bucketed aggregation (K == N, world_size > 1): ``phase`` 1 = early bucket ``[begin, end)`` (floats) on a few
        CTAs next to the remaining backward kernels, 2 = late bucket + completion of the step (csrc/fused_sync.cu)."""
        pb, gb = self._by_ptr[params.data_ptr()], self._by_ptr[grads.data_ptr()]
        self.lib.dm_fused_sync_bucket(
            self.ctrl.ptr_table(), pb.ptr_table(), gb.ptr_table(), self.ctx.rank, self.ctx.world_size, int(phase), begin, end,
            early_begin, early_end, lr0, decay_rate, int(decay_steps), self.timeout_ms, self.shadow, int(ctas),
            stream_ptr(stream), *self._mc_ptrs(pb, gb))

    def enqueue_bucket_v2(self, params: torch.Tensor, grads: torch.Tensor, g16, inbox, phase: int, fc1_begin: int,
                          fc1_end: int, lr0: float, decay_rate: float = 1.0, decay_steps: int = 1, ctas: int = 0,
                          stream: Optional[torch.cuda.Stream] = None) -> None:
        """Bucketed aggregation, bf16 wire (csrc/fused_bucket.cu).  ``phase`` 1: reduce the bf16 fc1 gradient buffer ``g16``
        in place over NVLink (NVLS or P2P) and apply SGD to the local fp32 fc1 weights -- a side branch of the step graph;
        ``phase`` 2: push the small bucket into every replica's ``inbox``, sum in rank order, SGD, close the step."""
        pb, gb = self._by_ptr[params.data_ptr()], self._by_ptr[grads.data_ptr()]
        on = self.use_nvls and self.ctx.world_size > 1
        mc_g16 = g16.multicast_ptr if on else 0
        mc_inbox = inbox.multicast_ptr if (on and inbox is not None) else 0
        self.lib.dm_bucket_sync(
            self.ctrl.ptr_table(), pb.ptr_table(), gb.ptr_table(), g16.ptr_table(),
            inbox.ptr_table() if inbox is not None else None, self.ctx.rank, self.ctx.world_size, int(phase), fc1_begin,
            fc1_end, params.numel(), lr0, decay_rate, int(decay_steps), self.timeout_ms, self.shadow, int(ctas),
            stream_ptr(stream), mc_g16, mc_inbox, int(self.late_ll), int(self.late_bf16))

    # ---- device-side interval mode (mode C, csrc/fused_interval.cu) ----------------------------------------------------------
    def interval_arm(self, interval_ms: float) -> None:
        """Start the interval clock on this replica (reference ``start_interval_updates``): first tick due in ``interval_ms``."""
        self.barrier()                       # replicas start their clocks together (each uses its own %globaltimer afterwards)
        self.interval_ns = int(float(interval_ms) * 1e6)      # what the device holds: the kernel truncates the same way
        self.lib.dm_interval_arm(self.ctrl.local_ptr, interval_ms, stream_ptr())
        torch.cuda.synchronize()
        self.barrier()

    def enqueue_interval_begin(self, params: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Start of an interval-mode iteration: adopt weights a committer has pushed (step counter, bf16 shadow)."""
        self.lib.dm_interval_begin(self.ctrl.local_ptr, params, self.shadow, params.numel(), stream_ptr(stream))

    def enqueue_interval_end(self, params: torch.Tensor, grads: torch.Tensor, acc: torch.Tensor, lr0: float,
                             decay_rate: float = 1.0, decay_steps: int = 1,
                             stream: Optional[torch.cuda.Stream] = None) -> None:
        """End of an interval-mode iteration: accumulate the gradient locally; after the tick's deadline try to commit the
        tick (mean of whatever every replica has accumulated) -- never blocks on another replica's progress."""
        pb, gb, ab = self._by_ptr[params.data_ptr()], self._by_ptr[grads.data_ptr()], self._by_ptr[acc.data_ptr()]
        mc = pb.multicast_ptr if (self.use_nvls and pb.multicast_ptr) else 0
        self.lib.dm_interval_end(self.ctrl.ptr_table(), pb.ptr_table(), gb.ptr_table(), ab.ptr_table(), self.ctx.rank,
                                 self.ctx.world_size, params.numel(), lr0, decay_rate, int(decay_steps), self.timeout_ms,
                                 int(self.ctas), stream_ptr(stream), mc)

    # ---- K > N gradients per update (count trigger, csrc/fused_interval.cu with COUNT) ---------------------------------------
    def kgtn_arm(self) -> None:
        """Start a fresh accumulation on this replica at its current global step (collective: every rank calls it)."""
        self.interval_arm(0.0)

    def enqueue_kgtn_begin(self, params: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Start of a K > N iteration: adopt weights a committer has pushed; gradients accumulated for the step after its
        contributors were frozen are counted as dropped."""
        self.lib.dm_kgtn_begin(self.ctrl.local_ptr, self.ctx.rank, params, self.shadow, params.numel(), stream_ptr(stream))

    def enqueue_kgtn_end(self, params: torch.Tensor, grads: torch.Tensor, acc: torch.Tensor, k: int, lr0: float,
                         decay_rate: float = 1.0, decay_steps: int = 1, stream: Optional[torch.cuda.Stream] = None) -> None:
        """End of a K > N iteration: accumulate the gradient locally; once ``k`` gradients computed on the current step's
        weights are accumulated across the replicas, the first replica to see it commits their mean."""
        pb, gb, ab = self._by_ptr[params.data_ptr()], self._by_ptr[grads.data_ptr()], self._by_ptr[acc.data_ptr()]
        nv = self.use_nvls and bool(pb.multicast_ptr) and bool(ab.multicast_ptr)
        self.lib.dm_kgtn_end(self.ctrl.ptr_table(), pb.ptr_table(), gb.ptr_table(), ab.ptr_table(), self.ctx.rank,
                             self.ctx.world_size, int(k), params.numel(), lr0, decay_rate, int(decay_steps), self.timeout_ms,
                             int(self.ctas), stream_ptr(stream), pb.multicast_ptr if nv else 0, ab.multicast_ptr if nv else 0)

    # ---- asynchronous SGD (csrc/fused_async.cu) ------------------------------------------------------------------------------
    def async_arm(self, master: torch.Tensor, params: torch.Tensor, stats: torch.Tensor,
                  ssp_stats: Optional[torch.Tensor] = None) -> None:
        """Start asynchronous SGD from the current weights and global step: the master copy ``master`` (an :meth:`allocate`
        arena) := ``params``, the staleness statistics ``stats`` (``dm_async_stats_bytes()`` bytes of device memory) zeroed.
        The chief's update counter is the ``global_step`` word that :meth:`set_global_step` sets.  Collective: every rank
        calls it, and no replica's first update can land before every copy holds the starting weights.  ``ssp_stats``
        (from :meth:`ssp_arm`): the staleness bound is armed too -- the clock board and the bound's statistics, with the
        clock, are zeroed, and no replica's first wait can read a clock of an earlier run."""
        torch.cuda.synchronize()
        self.barrier()
        master.copy_(params)
        stats.zero_()
        if ssp_stats is not None:
            self._ssp_board.view(torch.int32, 0, 32 * SSP_LINES).zero_()
            ssp_stats.zero_()
        torch.cuda.synchronize()
        self.barrier()

    def enqueue_async_begin(self, master: torch.Tensor, params: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Start of an asynchronous iteration: read the update counter r, pull my master copy into ``params`` and the bf16
        shadow."""
        self.lib.dm_async_begin(self.ctrl.ptr_table(), self.ctx.rank, master, params, self.shadow, params.numel(),
                                int(self.ctas), stream_ptr(stream))

    def enqueue_async_end(self, master: torch.Tensor, grads: torch.Tensor, stats: torch.Tensor, lr0: float,
                          decay_rate: float = 1.0, decay_steps: int = 1, stream: Optional[torch.cuda.Stream] = None) -> None:
        """End of an asynchronous iteration: take the ticket s of the update, add ``-fl(lr(s) * grads)`` to every replica's
        master copy (in-switch under the NVLS policy, else one reduction per copy).  Never waits for another replica."""
        mb = self._by_ptr[master.data_ptr()]
        mc = mb.multicast_ptr if (self.use_nvls and mb.multicast_ptr) else 0
        self.lib.dm_async_end(self.ctrl.ptr_table(), mb.ptr_table(), grads, stats, self.ctx.rank, self.ctx.world_size,
                              master.numel(), lr0, decay_rate, int(decay_steps), int(self.ctas), stream_ptr(stream), mc)

    @staticmethod
    def async_stats(stats: torch.Tensor) -> Dict:
        """Decode the staleness statistics (synchronises the device): ``updates``, ``hist`` (64 buckets, the last one
        counting tau >= 63), ``tau_sum``, ``tau_max`` and ``pairs``, the (r, s) of the last min(updates, 1024) updates, oldest
        first."""
        torch.cuda.synchronize()
        raw = stats.cpu().numpy()
        hist = raw[:256].view("<u4").astype(np.int64)
        updates = int(raw[268:272].view("<u4")[0])
        ring = raw[272:].view("<u4").reshape(-1, 2).astype(np.int64)
        j = np.arange(max(0, updates - len(ring)), updates)
        return dict(updates=updates, hist=hist.tolist(), tau_sum=int(raw[256:264].view("<u8")[0]),
                    tau_max=int(raw[264:268].view("<u4")[0]), pairs=ring[j % len(ring)])

    # ---- stale synchronous parallel (csrc/fused_async.cu) ----------------------------------------------------------------
    def ssp_arm(self) -> torch.Tensor:
        """Prepare the staleness bound: this replica's clock board (one 128-byte line per peer, symmetric, allocated on
        first use -- collective, like :meth:`allocate`) and a new statistics block (``dm_ssp_stats_bytes()`` bytes of
        device memory, which also holds the clock), returned.  :meth:`async_arm` with ``ssp_stats`` zeroes both."""
        if self._ssp_board is None:
            self._ssp_board = self.allocate_buffer(128 * SSP_LINES)
        return torch.zeros(int(self.lib.dm_ssp_stats_bytes()), dtype=torch.uint8, device=self.ctx.device)

    def enqueue_ssp_wait(self, stats: torch.Tensor, s: int, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Before :meth:`enqueue_async_begin`: wait until every peer that has not retired has applied at least c - ``s``
        updates, c = this replica's clock.  A wait longer than the watchdog sets the error word (3)."""
        self.lib.dm_ssp_wait(self._ssp_board.local_ptr, self.ctrl.local_ptr, stats, self.ctx.rank, self.ctx.world_size,
                             int(s), self.timeout_ms, stream_ptr(stream))

    def enqueue_ssp_publish(self, stats: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> None:
        """After :meth:`enqueue_async_end`: this replica's clock + 1, released into every replica's board."""
        self.lib.dm_ssp_publish(self._ssp_board.ptr_table(), stats, self.ctx.rank, self.ctx.world_size, 0,
                                stream_ptr(stream))

    def enqueue_ssp_retire(self, stats: torch.Tensor, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Once this replica's last iteration is enqueued: publish the retired clock, so no peer waits for it again."""
        self.lib.dm_ssp_publish(self._ssp_board.ptr_table(), stats, self.ctx.rank, self.ctx.world_size, 1,
                                stream_ptr(stream))

    @staticmethod
    def ssp_stats(stats: torch.Tensor) -> Dict:
        """Decode the bound's statistics (synchronises the device): ``clock`` (updates applied), ``waits``,
        ``wait_total_ns``, ``wait_max_ns``, ``lead_max`` and ``pairs``, the (c, min clock of the non-retired peers --
        0xFFFFFFFF: none) of the last min(clock + 1, 1024) pulls, oldest first."""
        torch.cuda.synchronize()
        raw = stats.cpu().numpy()
        w = raw[:16].view("<u4")
        ring = raw[32:].view("<u4").reshape(-1, 2).astype(np.int64)
        clock = int(w[0])
        j = np.arange(max(0, clock + 1 - len(ring)), clock + 1)
        pairs = ring[j % len(ring)]
        return dict(clock=clock, waits=int(w[1]), lead_max=int(w[2]), wait_total_ns=int(raw[16:24].view("<u8")[0]),
                    wait_max_ns=int(raw[24:32].view("<u8")[0]), pairs=pairs[pairs[:, 0] == j])

    # ---- local SGD (csrc/fused_local.cu) ---------------------------------------------------------------------------------
    def _local_mc(self, params: torch.Tensor) -> int:
        pb = self._by_ptr[params.data_ptr()]
        return pb.multicast_ptr if (self.use_nvls and pb.multicast_ptr and self.ctx.world_size > 1) else 0

    def enqueue_local_step(self, params: torch.Tensor, grads: torch.Tensor, period: int, lr0: float,
                           decay_rate: float = 1.0, decay_steps: int = 1, stream: Optional[torch.cuda.Stream] = None) -> None:
        """The local update of one iteration: ``params -= fp32(lr(s)) * grads`` and the bf16 shadow, s = this replica's
        global step, with the armed schedule.  Never waits for another replica."""
        self.lib.dm_local_apply(self.ctrl.ptr_table(), self.ctx.rank, params, grads, self.shadow, params.numel(),
                                int(period), lr0, decay_rate, int(decay_steps), int(self.ctas), stream_ptr(stream),
                                self._local_mc(params))

    def enqueue_local_average(self, params: torch.Tensor, stats: torch.Tensor, period: int, close: bool = True,
                              stream: Optional[torch.cuda.Stream] = None) -> None:
        """After :meth:`enqueue_local_step` (``close``): the step is closed, and when its global step is a multiple of
        ``period`` every replica's arena and shadow become the mean of all arenas, between two device barriers.  The
        NVLS policy picks the in-switch reduction, else the rank-ordered peer loads.  ``close=False, period=1``: one
        unconditional average that closes no step (the end of a run).  ``stats``: ``dm_local_stats_bytes()`` bytes."""
        pb = self._by_ptr[params.data_ptr()]
        self.lib.dm_local_average(self.ctrl.ptr_table(), pb.ptr_table(), self.shadow, stats, self.ctx.rank,
                                  self.ctx.world_size, params.numel(), int(period), int(bool(close)), self.timeout_ms,
                                  int(self.ctas), stream_ptr(stream), self._local_mc(params))

    @staticmethod
    def local_stats(stats: torch.Tensor) -> Dict:
        """Decode the averaging statistics (synchronises the device): ``rounds``, ``wait_total_ns``, ``wait_max_ns`` (the
        %globaltimer time of a round's two barriers, summed and at most)."""
        torch.cuda.synchronize()
        raw = stats.cpu().numpy()
        return dict(rounds=int(raw[0:4].view("<u4")[0]), wait_total_ns=int(raw[8:16].view("<u8")[0]),
                    wait_max_ns=int(raw[16:24].view("<u8")[0]))

    # ---- gossip SGD (csrc/fused_gossip.cu) ---------------------------------------------------------------------------------
    def gossip_arm(self, numel: int) -> torch.Tensor:
        """This replica's two send buffers of ``numel`` fp32 each (one symmetric allocation, on first use -- collective,
        like :meth:`allocate`) and a new, zeroed statistics block (``dm_gossip_stats_bytes()`` bytes), returned."""
        if self._gossip_send is None:
            self._gossip_send = self.allocate_buffer(2 * 4 * int(numel))
        return torch.zeros(int(self.lib.dm_gossip_stats_bytes()), dtype=torch.uint8, device=self.ctx.device)

    def enqueue_gossip_step(self, params: torch.Tensor, grads: torch.Tensor, stats: torch.Tensor, lr0: float,
                            decay_rate: float = 1.0, decay_steps: int = 1,
                            stream: Optional[torch.cuda.Stream] = None) -> None:
        """One gossip iteration after the gradient (after :meth:`gossip_arm`): the half step ``params - fp32(lr(s)) *
        grads`` into this replica's send buffer s % 2, s = its global step, with the armed schedule; the step is closed
        and the barrier with the two ring neighbours taken; then ``params`` and the shadow := the mean of the half steps
        of the neighbourhood, summed in rank order over the peer path."""
        self.lib.dm_gossip_apply(self.ctrl.ptr_table(), self.ctx.rank, params, grads, self._gossip_send.local_ptr,
                                 params.numel(), lr0, decay_rate, int(decay_steps), int(self.ctas), stream_ptr(stream))
        self.lib.dm_gossip_exchange(self.ctrl.ptr_table(), self._gossip_send.ptr_table(), params, self.shadow, stats,
                                    self.ctx.rank, self.ctx.world_size, params.numel(), self.timeout_ms, int(self.ctas),
                                    stream_ptr(stream))

    @staticmethod
    def gossip_stats(stats: torch.Tensor) -> Dict:
        """Decode the gossip statistics (synchronises the device): ``iterations``, ``waits`` (barriers at whose first
        poll a neighbour had not arrived), ``wait_total_ns``, ``wait_max_ns`` (%globaltimer time in the barriers) and
        ``t_pass``, the ring of the %globaltimer stamps at which the barrier of iteration s was passed, at s % 1024."""
        torch.cuda.synchronize()
        raw = stats.cpu().numpy()
        return dict(iterations=int(raw[0:4].view("<u4")[0]), waits=int(raw[4:8].view("<u4")[0]),
                    wait_total_ns=int(raw[8:16].view("<u8")[0]), wait_max_ns=int(raw[16:24].view("<u8")[0]),
                    t_pass=raw[32:].view("<u8").copy())

    @property
    def nvls_active(self) -> bool:
        return self.use_nvls and bool(self._buffers) and all(b.multicast_ptr for b in self._buffers[:2])

    def enqueue_straggler_delay(self, prob: float, usec: float, seed: int = 12345,
                                stream: Optional[torch.cuda.Stream] = None) -> None:
        self.lib.dm_straggler_delay(self.ctrl.local_ptr, prob, int(usec), seed, stream_ptr(stream))

    def arm_straggler(self, spec) -> None:
        """Sampled forms (``rank:exp|lognormal|profile:...``): upload the quantile table and allocate the sampler's state
        block (iteration counter + ring of drawn / spun delays).  Arming the spec that is already armed keeps its counter."""
        if not spec.sampled or getattr(self, "_strag_spec", None) is spec:
            return
        limit = straggler.delay_limit_ns(self.timeout_ms)
        if int(spec.table.max()) > limit:
            raise ValueError("--inject_straggler: the largest delay of %s, %.0f us, exceeds a quarter of this backend's "
                             "watchdog (%.0f us)" % (spec.dist, int(spec.table.max()) / 1e3, limit / 1e3))
        assert spec.table.shape == (straggler.TABLE_POINTS,) and spec.table.dtype == np.uint32
        assert int(self.lib.dm_straggler_state_bytes()) == straggler.STATE_BYTES
        self._strag_table = torch.from_numpy(spec.table.view(np.int32).copy()).to(self.ctx.device)
        self._strag_state = torch.zeros(straggler.STATE_BYTES, dtype=torch.uint8, device=self.ctx.device)
        self._strag_spec = spec

    def enqueue_straggler(self, spec, stream: Optional[torch.cuda.Stream] = None) -> None:
        """The injected delay of one iteration, stream-ordered: the fixed form (``rank:prob:usec``) through
        ``straggler_delay_kernel`` exactly as before, sampled forms through ``straggler_sample_kernel`` (armed first)."""
        if not spec.sampled:
            self.enqueue_straggler_delay(spec.prob, spec.usec, stream=stream)
            return
        if getattr(self, "_strag_spec", None) is not spec:
            raise RuntimeError("enqueue_straggler: arm_straggler(spec) has not been called for this spec")
        self.lib.dm_straggler_sample(self._strag_state, self._strag_table, spec.seed_mix, stream_ptr(stream))

    def straggler_samples(self):
        """``(j, drawn_ns, spun_ns)`` of the sampled iterations still in the device ring (the last 1024), oldest first;
        synchronises the device."""
        torch.cuda.synchronize()
        raw = self._strag_state.cpu().numpy()
        n = int(raw[:4].view("<u4")[0])
        drawn = raw[16:16 + 4 * straggler.RING].view("<u4")
        spun = raw[16 + 4 * straggler.RING:].view("<u8")
        j = np.arange(max(0, n - straggler.RING), n, dtype=np.int64)
        return j, drawn[j % straggler.RING].copy(), spun[j % straggler.RING].copy()

    def device_barrier(self, stream: Optional[torch.cuda.Stream] = None) -> None:
        """Stream-ordered barrier over NVLink flags (csrc/fused_sync.cu): every replica's stream passes it within a flag hop of
        the last replica reaching it -- aligns the replicas far tighter than a host-side barrier can."""
        if self.ctx.world_size > 1:
            self.lib.dm_device_barrier(self.ctrl.ptr_table(), self.ctx.rank, self.ctx.world_size,
                                       self.timeout_ms, stream_ptr(stream))

    def enqueue_stamp_arrive(self, stream: Optional[torch.cuda.Stream] = None) -> None:
        """cdf telemetry: "my gradient is complete" on the compute chain, before it joins the exchange branch."""
        self.lib.dm_stamp_arrive(self.ctrl.local_ptr, stream_ptr(stream))

    def enqueue_stamp_start(self, stream: Optional[torch.cuda.Stream] = None) -> None:
        self.lib.dm_stamp_start(self.ctrl.local_ptr, stream_ptr(stream))

    def drop_connect_(self, grads: torch.Tensor, keep_prob: float, step: int) -> None:
        # Applied inside the fused kernel's load stage (per contributor); just arm it.
        self.drop_keep = float(keep_prob)
        self.drop_seed = 0x2545F491

    def last_step_info(self, check: bool = False) -> StepInfo:
        st = self.read_status()
        if check:
            self.check_error(st)
        late = st["last_late"]
        return StepInfo(global_step=st["epoch"], accepted=not late, mask=st["last_mask"], count=st["last_count"],
                        stale=bool(late))

    def sync_step(self, params, grads, lr, local_step, k, delay_s: float = 0.0) -> StepInfo:
        self._refuse_host_rate("sync_step")
        if delay_s > 0:
            self.enqueue_straggler_delay(1.0, delay_s * 1e6)
        self.enqueue(params, grads, k, lr0=float(lr))
        return self.last_step_info(check=True)   # one device -> host read (synchronises)

    def interval_tick(self, params, acc, count, lr, tick) -> StepInfo:
        """Mode C tick: every rank joins; ranks with an empty accumulator contribute zeros and the
        divisor is the total number of accumulated gradients (mean of whatever arrived)."""
        self._refuse_host_rate("interval_tick")
        counts = self.all_gather_object(int(count))
        total = sum(counts)
        mask = sum(1 << i for i, c in enumerate(counts) if c > 0)
        if total == 0:
            return StepInfo(self.device_epoch, False, 0, 0, applied=False)
        # lr/total instead of lr/popcount: fold the ratio into lr0 (kernel divides by N contributors)
        self.enqueue(params, acc, self.ctx.world_size, lr0=float(lr) * self.ctx.world_size / total)
        info = self.last_step_info()
        self.check_error()
        return StepInfo(info.global_step, count > 0, mask, total)

    def close(self) -> None:
        torch.cuda.synchronize()
        self.barrier()
        for b in self._buffers + [self.ctrl]:
            b.close()
