"""Gradient-aggregation policies: the three synchronisation modes of the reference.

====================  =====================================================  =========================
mode                  reference                                              here
====================  =====================================================  =========================
A  K-of-N (default)   stock ``tf.train.SyncReplicasOptimizer`` selected at   :class:`SyncReplicasOptimizer`
                      src/distributed_train.py:185-188
B  full barrier +     ``TimeoutReplicasOptimizer`` with ``take_grad(N)``,     :class:`TimeoutReplicasOptimizer`
   timing ("cdf")     per-worker token queues, ``_wait_op`` run first         (``mode="cdf"``)
                      (sync_replicas_optimizer_modified.py:198-206,278-279,
                      370-371; distributed_train.py:305-307,344-345)
C  interval           ``take_grad(1)`` from a chief-side timer every          :class:`TimeoutReplicasOptimizer`
                      ``--interval_ms`` (…modified.py:208-215,373)            (``mode="interval"``)
====================  =====================================================  =========================

Optional gradient drop-connect (Bernoulli(p) 0/1 mask on every gradient element
before aggregation, no 1/p rescale, mode A only -- distributed_train.py:194-196,
202-203,414-416) and straggler injection (new; the reference relied on naturally
slow EC2 ``t2`` instances) are applied here, before the backend moves any bytes.
"""
from __future__ import annotations

import dataclasses
import random
import time
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch

from .backends import Backend, StepInfo
from .straggler import delay_limit_ns, parametric_table, profile_table, sample_ns, seed_mix


@dataclass
class StragglerSpec:
    """One replica's injected delay.  ``dist == "fixed"`` (``rank:prob:usec``): ``usec`` with probability ``prob``, decided
    by a hash of the global step.  Otherwise (``exp``, ``lognormal``, ``profile``) a delay drawn every iteration from the
    quantile ``table`` (ns, parallel/straggler.py) with the replica's stream key ``seed_mix``."""
    prob: float
    usec: float
    dist: str = "fixed"
    params: tuple = ()
    table: Optional[np.ndarray] = field(default=None, compare=False, repr=False)
    seed_mix: int = 0

    @property
    def sampled(self) -> bool:
        return self.dist != "fixed"


class StragglerMap(dict):
    """rank -> StragglerSpec; the key ``"*"`` stands for every rank (each draws from its own stream)."""

    def get(self, rank, default=None):
        if rank in self:
            return self[rank]
        return super().get("*", default)


_DISTS = {"exp": ("MEAN_US",), "lognormal": ("MEDIAN_US", "SIGMA"), "profile": ("PATH",)}


def _positive(item: str, name: str, text: str) -> float:
    try:
        v = float(text)
    except ValueError:
        raise ValueError("--inject_straggler %r: %s is not a number: %r" % (item, name, text))
    if not (np.isfinite(v) and v > 0):
        raise ValueError("--inject_straggler %r: %s must be a positive number, got %r" % (item, name, text))
    return v


def parse_straggler_spec(text: str, sync_timeout_ms: Optional[float] = None) -> Dict[int, StragglerSpec]:
    """Comma-separated list of
    ``rank:prob:usec`` (``"3:0.5:2000"`` -> rank 3 sleeps 2000 us with probability .5),
    ``rank:exp:MEAN_US``, ``rank:lognormal:MEDIAN_US:SIGMA`` or ``rank:profile:PATH`` (delays in us, ``.npy`` or text),
    where ``rank`` of the last three may be ``*`` (every replica).  Sampled forms compile to a quantile table whose largest
    point must stay within ``min(sync_timeout_ms / 4, 4 s)``."""
    out = StragglerMap()
    limit = delay_limit_ns(sync_timeout_ms)
    for item in filter(None, (s.strip() for s in (text or "").split(","))):
        head = item.split(":", 2)
        if len(head) == 3 and head[1] in _DISTS:
            rank_txt, dist, rest = head
            if rank_txt.strip() == "*":
                rank = "*"
            else:
                try:
                    rank = int(rank_txt)
                except ValueError:
                    raise ValueError("--inject_straggler %r: rank must be an integer or *, got %r" % (item, rank_txt))
                if rank < 0:
                    raise ValueError("--inject_straggler %r: rank must not be negative" % item)
            if dist == "profile":
                args = (rest,)
                table = profile_table(rest, limit)
            else:
                vals = rest.split(":")
                if len(vals) != len(_DISTS[dist]):
                    raise ValueError("--inject_straggler %r: wants rank:%s:%s" % (item, dist, ":".join(_DISTS[dist])))
                args = tuple(_positive(item, n, v) for n, v in zip(_DISTS[dist], vals))
                table = parametric_table(dist, args, limit)
            spec = StragglerSpec(1.0, 0.0, dist, args, table)
        else:
            parts = item.split(":")
            if len(parts) != 3:
                raise ValueError("--inject_straggler wants rank:prob:usec, rank:exp:MEAN_US, rank:lognormal:MEDIAN_US:SIGMA "
                                 "or rank:profile:PATH, got %r" % item)
            try:
                float(parts[1])
            except ValueError:
                raise ValueError("--inject_straggler %r: unknown distribution %r (known: %s)"
                                 % (item, parts[1], ", ".join(sorted(_DISTS))))
            rank = int(parts[0])
            spec = StragglerSpec(float(parts[1]), float(parts[2]))
        if rank in out or (out and (rank == "*" or "*" in out)):
            raise ValueError("--inject_straggler: rank %s is given twice (* stands for every rank)" % rank)
        out[rank] = spec
    return out


class _AggregatorBase:
    def __init__(self, backend: Backend, lr_schedule: Callable[[int], float], total_num_replicas: int,
                 straggler: Optional[Dict[int, StragglerSpec]] = None, seed: int = 0):
        self.backend = backend
        self.lr_schedule = lr_schedule
        self.total_num_replicas = int(total_num_replicas)
        self.local_step = 0          # global step of the weights my next gradient is computed from (X7)
        self.last_info: Optional[StepInfo] = None
        s = (straggler or {}).get(backend.ctx.rank)
        if s is not None and s.sampled:
            s = dataclasses.replace(s, seed_mix=seed_mix(seed, backend.ctx.rank))     # this replica's own stream
        self._straggler = s
        self._rng = random.Random(seed * 7919 + backend.ctx.rank)
        self._straggler_iter = 0
        self.straggler_delays_ns: List[int] = []     # sampled forms: what _delay_s handed out, one per local iteration
        self.accepted_steps = 0
        self.dropped_steps = 0

    @property
    def global_step(self) -> int:
        return self.local_step

    def _delay_s(self) -> float:
        s = self._straggler
        if s is not None and s.sampled:
            ns = int(sample_ns(s.table, s.seed_mix, self._straggler_iter)[0])
            self._straggler_iter += 1
            self.straggler_delays_ns.append(ns)
            return ns * 1e-9
        if s is not None and self._rng.random() < s.prob:
            return s.usec * 1e-6
        return 0.0

    def _account(self, info: StepInfo) -> StepInfo:
        self.last_info = info
        self.local_step = info.global_step
        if info.applied:
            if info.accepted:
                self.accepted_steps += 1
            else:
                self.dropped_steps += 1
        return info

    # API-shape parity with the reference's optimizer objects; the queue runner /
    # token machinery has no work left to do (SURVEY §2.5 X5, X6, X8).
    def get_chief_queue_runner(self):
        return None

    def get_init_tokens_op(self):
        return None


class SyncReplicasOptimizer(_AggregatorBase):
    """Mode A: synchronous SGD that commits on the first K of N gradients.  K > N: replicas compute several batches per
    update -- each step commits once at least K gradients computed on its weights are accumulated across the replicas, and
    the update is their mean over the number accumulated."""

    def __init__(self, backend: Backend, lr_schedule, replicas_to_aggregate: int, total_num_replicas: int,
                 drop_connect_probability: Optional[float] = None, straggler=None, seed: int = 0):
        super().__init__(backend, lr_schedule, total_num_replicas, straggler, seed)
        if replicas_to_aggregate < 1:
            raise ValueError("replicas_to_aggregate=%d must be >= 1" % replicas_to_aggregate)
        self.replicas_to_aggregate = int(replicas_to_aggregate)
        self.drop_connect_probability = drop_connect_probability
        self._dc_gen: Optional[torch.Generator] = None

    def _drop_connect(self, grads: torch.Tensor) -> torch.Tensor:
        p = self.drop_connect_probability
        if p is None:
            return grads
        if hasattr(self.backend, "drop_connect_"):
            self.backend.drop_connect_(grads, p, self.local_step)   # device-side hash mask
            return grads
        if self._dc_gen is None:
            self._dc_gen = torch.Generator(device="cpu")
            self._dc_gen.manual_seed(1009 * (self.backend.ctx.rank + 1))
        keep = (torch.rand(grads.shape, generator=self._dc_gen) < p).to(grads.dtype).to(grads.device)
        return grads.mul_(keep)

    def apply_gradients(self, params: torch.Tensor, grads: torch.Tensor) -> StepInfo:
        grads = self._drop_connect(grads)
        lr = self.lr_schedule(self.local_step)
        if self.replicas_to_aggregate > self.total_num_replicas:
            info = self.backend.accumulate_step(params, grads, lr, self.local_step, self.replicas_to_aggregate,
                                                delay_s=self._delay_s())
            self.last_info = info
            self.local_step = info.global_step
            self.accepted_steps += info.contributed      # gradients that entered a committed update
            return info
        info = self.backend.sync_step(params, grads, lr, self.local_step, self.replicas_to_aggregate,
                                      delay_s=self._delay_s())
        return self._account(info)


STALENESS_BUCKETS = 64         # staleness histogram: bucket b counts tau = b, the last one tau >= 63


def staleness_report(hist: Sequence[int], tau_sum: int, tau_max: int) -> Dict:
    """Updates applied, the histogram, mean, max and p50 / p99 of the staleness tau = s - r of one replica's updates.  The
    percentiles are read from the histogram: a value of 63 means >= 63."""
    hist = [int(h) for h in hist]
    assert len(hist) == STALENESS_BUCKETS
    n = sum(hist)

    def pct(q: float) -> int:
        need, run = max(1, int(np.ceil(q * n))), 0
        for b, h in enumerate(hist):
            run += h
            if run >= need:
                return b
        return 0
    return dict(updates=n, hist=hist, mean=(float(tau_sum) / n if n else 0.0), max=int(tau_max),
                p50=pct(0.5) if n else 0, p99=pct(0.99) if n else 0)


class AsyncSGDOptimizer(_AggregatorBase):
    """Asynchronous SGD (TF's asynchronous parameter-server training): every replica applies its own gradient as soon as it
    has it, at the learning rate of the global step its update produces, and nothing is averaged, dropped or waited for.
    The GPU path runs it on the device (csrc/fused_async.cu, see ``FusedBackend.enqueue_async_begin``); here, for the torch
    engine, it is implemented for one replica only, where it is plain SGD and every update has staleness 0.

    ``ssp_staleness`` = s >= 0 bounds it (stale synchronous parallel, ``--ssp_staleness``): no replica starts its
    iteration c before every peer that has not retired has applied c - s updates.  -1: unbounded.  One replica never
    waits, so here it changes nothing."""
    mode = "async"

    def __init__(self, backend: Backend, lr_schedule, total_num_replicas: int, straggler=None, seed: int = 0,
                 ssp_staleness: int = -1):
        super().__init__(backend, lr_schedule, total_num_replicas, straggler, seed)
        self.staleness_hist = [0] * STALENESS_BUCKETS
        self.tau_sum = self.tau_max = 0
        self.ssp_staleness = int(ssp_staleness)

    def apply_gradients(self, params: torch.Tensor, grads: torch.Tensor) -> StepInfo:
        if self.backend.ctx.world_size != 1:
            raise ValueError("--async_method with the torch engine is implemented for one replica, not %d"
                             % self.backend.ctx.world_size)
        info = self.backend.sync_step(params, grads, self.lr_schedule(self.local_step), self.local_step, 1,
                                      delay_s=self._delay_s())
        self.staleness_hist[0] += 1          # one replica: the update is made on the weights it was computed from
        return self._account(info)

    def staleness(self) -> Dict:
        return staleness_report(self.staleness_hist, self.tau_sum, self.tau_max)


def ssp_report(s: int, waits: int, wait_total_ns: int, wait_max_ns: int, lead_max: int, updates: int) -> Dict:
    """The staleness bound s of one replica, the iterations that waited for a peer, the time spent waiting, the largest
    clock lead over the slowest non-retired peer seen at a pull, and the updates the replica applied."""
    return dict(s=int(s), waits=int(waits), wait_total_ns=int(wait_total_ns), wait_max_ns=int(wait_max_ns),
                lead_max=int(lead_max), updates=int(updates))


def local_sgd_report(period: int, rounds: int, wait_total_ns: int, wait_max_ns: int) -> Dict:
    """H, the averaging rounds one replica took part in, and the time it spent in their barriers."""
    return dict(period=int(period), rounds=int(rounds), wait_total_s=int(wait_total_ns) * 1e-9,
                wait_max_s=int(wait_max_ns) * 1e-9, wait_mean_s=int(wait_total_ns) * 1e-9 / rounds if rounds else 0.0)


class LocalSGDOptimizer(_AggregatorBase):
    """Local SGD (periodic model averaging): every replica applies its own gradient to its own weights, at the learning
    rate of the global step, and after every ``period``-th global step every replica's weights become the mean of all
    replicas' weights.  The GPU path runs it on the device (csrc/fused_local.cu, see ``FusedBackend.enqueue_local_step``);
    here, for the torch engine, the average is an ``all_reduce`` of the weights over the process group, divided by N."""
    mode = "local"

    def __init__(self, backend: Backend, lr_schedule, total_num_replicas: int, period: int, straggler=None, seed: int = 0):
        super().__init__(backend, lr_schedule, total_num_replicas, straggler, seed)
        if int(period) < 1:
            raise ValueError("local SGD needs an averaging period of at least 1 step, got %d" % period)
        self.period = int(period)
        self.rounds = 0
        self.wait_total_ns = self.wait_max_ns = 0
        self.before_average: Optional[torch.Tensor] = None    # this replica's weights before the newest average

    def apply_gradients(self, params: torch.Tensor, grads: torch.Tensor) -> StepInfo:
        delay = self._delay_s()
        if delay > 0:
            time.sleep(delay)
        params.add_(grads, alpha=-float(self.lr_schedule(self.local_step)))
        step = self.local_step + 1
        if step % self.period == 0:
            self.average(params)
        return self._account(StepInfo(step, True, 1 << self.backend.ctx.rank, 1))

    def average(self, params: torch.Tensor) -> None:
        """Every replica's ``params`` := the mean of all of them (collective).  The time spent in the collective is this
        path's barrier wait."""
        n = self.backend.ctx.world_size
        self.before_average = params.detach().clone()
        if n > 1:
            t0 = time.perf_counter_ns()
            torch.distributed.all_reduce(params, op=torch.distributed.ReduceOp.SUM)
            params.div_(n)
            ns = time.perf_counter_ns() - t0
            self.wait_total_ns += ns
            self.wait_max_ns = max(self.wait_max_ns, ns)
        self.rounds += 1

    def report(self) -> Dict:
        return local_sgd_report(self.period, self.rounds, self.wait_total_ns, self.wait_max_ns)


class TimeoutReplicasOptimizer(_AggregatorBase):
    """Modes B ("cdf": full barrier + per-iteration timing) and C ("interval")."""

    def __init__(self, backend: Backend, lr_schedule, total_num_replicas: int, mode: str = "cdf",
                 interval_ms: int = 1000, straggler=None, seed: int = 0,
                 clock: Callable[[], float] = time.monotonic):
        super().__init__(backend, lr_schedule, total_num_replicas, straggler, seed)
        assert mode in ("cdf", "interval")
        self.mode = mode
        self.interval_s = interval_ms / 1000.0
        self._clock = clock
        self._acc: Optional[torch.Tensor] = None
        self._acc_count = 0
        self._tick = 0
        self._t0: Optional[float] = None
        self.dequeue_times: List[float] = []      # mode B telemetry (host clock)
        self.finish_times: List[float] = []

    # ---- mode B ---------------------------------------------------------------
    def wait_op(self) -> float:
        """Acquire half of the barrier: the reference's per-worker token dequeue
        (``_wait_op``, …modified.py:278-279).  With a commit protocol the token *is*
        the previous step's commit, which ``apply_gradients`` already waited for, so
        this only stamps the time (the event ``worker_dequeued_token`` reports)."""
        t = time.time()
        self.dequeue_times.append(t)
        return t

    def mark_finished(self) -> float:
        t = time.time()
        self.finish_times.append(t)
        return t

    # ---- mode C ---------------------------------------------------------------
    def start_interval_updates(self, t0: Optional[float] = None) -> None:
        """Arm the interval clock (reference ``start_interval_updates``, …modified.py:208-215).

        Deadlines are absolute: tick k fires at ``t0 + (k+1)*interval``.  All replicas
        live on one box and share ``CLOCK_MONOTONIC``, so the chief's t0 (shared at
        start-up) gives every replica the same deadlines without a timer thread."""
        if t0 is None:
            t0 = self.backend.all_gather_object(self._clock())[0]
        self._t0 = t0

    def _deadline(self, tick: int) -> float:
        assert self._t0 is not None, "call start_interval_updates() first"
        return self._t0 + (tick + 1) * self.interval_s

    def apply_gradients(self, params: torch.Tensor, grads: torch.Tensor, worker_id: int = 0,
                        collect_cdfs: bool = False) -> StepInfo:
        if self.mode == "cdf":
            lr = self.lr_schedule(self.local_step)
            info = self.backend.sync_step(params, grads, lr, self.local_step, self.total_num_replicas,
                                          delay_s=self._delay_s())
            return self._account(info)
        # interval: push into the local accumulator, never block on other replicas
        # until a deadline has passed.
        d = self._delay_s()
        if d > 0:
            time.sleep(d)
        if self._acc is None:
            self._acc = self.backend.allocate(grads.numel())   # symmetric on the fused backend
        self._acc.add_(grads)
        self._acc_count += 1
        info = StepInfo(self.local_step, False, 0, 0, applied=False)
        if self._clock() >= self._deadline(self._tick):
            # ONE tick per call (every replica joins tick t exactly once, in its first call after deadline t), and after a
            # late tick the next deadline is the first one still in the future *on the chief's clock* (exchanged inside the
            # tick) -- missed deadlines are skipped, never replayed, and no replica decides on its own to run another tick
            # (reference: the chief's timer sleeps the interval after each take_grad, …modified.py:208-215).
            lr = self.lr_schedule(self.local_step)
            res = self.backend.interval_tick(params, self._acc, self._acc_count, lr, self._tick)
            chief_now = getattr(self.backend, "last_chief_clock", None)
            nxt = self._tick + 1
            if chief_now is not None and self._t0 is not None:
                nxt = max(nxt, int((chief_now - self._t0) / self.interval_s))
            self._tick = nxt
            self._acc.zero_()
            self._acc_count = 0
            if res.applied:
                info = res
                self._account(res)
        self.last_info = info
        return info
