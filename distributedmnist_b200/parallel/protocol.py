"""K-of-N commit protocol: the executable specification of the device-side arrival bitmap.

What it replaces (reference, SURVEY §2.3 mode A / §2.5 X1-X8): per-variable
``ConditionalAccumulator``s on the parameter server that accept a gradient iff
``local_step >= accumulator_step`` and release the mean once ``>= K`` gradients
have arrived (sync_replicas_optimizer_modified.py:57-90), plus token queues that
carry the new global step back to the workers (:394-398).

The protocol, identical on every implementation (this host model, the
c10d-store version used by the CPU/gloo backend, and ``csrc/fused_sync.cu``):

* there is one *arrival bitmap* and one *commit word* per global step;
* a replica arriving with ``local_step == global_step`` ORs its bit into the
  bitmap; whoever first observes ``popcount >= K`` publishes the frozen bitmap as
  the step's commit mask (compare-and-swap, exactly one winner);
* every replica then reads the same mask: contributors are the set bits, the
  divisor is ``popcount(mask)`` (mean over the number actually accumulated,
  reference :72-81), replicas not in the mask are *late* -- their gradient is
  discarded but they still receive the update, so replicas never diverge;
* a replica arriving with ``local_step < global_step`` is *stale* (reference
  :59-62): dropped immediately, it fast-forwards to the current step.

Because the mask is a single word for the whole flat arena, the contributor set
is uniform across variables (the reference's per-variable accumulators allow
it to differ; SURVEY §2.3 note).
"""
from __future__ import annotations

import threading
import time
from dataclasses import dataclass
from fractions import Fraction
from typing import Dict, List, Optional


@dataclass
class Decision:
    step: int            # the global step this decision belongs to
    accepted: bool       # this replica's gradient is part of the mean
    stale: bool          # arrived with local_step < global_step (dropped before arrival)
    mask: int            # committed contributor bitmap of `step`
    count: int           # popcount(mask) == divisor
    global_step: int     # global step after the commit (what the replica moves on to)


def popcount(x: int) -> int:
    return bin(x).count("1")


class CommitBoard:
    """In-process, thread-safe model (one thread per replica in tests)."""

    def __init__(self, num_replicas: int, replicas_to_aggregate: int):
        assert 1 <= replicas_to_aggregate <= num_replicas <= 32
        self.n = num_replicas
        self.k = replicas_to_aggregate
        self._cv = threading.Condition()
        self._bitmap: Dict[int, int] = {}
        self._commit: Dict[int, int] = {}
        self._global_step = 0

    @property
    def global_step(self) -> int:
        with self._cv:
            return self._global_step

    def commit_mask(self, step: int) -> Optional[int]:
        with self._cv:
            return self._commit.get(step)

    def arrive(self, rank: int, local_step: int, timeout: Optional[float] = None,
               deadline_passed: Optional[bool] = None) -> Decision:
        """Replica ``rank`` finished the gradient it computed from step ``local_step`` weights.

        ``deadline_passed`` switches to interval semantics (mode C): the commit
        happens when the caller says the interval elapsed and >= 1 gradient is
        present, instead of when ``popcount >= K``.
        """
        bit = 1 << rank
        with self._cv:
            if local_step < self._global_step:
                m = self._commit.get(local_step, 0)
                return Decision(local_step, False, True, m, popcount(m), self._global_step)
            if local_step > self._global_step:
                raise RuntimeError("replica %d is ahead of the global step (%d > %d)"
                                   % (rank, local_step, self._global_step))
            bm = self._bitmap.get(local_step, 0) | bit
            self._bitmap[local_step] = bm
            ready = popcount(bm) >= self.k if deadline_passed is None else (deadline_passed and bm != 0)
            if ready and local_step not in self._commit:
                self._commit[local_step] = bm
                self._global_step = local_step + 1
                self._cv.notify_all()
            end = None if timeout is None else time.monotonic() + timeout
            while local_step not in self._commit:
                remaining = None if end is None else end - time.monotonic()
                if remaining is not None and remaining <= 0:
                    raise TimeoutError("step %d never committed (bitmap=%#x, K=%d)"
                                       % (local_step, self._bitmap.get(local_step, 0), self.k))
                self._cv.wait(remaining)
            m = self._commit[local_step]
            return Decision(local_step, bool(m & bit), False, m, popcount(m), self._global_step)


class StoreCommitBoard:
    """Same protocol over a c10d ``Store`` (TCPStore): multi-process CPU implementation.

    ``store.add`` is the atomic OR (each replica adds its own bit exactly once
    per step, so the sum equals the OR) and ``store.compare_set`` is the CAS that
    publishes the commit word -- the same two primitives the device kernel uses
    (``atom.or.sys`` / ``atom.cas.sys`` on the chief's control block).
    """

    def __init__(self, store, num_replicas: int, replicas_to_aggregate: int, prefix: str = "commit_board"):
        assert 1 <= replicas_to_aggregate <= num_replicas <= 32
        self.store = store
        self.n = num_replicas
        self.k = replicas_to_aggregate
        self.prefix = prefix

    def _k_arr(self, step: int) -> str:
        return "%s/arr/%d" % (self.prefix, step)

    def _k_commit(self, step: int) -> str:
        return "%s/commit/%d" % (self.prefix, step)

    def commit_mask(self, step: int) -> Optional[int]:
        key = self._k_commit(step)
        if not self.store.check([key]):
            return None
        return int(self.store.get(key).decode())

    def arrive(self, rank: int, local_step: int, timeout: Optional[float] = None,
               deadline_passed: Optional[bool] = None) -> Decision:
        bit = 1 << rank
        ckey = self._k_commit(local_step)
        if self.store.check([ckey]):
            m = int(self.store.get(ckey).decode())
            return Decision(local_step, False, True, m, popcount(m), local_step + 1)
        bm = int(self.store.add(self._k_arr(local_step), bit))
        ready = popcount(bm) >= self.k if deadline_passed is None else (deadline_passed and bm != 0)
        if ready:
            self.store.compare_set(ckey, "", str(bm))
        if timeout is not None:
            import datetime
            self.store.wait([ckey], datetime.timedelta(seconds=timeout))
        else:
            self.store.wait([ckey])
        m = int(self.store.get(ckey).decode())
        return Decision(local_step, bool(m & bit), False, m, popcount(m), local_step + 1)

    def gc(self, step: int) -> None:
        """Drop keys of steps older than ``step`` (best effort; bounded store growth)."""
        for key in (self._k_arr(step), self._k_commit(step)):
            try:
                self.store.delete_key(key)
            except Exception:
                pass


class BucketedExchange:
    """Executable specification of the bucketed, overlapped aggregation of ``csrc/fused_sync.cu`` (K == N).

    Threads play the replicas, numpy arrays the symmetric arenas, integer flag words (value = epoch + 1, monotonic) the
    control block.  ``early(rank)`` / ``late(rank)`` do exactly what ``fused_sync_early_kernel`` /
    ``fused_sync_late_kernel`` do, in the same order:

    * early: arrive_e all-to-all -> reduce my shard of the early bucket over every replica's gradient arena -> SGD ->
      store the new weights into EVERY replica's parameter arena -> done_e flags.  Does not wait for the peers' pushes.
    * late: arrive all-to-all -> one-shot: sum all contributions of the late ranges in rank order, update the local
      parameters only -> done flags (my reads of the peers' gradient arenas are complete) -> wait done_e of every peer
      (their early pushes have landed here) -> wait done of every peer (nobody still reads MY gradient arena, which the
      next step overwrites) -> epoch + 1.

    The model checks the two hazards the waits exist for: a reader must never see a gradient arena of another step
    (``grad_step``), and nobody may write a parameter range its owner still reads in the same step (``busy_early``).
    """

    def __init__(self, n: int, numel: int, early_range, lr: float = 0.1):
        import numpy as np
        self.np, self.n, self.numel, self.lr = np, n, numel, lr
        self.e0, self.e1 = early_range
        rng = np.random.default_rng(0)
        w0 = rng.standard_normal(numel).astype(np.float32)
        self.params = [w0.copy() for _ in range(n)]
        self.grads = [np.zeros(numel, np.float32) for _ in range(n)]
        self.grad_step = [-1] * n              # which step's gradients arena r currently holds
        self.busy_early = [False] * n          # replica r's compute still reads its early-range parameters
        self.early_from = [[-1] * n for _ in range(n)]   # [r][q]: step of the last early-bucket shard replica q pushed into r
        self.epoch = [0] * n
        self.arrive_e = [[0] * n for _ in range(n)]   # [owner][peer]
        self.done_e = [[0] * n for _ in range(n)]
        self.arrive = [[0] * n for _ in range(n)]
        self.done = [[0] * n for _ in range(n)]
        self._cv = threading.Condition()

    def _post(self, table, me: int, value: int) -> None:
        with self._cv:
            for q in range(self.n):
                table[q][me] = value
            self._cv.notify_all()

    def _wait(self, row, value: int, timeout: float = 10.0) -> None:
        end = time.monotonic() + timeout
        with self._cv:
            while not all(v >= value for v in row):
                left = end - time.monotonic()
                if left <= 0:
                    raise TimeoutError("flag wait timed out: %s < %d" % (row, value))
                self._cv.wait(left)

    def write_grads(self, r: int, g) -> None:
        """The backward pass of replica r overwrites its gradient arena for its current step."""
        self.grads[r][:] = g
        self.grad_step[r] = self.epoch[r]

    def early(self, r: int) -> None:
        np, n, ep = self.np, self.n, self.epoch[r]
        self._post(self.arrive_e, r, ep + 1)
        self._wait(self.arrive_e[r], ep + 1)
        size = self.e1 - self.e0
        shard = (size + n - 1) // n
        b, e = self.e0 + r * shard, min(self.e0 + (r + 1) * shard, self.e1)
        acc = np.zeros(max(e - b, 0), np.float32)
        for q in range(n):                                    # rank order: the same sum on every implementation
            assert self.grad_step[q] == ep, "replica %d read replica %d's gradients of step %d in step %d" % (r, q, self.grad_step[q], ep)
            acc += self.grads[q][b:e]
        nw = self.params[r][b:e] - np.float32(self.lr / n) * acc
        for q in range(n):
            assert not self.busy_early[q], "push into replica %d's early range while its compute still reads it" % q
            self.params[q][b:e] = nw
            self.early_from[q][r] = ep
        self._post(self.done_e, r, ep + 1)

    def late(self, r: int) -> None:
        np, n, ep = self.np, self.n, self.epoch[r]
        self._post(self.arrive, r, ep + 1)
        self._wait(self.arrive[r], ep + 1)
        for (b, e) in ((0, self.e0), (self.e1, self.numel)):
            acc = np.zeros(e - b, np.float32)
            for q in range(n):
                assert self.grad_step[q] == ep, "replica %d read replica %d's late gradients of step %d in step %d" % (r, q, self.grad_step[q], ep)
                acc += self.grads[q][b:e]
            self.params[r][b:e] -= np.float32(self.lr / n) * acc
        self._post(self.done, r, ep + 1)
        self._wait(self.done_e[r], ep + 1)
        # (the bf16 shadow refresh and the next forward pass read the early range from here on: every shard must be this step's)
        assert all(v == ep for v in self.early_from[r]), "replica %d reads early-bucket shards of steps %s in step %d" % (r, self.early_from[r], ep)
        self._wait(self.done[r], ep + 1)
        self.epoch[r] = ep + 1


# ----------------------------------------------------------------------------------------------------------------------
# Interval mode (mode C) -- executable model of csrc/fused_interval.cu
# ----------------------------------------------------------------------------------------------------------------------
class IntervalBoard:
    """Word-level model of the device-side interval protocol (one thread per replica in tests; every method body is one
    "memory operation" of the kernels and takes the lock, so threads interleave at exactly the granularity at which the
    kernels' system-scope loads / stores / CAS interleave on the GPUs under sequentially consistent fences).

    State per replica (the words of ``SyncCtrl``): ``epoch``, ``iv_state`` = (step tag, count), ``iv_busy``, the local copy of
    the commit ring, ``done`` flags; the chief's authoritative ``commit`` ring.  The accumulator is modelled as a float per
    replica plus an ``in_flight`` marker the committer must never observe while it reads (the property the Dekker pair
    ``busy := step+1; fence; read commit``  ||  ``write commit; fence; read busy`` provides).
    """

    def __init__(self, num_replicas: int, lr: float = 1.0):
        self.n = num_replicas
        self.lr = lr
        self._lock = threading.Lock()
        self.epoch = [0] * self.n
        self.state = [(1, 0)] * self.n             # (step + 1 tag, count)
        self.busy = [0] * self.n
        self.commit_local = [dict() for _ in range(self.n)]   # step -> (mask, committer)
        self.done = [[0] * self.n for _ in range(self.n)]     # done[q][p]: p's pushes for step s landed on q (value s+1)
        self.commit: Dict[int, tuple] = {}         # chief: step -> (mask, committer)
        self.acc = [0.0] * self.n
        self.in_flight = [False] * self.n
        self.weights = [0.0] * self.n
        self.ticks = []                            # (step, committer, mask, total)
        self.dropped = [0] * self.n
        self.accumulated = [0] * self.n
        self.lost = [0] * self.n                   # accumulated for a step whose mask was frozen a moment earlier (count was 0)

    # -- iv_adopt ------------------------------------------------------------------------------------------------------------
    def adopt(self, r: int) -> int:
        with self._lock:
            e, adopted = self.epoch[r], 0
            while e in self.commit_local[r]:
                mask, committer = self.commit_local[r][e]
                if self.done[r][committer] < e + 1:
                    break                          # its pushes are still landing
                tag, c = self.state[r]
                if tag == e + 1 and c > 0 and not (mask >> r) & 1:
                    self.lost[r] += c              # arrived after the mask was read: discarded with the step (reference: stale)
                e += 1
                adopted += 1
            if adopted:
                self.epoch[r] = e
                self.state[r] = (e + 1, 0)
            return adopted

    # -- iv_gate: busy := step+1; fence; commit word present? ------------------------------------------------------------------
    def gate_set_busy(self, r: int) -> int:
        with self._lock:
            self.busy[r] = self.epoch[r] + 1
            return self.epoch[r]

    def gate_check(self, r: int, e: int) -> bool:
        with self._lock:
            go = e not in self.commit_local[r]
            if not go:
                self.busy[r] = 0
                self.dropped[r] += 1
            return go

    # -- iv_accumulate (two operations so a reader could observe it half done) ---------------------------------------------------
    def accumulate_begin(self, r: int) -> None:
        with self._lock:
            self.in_flight[r] = True

    def accumulate_end(self, r: int, g: float) -> None:
        with self._lock:
            first = self.state[r][1] == 0
            self.acc[r] = g if first else self.acc[r] + g
            self.in_flight[r] = False

    # -- iv_close ---------------------------------------------------------------------------------------------------------------------
    def close(self, r: int, e: int) -> None:
        with self._lock:
            tag, c = self.state[r]
            assert tag == e + 1
            self.state[r] = (tag, c + 1)
            self.busy[r] = 0
            self.accumulated[r] += 1

    def try_commit(self, r: int, e: int) -> Optional[int]:
        """Deadline passed: read every replica's state word, CAS the chief's commit word.  Returns the mask if this replica won."""
        with self._lock:
            if e in self.commit:
                return None
        mask = 0
        for q in range(self.n):
            with self._lock:                        # one remote load per replica
                tag, c = self.state[q]
            if tag == e + 1 and c > 0:
                mask |= 1 << q
        with self._lock:                            # the CAS
            if e in self.commit:
                return None
            self.commit[e] = (mask, r)
        for q in range(self.n):
            with self._lock:                        # broadcast of the commit word, one store per replica
                self.commit_local[q][e] = (mask, r)
        return mask

    def collect(self, r: int, e: int, mask: int) -> int:
        """Committer: wait until no contributor is mid-accumulate for this step, then read the final counts."""
        total = 0
        for q in range(self.n):
            if not (mask >> q) & 1:
                continue
            while True:
                with self._lock:
                    if self.busy[q] != e + 1:
                        break
                time.sleep(0)
            with self._lock:
                tag, c = self.state[q]
                assert tag == e + 1, "a contributor moved on before its accumulator was read"
                total += c
        return total

    # -- iv_apply ----------------------------------------------------------------------------------------------------------------------
    def apply(self, r: int, e: int, mask: int, total: int) -> None:
        s = 0.0
        for q in range(self.n):
            if (mask >> q) & 1:
                with self._lock:
                    assert not self.in_flight[q], "committer read an accumulator while its owner was adding to it"
                    s += self.acc[q]
        with self._lock:
            new_w = self.weights[r] - self.lr * s / total
        for q in range(self.n):
            with self._lock:
                self.weights[q] = new_w
        with self._lock:
            self.ticks.append((e, r, mask, total))
        for q in range(self.n):
            with self._lock:
                self.done[q][r] = e + 1

    # -- one local iteration of replica r (what the step graph does) -----------------------------------------------------------------------
    def iteration(self, r: int, g: float, deadline_passed: bool, compute=lambda: None) -> None:
        self.adopt(r)
        compute()
        e = self.gate_set_busy(r)
        if not self.gate_check(r, e):
            return
        self.accumulate_begin(r)
        self.accumulate_end(r, g)
        self.close(r, e)
        if deadline_passed:
            mask = self.try_commit(r, e)
            if mask is not None:
                total = self.collect(r, e, mask)
                self.apply(r, e, mask, total)


# ----------------------------------------------------------------------------------------------------------------------
# K == N, bucketed (default path) -- executable model of csrc/fused_bucket.cu, explorable schedule by schedule
# ----------------------------------------------------------------------------------------------------------------------
class ProtocolHazard(AssertionError):
    """A replica consumed data of another step, or overwrote data its consumer had not read yet."""


class BucketV2Model:
    """Word-level model of ``bucket_early_kernel`` + ``bucket_late_ll_kernel`` (csrc/fused_bucket.cu).

    Every replica is a generator; each ``yield`` is one memory operation visible to the other replicas (a flag store, the
    loads of one element from all peers, the stores of one element to one peer, one LL line landing at ONE destination -- a
    multicast store reaches its destinations at different times) or a blocking wait (``yield predicate``).  A scheduler
    picks which runnable replica performs its next operation, so a test can enumerate EVERY interleaving of a small instance
    (:func:`explore_schedules`) or sample large ones.  The memory cells carry (step, kind) tags next to their values and every
    read checks them: the model fails with :class:`ProtocolHazard` exactly when the kernels would consume torn / stale data.

    What the model is for -- the three places where the kernels rely on an ordering argument instead of a flag:

    * the LL inbox has no "consumed" handshake: slot ``[parity][sender]`` is rewritten two steps later.  Safe because a sender
      can only reach step s + 2 after it received every peer's step s + 1 lines, which a peer sends only after its step-s
      kernel (and therefore its step-s polls) completed.  ``parities=1`` removes the double buffer and must fail.
    * the in-place reduction of the bf16 early bucket: rank r overwrites shard r of EVERY replica's buffer with the sum.  A
      replica may read its whole buffer only after ``done_e`` of all ranks, and may start the next backward pass (which
      overwrites the buffer with new gradients) only then too.  ``wait_done_e=False`` must fail.
    * gradients are read from peers only after ``arrive_e`` of that peer (``wait_arrive_e=False`` must fail).
    """

    def __init__(self, n: int, early_len: int, late_len: int, steps: int, parities: int = 2, wait_arrive_e: bool = True,
                 wait_done_e: bool = True, lr: float = 0.5):
        self.n, self.early_len, self.late_len, self.steps, self.parities, self.lr = n, early_len, late_len, steps, parities, lr
        self.wait_arrive_e, self.wait_done_e = wait_arrive_e, wait_done_e
        self.w_early = [[0.0] * early_len for _ in range(n)]
        self.w_late = [[0.0] * late_len for _ in range(n)]
        self.g16 = [[(-1, "none", 0.0)] * early_len for _ in range(n)]            # (step, "raw" | "sum", value)
        self.inbox = [[[[(0, 0.0)] * late_len for _ in range(n)] for _ in range(parities)] for _ in range(n)]   # [dst][parity][src][i] = (tag, v)
        self.consumed = [[[[0] * late_len for _ in range(n)] for _ in range(parities)] for _ in range(n)]      # highest tag dst has read
        self.arrive_e = [[0] * n for _ in range(n)]      # [owner][peer]
        self.done_e = [[0] * n for _ in range(n)]
        self.epoch = [0] * n

    @staticmethod
    def grad(r: int, step: int, i: int, late: bool) -> float:
        return float((r + 1) * (step + 1) + 3 * i + (100 if late else 0))         # small integers: sums are exact

    def expected(self, late: bool, i: int) -> float:
        return -self.lr / self.n * sum(self.grad(r, s, i, late) for r in range(self.n) for s in range(self.steps))

    # -- one replica ------------------------------------------------------------------------------------------------------
    def replica(self, r: int):
        n = self.n
        shard = (self.early_len + n - 1) // n
        b, e = min(r * shard, self.early_len), min((r + 1) * shard, self.early_len)
        for _ in range(self.steps):
            ep = self.epoch[r]
            # fc1_wgrad epilogue: my bf16 gradient of this step (local stores, but peers will read / overwrite these cells)
            for i in range(self.early_len):
                st, kind, _v = self.g16[r][i]
                if st == ep - 1 and kind == "raw" and ep > 0:
                    raise ProtocolHazard("replica %d starts step %d before shard of element %d was reduced" % (r, ep, i))
                self.g16[r][i] = (ep, "raw", self.grad(r, ep, i, False))
            if self.early_len:
                yield None
                # ---- bucket_early_kernel: exchange (operations on my own memory are not scheduling points of their own) ----------
                for q in range(n):
                    self.arrive_e[q][r] = ep + 1
                    if q != r:
                        yield None
                if self.wait_arrive_e:
                    yield (lambda: all(v >= ep + 1 for v in self.arrive_e[r]))
                for i in range(b, e):
                    total = 0.0
                    for q in range(n):                   # multimem.ld_reduce / N peer loads
                        st, kind, v = self.g16[q][i]
                        if (st, kind) != (ep, "raw"):
                            raise ProtocolHazard("replica %d reduced element %d of replica %d holding %s of step %d in step %d"
                                                 % (r, i, q, kind, st, ep))
                        total += v
                    self.g16[r][i] = (ep, "sum", total)  # (the kernel writes its own copy through the local path)
                    yield None
                    for q in range(n):                   # multimem.st: lands per destination
                        if q != r:
                            self.g16[q][i] = (ep, "sum", total)
                            yield None
                for q in range(n):
                    self.done_e[q][r] = ep + 1
                    if q != r:
                        yield None
                # ---- apply --------------------------------------------------------------------------------------------------
                if self.wait_done_e:
                    yield (lambda: all(v >= ep + 1 for v in self.done_e[r]))
                for i in range(self.early_len):
                    st, kind, v = self.g16[r][i]
                    if (st, kind) != (ep, "sum"):
                        raise ProtocolHazard("replica %d applied element %d holding %s of step %d in step %d" % (r, i, kind, st, ep))
                    self.w_early[r][i] -= self.lr / n * v
                yield None
            # ---- bucket_late_ll_kernel: push lines, poll, rank-ordered sum, SGD, epoch + 1 -----------------------------------------
            tag, par = ep + 1, ep % self.parities
            for q in range(n):
                if q == r:
                    continue
                for i in range(self.late_len):
                    old_tag = self.inbox[q][par][r][i][0]
                    if self.consumed[q][par][r][i] < old_tag:
                        raise ProtocolHazard("replica %d overwrote line %d (tag %d) in replica %d's inbox before it was read"
                                             % (r, i, old_tag, q))
                    self.inbox[q][par][r][i] = (tag, self.grad(r, ep, i, True))
                yield None
            for i in range(self.late_len):
                yield (lambda i=i: all(self.inbox[r][par][c][i][0] >= tag for c in range(n) if c != r))
                acc = 0.0
                for c in range(n):
                    if c == r:
                        acc += self.grad(r, ep, i, True)
                        continue
                    t, v = self.inbox[r][par][c][i]
                    if t != tag:
                        raise ProtocolHazard("replica %d polled line %d of replica %d: tag %d, wanted %d (overwritten)" % (r, i, c, t, tag))
                    self.consumed[r][par][c][i] = t
                    acc += v
                self.w_late[r][i] -= self.lr / n * acc
            self.epoch[r] = ep + 1

    # -- scheduler ----------------------------------------------------------------------------------------------------------
    def run(self, choose) -> None:
        """``choose(runnable_ranks) -> rank``.  Raises ``ProtocolHazard`` on a violated invariant or a deadlock."""
        gens = {r: self.replica(r) for r in range(self.n)}
        waiting = {}
        for r in list(gens):
            self._advance(r, gens, waiting)
        while gens:
            runnable = [r for r in sorted(gens) if r not in waiting or waiting[r]()]
            if not runnable:
                raise ProtocolHazard("deadlock: replicas %s wait forever (epochs %s)" % (sorted(gens), self.epoch))
            r = choose(runnable)
            waiting.pop(r, None)
            self._advance(r, gens, waiting)
        for r in range(self.n):
            for i in range(self.early_len):
                if self.w_early[r][i] != self.expected(False, i):
                    raise ProtocolHazard("replica %d early weight %d = %r, expected %r" % (r, i, self.w_early[r][i], self.expected(False, i)))
            for i in range(self.late_len):
                if self.w_late[r][i] != self.expected(True, i):
                    raise ProtocolHazard("replica %d late weight %d = %r, expected %r" % (r, i, self.w_late[r][i], self.expected(True, i)))

    @staticmethod
    def _advance(r, gens, waiting) -> None:
        try:
            w = next(gens[r])
        except StopIteration:
            del gens[r]
            return
        if w is not None:
            waiting[r] = w


class _Visited(Exception):
    """explore_schedules(dedup=True): the run reached a choice point whose state an earlier run has expanded."""


def explore_schedules(make_model, max_runs: int = 200000, dedup: bool = False) -> int:
    """Run ``make_model().run`` under EVERY schedule (depth-first over the scheduler's choice points, replaying prefixes).
    Returns the number of complete schedules; raises the first ``ProtocolHazard``.

    ``dedup``: the model's ``state()`` names everything its future depends on, so a choice point whose (state, runnable
    actors) an earlier run has already expanded is not expanded again and its run ends there.  Every reachable state and
    every transition is still visited -- what a model's per-step and end-of-run checks need -- without enumerating the
    exponentially many orders that lead to the same state.  The return value then counts runs, not schedules."""
    stack, runs, seen = [[]], 0, set()
    while stack:
        prefix = stack.pop()
        trace = []
        model = make_model()

        def choose(runnable, prefix=prefix, trace=trace, model=model):
            i = len(trace)
            if dedup and i >= len(prefix):
                key = (model.state(), tuple(runnable))
                if key in seen:
                    raise _Visited()
                seen.add(key)
            c = prefix[i] if i < len(prefix) else 0
            trace.append((c, len(runnable)))
            return runnable[c]

        try:
            model.run(choose)
        except _Visited:
            pass
        runs += 1
        if runs > max_runs:
            raise RuntimeError("more than %d schedules" % max_runs)
        for i in range(len(prefix), len(trace)):
            for alt in range(1, trace[i][1]):
                stack.append([t[0] for t in trace[:i]] + [alt])
    return runs


# ----------------------------------------------------------------------------------------------------------------------
# K < N (backup workers) -- word-level model of decide<KOFN> + fused_sync_sgd_kernel (csrc/fused_sync.cu)
# ----------------------------------------------------------------------------------------------------------------------
class KofNModel:
    """Every replica is a generator over the memory operations of its training loop (same scheduler as
    :class:`BucketV2Model`): read the parameter arena element by element (forward/backward), write the gradient arena, then
    the kernel -- local commit word, ``atomicOr`` into the chief's bitmap slot, CAS on the chief's commit word by whoever
    sees ``popcount >= K``, ``last_in_mask`` / ``global_step`` / broadcast of the commit word / wipe of the bitmap slot half
    a ring ahead, reduction of the owned shard over the masked contributors, push of the new weights to ALL replicas,
    ``done`` flags, the waits, fast-forward of late and stale replicas.

    Invariants checked while it runs (``ProtocolHazard`` otherwise):

    * a gradient that is ACCEPTED for step s was computed on exactly the weights of step s (a replica whose arena is being
      pushed into while it computes must always turn out late);
    * a team member only reads gradient arenas holding step-s gradients, and only pushes version s + 1 over version s;
    * the committed mask contains only replicas that really arrived for that step (no phantom bit from a recycled bitmap slot);
    * at the end every replica holds the same weights: the serial application of the committed means.

    The bitmap slots carry no tag (one ``atomicOr`` per arrival instead of a CAS loop); the committer of step s wipes the slot
    of step s + ring/2.  A replica that stalls for more than ring/2 global steps BETWEEN its commit-word read and its
    ``atomicOr`` therefore leaves a phantom bit -- with the shipped ring of 64 that is a stall of > 32 steps (~4 ms) between
    two instructions of one warp; the model shows it with ``ring=2`` (``tests/test_protocol.py``).  ``tagged=True`` models the
    designed fix (arrival word = (tag, bits), CAS loop, no wipe): no phantom bit under the same schedules.
    """

    def __init__(self, n: int, k: int, steps: int, ring: int = 8, numel: Optional[int] = None, lr: float = 0.5,
                 tagged: bool = False):
        assert 1 <= k <= n and ring >= 2 and ring % 2 == 0
        self.n, self.k, self.steps, self.ring, self.lr = n, k, steps, ring, lr
        self.tagged = tagged                                                # NEXT_STEPS item 7: (tag, bits) arrival words, CAS loop, no wipe
        self.bitmap_tag = [0] * ring
        self.numel = numel if numel is not None else n
        self.full = (1 << n) - 1
        self.params = [[(0, 0.0)] * self.numel for _ in range(n)]          # (version = number of updates applied, value)
        self.grads = [(-1, False, None)] * n                                # (step, computed on consistent step weights, values)
        self.epoch = [0] * n
        self.arrived = [-1] * n                                             # last step a replica ORed its bit for
        self.commit_local = [[(0, 0)] * ring for _ in range(n)]            # (tag, mask)
        self.done = [[0] * n for _ in range(n)]                             # [owner][peer]
        self.bitmap = [0] * ring                                            # chief
        self.commit = [(0, 0)] * ring                                       # chief
        self.last_in_mask = [0] * n                                         # chief
        self.global_step = 0                                                # chief
        self.log: Dict[int, int] = {}                                       # step -> committed mask
        self.at = [""] * n                                                  # program point labels for targeted schedulers
        self.accepted = [0] * n
        self.dropped = [0] * n

    @staticmethod
    def grad(r: int, step: int, i: int) -> float:
        return float((r + 1) + 7 * step + 3 * i)

    def replica(self, r: int):
        n, ring, bit = self.n, self.ring, 1 << r
        while self.epoch[r] < self.steps:
            ep = self.epoch[r]
            # ---- forward / backward on my parameter arena (peers may push into it concurrently) -------------------------------
            consistent = True
            for i in range(self.numel):
                consistent = consistent and self.params[r][i][0] == ep
                yield None
            self.grads[r] = (ep, consistent, [self.grad(r, ep, i) for i in range(self.numel)])
            yield None
            # ---- decide<KOFN> ----------------------------------------------------------------------------------------------
            slot, want = ep % ring, ep + 1
            cw = self.commit_local[r][slot]
            self.at[r] = "after_commit_word_read"
            yield None
            self.at[r] = ""
            if cw[0] < want:
                now = 0
                if not self.tagged:
                    self.bitmap[slot] |= bit                                # atomicOr_system
                    self.arrived[r] = ep
                    now = self.bitmap[slot] & self.full
                    yield None
                else:
                    while True:                                             # CAS loop on the (tag, bits) arrival word
                        seen = (self.bitmap_tag[slot], self.bitmap[slot])
                        yield None
                        if seen[0] > want:
                            break                                           # the slot already belongs to a later step: I am stale
                        new = (want, bit) if seen[0] < want else (want, seen[1] | bit)
                        if (self.bitmap_tag[slot], self.bitmap[slot]) == seen:
                            self.bitmap_tag[slot], self.bitmap[slot] = new
                            self.arrived[r] = ep
                            now = new[1] & self.full
                            yield None
                            break
                        yield None
                if popcount(now) >= self.k:
                    old = self.commit[slot]
                    yield None
                    if old[0] < want:
                        won = self.commit[slot] == old                      # atomicCAS_system
                        if won:
                            for q in range(n):
                                if (now >> q) & 1 and self.arrived[q] != ep:
                                    raise ProtocolHazard("step %d committed with a phantom bit of replica %d (it last arrived for step %d)"
                                                         % (ep, q, self.arrived[q]))
                            self.commit[slot] = (want, now)
                            self.log[ep] = now
                        yield None
                        if won:
                            for q in range(n):
                                if (now >> q) & 1:
                                    self.last_in_mask[q] = ep + 1
                            yield None
                            self.global_step = max(self.global_step, ep + 1)
                            yield None
                            for q in range(n):
                                self.commit_local[q][slot] = (want, now)
                                if q != r:
                                    yield None
                            if not self.tagged:
                                self.bitmap[(slot + ring // 2) % ring] = 0
                                yield None
                yield (lambda: self.commit_local[r][slot][0] >= want)
                cw = self.commit_local[r][slot]
            if cw[0] == want:
                mask, late = cw[1], not (cw[1] & bit)
            else:
                mask, late = 0, True                                        # committed a ring lap ago
            target = ep + 1
            if late:
                g = self.global_step
                yield None
                target = max(g, ep + 1)
            count = popcount(mask)
            if not late:
                step_g, ok, _vals = self.grads[r]
                if not ok:
                    raise ProtocolHazard("replica %d: gradient accepted for step %d was computed on weights of mixed steps" % (r, ep))
                # ---- reduce my shard over the contributors, SGD, push to every replica -----------------------------------------
                members = [q for q in range(n) if (mask >> q) & 1]
                my_idx = members.index(r)
                shard = (self.numel + count - 1) // count
                for i in range(my_idx * shard, min((my_idx + 1) * shard, self.numel)):
                    acc = 0.0
                    for q in members:
                        gs, _ok, vals = self.grads[q]
                        if gs != ep:
                            raise ProtocolHazard("replica %d read replica %d's gradient arena of step %d in step %d" % (r, q, gs, ep))
                        acc += vals[i]
                    yield None
                    ver, w = self.params[r][i]
                    if ver != ep:
                        raise ProtocolHazard("replica %d updates element %d at version %d in step %d" % (r, i, ver, ep))
                    new = (ep + 1, w - self.lr / count * acc)
                    for q in range(n):
                        if q != r and self.params[q][i][0] != ep:
                            raise ProtocolHazard("replica %d pushes step %d over version %d of element %d at replica %d"
                                                 % (r, ep, self.params[q][i][0], i, q))
                        self.params[q][i] = new
                        if q != r:
                            yield None
                for q in range(n):
                    self.done[q][r] = ep + 1
                    if q != r:
                        yield None
                self.accepted[r] += 1
            else:
                self.dropped[r] += 1
            # ---- wait until every team member's shard has landed in MY arena ------------------------------------------------------
            for q in range(n):
                need = (ep + 1) if (mask >> q) & 1 else 0
                if late:
                    need = self.last_in_mask[q]                             # fast-forward: everything committed so far
                    yield None
                yield (lambda q=q, need=need: self.done[r][q] >= need)
            self.epoch[r] = target

    def run(self, choose) -> None:
        gens = {r: self.replica(r) for r in range(self.n)}
        waiting = {}
        for r in list(gens):
            BucketV2Model._advance(r, gens, waiting)
        while gens:
            runnable = [r for r in sorted(gens) if r not in waiting or waiting[r]()]
            if not runnable:
                raise ProtocolHazard("deadlock: replicas %s wait forever (epochs %s, global step %d)" % (sorted(gens), self.epoch, self.global_step))
            r = choose(runnable)
            waiting.pop(r, None)
            BucketV2Model._advance(r, gens, waiting)
        # serial replay of the committed means
        assert sorted(self.log) == list(range(self.steps)), "committed steps %s" % sorted(self.log)
        w = [0.0] * self.numel
        for s in range(self.steps):
            members = [q for q in range(self.n) if (self.log[s] >> q) & 1]
            if len(members) < self.k:
                raise ProtocolHazard("step %d committed with %d < K contributors" % (s, len(members)))
            for i in range(self.numel):
                w[i] -= self.lr / len(members) * sum(self.grad(q, s, i) for q in members)
        for r in range(self.n):
            if self.params[r] != [(self.steps, v) for v in w]:
                raise ProtocolHazard("replica %d ends with %s, expected versions %d values %s" % (r, self.params[r], self.steps, w))


# ----------------------------------------------------------------------------------------------------------------------
# Weight snapshot of the in-training evaluation -- element-level model of csrc/eval_snapshot.cu against the chief's arena
# ----------------------------------------------------------------------------------------------------------------------
class SnapshotModel:
    """The chief's evaluator (``snap_select`` / ``snap_copy`` / ``snap_validate``) against writers that commit steps and push
    them into the chief's arena element by element, under the same scheduler as :class:`KofNModel`.

    Writers: replica ``g % n`` commits step g (commit word in slot (g - 1) % ring, tag g), pushes every element of the chief's
    arena as (version g, value), then releases its ``done`` = g.  A writer commits g only after ``done`` of g - 1 (in the
    kernels a team member of g + 1 is at epoch g, so g's pushes have landed).  ``interval=False`` moves ``global_step`` right
    after the commit (``decide<KOFN>``), ``interval=True`` after the pushes (``iv_apply``).

    Reader: ``attempts`` attempts, each select / copy / validate as the kernels do it (an attempt whose candidate's commit
    slot was already reused fails at once); an accepted one must hold every element at exactly the version of the step it
    reports (``ProtocolHazard`` otherwise).  ``validate=False`` / ``wait_done=False`` remove the two checks the design rests on.
    """

    def __init__(self, n: int, steps: int, numel: int, interval: bool = False, ring: int = 4, attempts: int = 1,
                 validate: bool = True, wait_done: bool = True):
        self.n, self.steps, self.numel, self.interval, self.ring = n, steps, numel, interval, ring
        self.attempts, self.validate, self.wait_done = attempts, validate, wait_done
        self.arena = [(0, self.value(0, i)) for i in range(numel)]        # the chief's parameter arena: (version, value)
        self.commit = [(0, 0)] * ring                                      # chief: (tag, writer)
        self.global_step = 0
        self.done = [0] * n                                                # chief's done[q]
        self.accepted: List[int] = []                                      # steps of accepted snapshots

    @staticmethod
    def value(g: int, i: int) -> float:
        return float(100 * g + i)

    def writer(self, r: int):
        for g in range(1, self.steps + 1):
            if g % self.n != r:
                continue
            yield (lambda g=g: g == 1 or max(self.done) >= g - 1)
            self.commit[(g - 1) % self.ring] = (g, r)                      # CAS by the committer
            yield None
            if not self.interval:
                self.global_step = max(self.global_step, g)
                yield None
            for i in range(self.numel):
                self.arena[i] = (g, self.value(g, i))                      # one weak push per element
                yield None
            if self.interval:
                self.global_step = max(self.global_step, g)
                yield None
            self.done[r] = g                                               # release after the system fence
            yield None

    def _walk(self, g: int) -> int:
        for _ in range(self.ring):
            if self.commit[g % self.ring][0] != g + 1:
                break
            g += 1
        return g

    def reader(self):
        for _attempt in range(self.attempts):
            # ---- snap_select ------------------------------------------------------------------------------------------------
            g = self.global_step
            yield None
            g = self._walk(g)
            yield None
            lap = False
            while g > 0:
                tag, w = self.commit[(g - 1) % self.ring]
                if tag > g:
                    lap = True                                             # slot already reused: the attempt fails
                    break
                if tag < g or not self.wait_done:
                    break
                if self.done[w] >= g:
                    break
                # blocked until g's writer releases done or a newer step commits
                yield (lambda g=g, w=w: self.done[w] >= g or self.commit[g % self.ring][0] == g + 1)
                g = self._walk(g)
            if lap:
                continue
            # ---- snap_copy --------------------------------------------------------------------------------------------------
            snap = []
            for i in range(self.numel):
                snap.append(self.arena[i])
                yield None
            # ---- snap_validate ----------------------------------------------------------------------------------------------
            if self.validate:
                tag = self.commit[g % self.ring][0]
                yield None
                if tag > g:
                    continue
            bad = [(i, v) for i, (v, x) in enumerate(snap) if v != g or x != self.value(g, i)]
            if bad:
                raise ProtocolHazard("snapshot accepted as step %d holds element %d of version %d" % (g, bad[0][0], bad[0][1]))
            self.accepted.append(g)
            return

    def run(self, choose) -> None:
        gens = {r: self.writer(r) for r in range(self.n)}
        gens[self.n] = self.reader()
        waiting = {}
        for r in list(gens):
            BucketV2Model._advance(r, gens, waiting)
        while gens:
            runnable = [r for r in sorted(gens) if r not in waiting or waiting[r]()]
            if not runnable:
                raise ProtocolHazard("deadlock: %s wait forever (global step %d)" % (sorted(gens), self.global_step))
            r = choose(runnable)
            waiting.pop(r, None)
            BucketV2Model._advance(r, gens, waiting)


# ----------------------------------------------------------------------------------------------------------------------
# K > N gradients per update -- word-level model of the count-triggered interval kernels (csrc/fused_interval.cu, COUNT)
# ----------------------------------------------------------------------------------------------------------------------
class CountTriggerModel:
    """:class:`IntervalBoard` with the count trigger, as generators for :func:`explore_schedules`.  Each replica runs
    ``iters`` iterations (one number, or one per replica).  The code between two ``yield`` s is one atomic step; the steps are

    * adopt (``iv_adopt``: move past every committed step whose pushes have landed, counting gradients accumulated after a
      step's mask was frozen as ``lost``), forward/backward on the adopted weights, the gate (``busy := e+1``; fence.sc;
      commit word present? -> dropped) and the start of ``iv_accumulate`` (``in_flight``);
    * the end of the accumulate and ``iv_close``: publish ``(step, count + 1)``, ``busy := 0``, fence.sc, read every
      replica's ``(step, count)`` word.  ``fence=False`` lets those reads overtake the two stores (a store buffer): the
      stores become visible one step later;
    * sum >= K: read + CAS of the chief's commit word and its broadcast;
    * committer: wait until no contributor is mid-accumulate (``busy_wait=False`` skips the wait), read the final counts and
      the accumulators, SGD, push to every replica, ``done`` flags, credit every contributor's ``accepted``.

    Invariants (``ProtocolHazard`` otherwise): every commit's total is >= K; every accumulated gradient it sums was computed
    on the committed step's weights; the committer never reads an accumulator mid-add nor one whose count is behind; steps
    commit in order, once each; at the end every replica holds the serial replay of the commits, no step has K gradients
    without a commit, the accepted counts add up to the commit totals, and every accumulated gradient is accepted, lost or
    still pending.  Values are ``Fraction`` s, so the replay is exact."""

    def __init__(self, n: int, k: int, iters, fence: bool = True, busy_wait: bool = True, lr=Fraction(1, 2)):
        self.n, self.k, self.fence, self.busy_wait, self.lr = n, k, fence, busy_wait, Fraction(lr)
        self.iters = list(iters) if isinstance(iters, (list, tuple)) else [int(iters)] * n
        self.epoch = [0] * n
        self.state = [(1, 0)] * n                          # iv_state: (step + 1, gradients accumulated for it)
        self.busy = [0] * n
        self.commit_local: List[Dict[int, tuple]] = [dict() for _ in range(n)]   # step -> (mask, committer)
        self.commit: Dict[int, tuple] = {}                 # the chief's commit ring
        self.done = [[0] * n for _ in range(n)]            # done[q][p]: p's pushes of step s landed on q (value s + 1)
        self.acc: List[list] = [[] for _ in range(n)]      # (step of the weights, value) of every gradient accumulated
        self.in_flight = [False] * n
        self.weights = [(0, Fraction(0))] * n              # (version = committed steps applied, value)
        self.commits: List[tuple] = []                     # (step, committer, mask, counts, total, gradient sum)
        self.accumulated, self.accepted, self.dropped, self.lost = [0] * n, [0] * n, [0] * n, [0] * n

    @staticmethod
    def grad(r: int, it: int) -> Fraction:
        return Fraction(10 * (r + 1) + it)

    def replica(self, r: int):
        n = self.n
        for it in range(self.iters[r]):
            # ---- adopt, forward/backward, gate, accumulate begins ----------------------------------------------------------
            e = self.epoch[r]
            while e in self.commit_local[r]:
                mask, who = self.commit_local[r][e]
                if self.done[r][who] < e + 1:
                    break
                tag, c = self.state[r]
                if e == self.epoch[r] and tag == e + 1 and c > 0 and not (mask >> r) & 1:
                    self.lost[r] += c
                    self.dropped[r] += c
                e += 1
            if e != self.epoch[r]:
                self.epoch[r], self.state[r] = e, (e + 1, 0)
            ver, _w = self.weights[r]
            if ver != e:
                raise ProtocolHazard("replica %d computes on weights of version %d at step %d" % (r, ver, e))
            if e in self.commit_local[r]:
                self.dropped[r] += 1                       # stale: computed on weights a commit is replacing
                yield None
                continue
            self.busy[r] = e + 1
            self.in_flight[r] = True
            yield None
            # ---- accumulate ends, close ----------------------------------------------------------------------------------
            tag, c = self.state[r]
            if tag != e + 1:
                raise ProtocolHazard("replica %d closes step %d holding the count of step %d" % (r, e, tag - 1))
            self.acc[r] = [(e, self.grad(r, it))] if c == 0 else self.acc[r] + [(e, self.grad(r, it))]
            self.in_flight[r] = False
            self.accumulated[r] += 1
            mine = (e + 1, c + 1)
            if self.fence:
                self.state[r], self.busy[r] = mine, 0
                seen = [mine if q == r else self.state[q] for q in range(n)]
                yield None
            else:
                seen = [mine if q == r else self.state[q] for q in range(n)]
                yield None
                self.state[r], self.busy[r] = mine, 0
                yield None
            if sum(cq for tq, cq in seen if tq == e + 1) < self.k:
                continue
            # ---- the trigger fired: CAS the chief's commit word, broadcast it ---------------------------------------------
            if e in self.commit:
                continue
            mask = sum(1 << q for q, (tq, cq) in enumerate(seen) if tq == e + 1 and cq > 0)
            self.commit[e] = (mask, r)
            for q in range(n):
                self.commit_local[q][e] = (mask, r)
            yield None
            # ---- committer: busy-wait, final counts, peer loads of the accumulators, SGD, push, done ------------------------
            if self.busy_wait:
                for q in range(n):
                    if (mask >> q) & 1 and q != r:
                        yield (lambda q=q: self.busy[q] != e + 1)
            counts, terms = [0] * n, []
            for q in range(n):
                if not (mask >> q) & 1:
                    continue
                tq, cq = self.state[q]
                if tq != e + 1:
                    raise ProtocolHazard("contributor %d of step %d moved on before its accumulator was read" % (q, e))
                if self.in_flight[q]:
                    raise ProtocolHazard("committer %d read replica %d's accumulator while it was adding to it" % (r, q))
                if len(self.acc[q]) != cq:
                    raise ProtocolHazard("replica %d's accumulator holds %d gradients, its count says %d" % (q, len(self.acc[q]), cq))
                for s, v in self.acc[q]:
                    if s != e:
                        raise ProtocolHazard("commit of step %d sums a gradient computed on the weights of step %d" % (e, s))
                    terms.append(v)
                counts[q] = cq
            total = sum(counts)
            if total < self.k:
                raise ProtocolHazard("step %d committed with %d < K = %d gradients" % (e, total, self.k))
            ver, w = self.weights[r]
            if ver != e:
                raise ProtocolHazard("committer %d of step %d holds weights of version %d" % (r, e, ver))
            new = (e + 1, w - self.lr * sum(terms) / total)
            for q in range(n):
                self.weights[q] = new
                self.done[q][r] = e + 1
                self.accepted[q] += counts[q]
            self.commits.append((e, r, mask, tuple(counts), total, sum(terms)))
            yield None

    def run(self, choose) -> None:
        gens = {r: self.replica(r) for r in range(self.n)}
        waiting = {}
        for r in list(gens):
            BucketV2Model._advance(r, gens, waiting)
        while gens:
            runnable = [r for r in sorted(gens) if r not in waiting or waiting[r]()]
            if not runnable:
                raise ProtocolHazard("deadlock: replicas %s wait forever (epochs %s)" % (sorted(gens), self.epoch))
            r = choose(runnable)
            waiting.pop(r, None)
            BucketV2Model._advance(r, gens, waiting)
        self.check_end()

    def check_end(self) -> None:
        steps = [c[0] for c in self.commits]
        if steps != list(range(len(steps))):
            raise ProtocolHazard("commits out of order or repeated: %s" % steps)
        w = Fraction(0)
        for (_e, _r, _m, _c, total, gsum) in self.commits:
            w -= self.lr * gsum / total
        for q in range(self.n):
            if self.weights[q] != (len(steps), w):
                raise ProtocolHazard("replica %d ends with %s, the serial replay gives %s" % (q, self.weights[q], (len(steps), w)))
        top = len(steps)
        pending = sum(c for t, c in self.state if t == top + 1)
        if pending >= self.k:
            raise ProtocolHazard("every replica has closed and step %d holds %d >= K = %d gradients without a commit"
                                 % (top, pending, self.k))
        if sum(self.accepted) != sum(c[4] for c in self.commits):
            raise ProtocolHazard("accepted %s do not add up to the commit totals" % self.accepted)
        for q in range(self.n):
            t, c = self.state[q]
            mask = self.commit.get(t - 1, (None,))[0]
            residual = c if mask is None or not (mask >> q) & 1 else 0   # pending, or lost but not adopted yet
            if self.accumulated[q] != self.accepted[q] + self.lost[q] + residual:
                raise ProtocolHazard("replica %d accumulated %d gradients: %d accepted, %d lost, %d pending"
                                     % (q, self.accumulated[q], self.accepted[q], self.lost[q], residual))


# ----------------------------------------------------------------------------------------------------------------------
# --target_accuracy -- host loops of N lock-step replicas against the stop word (csrc/eval_target.cu, train.py)
# ----------------------------------------------------------------------------------------------------------------------
class TargetStopModel:
    """N replicas with K = N: one host loop (``train.train``'s pipelined or non-pipelined loop) and one device stream each,
    as generators for :func:`run_random` / :func:`explore_schedules` (actors 0..N-1 are the hosts, N..2N-1 the devices).

    * host: launch step j; the chief enqueues a pass after it when ``j % every == 0`` or ``j > max``; wait for step j - 1
      (pipelined) or j (non-pipelined), read the host word, lower ``max`` to a stop step found there; stop launching once
      ``j > max``.
    * device: step j publishes its exchange (on the chief after the target test of the pass after step j - 1), waits for
      every replica's exchange of step j, then ``stop_publish`` copies the replica's stop word into its host word.  The
      chief's pass after step j reaches the target iff ``j >= reach``; its test stores S = j + ``margin`` into every
      replica's stop word if none is set.

    Invariants (``ProtocolHazard`` otherwise): no deadlock, every replica launches exactly the steps a run with
    ``--max_steps=S`` launches (S = min(max_steps, stop step)), and the chief enqueues exactly that run's passes."""

    def __init__(self, n: int, every: int, reach: int, margin: int, max_steps: int = 1000, pipelined: bool = True):
        self.n, self.every, self.reach, self.margin, self.max_steps, self.pipelined = n, every, reach, margin, max_steps, pipelined
        self.launched = [0] * n
        self.host_done = [False] * n
        self.exchanged = [0] * n       # newest step whose exchange the replica has published
        self.completed = [0] * n
        self.stop = [0] * n            # stop words (device)
        self.host_word = [0] * n       # page-locked copies (host)
        self.evals: List[int] = []     # steps after which the chief enqueued a pass

    def host(self, r: int):
        mx, j = self.max_steps, 0
        while True:
            j += 1
            self.launched[r] = j
            if r == 0 and (j % self.every == 0 or j > mx):
                self.evals.append(j)
            yield None
            wait = j - 1 if self.pipelined else j
            if wait > 0:
                yield (lambda w=wait: self.completed[r] >= w)
                if self.host_word[r]:
                    mx = min(mx, self.host_word[r])
            if j > mx:
                break
            yield None
        yield (lambda: self.completed[r] >= j)            # the step still in flight is drained
        self.host_done[r] = True

    def device(self, r: int):
        j = 0
        while True:
            yield (lambda: self.launched[r] > j or self.host_done[r])
            if self.launched[r] <= j:
                return
            j += 1
            self.exchanged[r] = j
            yield None
            yield (lambda s=j: all(e >= s for e in self.exchanged))
            self.host_word[r] = self.stop[r]
            self.completed[r] = j
            yield None
            if r == 0:
                # the pass after step j (if any) is known once step j + 1 is launched or the host has finished
                yield (lambda s=j: self.launched[0] > s or self.host_done[0])
                if j in self.evals and j >= self.reach and not self.stop[0]:
                    for q in range(self.n):
                        self.stop[q] = j + self.margin
                yield None

    def run(self, choose) -> None:
        n = self.n
        gens = {a: (self.host(a) if a < n else self.device(a - n)) for a in range(2 * n)}
        waiting = {}
        for a in list(gens):
            BucketV2Model._advance(a, gens, waiting)
        while gens:
            runnable = [a for a in sorted(gens) if a not in waiting or waiting[a]()]
            if not runnable:
                raise ProtocolHazard("deadlock: %s wait forever (launched %s, completed %s)"
                                     % (sorted(gens), self.launched, self.completed))
            a = choose(runnable)
            waiting.pop(a, None)
            BucketV2Model._advance(a, gens, waiting)
        first = next((j for j in range(1, self.max_steps + 2) if j >= self.reach and
                      (j % self.every == 0 or j > self.max_steps)), None)
        s = min(self.max_steps, first + self.margin) if first is not None else self.max_steps
        if self.launched != [s + 1] * n:
            raise ProtocolHazard("replicas launched %s steps, a run with --max_steps=%d launches %d"
                                 % (self.launched, s, s + 1))
        want = [j for j in range(1, s + 2) if j % self.every == 0 or j > s]
        if self.evals != want:
            raise ProtocolHazard("the chief enqueued passes after steps %s, a run with --max_steps=%d after %s"
                                 % (self.evals, s, want))


# ----------------------------------------------------------------------------------------------------------------------
# Stale synchronous parallel -- word-level model of ssp_wait / as_pull_step / as_pull / as_ticket / as_apply / ssp_publish
# (csrc/fused_async.cu) and of the training loop's stop rule with retirement
# ----------------------------------------------------------------------------------------------------------------------
SSP_RETIRED = 0xFFFFFFFF


class SSPModel:
    """N replicas running asynchronous SGD under the staleness bound s, as generators for :func:`explore_schedules`.

    Memory: ``counts[d][p]`` is the number of replica p's updates that have landed in replica d's master copy (with
    integer updates this is what the copy's slot p holds), ``board[d][p]`` peer p's clock in replica d's clock board,
    ``counter`` the chief's update counter.  One iteration of replica q with clock c is two atomic steps:

    * the wait (blocked until every peer's clock in q's board is >= c - s, or retired), the read of r and the pull of
      q's master copy -- as one step, the earliest the pull can happen: a copy's counts and the counter only grow, so a
      later read could only see more;
    * the ticket, the apply to every copy and the publication of c + 1 into every board -- as one step, the latest the
      ticket and the apply can happen before the release, which the kernels' fences order after them.

    The host's stop rule: the pipelined loop has launched iteration i + 1 when it reads iteration i's ticket t, and stops
    launching once t + 1 > ``max_steps``; replica q also stops after ``iters[q]`` iterations (a replica that stops early).
    A stopped replica publishes the retired clock into every board.

    Checked at every step (``ProtocolHazard`` otherwise), B1-B4 of DESIGN.md §4:
    B1 q's pull holds its own c updates, at least c - s of each peer it saw running, and every update of each peer it
    saw retired; B2 c - (smallest running peer clock seen) <= s; B3 tau = ticket - r <= (N - 1)(2s + 1); B4 no state
    in which every unfinished replica is blocked.  At the end: every copy holds every update, the tickets are 0 .. T - 1,
    and two replicas that both stopped by the stop rule differ by at most s + 3 updates.

    Mutants, each of which must fail: ``publish_before_apply`` (the clock is released before the update lands),
    ``retire=False`` and ``slack=1`` (the wait admits c - s - 1)."""

    def __init__(self, n: int, s: int, iters, max_steps: int = 1 << 30, publish_before_apply: bool = False,
                 retire: bool = True, slack: int = 0):
        self.n, self.s, self.iters, self.max_steps = n, s, list(iters), max_steps
        self.publish_before_apply, self.retire, self.slack = publish_before_apply, retire, slack
        self.counts = [[0] * n for _ in range(n)]
        self.board = [[0] * n for _ in range(n)]
        self.counter = 0
        self.clock = [0] * n           # updates q has applied and published
        self.r = [-1] * n              # r of q's current iteration, -1 between iterations
        self.stop_at = list(self.iters)   # iterations q runs: lowered by the stop rule
        self.by_rule = [False] * n     # q stopped by the stop rule (not by its own iteration count)
        self.tickets: List[int] = []
        self.done = [False] * n
        self.pc = [0] * n              # where q's generator stands: 0 wait, 1 pulled, 2 published (mutant), 3 applied

    def state(self):
        return (tuple(map(tuple, self.counts)), tuple(map(tuple, self.board)), self.counter, tuple(self.clock),
                tuple(self.r), tuple(self.stop_at), tuple(self.by_rule), tuple(self.done), tuple(self.pc))

    def replica(self, q: int):
        n, s = self.n, self.s
        peers = [p for p in range(n) if p != q]
        c = 0
        while c < self.stop_at[q]:
            self.pc[q] = 0
            yield (lambda c=c: all(self.board[q][p] + s + self.slack >= c for p in peers))
            seen = [self.board[q][p] for p in range(n)]
            pulled = list(self.counts[q])
            self.r[q] = self.counter
            if pulled[q] != c:
                raise ProtocolHazard("B1: replica %d pulled %d of its own updates in iteration %d" % (q, pulled[q], c))
            for p in peers:
                if seen[p] == SSP_RETIRED and pulled[p] != self.stop_at[p]:
                    raise ProtocolHazard("B1: replica %d saw %d retired but pulled %d of its %d updates"
                                         % (q, p, pulled[p], self.stop_at[p]))
                if seen[p] != SSP_RETIRED and pulled[p] < c - s:
                    raise ProtocolHazard("B1: replica %d pulled %d of replica %d's updates in iteration %d, s = %d"
                                         % (q, pulled[p], p, c, s))
            running = [seen[p] for p in peers if seen[p] != SSP_RETIRED]
            if running and c - min(running) > s:
                raise ProtocolHazard("B2: replica %d started iteration %d with peer clocks %s, s = %d" % (q, c, seen, s))
            self.pc[q] = 1
            yield None
            t = self.counter
            self.counter += 1
            self.tickets.append(t)
            if t - self.r[q] > (n - 1) * (2 * s + 1):
                raise ProtocolHazard("B3: replica %d pulled at r = %d and took ticket %d" % (q, self.r[q], t))
            self.r[q] = -1
            if self.publish_before_apply:
                for d in range(n):
                    self.board[d][q] = c + 1
                self.pc[q] = 2
                yield None
            for d in range(n):
                self.counts[d][q] += 1
            for d in range(n):
                self.board[d][q] = c + 1
            self.clock[q] = c + 1
            # the host read this iteration's ticket with the next one launched: stop after that one
            if t + 1 > self.max_steps and c + 2 < self.stop_at[q]:
                self.stop_at[q] = c + 2
                self.by_rule[q] = True
            c += 1
            self.pc[q] = 3
            yield None
        if self.retire:
            for d in range(n):
                self.board[d][q] = SSP_RETIRED
        self.done[q] = True

    def run(self, choose) -> None:
        gens = {q: self.replica(q) for q in range(self.n)}
        waiting = {}
        for q in list(gens):
            BucketV2Model._advance(q, gens, waiting)
        while gens:
            runnable = [q for q in sorted(gens) if q not in waiting or waiting[q]()]
            if not runnable:
                raise ProtocolHazard("B4: deadlock, replicas %s wait forever (clocks %s, boards %s)"
                                     % (sorted(gens), self.clock, self.board))
            q = choose(runnable)
            waiting.pop(q, None)
            BucketV2Model._advance(q, gens, waiting)
        for d in range(self.n):
            if self.counts[d] != self.clock:
                raise ProtocolHazard("replica %d's copy holds %s updates, the replicas applied %s" % (d, self.counts[d], self.clock))
        if sorted(self.tickets) != list(range(sum(self.clock))):
            raise ProtocolHazard("tickets %s are not a permutation" % sorted(self.tickets))
        ruled = [self.clock[q] for q in range(self.n) if self.by_rule[q]]
        if ruled and max(ruled) - min(ruled) > self.s + 3:
            raise ProtocolHazard("replicas stopped by the stop rule applied %s updates, s = %d" % (self.clock, self.s))


def run_random(make_model, seeds) -> int:
    """Run ``make_model().run`` once per seed, every choice drawn at random.  Returns the number of runs; raises the first
    ``ProtocolHazard``."""
    import random
    for seed in seeds:
        rng = random.Random(seed)
        make_model().run(lambda runnable: runnable[rng.randrange(len(runnable))])
    return len(seeds)
