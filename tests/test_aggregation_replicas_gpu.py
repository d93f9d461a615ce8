"""The multi-replica aggregation kernels run as N = 2 .. 8 replicas on ONE H100, in one process, and checked after every step
on every replica bit for bit against the exact emulation of ops/aggrefs.py: the fp32 weights, the bf16 shadow (RNE of the
weights), the replicas against each other, and the status words (epoch, last_mask, last_count, last_late, accepted and
dropped steps).  Every step also checks the weights against float64 within the fp32 bound of the sum, which keeps the
emulation honest too.

What only exists with several replicas is checked here: the contributor order of the sums, the shard split by the
committed count, the drop-connect seed of each contributor's rank, the late and stale fast-forward (also of the chief,
rank 0, which owns the arrival bitmap), the commit ring lapped by a replica away for more than SYNC_RING steps, the LL inbox
parity, the K > N credit and drop accounting and the local-SGD barriers.

The harness (:class:`_Replicas`) gives each replica a zeroed control block, params, grads and a bf16 shadow (and for the
bucketed kernels a bf16 gradient buffer and an LL inbox, for K > N an accumulator) as plain device memory, its own stream,
and 8-entry pointer tables.  Plain loads and stores through those pointers work within one device.

Co-residency.  A kernel that waits on a word another replica writes can only finish if that replica's kernel runs at the
same time, and on one GPU nothing promises that.  So:

* every step's grids, of every replica, fit on the GPU at once.  The waiting kernels (fused_sync_sgd_kernel,
  fused_sync_late_kernel, bucket_late_kernel, the LL late kernel) run 512-thread CTAs at most one per SM; the harness
  passes ``ctas = num_sms // (N * grids per step)`` or less and asserts ``N * grids * ctas <= num_sms``, so even if every
  CTA of every grid of a step took a whole SM they would all be resident;
* every kernel is loaded before replicas launch it together.  Kernels load lazily, at their first launch, and a load
  can wait for the kernels already running on the device: a replica spinning in a barrier would then hold up the host
  thread that is to launch the replica it waits for.  The aggregation entry points set a function attribute before
  their first launch, which loads their kernels; the local-SGD kernels are first launched on one replica of their own;
* the watchdog gets a short timeout (5 s);
* after every step every replica's ``error`` word is read; if one is set the test fails at once with every replica's
  handshake words and runs nothing further.

No replica is ordered by a delay or a sleep.  Where order matters (a late replica, the K > N schedules) the host launches
a replica's kernels only after the kernels they must follow have completed.

Not here: NVLS (it needs several devices), deadline-mode interval ticks (they depend on the wall clock), and a K > N
gradient accumulated after its step's mask froze.  That needs a commit to land between one replica's gate and close
kernels, which only concurrent iterations can produce; the serialized schedules below assert that it never happens in
them, and tests/_kgtn_worker.py accounts for it across GPUs."""
import ctypes

import numpy as np
import pytest
import torch

from _agg_exact_worker import RAGGED, _grad
from distributedmnist_b200.ops import aggrefs as A
from distributedmnist_b200.schedule import LearningRateSchedule

pytestmark = pytest.mark.gpu

SCHED = LearningRateSchedule(0.05, 1, 0.999)       # p = step: the step size changes every step
LR = (SCHED.initial_learning_rate, SCHED.decay_rate, SCHED.decay_steps)
TIMEOUT_MS = 5000.0
SYNC_RING = 64
STEP0 = 5000
LENET = 1665024
EPS = 2.0 ** -23

_STATUS = ("epoch", "error", "accepted_steps", "dropped_steps", "last_mask", "last_count", "last_late")
_WORDS = _STATUS + ("global_step", "arrive", "done", "arrive_e", "done_e", "commit_local", "bitmap", "commit",
                    "last_in_mask", "decided_tag", "decided_mask", "decided_late", "decided_target", "decider_claim",
                    "iv_state", "iv_busy")


def _lib():
    from distributedmnist_b200.ops.lib import load
    return load()


def _table(ptrs):
    return (ctypes.c_void_p * 8)(*([int(p) for p in ptrs] + [int(ptrs[0])] * (8 - len(ptrs))))


def _mask(ranks):
    return sum(1 << q for q in ranks)


def _param(spec, name):
    q = [p for p in spec.params if p.name == name][0]
    return q.offset, q.offset + q.numel


class _Replicas:
    """N replicas of the aggregation state in plain device memory of one GPU, with one stream each.  ``grids``: the number
    of grids one replica launches per step, for the co-residency budget."""

    def __init__(self, n, numel, grids=1, ctas=None, g16=0, inbox=0, acc=False, step0=STEP0, seed=5):
        lib = _lib()
        self.lib, self.n, self.numel = lib, n, numel
        self.sms = int(lib.dm_num_sms())
        self.ctas = max(1, self.sms // (n * grids)) if ctas is None else ctas
        assert n * grids * self.ctas <= self.sms, (n, grids, self.ctas, self.sms)
        self.off = {f: int(lib.dm_sync_ctrl_offset(f.encode())) for f in _WORDS}
        assert all(v >= 0 for v in self.off.values()), self.off
        w0 = (torch.randn(numel, generator=torch.Generator().manual_seed(seed)) * 0.05).cuda()
        cb = int(lib.dm_sync_ctrl_bytes())
        self.ctrl = [torch.zeros(cb, dtype=torch.uint8, device="cuda") for _ in range(n)]
        self.params = [w0.clone() for _ in range(n)]
        self.grads = [torch.zeros(numel, device="cuda") for _ in range(n)]
        self.shadow = [torch.empty(numel, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
        for q in range(n):
            lib.dm_f32_to_bf16(self.params[q], self.shadow[q], numel, None)
        self.streams = [torch.cuda.Stream() for _ in range(n)]
        self.ct = _table([c.data_ptr() for c in self.ctrl])
        self.pt = _table([p.data_ptr() for p in self.params])
        self.gt = _table([g.data_ptr() for g in self.grads])
        if g16:
            self.g16 = [torch.zeros(g16, dtype=torch.bfloat16, device="cuda") for _ in range(n)]
            self.g16t = _table([g.data_ptr() for g in self.g16])
        if inbox:
            self.inbox = [torch.zeros(inbox, dtype=torch.uint8, device="cuda") for _ in range(n)]
            self.it = _table([b.data_ptr() for b in self.inbox])
        if acc:
            self.acc = [torch.zeros(numel, device="cuda") for _ in range(n)]
            self.at = _table([a.data_ptr() for a in self.acc])
        self.step0 = step0
        for q in range(n):            # as FusedBackend.set_global_step; the host mirror stays null
            for f in ("epoch", "global_step", "decider_claim"):
                self.write(q, f, step0)
        torch.cuda.synchronize()

    def write(self, q, field, value):
        o = self.off[field]
        self.ctrl[q][o:o + 4].view(torch.int32).fill_(value)

    def sp(self, q):
        return ctypes.c_void_p(self.streams[q].cuda_stream)

    def set_grads(self, grads):
        """grads[q]: replica q's gradient (CPU float32 tensor) or None; complete on the device when this returns."""
        for q, g in enumerate(grads):
            if g is not None:
                self.grads[q].copy_(g)
        torch.cuda.synchronize()

    def _raw(self):
        return [c.cpu().numpy() for c in self.ctrl]

    def status(self, q, raw):
        return {f: int(raw[q][self.off[f]:self.off[f] + 4].view("<u4")[0]) for f in _STATUS}

    def dump(self, raw):
        lines = []
        for q, r in enumerate(raw):
            u32 = lambda o: int(r[o:o + 4].view("<u4")[0])            # noqa: E731
            u64 = lambda o: int(r[o:o + 8].view("<u8")[0])            # noqa: E731
            o = self.off
            ep = u32(o["epoch"])
            slots = sorted({(ep + d) % SYNC_RING for d in (-2, -1, 0, 1)})
            lines.append("replica %d: %s global_step=%d claim=%d decided(tag=%d mask=%#x late=%d target=%d) iv_state=%#x "
                         "iv_busy=%d" % (q, {f: u32(o[f]) for f in _STATUS}, u32(o["global_step"]), u32(o["decider_claim"]),
                                         u32(o["decided_tag"]), u32(o["decided_mask"]), u32(o["decided_late"]),
                                         u32(o["decided_target"]), u64(o["iv_state"]), u32(o["iv_busy"])))
            for f in ("arrive", "done", "arrive_e", "done_e"):
                lines.append("  %-8s per peer: %s" % (f, [u32(o[f] + 128 * p) for p in range(self.n)]))
            lines.append("  commit_local[slot] = (step+1, mask): %s" % {
                s: (u64(o["commit_local"] + 8 * s) >> 32, hex(u64(o["commit_local"] + 8 * s) & 0xFFFFFFFF)) for s in slots})
            if q == 0:
                lines.append("  chief bitmap: %s commit: %s last_in_mask: %s" % (
                    {s: hex(u32(o["bitmap"] + 4 * s)) for s in slots},
                    {s: (u64(o["commit"] + 8 * s) >> 32, hex(u64(o["commit"] + 8 * s) & 0xFFFFFFFF)) for s in slots},
                    [u32(o["last_in_mask"] + 4 * p) for p in range(self.n)]))
        return "\n".join(lines)

    def finish(self, what):
        """Wait for every replica's kernels; fail at once, with every replica's handshake words, if a watchdog fired."""
        torch.cuda.synchronize()
        raw = self._raw()
        if any(self.status(q, raw)["error"] for q in range(self.n)):
            pytest.fail("%s: watchdog error\n%s" % (what, self.dump(raw)), pytrace=False)
        return [self.status(q, raw) for q in range(self.n)]

    def check_weights(self, what, want, replicas=None, shadow=None):
        """fp32 weights of ``replicas`` (default: all) bit for bit equal to ``want``, and the shadow of ``shadow``
        (default: the same replicas) equal to RNE(want)."""
        replicas = range(self.n) if replicas is None else replicas
        wb, sb = A.bits(want), A.bf16_bits(want)
        for q in replicas:
            bad = np.flatnonzero(A.bits(self.params[q]) != wb)
            assert bad.size == 0, "%s: replica %d: %d of %d weights differ, first at %d: got %r, want %r" % (
                what, q, bad.size, wb.size, bad[0], A.f32(self.params[q])[bad[0]], want[bad[0]])
        for q in (replicas if shadow is None else shadow):
            sh = self.shadow[q].view(torch.int16).cpu().numpy().view(np.uint16)
            bad = np.flatnonzero(sh != sb)
            assert bad.size == 0, "%s: replica %d: %d of %d shadow elements differ from RNE(weights), first at %d" % (
                what, q, bad.size, sb.size, bad[0])


def _check_status(what, got, **want):
    bad = {f: (got[f], v) for f, v in want.items() if got[f] != v}
    assert not bad, "%s: status (got, want): %s" % (what, bad)


def _check_bound(what, w, terms, scale, got, rounded_sum=False):
    """|got - (w - scale * sum(terms))| in float64 within the fp32 roundings of the sequential sum and the update (and the
    sum's bf16 rounding when ``rounded_sum``)."""
    t = np.stack([np.asarray(x, np.float64) for x in terms])
    s = t.sum(0)
    exact = np.asarray(w, np.float64) - float(scale) * s
    bound = float(scale) * ((len(terms) - 1) * EPS * np.abs(t).sum(0) + (2.0 ** -8 * np.abs(s) if rounded_sum else 0.0))
    bound += EPS * np.abs(exact) + 1e-30
    excess = np.abs(np.asarray(got, np.float64) - exact) - bound
    assert excess.max() <= 0.0, "%s: %d weights outside the fp32 bound of the float64 update, worst by %g" % (
        what, int((excess > 0).sum()), excess.max())


# ---- fused_sync_sgd_kernel: K of N ------------------------------------------------------------------------------------
def _sync_run(R, k, schedule, tag, drop=None):
    """One step per schedule entry (team, late): the team's K replicas launch together; after their kernels have
    completed, the late replicas launch (they find the step committed and fast-forward).  Replicas in neither list stay
    away.  ``drop = (keep_prob, seed)``: drop-connect, each contributor's mask seeded by its rank."""
    n = R.n
    keep, seed = drop if drop is not None else (0.0, 0)
    E = R.step0                         # newest committed global step
    w = A.f32(R.params[0])
    epoch = [E] * n                     # each replica's epoch word
    acc, dropped = [0] * n, [0] * n
    masks = {}
    for s, (team, late) in enumerate(schedule):
        what = "%s step %d (team %s, late %s)" % (tag, s, list(team), list(late))
        assert len(team) == k and all(epoch[q] == E for q in team) and not set(team) & set(late)
        gs = [None] * n
        for q in team:
            gs[q] = _grad(100003 * tag_seed(tag) + 1000 * s + q, R.numel)
        R.set_grads(gs)
        for q in team:
            R.lib.dm_fused_sync_sgd(R.ct, R.pt, R.gt, q, n, k, R.numel, *LR, keep, seed, TIMEOUT_MS, R.shadow[q], R.ctas,
                                    R.sp(q), None, None)
        R.finish(what + " team")
        for q in late:
            R.lib.dm_fused_sync_sgd(R.ct, R.pt, R.gt, q, n, k, R.numel, *LR, keep, seed, TIMEOUT_MS, R.shadow[q], R.ctas,
                                    R.sp(q), None, None)
        st = R.finish(what)
        mask = _mask(team)
        scale = A.step_scale(SCHED, E, k)
        terms = []
        for q in sorted(team):           # rank order
            g = A.f32(gs[q])
            if drop is not None:
                g = np.where(A.drop_keep(seed, E, q, keep, g.size), g, np.float32(0))
            terms.append(g)
        want = A.sgd(w, A.seq_sum(terms), scale)
        _check_bound(what, w, terms, scale, want)
        w = want
        masks[E] = mask
        E += 1
        for q in team:
            epoch[q] = E
            acc[q] += 1
            _check_status("%s replica %d" % (what, q), st[q], epoch=E, last_mask=mask, last_count=k, last_late=0,
                          accepted_steps=acc[q], dropped_steps=dropped[q])
        for q in late:
            lapped = E - 1 - epoch[q] >= SYNC_RING      # its step's ring slot holds a newer commit: mask 0
            m = 0 if lapped else masks[epoch[q]]
            assert not (m >> q) & 1
            epoch[q] = E
            dropped[q] += 1
            _check_status("%s late replica %d" % (what, q), st[q], epoch=E, last_mask=m, last_count=bin(m).count("1"),
                          last_late=1, accepted_steps=acc[q], dropped_steps=dropped[q])
        # every arena holds the team's weights (the team pushes into all of them); launched replicas have a fresh shadow
        R.check_weights(what, w, shadow=list(team) + list(late))
    return epoch


def tag_seed(tag):
    return sum(ord(c) for c in tag) % 9973


ARENAS = {"ragged": RAGGED, "lenet": LENET}


@pytest.mark.parametrize("ctas", ["one", "max"])
@pytest.mark.parametrize("arena", list(ARENAS))
@pytest.mark.parametrize("n", [2, 3, 4, 5, 8])
def test_fused_sync_k_equals_n(n, arena, ctas):
    """Every replica contributes: the all-to-all arrival, shard i of count = N per team member, the rank-ordered sum.
    With one CTA per replica the grid-stride loops wrap many times."""
    R = _Replicas(n, ARENAS[arena], ctas=1 if ctas == "one" else None)
    _sync_run(R, n, [(list(range(n)), [])] * 4, "keqn-%s-%s-%d" % (arena, ctas, n))


@pytest.mark.parametrize("n,k", [(2, 2), (2, 1), (4, 4), (4, 3)])
def test_fused_sync_drop_connect(n, k):
    """The drop mask of contributor q is seeded with its rank q.  With K < N the team leaves out low ranks (the chief
    first), so a seed from the team index would differ."""
    R = _Replicas(n, RAGGED)
    sched = [(sorted(set(range(n)) - {(s + j) % n for j in range(n - k)}), [(s + j) % n for j in range(n - k)])
             for s in range(4)]
    _sync_run(R, k, sched, "drop-%d-%d" % (n, k), drop=(0.9, 0x1234567))


def _rotating(n, k, steps):
    """Step s leaves out the N - K replicas from s * (N - K) on (mod N), starting with the chief."""
    out = []
    for s in range(steps):
        late = [(s * (n - k) + j) % n for j in range(n - k)]
        out.append(([q for q in range(n) if q not in late], late))
    return out


@pytest.mark.parametrize("n,k", [(3, 2), (5, 3), (8, 5), (8, 7), (4, 1), (7, 6)])
def test_fused_sync_k_of_n_late_replicas(n, k):
    """K of N with N - K late replicas per step, launched after the team's kernels have completed: count = K runs from 1
    to 7, so shard = ceil(numel4 / count) splits the ragged arena at every count; the late set rotates through the chief."""
    R = _Replicas(n, RAGGED)
    sched = _rotating(n, k, 5)
    assert any(0 in late for _, late in sched)
    _sync_run(R, k, sched, "kofn-%d-%d" % (n, k))


@pytest.mark.parametrize("away", [0, 3])
def test_fused_sync_replica_away_three_steps(away):
    """Replica ``away`` (the chief, or the last rank) misses three steps, returns late in the fourth and fast-forwards four
    steps in one launch, then contributes again: it holds the team's weights and a fresh shadow, and counts as a
    contributor at the next step it arrives for."""
    n, k = 4, 3
    R = _Replicas(n, RAGGED)
    others = [q for q in range(n) if q != away]
    back = [q for q in range(n) if q != others[0]]
    sched = [(others, [])] * 3 + [(others, [away]), (back, [others[0]]), (others, [away])]
    epoch = _sync_run(R, k, sched, "away-%d" % away)
    assert len(set(epoch)) == 1


def test_fused_sync_replica_away_more_than_a_ring_lap():
    """Replica 2 is away for SYNC_RING + 2 steps: its step's commit slot has been reused, so it takes the "committed a ring
    lap ago" path (mask 0, late), fast-forwards to the newest step and contributes at the next one."""
    n, k = 3, 2
    R = _Replicas(n, 4 * 1031)
    laps = SYNC_RING + 2
    sched = [([0, 1], [])] * (laps - 1) + [([0, 1], [2]), ([1, 2], [0]), ([0, 2], [1])]
    _sync_run(R, k, sched, "ringlap")


# ---- csrc/fused_sync.cu bucketed kernels ------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [2, 4, 8])
def test_fused_sync_bucketed(n):
    """dm_fused_sync_bucket on the LeNet layout: phase 1 two-shot on the fc1 bucket (shard per rank, pushed to all), phase 2
    one-shot on the rest and the fc1 shadow; both rank-ordered fp32 sums."""
    from distributedmnist_b200.models import lenet_spec
    spec = lenet_spec()
    e0, e1 = _param(spec, "fc1_weights")
    numel = spec.arena_numel
    R = _Replicas(n, numel, grids=2)
    w = A.f32(R.params[0])
    for s in range(4):
        what = "bucket1 n=%d step %d" % (n, s)
        gs = [_grad(7000 + 1000 * s + q, numel) for q in range(n)]
        R.set_grads(gs)
        for q in range(n):
            R.lib.dm_fused_sync_bucket(R.ct, R.pt, R.gt, q, n, 1, e0, e1, e0, e1, *LR, TIMEOUT_MS, R.shadow[q], R.ctas,
                                       R.sp(q), None, None)
            R.lib.dm_fused_sync_bucket(R.ct, R.pt, R.gt, q, n, 2, 0, numel, e0, e1, *LR, TIMEOUT_MS, R.shadow[q], R.ctas,
                                       R.sp(q), None, None)
        st = R.finish(what)
        scale = A.step_scale(SCHED, STEP0 + s, n)
        terms = [A.f32(g) for g in gs]
        want = A.sgd(w, A.seq_sum(terms), scale)
        _check_bound(what, w, terms, scale, want)
        w = want
        R.check_weights(what, w)
        for q in range(n):
            _check_status("%s replica %d" % (what, q), st[q], epoch=STEP0 + s + 1, last_mask=(1 << n) - 1, last_count=n,
                          last_late=0, accepted_steps=s + 1, dropped_steps=0)


# ---- csrc/fused_bucket.cu (bf16 wire) -----------------------------------------------------------------------------------
@pytest.mark.parametrize("late", ["ll_bf16", "ll_fp32", "flags_fp32", "mlp"])
@pytest.mark.parametrize("n", [2, 4, 8])
def test_bucket_v2(n, late):
    """LeNet layout: early bucket fc1 (phase 1: in-place bf16 reduce + apply), late bucket over LL lines carrying bf16 or
    fp32, or data + flags.  MLP layout: early bucket fc2 exchanged (phase 3) and applied (phase 4) apart, the 3.3 MB late
    bucket through the fp32 kernel.  Four steps: the LL inbox parity alternates twice."""
    from distributedmnist_b200.models import lenet_spec, mlp_spec
    mlp = late == "mlp"
    spec = mlp_spec(3, 1024) if mlp else lenet_spec()
    e0, e1 = _param(spec, "fc2_weights" if mlp else "fc1_weights")
    numel = spec.arena_numel
    late_ll, late_bf16 = late != "flags_fp32", late in ("ll_bf16", "mlp")
    phases = (3, 4, 2) if mlp else (1, 2)
    R = _Replicas(n, numel, grids=len(phases), g16=e1 - e0, inbox=2 * n * (numel - (e1 - e0)) * 8)
    rounds = A.late_bucket_rounds_bf16(numel, e1 - e0, late_ll, late_bf16)
    assert rounds == (late == "ll_bf16")
    late_idx = np.r_[0:e0, e1:numel]
    w = A.f32(R.params[0])
    for s in range(4):
        what = "v2 %s n=%d step %d" % (late, n, s)
        gs = [_grad(9000 + 1000 * s + q, numel) for q in range(n)]
        g16 = [_grad(4000 + 777 * s + q, e1 - e0).to(torch.bfloat16) for q in range(n)]
        for q in range(n):
            R.g16[q].copy_(g16[q])
        R.set_grads(gs)
        for q in range(n):
            for ph in phases:
                R.lib.dm_bucket_sync(R.ct, R.pt, R.gt, R.g16t, R.it, q, n, ph, e0, e1, numel, *LR, TIMEOUT_MS, R.shadow[q],
                                     R.ctas, R.sp(q), None, None, int(late_ll), int(late_bf16))
        st = R.finish(what)
        scale = A.step_scale(SCHED, STEP0 + s, n)
        t16 = [A.f32(g.float()) for g in g16]
        want = A.bucket_step(w, [A.f32(g) for g in gs], t16, (e0, e1), scale, rounds)
        _check_bound(what + " early", w[e0:e1], t16, scale, want[e0:e1], rounded_sum=True)
        tl = [A.rne_bf16(A.f32(g)[late_idx]) if rounds else A.f32(g)[late_idx] for g in gs]
        _check_bound(what + " late", w[late_idx], tl, scale, want[late_idx])
        w = want
        R.check_weights(what, w)
        for q in range(n):
            _check_status("%s replica %d" % (what, q), st[q], epoch=STEP0 + s + 1, last_mask=(1 << n) - 1, last_count=n,
                          last_late=0, accepted_steps=s + 1, dropped_steps=0)


# ---- K > N (dm_kgtn_begin / dm_kgtn_end), serialized ------------------------------------------------------------------
def _kgtn_run(n, k, ops, tag):
    """``ops``: ("it", q) = replica q's whole iteration, ("b", q) its begin alone, ("e", q) its end alone.  The host runs
    one op at a time and waits for it, so every commit is deterministic; each committed step is rebuilt from the host's
    own record of which gradients each replica accumulated for it."""
    R = _Replicas(n, RAGGED, acc=True)
    for q in range(n):
        R.lib.dm_interval_arm(R.ctrl[q], 0.0, R.sp(q))
    R.finish(tag + " arm")
    E = STEP0
    w = A.f32(R.params[0])
    seen = [E] * n                          # the step each replica's last begin adopted
    cur = [[] for _ in range(n)]            # gradients accumulated for step E, in iteration order
    acc, dropped = [0] * n, [0] * n
    last = None                             # (mask, total) of the newest commit
    commits = 0
    flat = []
    for op, q in ops:
        flat += [("b", q), ("e", q)] if op == "it" else [(op, q)]
    for i, (op, q) in enumerate(flat):
        what = "%s op %d (%s %d)" % (tag, i, op, q)
        if op == "b":
            R.lib.dm_kgtn_begin(R.ctrl[q], q, R.params[q], R.shadow[q], R.numel, R.sp(q))
            st = R.finish(what)
            adopted = seen[q] < E
            seen[q] = E
            _check_status(what, st[q], epoch=E)
            if adopted:
                _check_status(what, st[q], last_mask=last[0], last_count=last[1])
            R.check_weights(what, w, shadow=[q])
        else:
            g = _grad(100003 * tag_seed(tag) + i, R.numel)
            R.set_grads([g if r == q else None for r in range(n)])
            R.lib.dm_kgtn_end(R.ct, R.pt, R.gt, R.at, q, n, k, R.numel, *LR, TIMEOUT_MS, R.ctas, R.sp(q), None, None)
            st = R.finish(what)
            stale = seen[q] < E              # a commit landed since this replica's begin: its gate drops the gradient
            if stale:
                dropped[q] += 1
            else:
                cur[q].append(A.f32(g))
                total = sum(len(c) for c in cur)
                if total >= k:               # this close saw K gradients: it commits and applies
                    mask = _mask([r for r in range(n) if cur[r]])
                    scale = A.step_scale(SCHED, E, total)
                    terms = [A.interval_accumulate(cur[r]) if cur[r] else None for r in range(n)]
                    want = A.fused_sync_step(w, terms, mask, scale)
                    _check_bound(what, w, [x for c in cur for x in c], scale, want)
                    w = want
                    for r in range(n):
                        acc[r] += len(cur[r])
                    cur = [[] for _ in range(n)]
                    last = (mask, total)
                    E += 1
                    commits += 1
            _check_status(what, st[q], last_late=int(stale))
            for r in range(n):
                _check_status("%s replica %d" % (what, r), st[r], accepted_steps=acc[r], dropped_steps=dropped[r])
            R.check_weights(what, w, shadow=[])
    for q in range(n):                       # every replica adopts the newest commit: no gradient was lost after a freeze
        R.lib.dm_kgtn_begin(R.ctrl[q], q, R.params[q], R.shadow[q], R.numel, R.sp(q))
    st = R.finish(tag + " final begin")
    R.check_weights(tag + " final", w)
    for q in range(n):
        _check_status("%s final replica %d" % (tag, q), st[q], epoch=E, accepted_steps=acc[q], dropped_steps=dropped[q])
    assert sum(acc) + sum(dropped) + sum(len(c) for c in cur) == sum(1 for op, _ in flat if op == "e")
    return commits, acc, dropped


@pytest.mark.parametrize("n", [2, 3, 4])
@pytest.mark.parametrize("extra", ["n+1", "2n+1"])
def test_kgtn_round_robin(n, extra):
    k = n + 1 if extra == "n+1" else 2 * n + 1
    commits, acc, dropped = _kgtn_run(n, k, [("it", i % n) for i in range(3 * k)], "kgtn-rr-%d-%d" % (n, k))
    assert commits == 3 and sum(acc) == 3 * k and not any(dropped)


def test_kgtn_uneven():
    """Replica 0 computes most gradients, and one step is replica 0's alone."""
    order = [0, 0, 0, 1, 0, 2, 0, 0, 0, 0, 0, 0, 2, 1, 0, 0]
    commits, acc, dropped = _kgtn_run(3, 4, [("it", q) for q in order], "kgtn-uneven")
    assert commits == 4 and acc == [12, 2, 2] and not any(dropped)


@pytest.mark.parametrize("q", [0, 2])
def test_kgtn_stale_gradient_is_dropped(q):
    """Replica q begins, the others commit the step, then q ends: its gate finds the step committed and drops the gradient
    (q = 0: the chief).  Its next iteration adopts the commit and contributes again."""
    n, k = 3, 3
    o = [r for r in range(n) if r != q]
    ops = [("b", q), ("it", o[0]), ("it", o[1]), ("it", o[0]), ("e", q),
           ("it", q), ("it", o[1]), ("it", q), ("it", o[0]), ("it", q), ("it", o[1])]
    commits, acc, dropped = _kgtn_run(n, k, ops, "kgtn-stale-%d" % q)
    assert commits == 3 and dropped[q] == 1 and sum(dropped) == 1 and acc[q] == 3


# ---- local SGD: dm_local_apply + dm_local_average with both barriers ------------------------------------------------------
def _load_local_kernels(lib):
    """One averaging iteration of a lone replica, whose barriers wait on nobody: every local-SGD kernel is loaded."""
    numel = 1024
    ctrl = torch.zeros(int(lib.dm_sync_ctrl_bytes()), dtype=torch.uint8, device="cuda")
    params, grads = torch.zeros(numel, device="cuda"), torch.zeros(numel, device="cuda")
    shadow = torch.empty(numel, dtype=torch.bfloat16, device="cuda")
    stats = torch.zeros(int(lib.dm_local_stats_bytes()), dtype=torch.uint8, device="cuda")
    ct = _table([ctrl.data_ptr()])
    lib.dm_local_apply(ct, 0, params, grads, shadow, numel, 1, *LR, 1, None, None)
    lib.dm_local_average(ct, _table([params.data_ptr()]), shadow, stats, 0, 1, numel, 1, 1, TIMEOUT_MS, 1, None, None)
    torch.cuda.synchronize()
    o = int(lib.dm_sync_ctrl_offset(b"error"))
    assert int(ctrl[o:o + 4].view(torch.int32).item()) == 0


@pytest.mark.parametrize("n", [2, 3, 4, 8])
def test_local_sgd_replicas(n):
    """H = 2 on N concurrent streams: every replica applies its own gradient; the averaging steps' two device barriers
    order the shard owners' reads and writes.  Replicas differ between averages and are bit-identical after each one,
    equal to aggrefs.local_average of the copies before it."""
    H, steps, step0 = 2, 5, 3001
    R = _Replicas(n, RAGGED, step0=step0)
    lib = R.lib
    _load_local_kernels(lib)
    stats = [torch.zeros(int(lib.dm_local_stats_bytes()), dtype=torch.uint8, device="cuda") for _ in range(n)]
    ws = [A.f32(R.params[q]) for q in range(n)]
    rounds = 0
    for j in range(steps):
        s = step0 + j
        what = "local n=%d step %d" % (n, s)
        gs = [_grad(3000 + 1000 * j + q, R.numel) for q in range(n)]
        R.set_grads(gs)
        for q in range(n):
            lib.dm_local_apply(R.ct, q, R.params[q], R.grads[q], R.shadow[q], R.numel, H, *LR, R.ctas, R.sp(q), None)
            lib.dm_local_average(R.ct, R.pt, R.shadow[q], stats[q], q, n, R.numel, H, 1, TIMEOUT_MS, R.ctas, R.sp(q), None)
        st = R.finish(what)
        scale = A.step_scale(SCHED, s, 1)
        ws = [A.sgd(ws[q], A.f32(gs[q]), scale) for q in range(n)]
        if (s + 1) % H == 0:
            avg = A.local_average(ws)
            mean = sum(x.astype(np.float64) for x in ws) / n
            bound = (n - 1) * EPS * sum(np.abs(x.astype(np.float64)) for x in ws) / n + EPS * np.abs(mean) + 1e-30
            assert (np.abs(avg.astype(np.float64) - mean) <= bound).all(), what
            ws = [avg] * n
            rounds += 1
        for q in range(n):
            R.check_weights("%s replica %d" % (what, q), ws[q], replicas=[q])
            _check_status("%s replica %d" % (what, q), st[q], epoch=s + 1, accepted_steps=j + 1, last_mask=1 << q,
                          last_count=1, last_late=0)
            assert int(stats[q][0:4].view(torch.int32).item()) == rounds, (what, q)
        same = len({A.bits(p).tobytes() for p in R.params}) == 1
        assert same == ((s + 1) % H == 0), (what, same)
    assert rounds == 3
