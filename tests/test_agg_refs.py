"""The exact emulation of the aggregation arithmetic (ops/aggrefs.py) separates right from subtly wrong: its single-rounding
fma agrees with exact rational arithmetic, an emulated correct kernel -- shards, float4 loops, the late bucket's compacted
index -- matches it bit for bit, and every seeded fault is caught.  CPU only."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from distributedmnist_b200.ops import aggrefs as A
from distributedmnist_b200.schedule import LearningRateSchedule

SCHED = LearningRateSchedule(0.05, 1, 0.999)
FIRST_STEP = 1000


# ---- exact rounding --------------------------------------------------------------------------------------------------
def _f32_of(q: Fraction) -> np.float32:
    """Round-to-nearest-even of an exact rational to fp32 (normal range)."""
    if q == 0:
        return np.float32(0.0)
    sign, q = (-1 if q < 0 else 1), abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    while Fraction(2) ** e > q:
        e -= 1
    while Fraction(2) ** (e + 1) <= q:
        e += 1
    m = q / Fraction(2) ** (e - 23)            # in [2^23, 2^24)
    n, rem = divmod(m.numerator, m.denominator)
    half = Fraction(rem, m.denominator)
    if half > Fraction(1, 2) or (half == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return np.float32(sign * n * 2.0 ** (e - 23))


# a * b + c whose float64 sum lands exactly on an fp32 midpoint while the exact value does not: rounding the float64 sum
# to fp32 (ties to even) goes the wrong way in both directions
MIDPOINT_CASES = [(1 + 2.0 ** -12, (1 - 2.0 ** -12 + 2.0 ** -24) * 2.0 ** -24, 1.0),         # exact: 1 + 2^-24 + 2^-60
                  (1 + 2.0 ** -20, (1 - 2.0 ** -20) * 2.0 ** -24, 1 + 2.0 ** -23)]          # 1 + 2^-23 + 2^-24 - 2^-64


def test_fma_rounds_once_like_exact_arithmetic():
    rng = np.random.default_rng(0)
    a = (rng.standard_normal(4000) * 2.0 ** rng.integers(-20, 20, 4000)).astype(np.float32)
    b = (rng.standard_normal(4000) * 2.0 ** rng.integers(-20, 20, 4000)).astype(np.float32)
    c = (rng.standard_normal(4000) * 2.0 ** rng.integers(-20, 20, 4000)).astype(np.float32)
    c[:1000] = -(a[:1000].astype(np.float64) * b[:1000]).astype(np.float32)       # heavy cancellation
    a = np.concatenate([a, np.float32([x for x, _, _ in MIDPOINT_CASES])])
    b = np.concatenate([b, np.float32([y for _, y, _ in MIDPOINT_CASES])])
    c = np.concatenate([c, np.float32([z for _, _, z in MIDPOINT_CASES])])
    got = A.fma_f32(a, b, c)
    want = np.array([_f32_of(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)],
                    dtype=np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # the midpoint cases are where the plain double-then-float rounding goes wrong
    naive = (a[-2:].astype(np.float64) * b[-2:] + c[-2:]).astype(np.float32)
    assert (naive != want[-2:]).all()


def test_bf16_rounding_is_rne():
    x = torch.randn(100000) * 3
    x[:8] = torch.tensor([1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 2.0 ** -8), 1 + 2.0 ** -9, 0.0, -0.0, 2.0 ** -126, 1e30])
    want = x.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(A.bf16_bits(x.numpy()), want)
    assert np.array_equal(A.rne_bf16(x.numpy()), x.to(torch.bfloat16).float().numpy())


def test_subnormals_are_refused():
    with pytest.raises(AssertionError, match="subnormal"):
        A.sgd(np.float32([1.0, 2.0 ** -130]), np.float32([1.0, 1.0]), 0.5)
    with pytest.raises(AssertionError, match="subnormal"):
        A.sgd(np.float32([2.0 ** -120]), np.float32([2.0 ** -120]), 0.99)       # 2^-120 - 0.99 * 2^-120


def test_step_size_is_the_host_schedule_rounded_once():
    for step in (0, 1, 999, 12345):
        for count in (1, 3, 7):
            assert A.step_scale(SCHED, step, count) == np.float32(0.05 * 0.999 ** step / count)
    mid = (1.0 + (1.0 + 2.0 ** -23)) / 2
    assert A.midpoint_distance_ulps(mid) == 0.0
    assert A.midpoint_distance_ulps(1.0) == 2.0 ** 27      # 1 - 2^-25 below, in units of 2^-52


# ---- emulated kernels ------------------------------------------------------------------------------------------------
def _kernel_fused_sync(w, grads, mask, lr, prev_shadow, drop=None, fault=None):
    """fused_sync_sgd_kernel seen from all ranks: team member m of `count` reduces float4 shard m over the contributors in
    mask order, applies SGD and pushes; the shadow is refreshed everywhere."""
    n4, contrib = w.size // 4, A.ranks(mask, len(grads))
    count = len(contrib)
    if fault == "recip":
        scale = np.float32(lr) * (np.float32(1) / np.float32(count))
    else:
        scale = np.float32(lr / count)
    W = w.reshape(n4, 4).copy()
    G = [g.reshape(n4, 4) for g in grads]
    keep = None
    if drop is not None:
        seed, step, p = drop
        keep = [A.drop_keep(seed, step, c if fault == "drop_wrong_rank" else contrib[c], p, w.size).reshape(n4, 4)
                for c in range(count)]
    shard = n4 // count if fault == "shard_skip" else -(-n4 // count)
    for m in range(count):
        begin = m * shard - (1 if fault == "shard_twice" and m > 0 else 0)
        rows = slice(begin, min(m * shard + shard, n4))
        acc = np.zeros_like(W[rows])
        for c in (reversed(range(count)) if fault == "reverse_order" else range(count)):
            v = G[contrib[c]][rows]
            acc = acc + (np.where(keep[c][rows], v, np.float32(0)) if keep is not None else v)
        W[rows] = W[rows] - scale * acc if fault == "unfused" else A.fma_f32(-scale, acc, W[rows])
    out = W.reshape(-1)
    shadow = (out.view(np.uint32) >> 16).astype(np.uint16) if fault == "trunc_shadow" else A.bf16_bits(out)
    if fault == "stale_shadow":
        shadow[200:204] = prev_shadow[200:204]
    return out, shadow


def _kernel_bucket(w, grads, g16, early, lr, late_bf16, fault=None):
    """csrc/fused_bucket.cu on every replica at once: the early bucket from the bf16-rounded rank-ordered sum of the bf16
    gradients, then the late bucket walked through its compacted index j -> arena float4 i, skipping the early range."""
    n4, b4, e4 = w.size // 4, early[0] // 4, early[1] // 4
    scale = np.float32(lr / len(grads))
    W = w.reshape(n4, 4).copy()
    W[b4:e4] = A.fma_f32(-scale, A.rne_bf16(A.seq_sum(g16)).reshape(-1, 4), W[b4:e4])
    j = np.arange(n4 - (e4 - b4))
    i = np.where(j <= b4 if fault == "late_index" else j < b4, j, j + (e4 - b4))
    acc = np.zeros((j.size, 4), np.float32)
    for g in grads:
        v = g.reshape(n4, 4)[i]
        acc = acc + (A.rne_bf16(v) if late_bf16 else v)
    W[i] = A.fma_f32(-scale, acc, W[i])
    out = W.reshape(-1)
    return out, A.bf16_bits(out)


N = 4
N4 = 3 * 37 + 2                 # not a multiple of the 3 contributors
GAP_MASK = 0b1101               # rank 1 missing: contributor position != rank from the second one on
EARLY = (4 * 20, 4 * 80)
DROP = (0x2545F491, 0.9)


def _grads(rng, n):
    """Magnitudes spread over 2^-6 .. 2^6, so that the order of the adds changes the rounded sums."""
    return [(rng.standard_normal(n) * 2.0 ** rng.integers(-6, 7, n)).astype(np.float32) for _ in range(N)]


def _mismatches(path, fault=None, steps=8):
    """Weights plus shadow elements where the emulated kernel departs from ops/aggrefs.py, summed over `steps` steps."""
    rng = np.random.default_rng(3)
    n = 4 * N4 if path != "bucket" else 4 * 100
    w = (rng.standard_normal(n) * 0.05).astype(np.float32)
    bad = 0
    for s in range(steps):
        step, grads = FIRST_STEP + s, _grads(rng, n)
        lr = SCHED(step)
        if path == "bucket":
            g16 = [A.rne_bf16(g[EARLY[0]:EARLY[1]] * 0.5) for g in grads]
            got, got_sh = _kernel_bucket(w, grads, g16, EARLY, lr, True, fault)
            want = A.bucket_step(w, grads, g16, EARLY, A.step_scale(SCHED, step, N), True)
        else:
            drop = (DROP[0], step, DROP[1]) if path == "drop" else None
            got, got_sh = _kernel_fused_sync(w, grads, GAP_MASK, lr, A.bf16_bits(w), drop, fault)
            want = A.fused_sync_step(w, grads, GAP_MASK, A.step_scale(SCHED, step, 3), drop)
        bad += int((A.bits(got) != A.bits(want)).sum()) + int((got_sh != A.bf16_bits(want)).sum())
        w = want
    return bad


@pytest.mark.parametrize("path", ["sync", "drop", "bucket"])
def test_emulated_correct_kernel_is_bit_exact(path):
    assert _mismatches(path) == 0


# (fault, path whose data must catch it)
FAULTS = [("reverse_order", "sync"), ("recip", "sync"), ("unfused", "sync"), ("stale_shadow", "sync"),
          ("trunc_shadow", "sync"), ("shard_skip", "sync"), ("shard_twice", "sync"), ("late_index", "bucket"),
          ("drop_wrong_rank", "drop")]


@pytest.mark.parametrize("fault,path", FAULTS)
def test_seeded_aggregation_fault_is_caught(fault, path):
    assert _mismatches(path, fault) > 0, "fault %s passed on the %s path" % (fault, path)


def test_interval_accumulator_is_sequential_with_the_first_gradient_overwriting():
    rng = np.random.default_rng(4)
    gs = _grads(rng, 64)
    want = gs[0].copy()
    for g in gs[1:]:
        want = want + g
    assert np.array_equal(A.bits(A.interval_accumulate(gs)), A.bits(want))
    assert not np.array_equal(A.bits(A.interval_accumulate(gs[::-1])), A.bits(want))
