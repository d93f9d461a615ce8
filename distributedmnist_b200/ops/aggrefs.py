"""Exact CPU emulation of the gradient-aggregation arithmetic (csrc/fused_sync.cu, csrc/fused_bucket.cu,
csrc/fused_interval.cu).

Not a float64 approximation.  Wherever the contributor order is known, a kernel's result is a deterministic function of
its inputs, and this module computes that function bit for bit with numpy float32 (IEEE round-to-nearest-even):

* **sums** -- sequential fp32 adds starting from +0.0, in rank (mask) order: the P2P paths, the late bucket and the
  interval apply over the accumulators.  The interval accumulator adds a replica's gradients in iteration order; the
  first one overwrites.
* **bf16** -- round-to-nearest-even of an fp32 value (``__floats2bfloat162_rn``).  The early bucket's P2P reduce sums
  every replica's bf16 gradient in fp32 in rank order and rounds the sum to bf16.  The LL-bf16 late bucket rounds every
  contribution, the replica's own included, to bf16 before the sum.
* **step size** -- ``fp32(lr(step) / count)`` with ``lr`` from :class:`~distributedmnist_b200.schedule.LearningRateSchedule`.
  The kernels evaluate the same expression in double and round once (``cta_scale`` in csrc/fused_sync.cuh).
* **update** -- ``fma(-scale, g, w)`` with a single rounding: every update loop compiles to FFMA.
* **shadow** -- RNE bf16 of the final fp32 weights over the whole arena.
* **drop-connect** -- contributor q's gradient masked by :func:`~distributedmnist_b200.models.dropout_keep_mask` with the
  kernel's seed mix ``seed + step * 0x9E3779B9 + q * 0x85EBCA77``, no rescale.

The kernels are built with flush-to-zero.  :func:`assert_no_subnormal` checks that no operand or result is subnormal,
where FTZ and IEEE arithmetic would differ; the emulation calls it on everything it computes.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence, Tuple

import numpy as np

FLT_MIN = 2.0 ** -126
_M32 = 0xFFFFFFFF


def f32(x) -> np.ndarray:
    """Contiguous float32 numpy copy of an array, a tensor (any device) or a scalar."""
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    return np.ascontiguousarray(np.asarray(x, dtype=np.float32))


def assert_no_subnormal(what: str, *arrays) -> None:
    for a in arrays:
        a = np.abs(np.asarray(a, dtype=np.float64))
        n = int(((a != 0) & (a < FLT_MIN)).sum())
        assert n == 0, "%s: %d subnormal values; the kernels flush them to zero, the emulation would not" % (what, n)


def bits(x) -> np.ndarray:
    """fp32 bit patterns (compare results with these: -0.0 != +0.0, NaN == NaN)."""
    return f32(x).view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------------
# roundings
# ---------------------------------------------------------------------------------------------------------------------
def rne_bf16(x) -> np.ndarray:
    """bf16 round-to-nearest-even of fp32 values, returned as the float32 numbers they are."""
    u = f32(x).view(np.uint32).astype(np.uint64)
    r = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return r.astype(np.uint32).view(np.float32)


def bf16_bits(x) -> np.ndarray:
    """uint16 patterns of ``rne_bf16(x)``: what a kernel's bf16 store of fp32 ``x`` writes."""
    return (rne_bf16(x).view(np.uint32) >> 16).astype(np.uint16)


def _is_f32_midpoint(s: np.ndarray) -> np.ndarray:
    """float64 values lying exactly halfway between two adjacent normal fp32 numbers: the 29 mantissa bits below fp32
    precision are 1000...0."""
    low = s.view(np.uint64) & np.uint64((1 << 29) - 1)
    return (low == np.uint64(1 << 28)) & (np.abs(s) >= FLT_MIN)


def fma_f32(a, b, c) -> np.ndarray:
    """``a * b + c`` in fp32 with ONE rounding (FFMA).  The product of two fp32 numbers is exact in float64; the sum
    ``s = RN64(p + c)`` is exact up to the two-sum error ``e``.  Rounding ``s`` to fp32 is then correct unless ``s`` lands
    exactly on an fp32 midpoint while the exact sum does not (``e != 0``): the exact sum lies on ``e``'s side of it."""
    a, b, c = np.broadcast_arrays(f32(a), f32(b), f32(c))
    p = a.astype(np.float64) * b.astype(np.float64)
    c = c.astype(np.float64)
    s = p + c
    bv = s - p
    e = (p - (s - bv)) + (c - bv)
    r = s.astype(np.float32)
    fix = _is_f32_midpoint(s) & (e != 0)
    if fix.any():
        r[fix] = np.nextafter(s[fix], np.where(e[fix] > 0, np.inf, -np.inf)).astype(np.float32)
    return r


def sgd(w, g, scale) -> np.ndarray:
    """The update of every aggregation kernel: ``w - scale * g`` as ``fma(-scale, g, w)``."""
    w, g = f32(w), f32(g)
    out = fma_f32(-np.float32(scale), g, w)
    assert_no_subnormal("sgd", w, g, out)
    return out


def seq_sum(terms: Sequence[np.ndarray]) -> np.ndarray:
    """Sequential fp32 sum from +0.0 in the given order."""
    acc = None
    for t in terms:
        t = f32(t)
        acc = np.zeros_like(t) if acc is None else acc
        acc = acc + t
        assert_no_subnormal("sum", acc)
    return acc


def ranks(mask: int, nranks: int = 32):
    return [q for q in range(nranks) if (mask >> q) & 1]


# ---------------------------------------------------------------------------------------------------------------------
# learning rate
# ---------------------------------------------------------------------------------------------------------------------
def step_scale(schedule, step: int, count: int) -> np.float32:
    """The kernels' step size: ``fp32(lr(step) / count)``, evaluated in double like the host schedule."""
    return np.float32(schedule(step) / count)


def midpoint_distance_ulps(x: float) -> float:
    """Distance of the double ``x`` from the nearest fp32 rounding boundary, in double ulps of ``x``.  Two evaluations of
    ``x`` that differ by less than this round to the same fp32 number."""
    f = np.float32(x)
    lo = (float(f) + float(np.nextafter(f, np.float32(-np.inf)))) / 2
    hi = (float(f) + float(np.nextafter(f, np.float32(np.inf)))) / 2
    return min(abs(x - lo), abs(hi - x)) / math.ulp(x)


# ---------------------------------------------------------------------------------------------------------------------
# drop-connect
# ---------------------------------------------------------------------------------------------------------------------
def drop_seed_mix(seed: int, step: int, rank: int) -> int:
    return (seed + step * 0x9E3779B9 + rank * 0x85EBCA77) & _M32


def drop_keep(seed: int, step: int, rank: int, keep_prob: float, n: int) -> np.ndarray:
    """Contributor ``rank``'s keep mask at ``step``, with the kernel's threshold (``models.lenet.dropout_threshold``)."""
    from ..models import dropout_keep_mask
    return dropout_keep_mask(drop_seed_mix(seed, step, rank), 1, n, keep_prob).view(-1).numpy()


# ---------------------------------------------------------------------------------------------------------------------
# the aggregation paths
# ---------------------------------------------------------------------------------------------------------------------
def fused_sync_step(w, grads: Sequence, mask: int, scale, drop: Optional[Tuple[int, int, float]] = None) -> np.ndarray:
    """fused_sync_sgd_kernel (peer-load path) and the interval apply: the contributors in ``mask`` summed in rank order
    (``grads[q]`` is rank q's arena), then SGD.  ``drop = (seed, step, keep_prob)`` masks every contributor first."""
    w = f32(w)
    terms = []
    for q in ranks(mask, len(grads)):
        g = f32(grads[q])
        if drop is not None:
            g = np.where(drop_keep(drop[0], drop[1], q, drop[2], g.size), g, np.float32(0))
        terms.append(g)
    return sgd(w, seq_sum(terms), scale)


def late_bucket_rounds_bf16(numel: int, early_len: int, late_ll: bool, late_bf16: bool) -> bool:
    """Does the late bucket of csrc/fused_bucket.cu carry bf16?  LL lines are used up to 1 MB of late bucket."""
    return bool(late_ll and late_bf16 and (numel - early_len) * 4 <= (1 << 20))


def bucket_step(w, grads: Sequence, g16: Sequence, early: Tuple[int, int], scale, late_bf16: bool) -> np.ndarray:
    """csrc/fused_bucket.cu, every replica contributing.  Early bucket ``[early)``: the fp32 rank-ordered sum of the
    replicas' bf16 gradients ``g16[q]``, rounded to bf16, then SGD.  Late bucket (the rest of the arena): the rank-ordered
    fp32 sum of the replicas' gradients -- each rounded to bf16 first when the LL lines carry bf16 -- then SGD."""
    w = f32(w)
    b, e = early
    out = w.copy()
    out[b:e] = sgd(w[b:e], rne_bf16(seq_sum([f32(x) for x in g16])), scale)
    late = np.r_[0:b, e:w.size]
    terms = [rne_bf16(f32(g)[late]) if late_bf16 else f32(g)[late] for g in grads]
    out[late] = sgd(w[late], seq_sum(terms), scale)
    return out


def interval_accumulate(grads_in_order: Sequence) -> np.ndarray:
    """iv_accumulate_kernel over one tick: the first gradient overwrites, each later one is added to it."""
    acc = f32(grads_in_order[0]).copy()
    for g in grads_in_order[1:]:
        acc = f32(g) + acc
        assert_no_subnormal("accumulate", acc)
    return acc


# ---------------------------------------------------------------------------------------------------------------------
# asynchronous SGD (csrc/fused_async.cu)
# ---------------------------------------------------------------------------------------------------------------------
def ftz(x) -> np.ndarray:
    """Subnormal fp32 values flushed to a zero of their sign, as the kernels' FTZ arithmetic flushes operands and results."""
    x = f32(x)
    return np.where(np.abs(x) < np.float32(FLT_MIN), np.copysign(np.float32(0), x), x).astype(np.float32)


def async_update(g, scale) -> np.ndarray:
    """The update as_apply_kernel adds to every master copy: ``-fl(scale * g)``, one fp32 product (``__fmul_rn``, FTZ)."""
    return -ftz(np.float32(scale) * ftz(g))


def async_apply(w, xs: Sequence) -> np.ndarray:
    """A master copy after the updates ``xs`` (each from :func:`async_update`) landed in that order: one fp32 add per
    update, with the FTZ of the in-memory reduction (``REDG.E.ADD.F32x4.FTZ.RN``)."""
    w = ftz(w)
    for x in xs:
        w = ftz(w + f32(x))
    return w
