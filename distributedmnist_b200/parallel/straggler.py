"""Sampled straggler delays: the quantile tables behind ``--inject_straggler rank:exp|lognormal|profile:...`` and the
host emulation of the device sampler (``straggler_sample_kernel``, csrc/fused_sync.cu).

A distribution is compiled on the host into TABLE_POINTS ``uint32`` nanosecond points at probabilities
``(i + 0.5) / TABLE_POINTS``.  The delay of iteration ``j`` of a replica is drawn in integer arithmetic only:
``u = hash_mix(seed_mix, j)`` (the finaliser of ``dropout_keep``, csrc/common.cuh), segment ``u >> 22``, position
``(u >> 6) & 0xFFFF`` inside it, linear interpolation between the segment's two points in 64-bit integers.  ``j`` counts
the replica's own iterations and ``seed_mix`` is derived from ``--seed`` and the rank, so every replica draws from a
stream of its own and the device and this emulation agree to the nanosecond.
"""
from __future__ import annotations

import os
from typing import Optional, Sequence

import numpy as np

TABLE_POINTS = 1025
RING = 1024                        # device ring of (drawn, spun) pairs, indexed by j % RING
STATE_BYTES = 16 + 4 * RING + 8 * RING
MAX_DELAY_NS = 4_000_000_000       # every point fits a uint32 nanosecond count
_M32 = 0xFFFFFFFF


def table_probs() -> np.ndarray:
    return (np.arange(TABLE_POINTS, dtype=np.float64) + 0.5) / TABLE_POINTS


def delay_limit_ns(sync_timeout_ms: Optional[float] = None) -> int:
    """Largest table point allowed: a quarter of the device watchdog (a drawn delay never gets near it), at most 4 s."""
    if sync_timeout_ms is None:
        return MAX_DELAY_NS
    return min(MAX_DELAY_NS, int(float(sync_timeout_ms) * 1e6 / 4))


def _to_table(points_us: np.ndarray, what: str, limit_ns: int) -> np.ndarray:
    ns = np.rint(np.asarray(points_us, dtype=np.float64) * 1e3)
    if not np.all(np.isfinite(ns)) or ns.min() < 0:
        raise ValueError("--inject_straggler %s: the quantile table has negative or non-finite points" % what)
    if ns.max() > limit_ns:
        raise ValueError("--inject_straggler %s: its largest delay, %.0f us, exceeds the limit of %.0f us "
                         "(--sync_timeout_ms / 4, at most 4 s)" % (what, ns.max() / 1e3, limit_ns / 1e3))
    return ns.astype(np.uint32)


def parametric_table(dist: str, params: Sequence[float], limit_ns: int = MAX_DELAY_NS) -> np.ndarray:
    """``exp`` (mean us) or ``lognormal`` (median us, sigma) -> quantile table via scipy's ``ppf``."""
    from scipy import stats
    if dist == "exp":
        law = stats.expon(scale=params[0])
    elif dist == "lognormal":
        law = stats.lognorm(s=params[1], scale=params[0])
    else:
        raise ValueError("--inject_straggler: unknown distribution %r" % dist)
    return _to_table(law.ppf(table_probs()), "%s:%s" % (dist, ":".join("%g" % p for p in params)), limit_ns)


def load_profile(path: str) -> np.ndarray:
    """Delays in microseconds from a ``.npy`` file or a whitespace-separated text file."""
    if not os.path.isfile(path):
        raise ValueError("--inject_straggler profile: no such file %r" % path)
    try:
        d = np.load(path) if path.endswith(".npy") else np.loadtxt(path, ndmin=1)
    except (OSError, ValueError) as e:
        raise ValueError("--inject_straggler profile %r: cannot read it (%s)" % (path, e))
    d = np.asarray(d, dtype=np.float64).reshape(-1)
    if d.size == 0 or not np.all(np.isfinite(d)) or d.min() < 0:
        raise ValueError("--inject_straggler profile %r: wants a non-empty list of finite, non-negative delays (us)" % path)
    return d


def profile_table(path: str, limit_ns: int = MAX_DELAY_NS) -> np.ndarray:
    return _to_table(np.quantile(load_profile(path), table_probs()), "profile:%s" % path, limit_ns)


def seed_mix(seed: int, rank: int) -> int:
    """Per-replica stream key from ``--seed`` and the rank (hashed, so neighbouring ranks' streams are unrelated)."""
    x = (int(seed) * 0x632BE5AB + int(rank) * 0x85EBCA77 + 0x53545247) & _M32
    return int(hash_mix(x, np.zeros(1, dtype=np.uint64))[0])


def hash_mix(seed: int, j) -> np.ndarray:
    """csrc/common.cuh ``hash_mix`` over an array of indices (uint64 holding 32-bit values)."""
    x = (np.asarray(j, dtype=np.uint64) * np.uint64(0x9E3779B1) + np.uint64(seed & _M32)) & np.uint64(_M32)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x85EBCA6B)) & np.uint64(_M32)
    x ^= x >> np.uint64(13)
    x = (x * np.uint64(0xC2B2AE35)) & np.uint64(_M32)
    x ^= x >> np.uint64(16)
    return x


def sample_ns(table: np.ndarray, mix: int, j) -> np.ndarray:
    """Delays (ns, uint32) of iterations ``j`` of the replica keyed ``mix``: what the device sampler draws."""
    u = hash_mix(mix, np.atleast_1d(np.asarray(j, dtype=np.uint64)) & np.uint64(_M32))
    seg = (u >> np.uint64(22)).astype(np.int64)
    frac = (u >> np.uint64(6)) & np.uint64(0xFFFF)
    t = np.asarray(table, dtype=np.uint64)
    lo, hi = t[seg], t[seg + 1]
    return (lo + (((hi - lo) * frac) >> np.uint64(16))).astype(np.uint32)
