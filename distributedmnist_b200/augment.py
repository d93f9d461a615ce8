"""Random affine augmentation of the training images (``--augment_max_shift``, ``--augment_max_rotation``,
``--augment_max_scale``): small shifts, rotations and zooms, as Keras's ``ImageDataGenerator`` and torchvision's
``RandomAffine`` provide them.  Training batches only: no evaluation is ever augmented, and labels are unchanged.

The transform, defined here once (csrc/augment.cu computes the same one in fp32 on the device):

* Row ``b`` of replica ``r`` at augmentation iteration ``i`` draws four uniforms ``u_k = (h_k >> 8) * 2^-24`` with
  ``h_k = hash_mix(hash_mix(seed_mix(seed, r), i), 4 b + k)``, ``hash_mix`` the murmur3 finaliser the dropout mask uses
  (models/lenet.py), keyed by a mixing constant of its own so the draws are independent of dropout's.  A row's draws do
  not depend on the batch size.
* ``theta = R pi/180 (2 u0 - 1)``, ``s = 1 + S (2 u1 - 1)``, ``tx = T (2 u2 - 1)``, ``ty = T (2 u3 - 1)``.
* Output pixel ``(x, y)`` samples the source bilinearly at the inverse map around the centre ``c = 13.5``:
  ``sx = c + a dx + b dy``, ``sy = c - b dx + a dy`` with ``a = cos(theta) / s``, ``b = sin(theta) / s``,
  ``dx = x - c - tx``, ``dy = y - c - ty``.  A tap outside ``[0, 27]^2`` reads the background ``BACKGROUND = -0.5``, the
  value of a zero pixel after data.py's ``(x - 127.5) / 255`` scaling.

Elastic distortion (``--augment_elastic_alpha``, ``--augment_elastic_sigma``; Simard, Steinkraus and Platt, "Best
practices for convolutional neural networks applied to visual document analysis", 2003), csrc/augment_elastic.cu:

* Row ``b`` of replica ``r`` at iteration ``i`` draws ``2 x 784`` uniforms ``v = 2 u - 1``, ``u = (h >> 8) * 2^-24``
  with ``h = hash_mix(hash_mix(E, i), 1568 b + 784 d + p)``, ``E = seed_mix(seed, r) + ELASTIC_MIX (mod 2^32)``, ``d``
  0 for the x component and 1 for y, ``p = 28 y + x``.  The batch is limited to ``MAX_ELASTIC_BATCH`` rows so that the
  index fits in u32.  The affine draws above do not change.
* Each component is smoothed by the normalised Gaussian of width ``sigma`` (:func:`gaussian_weights`, radius
  ``R = floor(4 sigma + 0.5)``, taps outside the image read 0: ``scipy.ndimage.gaussian_filter(v, sigma,
  mode="constant", cval=0, truncate=4)``) and scaled by ``alpha``: the displacement ``(ex, ey)`` in pixels.
* Output pixel ``(x, y)`` is first displaced to ``(x + ex, y + ey)``, which the affine inverse map above then takes
  in place of ``(x, y)``; the bilinear sample and the background are those above.

``i`` counts the replica's training iterations, so two iterations of one run never share draws.  A restarted run starts
it past the iterations that went into the restored global step (:func:`start_iteration`), so a one-replica run does
not replay the draws of the steps it restored; a multi-replica K > N run or an interval run can repeat some (see
there).  Nothing enters the checkpoint.

The numpy hash here is exact (integer arithmetic); :func:`warp` is the float64 warp.  The torch engine applies
:func:`augment_batch`; the tests compare the kernel's draws and pixels against both.
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import numpy as np

_M32 = 0xFFFFFFFF
CENTRE = 13.5
BACKGROUND = -0.5
MAX_SHIFT = 8.0                 # pixels
MAX_ROTATION = 180.0            # degrees
RANK_MIX = 0x297A2D39           # seed_mix(seed, r + 1) = seed_mix(seed, r) + RANK_MIX (mod 2^32)
# the elastic key's offset from the affine key; not k * RANK_MIX (mod 2^32) for |k| < 1024, so no replica's elastic key
# is any replica's affine key in a run of up to 1024 replicas
ELASTIC_MIX = 0x6A09E667
ELASTIC_DRAWS = 2 * 784         # draws per row: the x then the y component, pixel-major
MAX_ELASTIC_BATCH = 2 ** 32 // ELASTIC_DRAWS    # rows whose every draw index 1568 b + 784 d + p fits in u32
MAX_ALPHA = 64.0                # pixels
MIN_SIGMA, MAX_SIGMA = 0.5, 8.0     # the radius floor(4 sigma + 0.5) is then at most 32
DEFAULT_SIGMA = 4.0             # Simard et al.'s width


class Elastic(NamedTuple):
    alpha: float                # scale of the smoothed field, pixels
    sigma: float                # width of the Gaussian, pixels


class Ranges(NamedTuple):
    max_shift: float            # T, pixels
    max_rotation: float         # R, degrees
    max_scale: float            # S


def seed_mix(seed: int, rank: int) -> int:
    """The per-replica key of the draws (constants distinct from models/lenet.py's ``dropout_seed_mix``)."""
    return (seed * 0x2C1B3C6D + rank * RANK_MIX + 0x5BD1E995) & _M32


def hash_mix(key, idx):
    """csrc/common.cuh ``hash_mix`` on uint64 arrays (or ints) holding u32 values."""
    x = (np.asarray(idx, dtype=np.uint64) * np.uint64(0x9E3779B1) + np.uint64(key)) & np.uint64(_M32)
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x85EBCA6B)) & np.uint64(_M32)
    x ^= x >> np.uint64(13)
    x = (x * np.uint64(0xC2B2AE35)) & np.uint64(_M32)
    x ^= x >> np.uint64(16)
    return x


def uniforms(mix: int, iteration: int, rows: int) -> np.ndarray:
    """float64 ``[rows, 4]``: the draws ``u0..u3`` of rows ``0..rows-1`` at ``iteration`` (each a multiple of 2^-24 in
    [0, 1), exact in fp32)."""
    key = int(hash_mix(mix, int(iteration) & _M32))
    idx = (np.arange(rows, dtype=np.uint64)[:, None] * np.uint64(4) + np.arange(4, dtype=np.uint64)[None, :]) \
        & np.uint64(_M32)
    return (hash_mix(key, idx) >> np.uint64(8)).astype(np.float64) * 2.0 ** -24


def coefficients(u: np.ndarray, ranges: Ranges):
    """``(a, b, tx, ty)``, float64 ``[rows]`` each, of the draws ``u`` ``[rows, 4]``."""
    T, R, S = (float(v) for v in (ranges.max_shift, ranges.max_rotation, ranges.max_scale))
    theta = R * math.pi / 180.0 * (2.0 * u[:, 0] - 1.0)
    s = 1.0 + S * (2.0 * u[:, 1] - 1.0)
    return np.cos(theta) / s, np.sin(theta) / s, T * (2.0 * u[:, 2] - 1.0), T * (2.0 * u[:, 3] - 1.0)


def affine(theta, scale, tx, ty):
    """``(a, b, tx, ty)`` of a rotation by ``theta`` (radians) and a zoom ``scale``, as float64 arrays."""
    theta, scale = np.asarray(theta, dtype=np.float64), np.asarray(scale, dtype=np.float64)
    return np.cos(theta) / scale, np.sin(theta) / scale, np.asarray(tx, np.float64), np.asarray(ty, np.float64)


def gaussian_weights(sigma: float) -> np.ndarray:
    """float64 ``[R + 1]``: the normalised Gaussian's taps ``w_0 .. w_R`` (``w_-k = w_k``), ``R = floor(4 sigma + 0.5)``,
    ``w_k = exp(-k^2 / 2 sigma^2) / sum_{|j| <= R} exp(-j^2 / 2 sigma^2)`` (scipy.ndimage's ``truncate=4`` kernel)."""
    sigma = float(sigma)
    radius = int(4.0 * sigma + 0.5)
    w = np.exp(-0.5 / (sigma * sigma) * np.arange(-radius, radius + 1, dtype=np.float64) ** 2)
    return (w / w.sum())[radius:]


def elastic_uniforms(mix: int, iteration: int, rows: int) -> np.ndarray:
    """float64 ``[rows, 2, 784]``: the elastic draws ``v = 2 u - 1`` of rows ``0..rows-1`` at ``iteration`` under the
    replica's affine key ``mix`` (component 0: x, 1: y; each exact in fp32)."""
    if rows > MAX_ELASTIC_BATCH:
        raise ValueError("elastic distortion draws %d values per row: at most %d rows, got %d"
                         % (ELASTIC_DRAWS, MAX_ELASTIC_BATCH, rows))
    key = int(hash_mix((int(mix) + ELASTIC_MIX) & _M32, int(iteration) & _M32))
    idx = np.arange(rows * ELASTIC_DRAWS, dtype=np.uint64).reshape(rows, 2, 784)
    return (hash_mix(key, idx) >> np.uint64(8)).astype(np.float64) * 2.0 ** -23 - 1.0


def elastic_field(mix: int, iteration: int, rows: int, elastic: Elastic) -> np.ndarray:
    """float64 ``[rows, 2, 28, 28]``: the displacement ``(ex, ey)`` in pixels of rows ``0..rows-1`` at ``iteration``,
    ``alpha G V G^T`` with ``G`` the banded 28 x 28 matrix of :func:`gaussian_weights` (taps outside the image read 0)."""
    w = gaussian_weights(elastic.sigma)
    k = np.abs(np.arange(28)[:, None] - np.arange(28)[None, :])
    g = np.where(k < len(w), w[np.minimum(k, len(w) - 1)], 0.0)
    v = elastic_uniforms(mix, iteration, rows).reshape(rows, 2, 28, 28)
    return float(elastic.alpha) * (g @ v @ g.T)


def warp(images: np.ndarray, a, b, tx, ty, centre: float = CENTRE, field=None) -> np.ndarray:
    """The float64 warp of ``images`` (``[rows, 28, 28]`` or ``[rows, 784]``, row-major y, x) with per-row coefficients;
    returns float64 ``[rows, 28, 28]``.  ``centre``: the transform's is ``CENTRE`` (the tests warp about others to show
    that their bounds tell the two apart).  ``field``: None, or the elastic displacement ``[rows, 2, 28, 28]`` (or
    ``[rows, 2, 784]``) that moves each output pixel before the affine map."""
    img = np.asarray(images, dtype=np.float64).reshape(-1, 28, 28)
    n = img.shape[0]
    a, b, tx, ty = (np.broadcast_to(np.asarray(v, dtype=np.float64), (n,))[:, None, None] for v in (a, b, tx, ty))
    y, x = np.meshgrid(np.arange(28, dtype=np.float64), np.arange(28, dtype=np.float64), indexing="ij")
    if field is None:
        dx, dy = x[None] - centre - tx, y[None] - centre - ty
    else:
        f = np.asarray(field, dtype=np.float64).reshape(n, 2, 28, 28)
        dx, dy = (x[None] + f[:, 0]) - centre - tx, (y[None] + f[:, 1]) - centre - ty
    sx = centre + a * dx + b * dy
    sy = centre - b * dx + a * dy
    x0, y0 = np.floor(sx), np.floor(sy)
    fx, fy = sx - x0, sy - y0
    pad = np.pad(img, ((0, 0), (1, 1), (1, 1)), constant_values=BACKGROUND)     # index 0 and 29: background

    def tap(yy, xx):
        inside = (yy >= 0) & (yy <= 27) & (xx >= 0) & (xx <= 27)
        yi = np.where(inside, yy, -1).astype(np.int64) + 1
        xi = np.where(inside, xx, -1).astype(np.int64) + 1
        return pad[np.arange(n)[:, None, None], yi, xi]

    v00, v01, v10, v11 = tap(y0, x0), tap(y0, x0 + 1), tap(y0 + 1, x0), tap(y0 + 1, x0 + 1)
    return (1.0 - fy) * ((1.0 - fx) * v00 + fx * v01) + fy * ((1.0 - fx) * v10 + fx * v11)


def augment_batch(images: np.ndarray, mix: int, iteration: int, ranges: Ranges,
                  elastic: Optional[Elastic] = None) -> np.ndarray:
    """The augmented batch (float64 warp from the float64 coefficients and, with ``elastic``, the float64 field, rounded
    to fp32), in the shape of ``images``."""
    img = np.asarray(images)
    n = img.shape[0]
    u = uniforms(mix, iteration, n)
    field = None if elastic is None else elastic_field(mix, iteration, n, elastic)
    return warp(img, *coefficients(u, ranges), field=field).astype(np.float32).reshape(img.shape)


def start_iteration(restored_step: int, count_triggered: bool, k: int, n: int) -> int:
    """The first iteration a run restored at global step ``restored_step`` draws from (u32).

    A synchronous run with K <= N gradients per update (``count_triggered``: mode A; ``k``, ``n``: K and the number of
    replicas) computes at most one iteration per replica per global step, so its replicas used iterations below the
    restored step.  With K > N each step commits once K gradients computed on its weights are accumulated, and the start
    is ``k * restored_step``.  On one replica that is exact: every step takes exactly K iterations.

    With K > N on more than one replica it is not a bound.  A replica counts at most K iterations of a step (the close
    that brings its own count to K sees the sum reach K, so the step commits).  But once another replica has committed
    the step, this one keeps computing iterations on the step's weights until the committer's pushes have landed
    (``iv_adopt`` waits for the ``done`` flag), and the gate drops each of them; each still advances the counter.  How
    many such stale iterations run depends on timing, not on the global step, so a restarted multi-replica K > N run can
    repeat some draws of the run it restored.

    Interval and cdf runs start at the restored step.  An interval replica's iteration count follows a wall-clock
    deadline and is not a function of the global step either, so a restarted interval run can repeat draws too."""
    return (int(restored_step) * (int(k) if count_triggered and k > n else 1)) & _M32


def check_ranges(ranges: Ranges) -> None:
    """Raises ValueError unless every range is finite and within bounds."""
    for name, v, hi, closed in (("--augment_max_shift", ranges.max_shift, MAX_SHIFT, True),
                                ("--augment_max_rotation", ranges.max_rotation, MAX_ROTATION, True),
                                ("--augment_max_scale", ranges.max_scale, 1.0, False)):
        v = float(v)
        if not math.isfinite(v) or v < 0.0 or (v > hi if closed else v >= hi):
            raise ValueError("%s must be finite and lie in [0, %g%s (0 = off), got %r" % (name, hi, "]" if closed else ")", v))


def from_flags(flags) -> Optional[Ranges]:
    """The three ranges, or None when augmentation is off (all 0).  Raises ValueError on a value out of range."""
    r = Ranges(*(float(getattr(flags, "augment_" + k, 0.0) or 0.0) for k in ("max_shift", "max_rotation", "max_scale")))
    check_ranges(r)
    return r if any(r) else None


def check_elastic(elastic: Elastic) -> None:
    """Raises ValueError unless alpha and sigma are finite and within bounds."""
    a, s = float(elastic.alpha), float(elastic.sigma)
    if not math.isfinite(a) or not 0.0 <= a <= MAX_ALPHA:
        raise ValueError("--augment_elastic_alpha must be finite and lie in [0, %g] (0 = off), got %r" % (MAX_ALPHA, a))
    if not math.isfinite(s) or not MIN_SIGMA <= s <= MAX_SIGMA:
        raise ValueError("--augment_elastic_sigma must be finite and lie in [%g, %g], got %r" % (MIN_SIGMA, MAX_SIGMA, s))


def elastic_from_flags(flags) -> Optional[Elastic]:
    """``Elastic(alpha, sigma)``, or None when elastic distortion is off (alpha 0).  Raises ValueError on a value out of
    range, and on a sigma other than the default without an alpha: it would change nothing."""
    e = Elastic(float(getattr(flags, "augment_elastic_alpha", 0.0) or 0.0),
                float(getattr(flags, "augment_elastic_sigma", DEFAULT_SIGMA)))
    check_elastic(e)
    if e.alpha == 0.0:
        if e.sigma != DEFAULT_SIGMA:
            raise ValueError("--augment_elastic_sigma needs --augment_elastic_alpha > 0: without an alpha there is no "
                             "field for it to smooth")
        return None
    return e


def check_flags(flags) -> None:
    """The augmentation flags, checked before any device work starts."""
    from_flags(flags)
    elastic_from_flags(flags)


def describe(r: Ranges, elastic: Optional[Elastic] = None) -> str:
    s = "shift up to %g px, rotation up to %g degrees, zoom in [%g, %g]" % (r.max_shift, r.max_rotation,
                                                                          1.0 - r.max_scale, 1.0 + r.max_scale)
    if elastic is not None:
        s += ", elastic distortion alpha %g px, sigma %g px" % (elastic.alpha, elastic.sigma)
    return s
