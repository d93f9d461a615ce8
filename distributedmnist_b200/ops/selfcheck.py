"""Numerics self-checks of the sm_90a LeNet and MLP kernels against float64 references (``ops/refs.py``).

Each check returns ``(name, error, tolerance)`` tuples; ``tests/test_lenet_kernels_gpu.py``,
``tests/test_kernel_refs_gpu.py`` and ``tests/test_mlp_kernels_gpu.py`` assert on them and ``tools/gpu_diag_lenet.py`` prints them all (one GPU call gives the
full picture when bringing a kernel up).  Every kernel-level check runs on exact-grid data (bitwise comparisons) and on
continuous random data (precision bounds); see ``refs.py`` for the rule.  ``stale_B`` runs a slot-reduced kernel at
that batch first, so the check's own launch finds stale partial sums in the workspace and a ticket last reset by a
launch with a different CTA count.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ..models import dropout_keep_mask, dropout_seed_mix, get_model, lenet_forward, loss_and_accuracy
from ..models.lenet import dropout_threshold
from ..parallel.context import ReplicaContext
from ..parallel.fused import FusedBackend
from . import aggrefs as A
from . import gemm as G
from . import refs as R
from .lib import load, stream_ptr

Result = Tuple[str, float, float]
KINDS = ("grid", "rand")
BF = torch.bfloat16


def _gen(seed: int) -> torch.Generator:
    return torch.Generator(device="cpu").manual_seed(seed)


def _bf(t: torch.Tensor) -> torch.Tensor:
    return t.to(BF)


def _dev(*ts):
    return [t.cuda() for t in ts]


# ---------------------------------------------------------------------------------------------------------------------
# references of large batches, a chunk of rows at a time
# ---------------------------------------------------------------------------------------------------------------------
REF_ROWS = 1024        # batch rows per float64 reference evaluation: a conv1 activation of 1024 rows is 206 MB in float64


def row_slices(B: int) -> List[slice]:
    return [slice(r, min(B, r + REF_ROWS)) for r in range(0, B, REF_ROWS)]


def merge_row_chunks(parts: Sequence[List[Result]], rows: Sequence[int]) -> List[Result]:
    """The results of the same comparisons on row chunks of the same outputs, as if made on the whole outputs: counts add
    up, ``[inexact]`` fractions are weighted by rows (each row holds as many elements), ``[err/bound]`` ratios take the
    maximum.  A normwise ``[rel]`` error does not split into chunks and is refused."""
    if len(parts) == 1:
        return list(parts[0])
    merged: List[Result] = []
    for i, (name, _, tol) in enumerate(parts[0]):
        assert all(p[i][0] == name and p[i][2] == tol for p in parts), name
        vals = [p[i][1] for p in parts]
        if name.endswith("[inexact]"):
            v = sum(x * n for x, n in zip(vals, rows)) / sum(rows)
        elif name.endswith("[err/bound]"):
            v = max(vals)
        elif name.endswith("[rel]"):
            raise ValueError("%s: a normwise error does not split into row chunks" % name)
        else:
            v = sum(vals)
        merged.append((name, float(v), tol))
    return merged


def by_rows(fn, B: int, *rows: torch.Tensor) -> List[Result]:
    """``fn`` on chunks of REF_ROWS batch rows of each tensor in ``rows``, its results merged (:func:`merge_row_chunks`)."""
    slices = row_slices(B)
    return merge_row_chunks([fn(*(t[s] for t in rows)) for s in slices], [s.stop - s.start for s in slices])


def sum_by_rows(fn, B: int, *rows: torch.Tensor):
    """The float64 sum over chunks of REF_ROWS batch rows of ``fn``'s results (a tensor or a tuple of tensors): a weight
    gradient reference over the whole batch without the whole batch's float64 activations."""
    total = None
    for s in row_slices(B):
        r = fn(*(t[s] for t in rows))
        total = r if total is None else (tuple(a + b for a, b in zip(total, r)) if isinstance(r, tuple) else total + r)
    return total


# ---------------------------------------------------------------------------------------------------------------------
# launchers: one kernel, fresh outputs
# ---------------------------------------------------------------------------------------------------------------------
def run_conv1_fwd(x, w, b):
    """x [B,28,28] fp32, w [5,5,1,32] fp32, b [32] -> (pooled bf16 [B,14,14,32], code, the cleared junk range)."""
    B = x.shape[0]
    out = torch.zeros(B, 14, 14, 32, dtype=BF, device="cuda")
    code = torch.zeros(B, 14, 14, 32, dtype=torch.uint8, device="cuda")
    junk = torch.ones(100, device="cuda")
    load().dm_conv1_fwd_tc(x, w, b, out, code, B, junk, 100, None, 0, None, 0, stream_ptr())
    return out, code, junk


def run_conv1_wgrad(x, dpool, code, tc: bool = True):
    """``tc``: the wgmma kernel, the only conv1 weight gradient there is (False, the removed SIMT kernel, is an error)."""
    if not tc:
        raise ValueError("the SIMT conv1 weight-gradient kernel was removed: only tc=True exists")
    B = x.shape[0]
    gw, gb = torch.zeros(25, 32, device="cuda"), torch.zeros(32, device="cuda")
    load().dm_conv1_wgrad_tc(x, dpool, code, gw, gb, B, stream_ptr())
    return gw, gb


def _output(shape, dtype, guard: int = 0) -> torch.Tensor:
    """A zeroed output buffer; with ``guard`` > 0 the head of an allocation ``guard`` elements longer, all of it poison:
    NaN, or 0xFF for pooling codes (a code is an argmax position 0-3 plus the ReLU flag 4).  ``unwritten_results``
    then finds every element the kernel left alone and every element it wrote past the end."""
    if not guard:
        return torch.zeros(shape, dtype=dtype, device="cuda")
    n = int(np.prod(shape))
    fill = 0xFF if dtype == torch.uint8 else float("nan")
    return torch.full((n + guard,), fill, dtype=dtype, device="cuda")[:n].view(shape)


def unwritten_results(tag: str, t: torch.Tensor, guard: int) -> List[Result]:
    """Poison left inside ``t`` (elements never written) and guard elements past its end that are no longer poison
    (writes out of bounds); both must be 0.  ``t`` comes from ``_output(..., guard)``."""
    full = torch.as_strided(t, (t.numel() + guard,), (1,), t.storage_offset())
    poison = full == 0xFF if t.dtype == torch.uint8 else torch.isnan(full)
    n = t.numel()
    return [(tag + ".unwritten", float(poison[:n].sum()), 0.0),
            (tag + ".written_past_end", float((~poison[n:]).sum()), 0.0)]


def run_conv2_fwd(a1, w, b, guard: int = 0):
    """``guard``: see ``_output``."""
    B = a1.shape[0]
    out = _output((B, 7, 7, 64), BF, guard)
    code = _output((B, 7, 7, 64), torch.uint8, guard)
    load().dm_conv2_fwd(a1, w, b, out, code, B, stream_ptr())
    return out, code


def run_conv2_dgrad(dy, w, guard: int = 0):
    """``guard``: see ``_output``."""
    dx = _output((dy.shape[0], 14, 14, 32), BF, guard)
    load().dm_conv2_dgrad(dy, w, dx, dy.shape[0], stream_ptr())
    return dx


def run_conv2_wgrad(a1, dy):
    gw = torch.zeros(5, 5, 32, 64, device="cuda")
    load().dm_conv2_wgrad(a1, dy, gw, a1.shape[0], stream_ptr())
    return gw


FC1_SPLITS = 7


def run_fc1_fwd(a2, w1):
    """fc1 forward as the engine issues it: split-K over 7 CTAs, partial tiles stored side by side."""
    B = a2.shape[0]
    part = torch.full((FC1_SPLITS, B, 512), 7.0, device="cuda")         # every element must be overwritten
    G.gemm_bf16_raw(a2, w1, part, B, 512, 3136, 3136, 512, 512, False, True, G.EPI_STORE_F32, splits=FC1_SPLITS, bn=64,
                    split_stride=part.stride(0))
    return part


def run_fc2_fwd_bwd(parts, b1, w2, b2, labels, train: bool = True, mix0: int = 0, step: int = 0, keep_prob: float = 0.5):
    lib, B = load(), labels.shape[0]
    o = dict(dh=torch.zeros(B, 512, dtype=BF, device="cuda"), h=torch.zeros(B, 512, device="cuda"),
             dl=torch.zeros(B, 12, device="cuda"), la=torch.zeros(2, device="cuda"), logits=torch.zeros(B, 10, device="cuda"))
    st = torch.tensor([step], dtype=torch.int32, device="cuda")
    lib.dm_fc2_fwd_bwd(parts, parts.stride(0), parts.shape[0], b1, w2, b2, labels, o["dh"], o["h"], o["dl"], o["la"],
                       o["logits"], B, int(train), mix0, st, keep_prob, stream_ptr())
    return o


def run_fc2_wgrad(h, dl, dh):
    gw2, gb2, gb1 = torch.full((512, 10), 7.0, device="cuda"), torch.full((10,), 7.0, device="cuda"), \
        torch.full((512,), 7.0, device="cuda")                          # plain stores: stale contents must not matter
    load().dm_fc2_wgrad(h, dl, dh, gw2, gb2, gb1, h.shape[0], stream_ptr())
    return gw2, gb2, gb1


def run_fc1_wgrad(a2, dh, bf16_out: bool = False):
    """dW1 [3136,512] = a2^T dh (both MN-major, K = batch), 128-wide tiles as the engine issues it."""
    B = a2.shape[0]
    out = torch.full((3136, 512), 7.0, device="cuda").to(BF if bf16_out else torch.float32)
    G.gemm_bf16_raw(a2, dh, out, 3136, 512, B, 3136, 512, 512, True, True,
                    G.EPI_STORE_BF16 if bf16_out else G.EPI_STORE_F32, bn=128)
    return out


def run_fc1_wgrad_decay(a2, dh, w1, lam: float, bf16_out: bool = False, part=None):
    """dW1 + lambda W1 (dm_gemm_bf16_decay) as the engine issues it: (output, W^2 partial of each CTA).  ``w1``: the fp32
    weights, read through its data pointer as [3136][512] (a larger buffer holds rows the kernel must not read).  ``part``:
    the partials' workspace (default: a fresh NaN-filled one)."""
    lib, B = load(), a2.shape[0]
    out = torch.full((3136, 512), 7.0, device="cuda").to(BF if bf16_out else torch.float32)
    if part is None:
        part = torch.full((int(lib.dm_gemm_decay_ctas(3136, 512)),), float("nan"), dtype=torch.float64, device="cuda")
    lib.dm_gemm_bf16_decay(a2, dh, out, 3136, 512, B, 3136, 512, 512, int(bf16_out), w1, float(lam), part, stream_ptr())
    return out, part


def run_fc2_wgrad_decay(h, dl, dh, w2, b2, b1, lam: float, part=None):
    """fc2_wgrad<true>: (g_w2, g_b2, g_b1, W^2 partial of each CTA); stale output contents must not matter."""
    lib = load()
    gw2, gb2, gb1 = torch.full((512, 10), 7.0, device="cuda"), torch.full((10,), 7.0, device="cuda"), \
        torch.full((512,), 7.0, device="cuda")
    if part is None:
        part = torch.full((int(lib.dm_fc2_wgrad_decay_ctas()),), float("nan"), dtype=torch.float64, device="cuda")
    lib.dm_fc2_wgrad_decay(h, dl, dh, gw2, gb2, gb1, h.shape[0], w2, b2, b1, float(lam), part, stream_ptr())
    return gw2, gb2, gb1, part


def run_fc1_dgrad_unpool(dh, w1, code2, guard: int = 0):
    """``guard``: see ``_output`` (without it dy2 starts out as 7, which every element must overwrite)."""
    B = dh.shape[0]
    if guard:
        dy = _output((B, 14, 14, 64), BF, guard)
    else:
        dy = torch.full((B, 14, 14, 64), 7.0, dtype=BF, device="cuda")
    gb = torch.zeros(64, device="cuda")
    load().dm_fc1_dgrad_unpool(dh, w1, code2, dy, gb, B, stream_ptr())
    return dy, gb


def _codes(g, shape) -> torch.Tensor:
    return (torch.randint(0, 4, shape, generator=g) | (torch.randint(0, 2, shape, generator=g) << 2)).to(torch.uint8)


def prime_workspace(kernel: str, B: int, seed: int = 99) -> None:
    """One launch of a slot-reduced kernel at batch B on random data, result discarded: leaves B-sized partial sums in its
    workspace and a ticket reset by a launch of that CTA count."""
    g = _gen(seed)
    if kernel == "conv1_wgrad_tc":
        x, dp, c = _dev(torch.rand(B, 28, 28, generator=g) - 0.5, _bf(torch.randn(B, 14, 14, 32, generator=g)),
                        _codes(g, (B, 14, 14, 32)))
        run_conv1_wgrad(x, dp, c)
    elif kernel == "conv2_wgrad":
        a1, dy = _dev(_bf(torch.rand(B, 14, 14, 32, generator=g)), _bf(torch.randn(B, 14, 14, 64, generator=g)))
        run_conv2_wgrad(a1, dy)
    elif kernel == "fc1_dgrad_unpool":
        dh, w1, c = _dev(_bf(torch.randn(B, 512, generator=g)), _bf(torch.randn(3136, 512, generator=g) * 0.05),
                         _codes(g, (B, 3136)))
        run_fc1_dgrad_unpool(dh, w1, c)
    elif kernel == "fc2_fwd_bwd":
        parts, b1, w2, b2, lab = _dev(torch.randn(1, B, 512, generator=g), torch.randn(512, generator=g),
                                      torch.randn(512, 10, generator=g), torch.randn(10, generator=g),
                                      torch.randint(0, 10, (B,), generator=g))
        run_fc2_fwd_bwd(parts, b1, w2, b2, lab)
    else:
        raise ValueError(kernel)


# ---------------------------------------------------------------------------------------------------------------------
# data with pooling ties, exact zeros and all-negative windows
# ---------------------------------------------------------------------------------------------------------------------
def mnist_like(g: torch.Generator, B: int) -> torch.Tensor:
    """[B,28,28] images as MNIST normalises them: an exact -0.5 background and a few strokes (values k/8, mostly 0.5)."""
    x = torch.full((B, 28, 28), -0.5)
    for b in range(B):
        for _ in range(3):
            r, c = (int(v) for v in torch.randint(2, 24, (2,), generator=g))
            n = int(torch.randint(4, 14, (1,), generator=g))
            val = float(torch.randint(0, 9, (1,), generator=g)) / 8 - 0.5 if int(torch.randint(0, 3, (1,), generator=g)) == 0 else 0.5
            if int(torch.randint(0, 2, (1,), generator=g)):
                x[b, r:r + 2, c:min(28, c + n)] = val
            else:
                x[b, r:min(28, r + n), c:c + 2] = val
    return x


def _conv1_data(kind: str, g, B: int):
    if kind == "rand":
        return torch.rand(B, 28, 28, generator=g) - 0.5, torch.randn(5, 5, 1, 32, generator=g) * 0.1, \
            torch.randn(32, generator=g) * 0.1
    w = R.grid(g, (5, 5, 1, 32), -16, 16, 64)
    b = R.grid(g, (32,), -16, 16, 64)
    if kind == "grid":
        return R.grid(g, (B, 28, 28), -4, 4, 8), w, b
    # edges: constant background -> ties in every background window; channels 0-7 cancel the background exactly (a
    # pre-activation of 0: ReLU flag off), channels 8-15 can never become positive (all-negative windows)
    s = w.sum((0, 1, 2))
    b[:8] = 0.5 * s[:8]
    b[8:16] = -4.0
    return mnist_like(g, B), w, b


def _conv2_data(kind: str, g, B: int):
    if kind == "rand":
        return _bf(torch.rand(B, 14, 14, 32, generator=g)), _bf(torch.randn(5, 5, 32, 64, generator=g) * 0.05), \
            torch.randn(64, generator=g) * 0.1
    w = R.grid(g, (5, 5, 32, 64), -8, 8, 64)
    b = R.grid(g, (64,), -32, 32, 64)
    if kind == "grid":
        return _bf(R.grid(g, (B, 14, 14, 32), 0, 4)), _bf(w), b
    # edges: per-channel constant background with a few blocks; channels 0-15 cancel the background exactly, 16-31 stay
    # negative everywhere
    bg = R.grid(g, (32,), 0, 2)
    a1 = bg.expand(B, 14, 14, 32).clone()
    for bi in range(B):
        r, c = (int(v) for v in torch.randint(0, 10, (2,), generator=g))
        a1[bi, r:r + 4, c:c + 3, :] = R.grid(g, (32,), 0, 4)
    s = (w * bg[None, None, :, None]).sum((0, 1, 2))
    b[:16] = -s[:16]
    b[16:32] = -(w.abs().sum((0, 1, 2))[16:32] * 4 + 1.0 / 64)
    return _bf(a1), _bf(w), b


# ---------------------------------------------------------------------------------------------------------------------
# kernel checks
# ---------------------------------------------------------------------------------------------------------------------
def _pool_results(tag: str, kind: str, out, code, z, za, bias, n_terms: int) -> List[Result]:
    ref = R.pool_fwd(z, bias)
    slack = R.windows(R.fp32_slack(za, n_terms))
    # the kernel adds the bias to its fp32 maximum (one more rounding); a near-tie may select the runner-up
    out_slack = 2 * slack.max(dim=-1).values + 2.0 ** -23 * ref["pre"].abs()
    res = R.compare(tag + ".out", "grid" if kind == "edges" else kind, out, ref["out"], out_slack)
    if kind == "edges":     # the data must actually hold what it is for
        ties = int((ref["win"] == ref["win"].max(dim=-1, keepdim=True).values).sum(-1).gt(1).sum())
        zeros, negative = int((ref["pre"] == 0).sum()), int((ref["win"].max(dim=-1).values + bias.double() < 0).sum())
        res.append((tag + ".edge_cases_missing(ties,zeros,all_negative)", float((ties == 0) + (zeros == 0) + (negative == 0)), 0.0))
    return res + R.cmp_pool(tag, "grid" if kind == "edges" else kind, code, ref, slack)


def conv1_fwd_results(tag: str, kind: str, x, w, b, out, code) -> List[Result]:
    """conv1_fwd's pooled output and codes from images x [B,28,28] fp32, weights w [5,5,1,32] fp32, bias b."""
    w = w.to(BF)                    # the kernel rounds its operands to bf16 (grid values are bf16 numbers already)

    def rows(x, out, code):
        x = x.to(BF)
        z = R.conv5x5(x[..., None], w)
        za = R.conv5x5(x.abs()[..., None], w.abs())
        if kind != "rand":
            R.assert_exact_grid(za + b.abs().double().max(), 1.0 / 512, tag)
        return _pool_results(tag, kind, out, code, z, za, b, 25)
    return by_rows(rows, x.shape[0], x, out, code)


def check_conv1_fwd(B: int = 8, seed: int = 0, kinds: Sequence[str] = KINDS) -> List[Result]:
    res: List[Result] = []
    for kind in kinds:
        tag = "conv1_fwd_tc.%s" % kind
        x, w, b = _conv1_data(kind, _gen(seed), B)
        x, w, b = _dev(x, w, b)
        out, code, junk = run_conv1_fwd(x, w, b)
        res += conv1_fwd_results(tag, kind, x, w, b, out, code)
        res.append((tag + ".zeroing", float(junk.abs().max()), 0.0))
    return res


check_conv1_fwd_tc = check_conv1_fwd       # the name the kernel tests call it by


def check_conv1_wgrad(B: int = 8, seed: int = 7, kinds: Sequence[str] = KINDS, stale_B: int = 0) -> List[Result]:
    """conv1 weight/bias gradient fused with the maxpool1/ReLU1 backward."""
    res: List[Result] = []
    for kind in kinds:
        tag = "conv1_wgrad_tc.%s" % kind
        g = _gen(seed)
        if kind == "rand":
            x, dp = torch.rand(B, 28, 28, generator=g) - 0.5, _bf(torch.randn(B, 14, 14, 32, generator=g) * 0.1)
        else:
            x, dp = R.grid(g, (B, 28, 28), -4, 4, 8), _bf(R.grid(g, (B, 14, 14, 32), -4, 4))
        x, dp, code = _dev(x, dp, _codes(g, (B, 14, 14, 32)))
        if stale_B:
            prime_workspace("conv1_wgrad_tc", stale_B)
        gw, gb = run_conv1_wgrad(x, dp, code)
        res += conv1_wgrad_results(tag, kind, x, dp, code, gw, gb)
    return res


def conv1_wgrad_results(tag: str, kind: str, x, dp, code, gw, gb) -> List[Result]:
    """conv1 weight [25,32] / bias gradients from images x [B,28,28] fp32, d pool1 output dp and pool1 codes."""
    xr = x.to(BF)                       # the kernel rounds the images to bf16
    rw, rb = sum_by_rows(R.conv1_wgrad, x.shape[0], xr, dp, code)
    if kind == "grid":
        aw, ab = sum_by_rows(lambda x, d, c: R.conv1_wgrad(x.abs(), d.abs(), c), x.shape[0], xr, dp, code)
        R.assert_exact_grid(aw, 1.0 / 8, tag + ".g_w")
        R.assert_exact_grid(ab, 1.0, tag + ".g_b")
    return R.compare(tag + ".g_w", kind, gw, rw) + R.compare(tag + ".g_b", kind, gb, rb)


def conv2_fwd_results(tag: str, kind: str, a1, w, b, out, code) -> List[Result]:
    """conv2_fwd's pooled output and codes [B,7,7,64] from a1 and the bf16 weights w."""
    def rows(a1, out, code):
        z, za = R.conv5x5(a1, w), R.conv5x5(a1.abs(), w.abs())
        if kind != "rand":
            R.assert_exact_grid(za + b.abs().double().max(), 1.0 / 64, tag)
        return _pool_results(tag, kind, out, code, z, za, b, 800)
    return by_rows(rows, a1.shape[0], a1, out, code)


def check_conv2_fwd(B: int = 8, seed: int = 1, kinds: Sequence[str] = KINDS, guard: int = 0) -> List[Result]:
    """``guard`` > 0: the outputs start out as poison with a poisoned guard tail (``_output``), and the check also counts
    elements left unwritten or written past the end."""
    res: List[Result] = []
    for kind in kinds:
        tag = "conv2_fwd.%s" % kind
        a1, w, b = _dev(*_conv2_data(kind, _gen(seed), B))
        out, code = run_conv2_fwd(a1, w, b, guard)
        res += conv2_fwd_results(tag, kind, a1, w, b, out, code)
        if guard:
            res += unwritten_results(tag + ".out", out, guard) + unwritten_results(tag + ".code", code, guard)
    return res


def conv2_dgrad_results(tag: str, kind: str, dy, w, dx) -> List[Result]:
    def rows(dy, dx):
        ref, ra = R.conv5x5_dgrad(dy, w), R.conv5x5_dgrad(dy.abs(), w.abs())
        if kind == "grid":
            R.assert_exact_grid(ra, 1.0 / 64, tag)
        return R.compare(tag, kind, dx, ref, R.fp32_slack(ra, 1600))
    return by_rows(rows, dy.shape[0], dy, dx)


def check_conv2_dgrad(B: int = 8, seed: int = 2, kinds: Sequence[str] = KINDS, guard: int = 0) -> List[Result]:
    """``guard``: as in ``check_conv2_fwd``."""
    res: List[Result] = []
    for kind in kinds:
        tag = "conv2_dgrad.%s" % kind
        g = _gen(seed)
        if kind == "rand":
            dy, w = _bf(torch.randn(B, 14, 14, 64, generator=g) * 0.1), _bf(torch.randn(5, 5, 32, 64, generator=g) * 0.05)
        else:
            dy, w = _bf(R.grid(g, (B, 14, 14, 64), -4, 4)), _bf(R.grid(g, (5, 5, 32, 64), -8, 8, 64))
        dy, w = _dev(dy, w)
        dx = run_conv2_dgrad(dy, w, guard)
        res += conv2_dgrad_results(tag, kind, dy, w, dx)
        if guard:
            res += unwritten_results(tag + ".dx", dx, guard)
    return res


def conv2_wgrad_results(tag: str, kind: str, a1, dy, gw) -> List[Result]:
    B = a1.shape[0]
    ref = sum_by_rows(R.conv5x5_wgrad, B, a1, dy)
    if kind == "grid":
        R.assert_exact_grid(sum_by_rows(lambda a, d: R.conv5x5_wgrad(a.abs(), d.abs()), B, a1, dy), 1.0, tag)
    return R.compare(tag, kind, gw, ref)


def check_conv2_wgrad(B: int = 8, seed: int = 3, kinds: Sequence[str] = KINDS, stale_B: int = 0) -> List[Result]:
    res: List[Result] = []
    for kind in kinds:
        tag = "conv2_wgrad.%s" % kind
        g = _gen(seed)
        if kind == "rand":
            a1, dy = _bf(torch.rand(B, 14, 14, 32, generator=g)), _bf(torch.randn(B, 14, 14, 64, generator=g) * 0.1)
        else:
            a1, dy = _bf(R.grid(g, (B, 14, 14, 32), 0, 3)), _bf(R.grid(g, (B, 14, 14, 64), -3, 3))
        a1, dy = _dev(a1, dy)
        if stale_B:
            prime_workspace("conv2_wgrad", stale_B)
        res += conv2_wgrad_results(tag, kind, a1, dy, run_conv2_wgrad(a1, dy))
    return res


def _fc2_inputs(kind: str, g, B: int):
    """(b1, w2, b2, labels) for the fc2 kernels."""
    if kind == "rand":
        return (torch.randn(512, generator=g) * 0.1, torch.randn(512, 10, generator=g) * 0.1,
                torch.randn(10, generator=g) * 0.1, torch.randint(0, 10, (B,), generator=g))
    return (R.grid(g, (512,), -16, 16, 64), R.grid(g, (512, 10), -8, 8, 64), R.grid(g, (10,), -16, 16, 64),
            torch.randint(0, 10, (B,), generator=g))


def _fc2_results(tag: str, kind: str, o: Dict[str, torch.Tensor], ref: Dict[str, torch.Tensor], w2, B: int,
                 train: bool, decay_loss: Optional[float] = None) -> List[Result]:
    """fc2_fwd_bwd outputs.  logits and activations follow the data kind (exact on grid data, where the fc1 sum, bias,
    x2 dropout scale and fc2 products are all grid numbers).  Loss, d logits and d h go through exp/log (the kernel uses
    the fast __expf/__logf) and are compared by the continuous rule on both kinds.  The accuracy is exact, except for
    rows whose top two reference logits are closer than the logits' fp32 error.  A training step stores no logits: with
    ``o["logits"]`` None they are judged through the loss and the accuracy alone.  ``decay_loss``: lambda R of an L2
    weight decay, which weight_decay_loss has added to the loss word: the word must then be CE + lambda R within the CE
    bound plus one fp32 ulp (the rounding of fp32(lambda R) and of the add)."""
    res: List[Result] = []
    la = o["la"].double()
    if kind == "grid":
        # h: fc1 sum + bias in units of 1/64, times 2 under dropout (keep 0.5); w2 in units of 1/64
        R.assert_exact_grid(ref["h"].abs() @ w2.abs().double() + 1, 1.0 / (2048 if train else 4096), tag + ".logits")
    if o.get("logits") is not None:
        res += R.compare(tag + ".logits", kind, o["logits"], ref["logits"])
    if decay_loss is None:
        res += R.cmp_fp32(tag + ".loss", la[0:1], ref["loss"].reshape(1))
    else:
        ce = float(ref["loss"])
        want = ce + decay_loss
        res.append((tag + ".loss(CE + lambda R)", abs(float(la[0]) - want), R.REL_FP32 * abs(ce) + 2.0 ** -23 * abs(want)))
    lg_slack = R.fp32_slack(ref["h"].abs() @ w2.abs().double(), 512).max(dim=1).values
    ok = ref["gap"] > 2 * lg_slack
    res.append((tag + ".acc", abs(float(la[1]) - float(ref["acc"])) * B - float((~ok).sum()), 0.5))
    if train:
        res += R.compare(tag + ".h_act", kind, o["h"], ref["h"])
        res += R.cmp_fp32(tag + ".dlogits", o["dl"], ref["dl"])
        # d h = sum_c dlogits_c w2[:, c] often cancels to a tiny value, so the one-ulp rule gets the dlogits error as
        # slack.  The kernel's softmax uses __expf (relative error about 2^-22 (1 + |x|) for x = logit - max) and p - 1 for
        # the label class loses p's absolute error: |error of dlogits_c| <= (eps_row p_c + 2^-23) / B.
        lg = ref["logits"]
        eps_row = 2.0 ** -20 * (1.0 + (lg.max(dim=1).values - lg.min(dim=1).values))
        p = torch.softmax(lg, dim=1)
        dl_err = (eps_row[:, None] * p + 2.0 ** -23) / B
        dh_slack = 2 * (dl_err @ w2.abs().double().t() + R.fp32_slack(ref["dl"][:, :10].abs() @ w2.abs().double().t(), 10))
        res += R.cmp_bf16(tag + ".dh", o["dh"], ref["dh"], dh_slack)
    return res


_M32 = 0xFFFFFFFF
_GOLDEN, _STEP_MIX = 0x9E3779B1, 0x9E3779B9        # csrc/common.cuh hash_mix, csrc/lenet_simt.cu per-step seed


def _unhash(u: int) -> int:
    """Inverse of the murmur3 32-bit finaliser in ``hash_mix``: the x with fmix32(x) == u (each step is a bijection)."""
    x = u ^ (u >> 16)
    x = (x * pow(0xC2B2AE35, -1, 1 << 32)) & _M32
    x ^= (x >> 13) ^ (x >> 26)
    x = (x * pow(0x85EBCA6B, -1, 1 << 32)) & _M32
    return x ^ (x >> 16)


def check_fc2_loss(B: int = 64, seed: int = 4, stale_B: int = 0, keep_prob: float = 0.5,
                   probe: Optional[int] = None) -> List[Result]:
    """fc2_fwd_bwd on three hand-made split-K partials, then fc2_wgrad on what it saved (continuous data).  The keep
    pattern of the dropout must match the host mask exactly.  ``probe`` = -1 / 0 / +1: the seed is chosen so that one
    element (with a positive pre-activation) hashes to exactly threshold - 1 / threshold / threshold + 1, the values
    where an off-by-one threshold on either side changes the decision."""
    g = _gen(seed)
    h_pre = torch.randn(B, 512, generator=g)
    b1, w2, b2, labels = _fc2_inputs("rand", g, B)
    step, mix0 = 7, dropout_seed_mix(123, 0, 2)
    thresh = dropout_threshold(keep_prob)
    if probe is not None:
        r, j = B // 2, 77
        h_pre[r, j] = h_pre[r, j].abs() + 1.0 + b1[j].abs()
        target = thresh + probe
        assert 0 <= target < 1 << 24, "threshold %d + %d is not a 24-bit hash value" % (thresh, probe)
        mix = (_unhash((target << 8) | 0x5A) - (r * 512 + j) * _GOLDEN) & _M32
        mix0 = (mix - step * _STEP_MIX) & _M32
    mix = (mix0 + step * _STEP_MIX) & _M32
    h_pre, b1, w2, b2, labels = _dev(h_pre, b1, w2, b2, labels)
    parts = torch.stack([h_pre * 0.5, h_pre * 0.25, h_pre * 0.25]).contiguous()   # exact split of h_pre
    if stale_B:
        prime_workspace("fc2_fwd_bwd", stale_B)
    o = run_fc2_fwd_bwd(parts, b1, w2, b2, labels, True, mix0, step, keep_prob)
    keep = dropout_keep_mask(mix, B, 512, keep_prob, device="cuda")
    ref = R.fc2_fwd_bwd(h_pre, b1, w2, b2, labels, keep, keep_prob)
    res = _fc2_results("fc2.rand", "rand", o, ref, w2, B, True)
    hp, ha = h_pre.double() + b1.double(), h_pre.double().abs() + b1.double().abs()
    res += keep_pattern_results("fc2.keep_pattern(keep=%g)" % keep_prob, o["h"], ref["h"], hp, 4 * R.FP32_UNIT * ha)
    if probe is not None:
        res.append(("fc2.probe(thresh%+d)_decision" % probe, float(bool(o["h"][r, j] != 0) != (probe < 0)), 0.0))
    return res + fc2_wgrad_results("fc2_wgrad", o["h"], o["dl"], o["dh"], *run_fc2_wgrad(o["h"], o["dl"], o["dh"]))


def keep_pattern_results(tag: str, h, ref_h, hp, slack) -> List[Result]:
    """The dropout keep pattern, exactly: apart from pre-activations ``hp`` within ``slack`` (the kernel's fp32 error) of
    zero, h != 0 iff ReLU and the mask keep."""
    settled = hp.abs() > slack
    return [(tag, float((((h != 0) != (ref_h != 0)) & settled).sum()), 0.0)]


def fc2_wgrad_results(tag: str, h, dl, dh, gw2, gb2, gb1) -> List[Result]:
    """fc2_wgrad on continuous data: fc2 weight / bias and fc1 bias gradients from h_act, dlogits and dh."""
    rw2, rb2, rb1 = R.fc2_wgrad(h, dl, dh)
    return R.cmp_fp32(tag + ".g_w2", gw2, rw2) + R.cmp_fp32(tag + ".g_b2", gb2, rb2) + R.cmp_fp32(tag + ".g_b1", gb1, rb1)


def fc1_fwd_results(tag: str, kind: str, a2, w1, part) -> List[Result]:
    """The fc1 GEMM's 7 split-K partials [7,B,512] from a2 [B,3136] and the bf16 weights w1 [3136,512]."""
    res: List[Result] = []
    # split z owns k-blocks [49 z / 7, 49 (z + 1) / 7) of 64
    for z in range(FC1_SPLITS):
        k0, k1 = 64 * (49 * z // FC1_SPLITS), 64 * (49 * (z + 1) // FC1_SPLITS)
        rz = a2[:, k0:k1].double() @ w1[k0:k1].double()
        res += R.compare("%s.partial%d" % (tag, z), kind, part[z], rz)
    if kind == "grid":
        R.assert_exact_grid(a2.double().abs() @ w1.double().abs(), 1.0 / 64, tag + ".gemm")
    return res


def check_fc1_fwd(B: int = 64, seed: int = 16, kinds: Sequence[str] = KINDS, train: bool = True) -> List[Result]:
    """fc1 forward as the engine runs it: the GEMM with 7 strided split-K partials, then fc2_fwd_bwd summing them."""
    res: List[Result] = []
    for kind in kinds:
        tag = "fc1_fwd.%s" % kind
        g = _gen(seed)
        if kind == "rand":
            a2, w1 = _bf(torch.rand(B, 3136, generator=g)), _bf(torch.randn(3136, 512, generator=g) * 0.02)
        else:
            a2, w1 = _bf(R.grid(g, (B, 3136), 0, 1)), _bf(R.grid(g, (3136, 512), -8, 8, 64))
        b1, w2, b2, labels = _fc2_inputs(kind, g, B)
        a2, w1, b1, w2, b2, labels = _dev(a2, w1, b1, w2, b2, labels)
        part = run_fc1_fwd(a2, w1)
        res += fc1_fwd_results(tag, kind, a2, w1, part)
        hsum = a2.double() @ w1.double()
        mix0 = dropout_seed_mix(seed, 0, 0)
        o = run_fc2_fwd_bwd(part, b1, w2, b2, labels, train, mix0, 3, 0.5)
        keep = dropout_keep_mask(dropout_seed_mix(seed, 3, 0), B, 512, 0.5, device="cuda") if train else None
        ref = R.fc2_fwd_bwd(hsum, b1, w2, b2, labels, keep, 0.5)
        res += _fc2_results("fc2_fwd_bwd.%s" % kind, kind, o, ref, w2, B, train)
    return res


def check_fc2_wgrad(B: int = 64, seed: int = 17) -> List[Result]:
    """fc2_wgrad on grid-valued h_act / dlogits / dh: exact."""
    g = _gen(seed)
    h = R.grid(g, (B, 512), 0, 16, 8) * (torch.rand(B, 512, generator=g) < 0.5)
    dl = torch.zeros(B, 12)
    dl[:, :10] = R.grid(g, (B, 10), -32, 32, 64)
    dh = _bf(R.grid(g, (B, 512), -64, 64, 64))
    h, dl, dh = _dev(h, dl, dh)
    gw2, gb2, gb1 = run_fc2_wgrad(h, dl, dh)
    rw2, rb2, rb1 = R.fc2_wgrad(h, dl, dh)
    aw2, ab2, ab1 = R.fc2_wgrad(h.abs(), dl.abs(), dh.abs())
    R.assert_exact_grid(aw2, 1.0 / 512, "fc2_wgrad.g_w2")
    R.assert_exact_grid(ab2, 1.0 / 64, "fc2_wgrad.g_b2")
    R.assert_exact_grid(ab1, 1.0 / 64, "fc2_wgrad.g_b1")
    return R.cmp_exact("fc2_wgrad.grid.g_w2", gw2, rw2) + R.cmp_exact("fc2_wgrad.grid.g_b2", gb2, rb2) + \
        R.cmp_exact("fc2_wgrad.grid.g_b1", gb1, rb1)


def check_fc1_wgrad(B: int = 64, seed: int = 18, kinds: Sequence[str] = KINDS) -> List[Result]:
    """fc1 weight gradient GEMM (a2^T dh, K = batch) with fp32 output (single-kernel aggregation) and bf16 output (the
    bucketed aggregation's wire buffer)."""
    res: List[Result] = []
    for kind in kinds:
        g = _gen(seed)
        if kind == "rand":
            a2, dh = _bf(torch.rand(B, 3136, generator=g)), _bf(torch.randn(B, 512, generator=g) * 0.01)
        else:
            a2, dh = _bf(R.grid(g, (B, 3136), 0, 2)), _bf(R.grid(g, (B, 512), -64, 64, 64))
        a2, dh = _dev(a2, dh)
        for bf in (False, True):
            out = run_fc1_wgrad(a2, dh, bf)
            res += fc1_wgrad_results("fc1_wgrad.%s.%s" % (kind, "bf16" if bf else "f32"), kind, a2, dh, out)
    return res


def fc1_wgrad_results(tag: str, kind: str, a2, dh, out) -> List[Result]:
    """dW1 = a2^T dh, stored as fp32 (gradient arena) or bf16 (the bucketed aggregation's wire buffer)."""
    ref = a2.double().t() @ dh.double()
    ra = a2.double().abs().t() @ dh.double().abs()
    if kind == "grid":
        R.assert_exact_grid(ra, 1.0 / 64, "fc1_wgrad")
    return R.compare(tag, kind, out, ref, R.fp32_slack(ra, a2.shape[0]))


# ---------------------------------------------------------------------------------------------------------------------
# L2 weight decay (--weight_decay): the decayed epilogues of fc1_wgrad / fc2_wgrad, their W^2 partials, weight_decay_loss
# ---------------------------------------------------------------------------------------------------------------------
DECAY_LAMS = (5e-4, 0.0123, 2.0 ** -4)
DECAY_PART_REL = 1e-12         # sums of exact squares in double: another order moves them by ~n * 2^-53


def _lam32(lam) -> float:
    return float(np.float32(lam))


def decayed_bound(abs_sum, n_terms: int, lam: float, v, ref):
    """Elementwise error bound of a decayed fp32 output fma(lambda, v, acc) against the float64 ``ref`` = plain +
    lambda v: the fp32 bound of a sum of ``n_terms`` terms whose magnitudes add up to ``abs_sum`` + lambda |v|, plus the
    fma's one rounding."""
    return R.fp32_slack(abs_sum.to(R.F64) + lam * v.to(R.F64).abs(), n_terms) + 2.0 ** -24 * ref.abs()


def decayed_results(tag: str, kind: str, got, plain_ref, abs_sum, n_terms: int, lam: float, v) -> List[Result]:
    """One decayed output ``got`` = fma(lambda, v, plain accumulator), stored fp32 or bf16.  ``plain_ref``: the float64
    reference of the undecayed value, ``abs_sum`` its sum of |terms| over ``n_terms`` terms, ``v`` the fp32 variable.
    Grid data (the accumulator is exact): bit for bit against the single-rounding emulation fma_f32(lambda, v, plain), then
    RNE for bf16.  Continuous data: elementwise against plain + lambda v within :func:`decayed_bound`; a bf16 output must
    lie within RNE of that interval."""
    lam = _lam32(lam)
    if kind == "grid":
        want = A.fma_f32(np.float32(lam), A.f32(v), A.f32(plain_ref.to(torch.float32)))
        if got.dtype == BF:
            bad = got.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16) != A.bf16_bits(want)
        else:
            bad = A.bits(got) != A.bits(want)
        return [(tag + "[fma bits]", float(bad.sum()), 0.0)]
    ref = plain_ref.to(R.F64) + lam * v.to(R.F64)
    bound = decayed_bound(abs_sum, n_terms, lam, v, ref)
    if got.dtype == BF:
        return R.cmp_bf16_bound(tag, got, ref, bound)
    return R.cmp_bound(tag, got, ref, bound)


def decay_visible(tag: str, abs_sum, n_terms: int, lam: float, v, plain_ref) -> Result:
    """Premise of a continuous-data decay check: somewhere lambda |v| exceeds twice :func:`decayed_bound`, so an output
    without its decay term would fail the check."""
    lam = _lam32(lam)
    ref = plain_ref.to(R.F64) + lam * v.to(R.F64)
    seen = bool((lam * v.to(R.F64).abs() > 2 * decayed_bound(abs_sum, n_terms, lam, v, ref)).any())
    return (tag + ".decay_term_detectable", 0.0 if seen else 1.0, 0.0)


def fc1_wgrad_decay_results(tag: str, kind: str, a2, dh, out, lam: float, w1) -> List[Result]:
    """dW1 + lambda W1 (fp32 arena or bf16 wire) from a2 [B,3136], dh [B,512] and the fp32 weights w1 [3136,512]."""
    ref = a2.double().t() @ dh.double()
    ra = a2.double().abs().t() @ dh.double().abs()
    return decayed_results(tag, kind, out, ref, ra, a2.shape[0], lam, w1)


def fc2_wgrad_decay_results(tag: str, kind: str, h, dl, dh, gw2, gb2, gb1, lam: float, w2, b2, b1) -> List[Result]:
    """fc2_wgrad<true>: g_w2 / g_b2 / g_b1 + lambda w2 / b2 / b1 from h_act, dlogits, dh and the fp32 variables."""
    B = h.shape[0]
    (rw2, rb2, rb1), (aw2, ab2, ab1) = R.fc2_wgrad(h, dl, dh), R.fc2_wgrad(h.abs(), dl.abs(), dh.abs())
    return decayed_results(tag + ".g_w2", kind, gw2, rw2, aw2, B, lam, w2) + \
        decayed_results(tag + ".g_b2", kind, gb2, rb2, ab2, B, lam, b2) + \
        decayed_results(tag + ".g_b1", kind, gb1, rb1, ab1, B, lam, b1)


def fc1_decay_partials(w1) -> torch.Tensor:
    """float64 W^2 sums of dm_gemm_bf16_decay's CTAs for W1 [3136,512]: CTA (x = 128-row tile, y = 128-column tile) at
    y * 25 + x.  The last row tile holds 64 rows."""
    sq = torch.zeros(3200, 512, dtype=R.F64, device=w1.device)
    sq[:3136] = w1.double() ** 2
    return sq.reshape(25, 128, 4, 128).sum((1, 3)).t().reshape(-1)


def fc2_decay_partials(w2, b2, b1) -> torch.Tensor:
    """float64 sums of squares of fc2_wgrad<true>'s 64 CTAs: CTA c owns w2 rows and b1 entries 8c .. 8c + 7, CTA 0 also
    b2."""
    s = (w2.double() ** 2).reshape(64, 80).sum(1) + (b1.double() ** 2).reshape(64, 8).sum(1)
    s[0] += (b2.double() ** 2).sum()
    return s


def decay_partials_results(tag: str, got, want) -> List[Result]:
    """W^2 partials or R against their float64 sums, each within DECAY_PART_REL of its value (a zero one exactly)."""
    return R.cmp_bound(tag, got.reshape(-1), want.reshape(-1), DECAY_PART_REL * want.reshape(-1).abs())


def weight_decay_loss_emulated(part, n: int, lam: float, loss: float):
    """csrc/weight_decay.cu on the host, in its order: lane l sums partials l, l + 32, ... in double, the xor butterfly
    (16, 8, 4, 2, 1), R = 0.5 * lane 0's sum; the loss word becomes fp32(loss + fp32(double(lambda) * R)).  Returns
    (R, new loss word) as numpy float64 / float32."""
    part = np.asarray(part, dtype=np.float64)
    lanes = [np.float64(0.0)] * 32
    for lane in range(32):
        s = np.float64(0.0)
        for i in range(lane, n, 32):
            s = s + part[i]
        lanes[lane] = s
    for off in (16, 8, 4, 2, 1):
        lanes = [lanes[i] + lanes[i ^ off] for i in range(32)]
    r = np.float64(0.5) * lanes[0]
    term = np.float32(np.float64(np.float32(lam)) * r)
    return r, np.float32(np.float32(loss) + term)


def _fc1_decay_inputs(kind: str, g, B: int):
    """(a2, dh, W1) on the data of :func:`check_fc1_wgrad`; W1 continuous, or on a k/64 grid."""
    if kind == "rand":
        return _bf(torch.rand(B, 3136, generator=g)), _bf(torch.randn(B, 512, generator=g) * 0.01), \
            torch.randn(3136, 512, generator=g)
    return _bf(R.grid(g, (B, 3136), 0, 2)), _bf(R.grid(g, (B, 512), -64, 64, 64)), R.grid(g, (3136, 512), -64, 64, 64)


def check_fc1_wgrad_decay(B: int = 64, seed: int = 18, kinds: Sequence[str] = KINDS,
                          lams: Sequence[float] = DECAY_LAMS) -> List[Result]:
    """dW1 + lambda W1 with the fp32 and the bf16 epilogue, and each CTA's W^2 partial.  W1 lives in the first 3136 rows
    of a buffer whose 64 rows after them hold 1024: the last row tile is half empty, and its missing rows must neither be
    read into the partial nor stored."""
    res: List[Result] = []
    for kind in kinds:
        g = _gen(seed)
        a2, dh, w = _fc1_decay_inputs(kind, g, B)
        wbuf = torch.full((3200, 512), 1024.0)
        wbuf[:3136] = w
        a2, dh, wbuf = _dev(a2, dh, wbuf)
        w = wbuf[:3136]
        ra = a2.double().abs().t() @ dh.double().abs()
        if kind == "grid":
            R.assert_exact_grid(ra, 1.0 / 64, "fc1_wgrad_decay")
        want_part = fc1_decay_partials(w)
        for lam in lams:
            for bf in (False, True):
                tag = "fc1_wgrad_decay.%s.%s.lam%g" % (kind, "bf16" if bf else "f32", lam)
                out, part = run_fc1_wgrad_decay(a2, dh, wbuf, lam, bf)
                res += fc1_wgrad_decay_results(tag, kind, a2, dh, out, lam, w)
                res += decay_partials_results(tag + ".w2_partials", part, want_part)
            if kind == "rand":
                res.append(decay_visible("fc1_wgrad_decay.rand.lam%g" % lam, ra, B, lam, w, a2.double().t() @ dh.double()))
    return res


def _fc2_decay_inputs(kind: str, g, B: int):
    """(h, dl, dh, w2, b2, b1): the grid data of :func:`check_fc2_wgrad` with the grid variables of :func:`_fc2_inputs`,
    or continuous data."""
    dl = torch.zeros(B, 12)
    if kind == "rand":
        h = torch.relu(torch.randn(B, 512, generator=g))
        dl[:, :10] = torch.randn(B, 10, generator=g) * 0.01
        dh = _bf(torch.randn(B, 512, generator=g) * 0.01)
        w2, b2, b1 = (torch.randn(*s, generator=g) for s in ((512, 10), (10,), (512,)))
        return h, dl, dh, w2, b2, b1
    h = R.grid(g, (B, 512), 0, 16, 8) * (torch.rand(B, 512, generator=g) < 0.5)
    dl[:, :10] = R.grid(g, (B, 10), -32, 32, 64)
    dh = _bf(R.grid(g, (B, 512), -64, 64, 64))
    b1, w2, b2, _ = _fc2_inputs("grid", g, B)
    return h, dl, dh, w2, b2, b1


def check_fc2_wgrad_decay(B: int = 64, seed: int = 17, kinds: Sequence[str] = KINDS,
                          lams: Sequence[float] = DECAY_LAMS) -> List[Result]:
    """fc2_wgrad<true>'s g_w2 / g_b2 / g_b1 and each CTA's sum of squares (b2 in CTA 0's only)."""
    res: List[Result] = []
    for kind in kinds:
        h, dl, dh, w2, b2, b1 = _dev(*_fc2_decay_inputs(kind, _gen(seed), B))
        aw2, ab2, ab1 = R.fc2_wgrad(h.abs(), dl.abs(), dh.abs())
        if kind == "grid":
            R.assert_exact_grid(aw2, 1.0 / 512, "fc2_wgrad_decay.g_w2")
            R.assert_exact_grid(ab2, 1.0 / 64, "fc2_wgrad_decay.g_b2")
            R.assert_exact_grid(ab1, 1.0 / 64, "fc2_wgrad_decay.g_b1")
        want_part = fc2_decay_partials(w2, b2, b1)
        for lam in lams:
            tag = "fc2_wgrad_decay.%s.lam%g" % (kind, lam)
            gw2, gb2, gb1, part = run_fc2_wgrad_decay(h, dl, dh, w2, b2, b1, lam)
            res += fc2_wgrad_decay_results(tag, kind, h, dl, dh, gw2, gb2, gb1, lam, w2, b2, b1)
            res += decay_partials_results(tag + ".w2_partials", part, want_part)
            if kind == "rand":
                rw2 = R.fc2_wgrad(h, dl, dh)[0]
                res.append(decay_visible(tag, aw2, B, lam, w2, rw2))
    return res


def check_weight_decay_workspace(B: int = 129, seed: int = 19, lam: float = 0.0123) -> List[Result]:
    """The engine's decay workspace (fc1 partials, fc2 partials, R) filled by two rounds of both weight-gradient kernels on
    different weights, then weight_decay_loss: every partial and R must be the second round's, within DECAY_PART_REL of
    float64, and the loss word must be the kernel's order emulated from the stored partials, bit for bit."""
    lib = load()
    n1, n2 = int(lib.dm_gemm_decay_ctas(3136, 512)), int(lib.dm_fc2_wgrad_decay_ctas())
    ws = torch.full((n1 + n2 + 1,), float("nan"), dtype=torch.float64, device="cuda")
    g = _gen(seed)
    a2, dh, _ = _fc1_decay_inputs("rand", g, B)
    h, dl, dh2, _, _, _ = _fc2_decay_inputs("rand", g, B)
    a2, dh, h, dl, dh2 = _dev(a2, dh, h, dl, dh2)
    for scale in (0.05, 0.2):
        w1, w2, b2, b1 = _dev(*(torch.randn(*s, generator=g) * scale for s in ((3136, 512), (512, 10), (10,), (512,))))
        run_fc1_wgrad_decay(a2, dh, w1, lam, part=ws[:n1])
        run_fc2_wgrad_decay(h, dl, dh2, w2, b2, b1, lam, part=ws[n1:n1 + n2])
    la = torch.tensor([2.5, 0.25], device="cuda")
    lib.dm_weight_decay_loss(ws, n1 + n2, float(lam), la, stream_ptr())
    torch.cuda.synchronize()
    want = torch.cat([fc1_decay_partials(w1), fc2_decay_partials(w2, b2, b1)])
    r, loss = weight_decay_loss_emulated(ws[:n1 + n2].cpu().numpy(), n1 + n2, lam, 2.5)
    got = la.cpu().numpy()
    return decay_partials_results("decay_ws.partials", ws[:n1 + n2], want) + \
        decay_partials_results("decay_ws.R", ws[n1 + n2:], want.sum().reshape(1) / 2) + \
        [("decay_ws.R_bits_vs_emulation", float(ws[n1 + n2].item() != r), 0.0),
         ("decay_ws.loss_bits_vs_emulation", float(got[0].tobytes() != loss.tobytes()), 0.0),
         ("decay_ws.acc_changed", float(got[1] != np.float32(0.25)), 0.0)]


def check_weight_decay_loss(n: int, seed: int = 20, lams: Sequence[float] = DECAY_LAMS) -> List[Result]:
    """weight_decay_loss alone on n partials spread over 40 binades (so that another summation order would round
    differently): part[n] and the loss word bit for bit against :func:`weight_decay_loss_emulated`; the partials and the
    accuracy word untouched."""
    lib, res = load(), []
    g = _gen(seed)
    vals = torch.rand(n, generator=g, dtype=torch.float64) * torch.exp2(torch.randint(-20, 21, (n,), generator=g).double())
    loss0, acc0 = np.float32(2.3025851), np.float32(0.375)
    for lam in lams:
        tag = "weight_decay_loss.n%d.lam%g" % (n, lam)
        part = torch.cat([vals, torch.tensor([float("nan")], dtype=torch.float64)]).cuda()
        la = torch.tensor([float(loss0), float(acc0)], dtype=torch.float32, device="cuda")
        lib.dm_weight_decay_loss(part, n, float(lam), la, stream_ptr())
        torch.cuda.synchronize()
        r, loss = weight_decay_loss_emulated(vals.numpy(), n, lam, loss0)
        got, p = la.cpu().numpy(), part.cpu().numpy()
        res += [(tag + ".partials_changed", float((p[:n].view(np.uint64) != vals.numpy().view(np.uint64)).sum()), 0.0),
                (tag + ".R_bits", float(p[n:].tobytes() != np.float64(r).tobytes()), 0.0),
                (tag + ".loss_bits", float(got[0].tobytes() != loss.tobytes()), 0.0),
                (tag + ".acc_changed", float(got[1].tobytes() != acc0.tobytes()), 0.0)]
    return res


# ---- random affine augmentation (augment.py, csrc/augment.cu) ---------------------------------------------------------
AUG_U = 2.0 ** -24
AUG_PREMISE_ROWS = 256         # rows the premise checks of augment_results warp (a large batch's would only cost time)


def augment_pixel_bound(coef, coef_ulps: int = 0, field=None, field_err=None) -> np.ndarray:
    """Per-pixel bound on |augment_affine - float64 warp of the fp32 coefficients ``coef``| ([B, 4]: a, b, tx, ty),
    float64 [B, 784].

    The kernel computes dx = fl(xc - tx) (xc = x - 13.5 exact), t = fma(b, dy, 13.5), sx = fma(a, dx, t) and likewise sy,
    each with one rounding, so with u = 2^-24: |dx_f - dx| <= u |dx|, and
        |sx_f - sx| <= |a| u |dx| + |b| u |dy| + u |t| + u |sx|   (to first order in u; the factor 1.001 covers the rest)
    and the same for sy with (a, -b).  Clamping sx, sy to [-2, 29] is 1-Lipschitz and changes nothing where a tap could
    be inside the image.  Bilinear interpolation with the background -0.5 is continuous in (sx, sy) and, for pixel values
    in [-0.5, 0.5], Lipschitz with constant <= 1 per axis (each slope is a difference of two such values), also across
    cell boundaries, so the sample point's error costs at most |sx_f - sx| + |sy_f - sy|.  The blend top = fma(fx, v01 -
    v00, v00), bot likewise, out = fma(fy, bot - top, top) with fx, fy exact adds at most 3u (|v| <= 0.5: each difference
    is rounded to within u/2, each fma to within u/4, and the errors of top and bot enter out with weights summing to 1);
    4u is used.  The float64 reference itself is exact to ~1e-15.

    ``coef_ulps``: the kernel's coefficients may each differ from ``coef`` by that many fp32 ulps (<= 2^-23 |c| each):
    its double ``sincos`` and numpy's may round to different fp32 neighbours near a tie.  Since sx = c + a dx + b dy with
    dx = x - c - tx, a change of e |a|, e |b|, e |tx|, e |ty| moves sx by at most e (|a| (|dx| + |tx|) + |b| (|dy| + |ty|))
    and sy by e (|b| (|dx| + |tx|) + |a| (|dy| + |ty|)), which the same Lipschitz argument adds to the bound.

    ``field``: the elastic displacement [B, 2, 784] (augment_elastic; fp32 values) the bound is taken around.  That
    kernel computes dx = fl(fl(xc + ex) - tx), two roundings: |dx_f - dx| <= u (|xc + ex| + |dx|), which enters sx with
    weight |a| and sy with |b| (dy likewise with |b|, |a|).  ``field_err``: [B, 2, 784] bound on |kernel field - field|;
    a change of the displacement by (fx, fy) moves sx by |a| fx + |b| fy and sy by |b| fx + |a| fy."""
    a, b, tx, ty = (np.asarray(coef, dtype=np.float64)[:, k][:, None] for k in range(4))
    y, x = np.divmod(np.arange(784, dtype=np.float64), 28)
    dx, dy = x[None] - 13.5 - tx, y[None] - 13.5 - ty
    if field is not None:
        f = np.asarray(field, dtype=np.float64).reshape(-1, 2, 784)
        dx, dy = (x[None] - 13.5 + f[:, 0]) - tx, (y[None] - 13.5 + f[:, 1]) - ty
    tsx, tsy = b * dy + 13.5, -b * dx + 13.5
    sx, sy = a * dx + tsx, a * dy + tsy
    bsx = AUG_U * (np.abs(a * dx) + np.abs(b * dy) + np.abs(tsx) + np.abs(sx))
    bsy = AUG_U * (np.abs(a * dy) + np.abs(b * dx) + np.abs(tsy) + np.abs(sy))
    if field is not None:
        rx, ry = AUG_U * np.abs(x[None] - 13.5 + f[:, 0]), AUG_U * np.abs(y[None] - 13.5 + f[:, 1])
        if field_err is not None:
            fe = np.asarray(field_err, dtype=np.float64).reshape(-1, 2, 784)
            rx, ry = rx + fe[:, 0], ry + fe[:, 1]
        bsx = bsx + np.abs(a) * rx + np.abs(b) * ry
        bsy = bsy + np.abs(b) * rx + np.abs(a) * ry
    if coef_ulps:
        e = coef_ulps * 2.0 ** -23
        ax, by = np.abs(dx) + np.abs(tx), np.abs(dy) + np.abs(ty)
        bsx = bsx + e * (np.abs(a) * ax + np.abs(b) * by)
        bsy = bsy + e * (np.abs(b) * ax + np.abs(a) * by)
    return 1.001 * (bsx + bsy) + 4 * AUG_U + 1e-12


def augment_coefficients(mix: int, iteration: int, B: int, ranges) -> np.ndarray:
    """[B, 4] (a, b, tx, ty) of rows 0..B-1 at ``iteration``: the float64 coefficients rounded to fp32, as float64."""
    from .. import augment as AU
    c = np.stack(AU.coefficients(AU.uniforms(mix, iteration, B), ranges), axis=1)
    return c.astype(np.float32).astype(np.float64)


def augment_results(tag: str, fed, got, mix: int, iteration: int, ranges, elastic=None) -> List[Result]:
    """One augmented step's buffer ``got`` [B, 784] against ``augment.warp`` of the batch it was ``fed`` (fp32, [B, 784]
    or [B, 28, 28], values in [-0.5, 0.5]) with the draws of ``iteration`` under ``mix``, the coefficients rounded to fp32,
    within :func:`augment_pixel_bound` widened by one ulp of each coefficient.

    Premise: the warps of iterations ``iteration`` +- 1, of the next rank's mix and about the centre 14.0 each differ from
    the reference by more than the bound on some pixel of the first ``AUG_PREMISE_ROWS`` rows, so a step that drew from a
    neighbouring iteration, used another replica's key or shifted the centre by half a pixel fails the check.

    ``elastic``: the ``augment.Elastic`` the step was armed with; see :func:`elastic_augment_results`."""
    if elastic is not None:
        return elastic_augment_results(tag, fed, got, mix, iteration, ranges, elastic)
    from .. import augment as AU
    x = (fed.detach().cpu().numpy() if torch.is_tensor(fed) else np.asarray(fed)).astype(np.float64)
    B = x.shape[0]
    x = x.reshape(B, 784)
    c = augment_coefficients(mix, iteration, B, ranges)
    want = AU.warp(x, *c.T).reshape(B, 784)
    bound = augment_pixel_bound(c, coef_ulps=1)
    g = got.detach().reshape(B, 784)
    res = R.cmp_bound(tag, g, torch.from_numpy(want).to(g.device), torch.from_numpy(bound).to(g.device))
    n = min(B, AUG_PREMISE_ROWS)
    xs = x[:n]
    alts = (("iteration_minus_1", AU.warp(xs, *augment_coefficients(mix, iteration - 1, n, ranges).T)),
            ("iteration_plus_1", AU.warp(xs, *augment_coefficients(mix, iteration + 1, n, ranges).T)),
            ("next_rank", AU.warp(xs, *augment_coefficients((mix + AU.RANK_MIX) & 0xFFFFFFFF, iteration, n, ranges).T)),
            ("centre_14", AU.warp(xs, *c[:n].T, centre=14.0)))
    for name, alt in alts:
        seen = bool((np.abs(alt.reshape(n, 784) - want[:n]) > bound[:n]).any())
        res.append(("%s.premise.%s_detectable" % (tag, name), 0.0 if seen else 1.0, 0.0))
    return res


def elastic_field_f32(mix: int, iteration: int, B: int, elastic) -> np.ndarray:
    """[B, 2, 784] float64 ``augment.elastic_field`` rounded to fp32: the field augment_elastic computes, each component
    within :func:`elastic_field_err` of it."""
    from .. import augment as AU
    return AU.elastic_field(mix, iteration, B, elastic).reshape(B, 2, 784).astype(np.float32).astype(np.float64)


def elastic_field_err(field, elastic) -> np.ndarray:
    """Bound on |augment_elastic's field - ``field``| per component: one fp32 ulp (<= 2^-23 |e|), and alpha 2^-44 for
    the double passes of the kernel and of the float64 reference where the field nearly cancels (csrc/augment_elastic.cu
    derives < alpha 2^-45 for each)."""
    return 2.0 ** -23 * np.abs(field) + float(elastic.alpha) * 2.0 ** -44


def elastic_augment_results(tag: str, fed, got, mix: int, iteration: int, ranges, elastic) -> List[Result]:
    """An elastic step's buffer ``got`` [B, 784] against ``augment.warp`` of the batch it was ``fed`` with the
    coefficients and the field of ``iteration`` under ``mix``, each rounded to fp32, within :func:`augment_pixel_bound`
    widened by one ulp of each coefficient and of each field component (:func:`elastic_field_err`).

    Premise: the warps of iterations ``iteration`` +- 1, of the next rank's mix, with the field's x and y components
    swapped, without the field, and with sigma 1.25 times as wide each differ from the reference by more than the bound
    on some pixel of the first ``AUG_PREMISE_ROWS`` rows."""
    from .. import augment as AU
    x = (fed.detach().cpu().numpy() if torch.is_tensor(fed) else np.asarray(fed)).astype(np.float64)
    B = x.shape[0]
    x = x.reshape(B, 784)
    c = augment_coefficients(mix, iteration, B, ranges)
    f = elastic_field_f32(mix, iteration, B, elastic)
    want = AU.warp(x, *c.T, field=f).reshape(B, 784)
    bound = augment_pixel_bound(c, coef_ulps=1, field=f, field_err=elastic_field_err(f, elastic))
    g = got.detach().reshape(B, 784)
    res = R.cmp_bound(tag, g, torch.from_numpy(want).to(g.device), torch.from_numpy(bound).to(g.device))
    n = min(B, AUG_PREMISE_ROWS)
    xs, cn, fn = x[:n], c[:n].T, f[:n]
    nxt = (mix + AU.RANK_MIX) & 0xFFFFFFFF
    wide = AU.Elastic(elastic.alpha, 1.25 * elastic.sigma)
    alts = (("iteration_minus_1", AU.warp(xs, *augment_coefficients(mix, iteration - 1, n, ranges).T,
                                          field=elastic_field_f32(mix, iteration - 1, n, elastic))),
            ("iteration_plus_1", AU.warp(xs, *augment_coefficients(mix, iteration + 1, n, ranges).T,
                                         field=elastic_field_f32(mix, iteration + 1, n, elastic))),
            ("next_rank", AU.warp(xs, *augment_coefficients(nxt, iteration, n, ranges).T,
                                  field=elastic_field_f32(nxt, iteration, n, elastic))),
            ("swapped_components", AU.warp(xs, *cn, field=fn[:, ::-1])),
            ("no_field", AU.warp(xs, *cn)),
            ("sigma_1.25", AU.warp(xs, *cn, field=elastic_field_f32(mix, iteration, n, wide))))
    for name, alt in alts:
        seen = bool((np.abs(alt.reshape(n, 784) - want[:n]) > bound[:n]).any())
        res.append(("%s.premise.%s_detectable" % (tag, name), 0.0 if seen else 1.0, 0.0))
    return res


def fc1_dgrad_results(tag: str, kind: str, dh, w1, code, dy, gb) -> List[Result]:
    """fc1_dgrad_unpool's dy2 [B,14,14,64] and conv2 bias gradient from dh, the bf16 weights w1 and the pool2 codes."""
    slices = row_slices(dh.shape[0])
    parts, rgb, agb = [], 0.0, 0.0
    for s in slices:
        rdy, g = R.fc1_dgrad_unpool(dh[s], w1, code[s])
        ady, _ = R.fc1_dgrad_unpool(dh[s].abs(), w1.abs(), code[s])
        if kind == "grid":
            R.assert_exact_grid(ady, 1.0 / 64, tag + ".dy")
        parts.append(R.compare(tag + ".dy", kind, dy[s], rdy, R.fp32_slack(ady, 512)))
        rgb, agb = rgb + g, agb + rdy.abs().sum((0, 1, 2))
    if kind == "grid":
        # the bias gradient adds the exact fp32 values: its partial sums are bounded by the sum of their magnitudes
        R.assert_exact_grid(agb, 1.0 / 64, tag + ".g_bias")
    return merge_row_chunks(parts, [s.stop - s.start for s in slices]) + R.compare(tag + ".g_bias", kind, gb, rgb)


def check_fc1_dgrad_unpool(B: int = 200, seed: int = 6, kinds: Sequence[str] = KINDS, stale_B: int = 0,
                           guard: int = 0) -> List[Result]:
    """fc1 dgrad GEMM with the maxpool2/ReLU2 backward + conv2 bias gradient fused into its epilogue.  ``guard``: as in
    ``check_conv2_fwd``, for dy2.  The grid weights are k/64 with |k| <= 8, or <= 4 above 8192 rows: the bias gradient
    sums about 25 B values of dy2 per channel, and its exact partial sums must stay below 2^24 units of 1/64."""
    res: List[Result] = []
    for kind in kinds:
        tag = "fc1_dgrad_unpool.%s" % kind
        g = _gen(seed)
        if kind == "rand":
            dh, w1 = _bf(torch.randn(B, 512, generator=g) * 0.1), _bf(torch.randn(3136, 512, generator=g) * 0.05)
        else:
            wk = 8 if B <= 8192 else 4
            dh, w1 = _bf(R.grid(g, (B, 512), -1, 1)), _bf(R.grid(g, (3136, 512), -wk, wk, 64))
        dh, w1, code = _dev(dh, w1, _codes(g, (B, 3136)))
        if stale_B:
            prime_workspace("fc1_dgrad_unpool", stale_B)
        dy, gb = run_fc1_dgrad_unpool(dh, w1, code, guard)
        res += fc1_dgrad_results(tag, kind, dh, w1, code, dy, gb)
        if guard:
            res += unwritten_results(tag + ".dy", dy, guard)
    return res


def _engine(B: int, seed: int = 5):
    from ..engine_cuda import CudaLeNetEngine
    ctx = ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none")
    be = FusedBackend(ctx)
    return CudaLeNetEngine(B, be, seed=seed, rank=0, use_graph=False), be


# Per-tensor L2 bound of (gradients of the bf16-operand tensor-core step) vs (gradients of a PLAIN fp32 model, TF32 off).
# This is not a kernel-accuracy figure -- against the bf16-emulating reference every tensor agrees to <= 0.44 % (above) -- but
# the distance between bf16 and fp32 *training arithmetic*: activations rounded to bf16 flip ReLU / max-pool decisions, and the
# flips accumulate towards the input, so the bounds grow towards conv1 (several percent there, well under 1 % at fc2).
# A wrong tap, a transposed tile or a dropped bias shows up as O(1).
FP32_GRAD_TOLS = {"conv1_weights": 0.30, "conv1_biases": 0.15, "conv2_weights": 0.15, "conv2_biases": 0.15,
                  "fc1_weights": 0.12, "fc1_biases": 0.12, "fc2_weights": 0.03, "fc2_biases": 0.03}


def check_end_to_end(B: int = 64, seed: int = 5, images: str = "rand", lam: float = 0.0) -> List[Result]:
    """Whole forward+backward through the CUDA engine vs torch autograd on the bf16-emulating reference.
    ``images="mnist"``: an exact -0.5 background with strokes, so many pooling windows hold equal maxima and the
    backward pass routes gradients through the first-max tie-break in both conv layers.  ``lam``: L2 weight decay armed
    on the engine; both references then differentiate CE + lambda R (``refs.weight_decay_terms``), and each decayed
    variable's lambda v must be a larger share of its gradient than that variable's FP32_GRAD_TOLS, so a missing or
    misplaced decay term fails."""
    eng, be = _engine(B, seed)
    spec, _ = get_model("lenet")
    if lam:
        eng.arm_weight_decay(lam)

    def regularised(loss, flat):
        return loss + _lam32(lam) * R.weight_decay_terms(spec, flat, lam)[0] if lam else loss
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.rand(B, 28, 28, 1, generator=g) - 0.5) if images == "rand" else mnist_like(g, B)[..., None]
    y = torch.randint(0, 10, (B,), generator=g)
    eng.load_batch(x.numpy(), y.numpy())
    eng.forward_backward(0)
    torch.cuda.synchronize()
    loss, acc = eng.loss_acc()
    # reference on the same weights
    flat = eng.params.detach().clone().requires_grad_(True)
    mask = dropout_keep_mask(dropout_seed_mix(seed, 0, 0), B, 512, 0.5, device="cuda")
    logits = lenet_forward(spec.views(flat), x.cuda(), train=True, keep_mask=mask, emulate_bf16=True,
                           conv1_bf16=True)
    rloss, racc = loss_and_accuracy(logits, y.cuda())
    rloss = regularised(rloss, flat)
    rloss.backward()
    out: List[Result] = [("e2e.loss", abs(loss - rloss.item()), 0.02 * max(1.0, abs(rloss.item()))),
                         ("e2e.acc", abs(acc - racc.item()), 2.0 / B + 1e-6)]
    gv, rv = spec.views(eng.grads), spec.views(flat.grad)
    for name in rv:
        scale = rv[name].abs().max().item() + 1e-8
        # a wrong tap / transposed tile shows up as O(1)
        out.append(("e2e.grad.%s(rel)" % name, (gv[name] - rv[name]).abs().max().item() / scale, 0.02))
    # the same gradients against a PLAIN fp32 reference (no bf16 emulation anywhere): the remaining difference is the bf16
    # rounding of the tensor-core operands, bounded per tensor in the L2 norm
    flat32 = eng.params.detach().clone().requires_grad_(True)
    tf32_conv, tf32_mm = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False      # a real fp32 reference
    try:
        logits32 = lenet_forward(spec.views(flat32), x.cuda(), train=True, keep_mask=mask, emulate_bf16=False, conv1_bf16=False)
        rloss32, _ = loss_and_accuracy(logits32, y.cuda())
        rloss32 = regularised(rloss32, flat32)
        rloss32.backward()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32_conv, tf32_mm
    r32 = spec.views(flat32.grad)
    terms = R.weight_decay_terms(spec, eng.params.detach(), lam)[1] if lam else {}
    for name in r32:
        num = (gv[name].double() - r32[name].double()).norm().item()
        den = r32[name].double().norm().item() + 1e-12
        tol = FP32_GRAD_TOLS.get(name, 0.3)
        out.append(("e2e.grad_vs_fp32.%s(L2 rel)" % name, num / den, tol))
        if name in terms:
            share = terms[name].norm().item() / den
            out.append(("e2e.decay_share_vs_tol.%s(tol/share)" % name, tol / share, 1.0))
    out.append(("e2e.loss_vs_fp32", abs(loss - rloss32.item()), 0.02 * max(1.0, abs(rloss32.item()))))
    # padding of the gradient arena must stay zero (the fused kernel reduces the whole arena)
    out.append(("e2e.grad.padding", eng.grads[~spec.valid_mask().cuda()].abs().max().item(), 1e-12))
    return out


def check_bucketed_step_matches_single_kernel(B: int = 64, steps: int = 6, seed: int = 31, model: str = "lenet",
                                              hidden: int = 256) -> List[Result]:
    """One replica, whole graph-replayed training steps: bucketed aggregation (csrc/fused_bucket.cu: fc1 gradient as bf16,
    applied by the early kernel under the backward pass; small bucket by the late kernel) vs the single fused kernel."""
    import os
    from ..parallel.aggregators import SyncReplicasOptimizer
    from ..schedule import LearningRateSchedule
    g = torch.Generator(device="cpu").manual_seed(seed)
    xs = torch.rand(steps, B, 28, 28, generator=g) - 0.5
    ys = torch.randint(0, 10, (steps, B), generator=g)
    runs = {}
    old = os.environ.get("DMNIST_BUCKET")
    try:
        for mode in ("2", "0"):
            os.environ["DMNIST_BUCKET"] = mode
            if model == "lenet":
                eng, be = _engine(B, seed)
            else:
                from ..engine_cuda import CudaMlpEngine
                be = FusedBackend(ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none"))
                eng = CudaMlpEngine(model, B, be, hidden=hidden, seed=seed, use_graph=True)
            eng.use_graph = True
            eng.attach_optimizer(SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 2, 0.5), 1, 1))
            losses = []
            p_init = eng.params.clone()
            for s in range(steps):
                eng.load_batch(xs[s], ys[s])
                eng.train_step()
                losses.append(eng.loss_acc()[0])
                if s == 0:
                    torch.cuda.synchronize()
                    p_first, g_first = eng.params.clone(), eng.grads.clone()
            torch.cuda.synchronize()
            be.check_error()
            runs[mode] = (eng.params.clone(), eng.shadow.float().clone(), losses, eng.step_info().global_step,
                          bool(eng._bucket_v2), p_first, p_init, g_first)
            e0, e1 = eng._bucket_early
            lr0 = eng._opt_args["lr0"]
            if mode == "2":
                # the LeNet late bucket (236 KB) travels as LL lines, which carry bf16 gradients unless DMNIST_LATE_BF16=0
                late_bf16 = be.late_ll and be.late_bf16
    finally:
        if old is None:
            os.environ.pop("DMNIST_BUCKET", None)
        else:
            os.environ["DMNIST_BUCKET"] = old
    (p2, s2, l2, st2, v2, f2, i2, g2), (p0, _s0, l0, st0, v0, f0, i0, g0) = runs["2"], runs["0"]
    pmax = p0.abs().max().item()
    upd = (f0 - i0).abs()
    tag = "bucket_v2" if model == "lenet" else "bucket_v2.%s" % model
    early = torch.zeros_like(f0, dtype=torch.bool)
    early[e0:e1] = True
    res: List[Result] = []
    if model == "lenet":
        # The LeNet step is bit-reproducible, so both paths hand the aggregation bitwise-equal gradients, and the first
        # update is rebuilt here to the bit.  On one replica both compute p - (lr / 1) * g as one fused multiply-add (lr of
        # step 0 = lr0 exactly).  They differ only in which g: the single kernel takes the fp32 gradient; the bucketed path
        # takes fc1's gradient as the bf16 the fc1_wgrad epilogue stores (RNE of the same fp32 accumulator), and the rest
        # (the late bucket) as bf16 too when its LL lines carry bf16 (csrc/fused_bucket.cu bucket_late_ll_kernel<true>
        # rounds the replica's own contribution exactly as its peers would see it).
        late_bits = float((g2 != g0)[~early].sum())
        scale = float(torch.tensor(lr0, dtype=torch.float32))

        def sgd(p, g):      # fma(-scale, g, p): the product is exact in float64, the difference rounds once to fp32
            return (p.double() - scale * g.double()).float()
        g0r = R.rne_bf16(g0).float()
        gb = torch.where(early | torch.tensor(bool(late_bf16), device=g0.device), g0r, g0)
        res += [(tag + ".init_bits_differ", float((i2 != i0).sum()), 0.0),
                (tag + ".first_step_single_bits_vs_expected", float((f0 != sgd(i0, g0)).sum()), 0.0),
                (tag + ".first_step_bucketed_bits_vs_expected", float((f2 != sgd(i2, gb)).sum()), 0.0)]
        first_excess = 0.0
    else:
        # the MLP gradients are accumulated with fp32 atomics, so two runs differ in the last bits everywhere
        late_bits = 0.0
        allow = upd * 2.0 ** -8 + 1e-6 * pmax
        first_excess = ((f2 - f0).abs() - allow).max().item()
    # later steps amplify the fc1 difference through ReLU / max-pool / dropout decisions: the final comparison is loose
    return res + [
            (tag + ".enabled", 0.0 if (v2 and not v0) else 1.0, 0.5),
            (tag + ".steps", abs(st2 - steps) + abs(st0 - steps), 0.5),
            (tag + ".first_step_late_gradient_bits_differ", late_bits, 0.0),
            (tag + ".first_step_excess", max(first_excess, 0.0) / pmax, 0.0),
            (tag + ".first_update(rel, info)", upd.max().item() / pmax, 1e9),
            (tag + ".params_vs_single(rel)", (p2 - p0).abs().max().item() / pmax, 0.05),
            (tag + ".shadow(rel)", (s2 - p2).abs().max().item() / pmax, 0.01),
            (tag + ".loss", max(abs(a - b) for a, b in zip(l2, l0)), 0.02)]


def check_bucketed_mlp_step_matches_single_kernel() -> List[Result]:
    return (check_bucketed_step_matches_single_kernel(B=128, steps=4, seed=41, model="mlp3", hidden=256)
            + check_bucketed_step_matches_single_kernel(B=96, steps=3, seed=42, model="mlp2", hidden=128))


def lenet_eval_f64(p: Dict[str, torch.Tensor], pb: Dict[str, torch.Tensor], images: torch.Tensor,
                   labels: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Float64 inference forward with the engine's storage roundings: conv1 operands as bf16 (the wgmma conv1 rounds them),
    a1 / a2 stored as bf16, conv2 / fc1 weights from the bf16 shadow ``pb``, fc2 in fp32 weights, no dropout."""
    B = images.shape[0]
    z1 = R.conv5x5(images.to(BF)[..., None], p["conv1_weights"].to(BF))
    a1 = R.rne_bf16(R.pool_fwd(z1, p["conv1_biases"])["out"])
    z2 = R.conv5x5(a1, pb["conv2_weights"])
    a2 = R.rne_bf16(R.pool_fwd(z2, p["conv2_biases"])["out"]).reshape(B, 3136)
    return R.fc2_fwd_bwd(a2 @ pb["fc1_weights"].double(), p["fc1_biases"], p["fc2_weights"], p["fc2_biases"], labels,
                         None, 1.0)


# Inference bounds.  The float64 forward above rounds to bf16 exactly where the kernels store bf16, so the two differ only
# where the kernels' fp32 accumulation moves an activation across a bf16 rounding boundary (a one-ulp flip in a small
# fraction of a1 / a2).  Estimated: such flips move a logit by about 1e-4 of the row's largest logit.  The check measures
# the actual deviation of the kernel's logits and requires it below EVAL_LOGIT_BOUND (relative to 1 + the row's largest
# |logit|); the accuracy is then exact on every row whose top two reference logits are more than twice the measured
# deviation apart, and those must be nearly all rows.
EVAL_LOGIT_BOUND = 2.0 ** -7
EVAL_LOSS_REL = 2.0 ** -10
EVAL_MAX_NEAR_TIES = 0.02      # fraction of rows the accuracy comparison may leave out


def check_evaluate(B: int = 1000, n: int = 2500, seed: int = 23) -> List[Result]:
    """``CudaLeNetEngine.evaluate`` (the evaluator's batch 1000; the last batch is partial) vs the float64 forward."""
    eng, _ = _engine(B, seed)
    g = _gen(seed)
    x = mnist_like(g, n)
    y = torch.randint(0, 10, (n,), generator=g)
    loss, acc = eng.evaluate(x.numpy(), y.numpy())
    xd, yd = x.cuda(), y.cuda()
    ref = lenet_eval_f64(eng.p, eng.pb, xd, yd)
    # the kernels' logits, batch by batch as evaluate() runs them
    got = torch.cat([eng.forward_logits(xd[s:s + B], yd[s:s + B], False) for s in range(0, n, B)]).double()
    return _eval_results("evaluate", loss, acc, got, ref, yd)


def _eval_results(tag: str, loss: float, acc: float, got: torch.Tensor, ref: Dict[str, torch.Tensor], yd) -> List[Result]:
    """evaluate()'s (loss, accuracy) and the kernels' logits ``got`` vs a float64 forward ``ref`` (see the bounds above)."""
    lg, n = ref["logits"], yd.shape[0]
    dev = (got - lg).abs().max(dim=1).values
    dev_rel = float((dev / (1.0 + lg.abs().max(dim=1).values)).max())
    near = ref["gap"] <= 2 * float(dev.max())            # argmax may differ only here
    hits = (lg.argmax(dim=1) == yd) & ~near
    lo, hi = float(hits.sum()) / n, float((hits | near).sum()) / n
    acc_excess = max(lo - acc, acc - hi, 0.0) * n
    return [(tag + ".logit_deviation(rel)", dev_rel, EVAL_LOGIT_BOUND),
            (tag + ".loss(rel)", abs(loss - float(ref["loss"])) / float(ref["loss"]), EVAL_LOSS_REL),
            (tag + ".acc(rows outside near-ties)", acc_excess, 1e-6),
            (tag + ".near_tie_fraction", float(near.sum()) / n, EVAL_MAX_NEAR_TIES)]


def check_training_reduces_loss(B: int = 128, steps: int = 40) -> List[Result]:
    from ..data import make_synthetic_mnist
    from ..parallel.aggregators import SyncReplicasOptimizer
    from ..schedule import LearningRateSchedule
    eng, be = _engine(B, 11)
    eng.use_graph = True
    opt = SyncReplicasOptimizer(be, LearningRateSchedule(0.05, 1000, 1.0), 1, 1)
    eng.attach_optimizer(opt)
    trx, try_, _, _ = make_synthetic_mnist(B * 8, 16, seed=3)
    losses = []
    for s in range(steps):
        i = (s % 8) * B
        eng.load_batch(trx[i:i + B], try_[i:i + B])
        eng.train_step()
        losses.append(eng.loss_acc()[0])
    info = eng.step_info()
    first, last = sum(losses[:5]) / 5, sum(losses[-5:]) / 5
    return [("train.loss_ratio(last/first)", last / first, 0.7), ("train.steps_missing", abs(info.global_step - steps), 0.5),
            ("train.nan", float(any(l != l for l in losses)), 0.5)]


def check_mlp_end_to_end(model: str = "mlp3", B: int = 256, hidden: int = 256, seed: int = 21) -> List[Result]:
    """CudaMlpEngine forward+backward vs torch autograd on the bf16-emulating reference."""
    from ..engine_cuda import CudaMlpEngine
    from ..models import mlp_forward
    ctx = ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none")
    eng = CudaMlpEngine(model, B, FusedBackend(ctx), hidden=hidden, seed=seed, use_graph=False)
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = (torch.rand(B, 28, 28, 1, generator=g) - 0.5)
    y = torch.randint(0, 10, (B,), generator=g)
    eng.load_batch(x.numpy(), y.numpy())
    eng.forward_backward(0)
    torch.cuda.synchronize()
    loss, acc = eng.loss_acc()
    flat = eng.params.detach().clone().requires_grad_(True)
    logits = mlp_forward(eng.spec.views(flat), x.cuda(), emulate_bf16=True)
    rloss, racc = loss_and_accuracy(logits, y.cuda())
    rloss.backward()
    out: List[Result] = [("%s.loss" % model, abs(loss - rloss.item()), 0.02 * max(1.0, abs(rloss.item()))),
                         ("%s.acc" % model, abs(acc - racc.item()), 2.0 / B + 1e-6)]
    gv, rv = eng.spec.views(eng.grads), eng.spec.views(flat.grad)
    for name in rv:
        scale = rv[name].abs().max().item() + 1e-8
        out.append(("%s.grad.%s(rel)" % (model, name), (gv[name] - rv[name]).abs().max().item() / scale, 0.06))
    out.append(("%s.grad.padding" % model, eng.grads[~eng.spec.valid_mask().cuda()].abs().max().item(), 1e-12))
    el, ea = eng.evaluate(x.numpy(), y.numpy())
    out.append(("%s.eval_loss" % model, abs(el - rloss.item()), 0.02 * max(1.0, abs(rloss.item()))))
    return out


def check_mlp2_end_to_end() -> List[Result]:
    return check_mlp_end_to_end("mlp2", B=96, hidden=128, seed=22)


# ---------------------------------------------------------------------------------------------------------------------
# MLP kernels (csrc/mlp_simt.cu, the input conversion) and the MLP step, stage by stage
# ---------------------------------------------------------------------------------------------------------------------
XN_PAD = 64
SENTINEL = 7.0          # prefilled into every output buffer: an element a kernel should write but does not stays 7


def _randint(g: torch.Generator, shape, lo: int, hi: int, denom: int = 1) -> torch.Tensor:
    """:func:`refs.grid` on the generator's own device (the large MLP shapes are generated on the GPU)."""
    return torch.randint(lo, hi + 1, tuple(shape), generator=g, device=g.device).to(torch.float32) / denom


def run_dense10_xent(h, w, b, labels, train: bool, g_b0, la0, logits: bool = True) -> Dict[str, torch.Tensor]:
    """One dense10_xent launch.  dh, dl_pad and logits start as SENTINEL; g_b and loss_acc start at g_b0 / la0 (the
    kernel adds to them)."""
    B, H = h.shape
    dev = h.device
    o = dict(dh=torch.full((B, H), SENTINEL, dtype=BF, device=dev), dl_pad=torch.full((B, XN_PAD), SENTINEL, dtype=BF, device=dev),
             g_b=g_b0.clone(), la=la0.clone(), logits=torch.full((B, 10), SENTINEL, device=dev) if logits else None)
    load().dm_dense10_xent(h, w, b, labels, o["dh"], o["dl_pad"], o["g_b"], o["la"], o["logits"], B, H, int(train),
                           stream_ptr())
    return o


def run_relu_bwd_colsum(dh, h, mode: str, g0) -> Tuple[Optional[torch.Tensor], torch.Tensor]:
    """``mode``: "inplace" (dpre = dh, the engine's use), "out" (a separate SENTINEL-filled dpre) or "none" (h = null: no
    store, column sums of dh only).  Returns (dpre or None, g_bias started at g0)."""
    B, H = dh.shape
    g = g0.clone()
    if mode == "none":
        d, hp = None, None
    elif mode == "inplace":
        d, hp = dh.clone(), h
    else:
        d, hp = torch.full_like(dh, SENTINEL), h
    src = d if mode == "inplace" else dh
    load().dm_relu_bwd_colsum(src, hp, d, g, B, H, stream_ptr())
    return d, g


def _dense10_data(kind: str, g: torch.Generator, B: int, H: int):
    """(h bf16 [B,H], w fp32 [H,10], b [10], labels [B]).  Rows 1 mod 5 carry logits near +80 and rows 3 mod 5 near -80
    (hidden units H-1 / H-2 at 64, weights of magnitude 1 .. 1.5): exp overflows / underflows there unless the row
    maximum is subtracted first.  Grid data: h = k/8 in [0, 2] (about half exact zeros), w = k/64; classes 3 and 7 have
    identical weights and bias, so they tie exactly in every row and the first-max rule decides the accuracy wherever
    they lead (the even rows are labelled 3: a hit for the first maximum, a miss for the last)."""
    dev = g.device
    rows = torch.arange(B, device=dev)
    if kind == "grid":
        h = _randint(g, (B, H), 0, 16, 8) * (torch.rand(B, H, generator=g, device=dev) < 0.5)
        w = _randint(g, (H, 10), -8, 8, 64)
        b = _randint(g, (10,), -16, 16, 64)
        big = _randint(g, (10,), 64, 96, 64)
    else:
        h = torch.relu(torch.randn(B, H, generator=g, device=dev))
        w = torch.randn(H, 10, generator=g, device=dev) * 0.05
        b = torch.randn(10, generator=g, device=dev) * 0.1
        big = 1.0 + 0.5 * torch.rand(10, generator=g, device=dev)
    h[:, H - 1] = torch.where(rows % 5 == 1, torch.full_like(h[:, 0], 64.0), h[:, H - 1])
    h[:, H - 2] = torch.where(rows % 5 == 3, torch.full_like(h[:, 0], 64.0), h[:, H - 2])
    w[H - 1], w[H - 2] = big, -big
    labels = torch.randint(0, 10, (B,), generator=g, device=dev)
    if kind == "grid":
        w[:, 7] = w[:, 3]
        b[3] = b[7] = 0.25
        labels = torch.where(rows % 2 == 0, torch.full_like(labels, 3), labels)
    return h.to(BF), w, b, labels


def _dense10_results(tag: str, kind: str, o: Dict[str, Optional[torch.Tensor]], h, w, b, labels, g_b0, la0, train: bool,
                     logit_unit: float, pad_value: float = SENTINEL) -> List[Result]:
    """dense10_xent outputs vs :func:`refs.dense10_xent`.  Logits: exact on grid data (the premise is asserted), within
    the fp32 bound otherwise.  Loss, dl, g_b and dh go through exp / log: bounded on both kinds (bf16 ones by
    :func:`refs.cmp_bf16_bound`; masked dh elements must be exactly zero).  Accuracy: exact on grid
    data and for a power-of-two B (every partial sum of 1/B terms is an fp32 number), else within the fp32 sum bound;
    on continuous data rows whose top two logits are within twice the logit bound may go either way.  ``pad_value``: what
    dl_pad columns 16..63 held before the launch (the kernel never writes them)."""
    B = h.shape[0]
    ref = R.dense10_xent(h, w, b, labels)
    res: List[Result] = []
    grid = kind == "grid"
    if grid:
        R.assert_exact_grid(ref["logit_abs"], logit_unit, tag + ".logits")
    if o.get("logits") is not None:
        res += R.cmp_bound(tag + ".logits", o["logits"], ref["logits"], 0.0 if grid else ref["logit_err"][:, None])
    la, la0 = o["la"].double(), la0.double()
    inv = float(np.float32(1.0) / np.float32(B))                        # the host's 1.f / B
    terms = ref["loss_terms"] / B
    res += R.cmp_bound(tag + ".loss", la[0], la0[0] + terms.sum(),
                       ref["term_err"].sum() + R.fp32_slack(la0[0].abs() + terms.abs().sum(), B + 1))
    near = torch.zeros_like(ref["hits"]) if grid else ref["gap"] <= 2 * ref["logit_err"]
    lo, hi = float((ref["hits"] & ~near).sum()), float((ref["hits"] | near).sum())
    acc_bound = 0.0 if B & (B - 1) == 0 else float(R.fp32_slack(la0[1].abs() + hi * inv, B + 1))
    a, a0 = float(la[1]), float(la0[1])
    res.append((tag + ".acc", max(a0 + lo * inv - a, a - a0 - hi * inv, 0.0), acc_bound))
    if not train:
        untouched = (o["dh"].double() != SENTINEL).sum() + (o["dl_pad"].double() != SENTINEL).sum() + (o["g_b"] != g_b0).sum()
        return res + [(tag + ".eval_wrote(dh,dl_pad,g_b)", float(untouched), 0.0)]
    dl_pad = o["dl_pad"]
    res += R.cmp_bf16_bound(tag + ".dl_pad", dl_pad[:, :10], ref["dl"], ref["dl_err"])
    res.append((tag + ".dl_pad[10:16]_nonzero", float((dl_pad[:, 10:16].double() != 0).sum()), 0.0))
    res.append((tag + ".dl_pad[16:]_changed", float((dl_pad[:, 16:].double() != pad_value).sum()), 0.0))
    res += R.cmp_bound(tag + ".g_b", o["g_b"], g_b0.double() + ref["dl"].sum(0),
                       ref["dl_err"].sum(0) + R.fp32_slack(g_b0.double().abs() + ref["dl"].abs().sum(0), B + 1))
    # dh = sum_c dl_c w[j,c]: the dl error through w, the 10-term fp32 sum, a result flushed below 2^-126
    wa = w.double().abs()
    dh_bound = ref["dl_err"] @ wa.t() + R.fp32_slack(ref["dl"].abs() @ wa.t(), 10) + R.FTZ
    res += R.cmp_bf16_bound(tag + ".dh", o["dh"], ref["dh"], torch.where(ref["on"], dh_bound, torch.zeros_like(dh_bound)))
    res.append((tag + ".dh.relu_mask", float(((o["dh"].double() != 0) & ~ref["on"]).sum()), 0.0))
    return res


def check_dense10_xent(B: int = 1000, H: int = 192, seed: int = 60, kinds: Sequence[str] = KINDS,
                       train: bool = True) -> List[Result]:
    """dense10_xent at batch B, width H: sentinel-filled outputs, non-zero starting g_b and loss_acc."""
    res: List[Result] = []
    for kind in kinds:
        tag = "dense10_xent.%s.B%d.H%d.%s" % (kind, B, H, "train" if train else "eval")
        g = torch.Generator(device="cuda").manual_seed(seed)
        h, w, b, labels = _dense10_data(kind, g, B, H)
        g_b0 = _randint(g, (10,), -16, 16, 64)
        la0 = torch.tensor([0.5, 0.25], device="cuda")
        o = run_dense10_xent(h, w, b, labels, train, g_b0, la0)
        res += _dense10_results(tag, kind, o, h, w, b, labels, g_b0, la0, train, 1.0 / 512)
        if kind == "grid" and B >= 64:          # the data must hold the ties it is for
            ref_gap = R.dense10_xent(h, w, b, labels)["gap"]
            ties = int(((ref_gap == 0) & (labels == 3)).sum())
            res.append((tag + ".tie_rows_missing", float(ties == 0), 0.0))
    return res


def _colsum_data(kind: str, g: torch.Generator, B: int, H: int):
    """(dh bf16, h bf16).  h holds exact +0 and -0 (masked) and 2^-126, the smallest normal bf16 (kept), at fixed
    positions where dh is 1.  (The kernels run with flush-to-zero, and no stage produces a subnormal activation.)"""
    dev = g.device
    if kind == "grid":
        dh, h = _randint(g, (B, H), -64, 64, 64), _randint(g, (B, H), -2, 2)
    else:
        dh, h = torch.randn(B, H, generator=g, device=dev) * 0.1, torch.randn(B, H, generator=g, device=dev)
    flat_dh, flat_h = dh.view(-1), h.view(-1)
    for k, v in enumerate((0.0, -0.0, 2.0 ** -126)):
        flat_h[k::7] = v
        flat_dh[k::7] = 1.0
    return dh.to(BF), h.to(BF)


def _colsum_results(tag: str, kind: str, dh, h, mode: str, dpre, g, g0) -> List[Result]:
    """dpre: the selection, exact.  g_bias = g0 + column sums of dpre: exact on grid data, fp32-bounded otherwise."""
    rd, rs, ra = R.relu_bwd_colsum(dh, None if mode == "none" else h)
    res: List[Result] = []
    if dpre is not None:
        res += R.cmp_exact(tag + ".dpre", dpre, rd)
    ref, a = g0.double() + rs, g0.double().abs() + ra
    if kind == "grid":
        R.assert_exact_grid(a, 1.0 / 64, tag + ".g_bias")
        res += R.cmp_exact(tag + ".g_bias", g, ref)
    else:
        res += R.cmp_bound(tag + ".g_bias", g, ref, R.fp32_slack(a, dh.shape[0] + 1))
    return res


def check_relu_bwd_colsum(B: int = 257, H: int = 66, seed: int = 61, kinds: Sequence[str] = KINDS,
                          modes: Sequence[str] = ("inplace", "out", "none")) -> List[Result]:
    """relu_bwd_colsum, masked in place, masked into a separate buffer and unmasked (h = null), from a non-zero g_bias."""
    res: List[Result] = []
    for kind in kinds:
        g = torch.Generator(device="cuda").manual_seed(seed)
        dh, h = _colsum_data(kind, g, B, H)
        g0 = _randint(g, (H,), -16, 16, 64)
        if kind == "grid" and B * H >= 3:   # the data must hold its edge values
            on = (h.view(-1)[:3].double() > 0).tolist()
            res.append(("relu_bwd_colsum.edges(+0,-0,min_normal)", float(on != [False, False, True]), 0.0))
        for mode in modes:
            d, gb = run_relu_bwd_colsum(dh, h, mode, g0)
            res += _colsum_results("relu_bwd_colsum.%s.B%d.H%d.%s" % (kind, B, H, mode), kind, dh, h, mode, d, gb, g0)
    return res


def check_f32_to_bf16(B: int = 3, seed: int = 62) -> List[Result]:
    """dm_f32_to_bf16 on B images' worth of values (n = 784 B): bit for bit round-to-nearest-even.  Random finite normal
    fp32 bit patterns and +-0; a quarter of them exact ties (low half 0x8000), a quarter one below / above a tie."""
    n = B * 784
    g = _gen(seed)
    hi = torch.randint(0, 1 << 16, (n,), generator=g, dtype=torch.int64)
    lo = torch.randint(0, 1 << 16, (n,), generator=g, dtype=torch.int64)
    lo[0::4] = 0x8000
    lo[1::4] = torch.where(lo[1::4] < 0x8000, torch.full_like(lo[1::4], 0x7FFF), torch.full_like(lo[1::4], 0x8001))
    e = (hi >> 7) & 0xFF
    hi = torch.where((e == 0) | (e == 0xFF), (hi & 0x807F) | (127 << 7), hi)     # no subnormals, infinities or NaNs
    hi[:2], lo[:2] = torch.tensor([0x0000, 0x8000]), 0                            # +0, -0
    bits = (hi << 16) | lo
    x = torch.where(bits >= 1 << 31, bits - (1 << 32), bits).to(torch.int32).view(torch.float32)
    xd = x.cuda()
    out = torch.full((n,), SENTINEL, dtype=BF, device="cuda")
    load().dm_f32_to_bf16(xd, out, n, stream_ptr())
    want = x.to(BF).view(torch.int16)
    return [("f32_to_bf16.n%d.bits_differ" % n, float((out.cpu().view(torch.int16) != want).sum()), 0.0)]


def _mlp_engine(model: str, B: int, hidden: int, seed: int):
    from ..engine_cuda import CudaMlpEngine
    ctx = ReplicaContext(0, 1, 0, torch.device("cuda", 0), "none")
    return CudaMlpEngine(model, B, FusedBackend(ctx), hidden=hidden, seed=seed, use_graph=False)


def _dgrad_results(tag: str, dh_in, w16, h, dh_out, g_bias, g_bias0) -> List[Result]:
    """A hidden layer's data gradient: dh_out = mask_h(RNE(dh_in w16^T)) on the bf16 shadow w16 (one ulp, with the fp32
    sum bound as slack; masked elements exactly zero), then g_bias = g_bias0 + column sums of the stored dh_out."""
    ref, ra = R.mlp_dgrad(dh_in, w16, h)
    res = R.cmp_bf16(tag, dh_out, ref, R.fp32_slack(ra, dh_in.shape[1]) + 2.0 ** -23 * ref.abs())
    res.append((tag + ".relu_mask", float(((dh_out.double() != 0) & (h.double() <= 0)).sum()), 0.0))
    _, cs, ca = R.relu_bwd_colsum(dh_out, None)
    return res + R.cmp_bound(tag + ".g_bias", g_bias, g_bias0.double() + cs,
                             R.fp32_slack(ca + g_bias0.double().abs(), dh_out.shape[0] + 1))


def _mlp_step_results(tag: str, kind: str, eng, images, labels) -> List[Result]:
    """One ``forward_backward`` of a CudaMlpEngine (``eng``: the engine, or a step's record with the same attributes, see
    ``ops/trajectory.py``), every stage against its float64 reference computed from the engine's
    own input buffers for that stage (x16, h[i], dh[i], dl_pad, the shadow pb, the fp32 arena p): one stage's rounding
    never loosens the next stage's bound, and bf16 inputs keep the forward stages exact on grid data.  Everything
    downstream of the softmax is continuous on both kinds and held to fp32 bounds."""
    p, pb, gr, L, B = eng.p, eng.pb, eng.g, eng.n_layers, eng.batch_size
    res = R.cmp_exact(tag + ".x16", eng.x16, images)                       # RNE of the fp32 images
    src = eng.x16
    for i in range(1, L):
        ref, ra = R.mlp_hidden(src, pb["fc%d_weights" % i], p["fc%d_biases" % i])
        if kind == "grid":                      # images k/8, weights k/8, biases k/64
            R.assert_exact_grid(ra, 2.0 ** -(3 + 3 * i), "%s.h%d" % (tag, i))
        res += R.compare("%s.h%d" % (tag, i), kind, eng.h[i - 1], ref, R.fp32_slack(ra, src.shape[1] + 1) + 2.0 ** -23 * ref.abs())
        src = eng.h[i - 1]
    zeros = torch.zeros(10, device=src.device)
    o = dict(dh=eng.dh[-1], dl_pad=eng.dl_pad, g_b=gr["fc%d_biases" % L], la=eng.d_loss_acc, logits=None)
    res += _dense10_results(tag + ".dense10_xent", kind, o, src, p["fc%d_weights" % L], p["fc%d_biases" % L], labels,
                            zeros, zeros[:2], True, 2.0 ** -(3 + 3 * L), pad_value=0.0)
    def wgrad(name, got, ref, bound):
        # the bucketed aggregation's early layer leaves its GEMM as bf16 (the wire buffer): RNE of the bounded fp32 value
        return (R.cmp_bf16_bound if got.dtype == BF else R.cmp_bound)(name, got, ref, bound)
    dl = eng.dl_pad[:, :10].double()
    res += wgrad("%s.g_fc%d_weights" % (tag, L), gr["fc%d_weights" % L], src.double().t() @ dl,
                 R.fp32_slack(src.double().abs().t() @ dl.abs(), B))
    _, cs, ca = R.relu_bwd_colsum(eng.dh[-1], None)
    res += R.cmp_bound("%s.g_fc%d_biases" % (tag, L - 1), gr["fc%d_biases" % (L - 1)], cs, R.fp32_slack(ca, B + 1))
    for i in range(L - 1, 0, -1):
        below = eng.h[i - 2] if i > 1 else eng.x16
        d = eng.dh[i - 1].double()
        res += wgrad("%s.g_fc%d_weights" % (tag, i), gr["fc%d_weights" % i], below.double().t() @ d,
                     R.fp32_slack(below.double().abs().t() @ d.abs(), B))
        if i > 1:
            res += _dgrad_results("%s.dh%d" % (tag, i - 1), eng.dh[i - 1], pb["fc%d_weights" % i], eng.h[i - 2],
                                  eng.dh[i - 2], gr["fc%d_biases" % (i - 1)], zeros[:1])
    res.append((tag + ".grad_padding", float(eng.grads[~eng.spec.valid_mask().to(eng.grads.device)].abs().max()), 0.0))
    return res


def check_mlp_step(model: str = "mlp3", B: int = 96, hidden: int = 192, seed: int = 63,
                   kinds: Sequence[str] = KINDS) -> List[Result]:
    """CudaMlpEngine.forward_backward, stage by stage.  Grid data: the parameters are overwritten with grid values
    (weights k/8 in [-1, 1], biases k/64) and the shadow refreshed; continuous data: the engine's own initialisation."""
    res: List[Result] = []
    for kind in kinds:
        eng = _mlp_engine(model, B, hidden, seed)
        g = _gen(seed)
        if kind == "grid":
            for name, t in eng.p.items():
                t.copy_(R.grid(g, t.shape, -1, 1, 8) if name.endswith("weights") else R.grid(g, t.shape, -16, 16, 64))
            eng.params_updated()
            x = R.grid(g, (B, 784), -4, 4, 8)
        else:
            x = torch.rand(B, 784, generator=g) - 0.5
        y = torch.randint(0, 10, (B,), generator=g)
        eng.load_batch(x.numpy(), y.numpy())
        eng.forward_backward(0)
        torch.cuda.synchronize()
        res += _mlp_step_results("mlp_step.%s.B%d.H%d.%s" % (model, B, hidden, kind), kind, eng, x.cuda(), y.cuda())
        del eng
    return res


def check_mlp_evaluate(model: str = "mlp3", hidden: int = 1024, B: int = 1000, n: int = 2500, seed: int = 64) -> List[Result]:
    """``CudaMlpEngine.evaluate`` (the evaluator's batch 1000; the last batch is partial) vs :func:`refs.mlp_step_f64`."""
    eng = _mlp_engine(model, B, hidden, seed)
    g = _gen(seed)
    x = mnist_like(g, n).reshape(n, 784)
    y = torch.randint(0, 10, (n,), generator=g)
    loss, acc = eng.evaluate(x.numpy(), y.numpy())
    xd, yd = x.cuda(), y.cuda()
    ref = R.mlp_step_f64(eng.p, eng.pb, xd, yd, eng.n_layers)
    got = []
    with torch.no_grad():
        for s in range(0, n, B):               # the kernels' logits, batch by batch as evaluate() runs them
            m = min(B, n - s)
            out = torch.full((m, 10), SENTINEL, device="cuda")
            eng.d_loss_acc.zero_()
            eng._forward(xd[s:s + m].contiguous(), yd[s:s + m].contiguous(), m, False, logits_out=out)
            got.append(out)
    return _eval_results("mlp_evaluate", loss, acc, torch.cat(got).double(), ref, yd)


ALL_CHECKS = [check_conv1_fwd, check_conv1_wgrad, check_conv2_fwd, check_conv2_dgrad, check_conv2_wgrad, check_fc2_loss, check_fc1_fwd, check_fc2_wgrad, check_fc1_wgrad, check_fc1_dgrad_unpool,
              check_evaluate,
              check_end_to_end, check_bucketed_step_matches_single_kernel, check_bucketed_mlp_step_matches_single_kernel,
              check_training_reduces_loss, check_mlp_end_to_end, check_mlp2_end_to_end,
              check_dense10_xent, check_relu_bwd_colsum, check_f32_to_bf16, check_mlp_step, check_mlp_evaluate]
