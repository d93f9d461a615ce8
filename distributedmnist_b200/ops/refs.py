"""Float64 references of the LeNet and MLP step kernels and the one rule every kernel check compares by.

The references compute in float64 (TF32 never applies), on whatever device their inputs live on, and round to bf16 only
where a kernel stores bf16 (round-to-nearest-even, as ``__floats2bfloat162_rn``).  Layouts are the kernels' own: NHWC
activations, HWIO weights, pooling codes ``(dy * 2 + dx) | ReLU-active << 2``.

The checks run every kernel on two kinds of data:

* **grid** -- values on a coarse binary grid (small integers, k/8, k/64) so that every product and every partial sum is
  an exact fp32 number.  The result then does not depend on the summation order: fp32 outputs equal the reference bit
  for bit, bf16 outputs equal RNE(reference), pooling codes and ReLU flags match exactly.  :func:`assert_exact_grid`
  verifies the premise on the data actually used: the sum of the absolute terms of every output (which bounds every
  partial sum, in any order) stays below 2^24 grid units.  This catches structural faults with zero tolerance: a
  dropped tap, a lost or doubled tile or split, a stale workspace slot, the wrong tie-break.
* **rand** -- continuous random values.  fp32 outputs must agree with float64 to a normwise relative error of 2^-12
  (fp32 accumulation lands near 2^-16; a partial sum stored as bf16 near 2^-9); bf16 outputs must be within one bf16 ulp
  of RNE(reference) and exactly equal in at least 99 % of the elements; pooling codes may differ only where the top two
  window values are within the fp32 error bound of each other.

Every comparison returns ``(name, error, tolerance)`` tuples; a check passes when ``error <= tolerance`` for all of them.
Nothing here needs a GPU: ``tests/test_refs.py`` runs the rule against emulated kernels and seeded faults on the CPU.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

Result = Tuple[str, float, float]

F64 = torch.float64
REL_FP32 = 2.0 ** -12          # normwise bound, fp32 outputs on continuous data
BF16_INEXACT = 0.01            # fraction of bf16 outputs allowed to differ from RNE(reference) by one ulp
GRID_LIMIT = 2 ** 24           # fp32 integers are exact below this many grid units
# Error bound of an fp32 sum of n exact products, in any order: (n + 2) * 2^-23 * sum |terms|.  2^-23 rather than 2^-24:
# tensor-core accumulation is not guaranteed to round to nearest.
FP32_UNIT = 2.0 ** -23


# ---------------------------------------------------------------------------------------------------------------------
# data
# ---------------------------------------------------------------------------------------------------------------------
def grid(g: torch.Generator, shape, lo: int, hi: int, denom: int = 1) -> torch.Tensor:
    """fp32 tensor of k / denom, k uniform in [lo, hi] (CPU; move it where needed)."""
    return torch.randint(lo, hi + 1, tuple(shape), generator=g).to(torch.float32) / denom


def rne_bf16(x: torch.Tensor) -> torch.Tensor:
    """bf16 round-to-nearest-even of ``x``, as float64.  float64 -> fp32 -> bf16: exact-then-RNE on grid data; on
    continuous data the kernels round their fp32 value the same way."""
    return x.to(torch.float32).to(torch.bfloat16).to(F64)


def assert_exact_grid(abs_sum: torch.Tensor, unit: float, what: str) -> float:
    """``abs_sum``: per-output sum of |terms| (float64).  Every partial sum of those terms is a multiple of ``unit`` no
    larger than abs_sum, so it is an exact fp32 number while abs_sum / unit < 2^24.  Returns the largest count of units."""
    units = float(abs_sum.max()) / unit if abs_sum.numel() else 0.0
    assert units < GRID_LIMIT, "%s: grid data reaches %.3g units >= 2^24, fp32 sums would round" % (what, units)
    return units


def fp32_slack(abs_sum: torch.Tensor, n_terms: int) -> torch.Tensor:
    return (n_terms + 2) * FP32_UNIT * abs_sum


# ---------------------------------------------------------------------------------------------------------------------
# comparisons
# ---------------------------------------------------------------------------------------------------------------------
def cmp_exact(name: str, got: torch.Tensor, ref: torch.Tensor) -> List[Result]:
    """Bitwise for fp32 outputs on grid data, ``rne_bf16(ref)`` for bf16 ones: the count of differing elements."""
    r = rne_bf16(ref) if got.dtype == torch.bfloat16 else ref.to(F64)
    return [(name + "[exact]", float((got.to(F64) != r).sum()), 0.0)]


def cmp_fp32(name: str, got: torch.Tensor, ref: torch.Tensor) -> List[Result]:
    ref = ref.to(F64)
    num = float((got.to(F64) - ref).norm())
    den = float(ref.norm())
    return [(name + "[rel]", num / den if den > 0 else num, REL_FP32)]


def _ordered(b: torch.Tensor) -> torch.Tensor:
    """bf16 bit patterns -> integers in value order (adjacent bf16 numbers differ by 1, +0 == -0)."""
    i = b.contiguous().view(torch.int16).to(torch.int32)
    return torch.where(i < 0, -(i & 0x7FFF), i)


def cmp_bf16(name: str, got: torch.Tensor, ref: torch.Tensor, slack: Optional[torch.Tensor] = None) -> List[Result]:
    """Continuous data: within one bf16 ulp of RNE(ref) everywhere, exactly RNE(ref) in >= 99 %.  ``slack``: the
    fp32 error bound of the kernel's value before rounding; where the reference itself lies within that of a rounding
    boundary two ulps can separate honest results, so an element also passes if |got - ref| <= slack."""
    assert got.dtype == torch.bfloat16
    ref = ref.to(F64)
    d = (_ordered(got) - _ordered(rne_bf16(ref).to(torch.bfloat16))).abs()
    far = d > 1
    if slack is not None:
        far &= (got.to(F64) - ref).abs() > slack
    n = max(got.numel(), 1)
    return [(name + "[>1ulp]", float(far.sum()), 0.0), (name + "[inexact]", float((d != 0).sum()) / n, BF16_INEXACT)]


def compare(name: str, kind: str, got: torch.Tensor, ref: torch.Tensor, slack: Optional[torch.Tensor] = None) -> List[Result]:
    """The rule: exact on grid data, by output dtype on continuous data."""
    if kind == "grid":
        return cmp_exact(name, got, ref)
    if got.dtype == torch.bfloat16:
        return cmp_bf16(name, got, ref, slack)
    return cmp_fp32(name, got, ref)


# ---------------------------------------------------------------------------------------------------------------------
# pooling
# ---------------------------------------------------------------------------------------------------------------------
def windows(z: torch.Tensor) -> torch.Tensor:
    """NHWC [B,H,W,C] -> [B,H/2,W/2,C,4], window position p = dy * 2 + dx."""
    B, H, W, C = z.shape
    return z.reshape(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(B, H // 2, W // 2, C, 4)


def first_max(win: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(max, index of its FIRST occurrence) over the last dim -- PyTorch's max-pool rule, spelled out."""
    mx = win.max(dim=-1).values
    eq = win == mx[..., None]
    idx = torch.full(mx.shape, 3, dtype=torch.long, device=win.device)
    for p in (2, 1, 0):
        idx = torch.where(eq[..., p], torch.full_like(idx, p), idx)
    return mx, idx


def decode(code: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    c = code.to(torch.int32)
    return (c & 3).long(), ((c >> 2) & 1).bool()


def encode(idx: torch.Tensor, act: torch.Tensor) -> torch.Tensor:
    return (idx | (act.long() << 2)).to(torch.uint8)


def pool_fwd(z: torch.Tensor, bias: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Max-pool 2x2 / bias / ReLU of the conv pre-activation ``z`` (no bias, float64 NHWC)."""
    win = windows(z)
    mx, idx = first_max(win)
    pre = mx + bias.to(F64)
    act = pre > 0
    return dict(win=win, idx=idx, act=act, pre=pre, out=torch.where(act, pre, torch.zeros_like(pre)),
                code=encode(idx, act))


def cmp_pool(name: str, kind: str, code: torch.Tensor, ref: Dict[str, torch.Tensor],
             slack: Optional[torch.Tensor] = None) -> List[Result]:
    """Pooling codes.  Grid: exact.  Continuous: an index may differ only where the top two window values are within
    2 * slack (the kernel's fp32 error bound per window value) of each other, a ReLU flag only where |pre| <= slack."""
    idx, act = decode(code)
    bad_idx, bad_act = idx != ref["idx"], act != ref["act"]
    if kind != "grid":
        s = slack.max(dim=-1).values if slack is not None else torch.zeros_like(ref["pre"])
        top2 = ref["win"].topk(2, dim=-1).values
        bad_idx &= (top2[..., 0] - top2[..., 1]) > 2 * s
        bad_act &= ref["pre"].abs() > s
    return [(name + ".argmax", float(bad_idx.sum()), 0.0), (name + ".relu_flag", float(bad_act.sum()), 0.0)]


def unpool(vals: torch.Tensor, code: torch.Tensor) -> torch.Tensor:
    """Max-pool/ReLU backward: ``vals`` [B,h,w,C] -> [B,2h,2w,C], each value where its code points, if ReLU was active."""
    idx, act = decode(code)
    B, h, w, C = vals.shape
    masked = vals.to(F64) * act
    out = torch.zeros(B, h, 2, w, 2, C, dtype=F64, device=vals.device)
    for q in range(4):
        out[:, :, q >> 1, :, q & 1, :] = masked * (idx == q)
    return out.reshape(B, 2 * h, 2 * w, C)


# ---------------------------------------------------------------------------------------------------------------------
# references (float64; ``*_abs`` variants give the per-output sum of |terms| for the grid premise and the fp32 bounds)
# ---------------------------------------------------------------------------------------------------------------------
def conv5x5(x: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """SAME 5x5 convolution, NHWC x [B,H,W,Ci], HWIO w [5,5,Ci,Co] -> [B,H,W,Co] float64, no bias."""
    return F.conv2d(x.to(F64).permute(0, 3, 1, 2), w.to(F64).permute(3, 2, 0, 1), padding=2).permute(0, 2, 3, 1)


def conv5x5_dgrad(dy: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """d input of :func:`conv5x5`: dy [B,H,W,Co] -> [B,H,W,Ci]."""
    B, H, W, _ = dy.shape
    dx = torch.nn.grad.conv2d_input((B, w.shape[2], H, W), w.to(F64).permute(3, 2, 0, 1), dy.to(F64).permute(0, 3, 1, 2),
                                    padding=2)
    return dx.permute(0, 2, 3, 1)


def conv5x5_wgrad(x: torch.Tensor, dy: torch.Tensor) -> torch.Tensor:
    """d weights of :func:`conv5x5`: -> HWIO [5,5,Ci,Co]."""
    gw = torch.nn.grad.conv2d_weight(x.to(F64).permute(0, 3, 1, 2), (dy.shape[3], x.shape[3], 5, 5),
                                     dy.to(F64).permute(0, 3, 1, 2), padding=2)
    return gw.permute(2, 3, 1, 0)


def conv1_wgrad(x: torch.Tensor, dpool: torch.Tensor, code: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """conv1 weight [25,32] and bias [32] gradients through the max-pool/ReLU backward; x [B,28,28]."""
    dy = unpool(dpool, code)
    gw = conv5x5_wgrad(x.to(F64)[..., None], dy).reshape(25, 32)
    return gw, dy.sum((0, 1, 2))


def fc1_dgrad_unpool(dh: torch.Tensor, w1: torch.Tensor, code2: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(dy2 [B,14,14,64] before its bf16 store, conv2 bias gradient [64]).  The kernel sums the fp32 values it scatters,
    not their bf16 roundings, so the bias gradient is the exact sum here."""
    B = dh.shape[0]
    dx = (dh.to(F64) @ w1.to(F64).t()).reshape(B, 7, 7, 64)
    dy = unpool(dx, code2.reshape(B, 7, 7, 64))
    return dy, dy.sum((0, 1, 2))


def fc2_fwd_bwd(hsum: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor, b2: torch.Tensor, labels: torch.Tensor,
                keep: Optional[torch.Tensor], keep_prob: float) -> Dict[str, torch.Tensor]:
    """fc1 bias + ReLU (+ dropout when ``keep`` is given), fc2, mean softmax CE, accuracy, d logits [B,12] and d fc1
    pre-activation (before its bf16 store).  ``hsum``: the fc1 GEMM result without bias.  The dropout scale is the
    kernel's fp32 ``1.f / keep_prob`` of an fp32 ``keep_prob``, not the float64 1 / keep_prob (under --use_fast_math
    the kernel's reciprocal is ``rcp.approx``, within one ulp of this; exact for powers of two)."""
    hp = hsum.to(F64) + b1.to(F64)
    on = hp > 0
    inv_keep = 1.0
    if keep is not None:
        on &= keep
        inv_keep = float(np.float32(1.0) / np.float32(keep_prob))
    h = torch.where(on, hp * inv_keep, torch.zeros_like(hp))
    logits = h @ w2.to(F64) + b2.to(F64)
    B = logits.shape[0]
    lse = torch.logsumexp(logits, dim=1)
    lab = labels.long()
    loss = (lse - logits.gather(1, lab[:, None])[:, 0]).mean()
    mx, _ = logits.max(dim=1)
    first = (logits == mx[:, None]).to(torch.int8).argmax(dim=1)       # int8: argmax of 0/1 returns the first 1
    acc = (first == lab).to(F64).mean()
    p = torch.softmax(logits, dim=1)
    dl = (p - F.one_hot(lab, 10).to(F64)) / B
    dh = torch.where(on, (dl @ w2.to(F64).t()) * inv_keep, torch.zeros_like(hp))
    dl12 = torch.zeros(B, 12, dtype=F64, device=dl.device)
    dl12[:, :10] = dl
    return dict(h=h, logits=logits, loss=loss, acc=acc, dl=dl12, dh=dh, gap=_top2_gap(logits))


def _top2_gap(logits: torch.Tensor) -> torch.Tensor:
    t = logits.topk(2, dim=1).values
    return t[:, 0] - t[:, 1]


def fc2_wgrad(h: torch.Tensor, dl: torch.Tensor, dh: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """fc2 weight [512,10] / bias [10] and fc1 bias [512] gradients; dh is summed as the bf16 values the kernel reads."""
    h, dl = h.to(F64), dl.to(F64)[:, :10]
    return h.t() @ dl, dl.sum(0), dh.to(F64).sum(0)


def weight_decay_terms(spec, p, lam: float) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
    """L2 weight decay (``weight_decay.py``) of the weights ``p`` (flat arena or ``spec.views`` dict): ``(R, terms)``,
    R = sum of v^2 / 2 over the decayed variables and ``terms[name]`` = lambda * v, the decayed variable's gradient term,
    both float64.  lambda is taken as the fp32 value the engines use (``weight_decay.value``)."""
    from types import SimpleNamespace
    from .. import weight_decay
    lam = weight_decay.value(SimpleNamespace(weight_decay=lam))
    views = spec.views(p) if isinstance(p, torch.Tensor) else p
    qs = weight_decay.decayed(spec)
    r = sum((views[q.name].to(F64) ** 2).sum() for q in qs) * 0.5
    return r, {q.name: lam * views[q.name].to(F64) for q in qs}


# ---------------------------------------------------------------------------------------------------------------------
# MLP (csrc/mlp_simt.cu for the output layer and the bias gradients; hidden layers and weight gradients on the wgmma GEMM)
# ---------------------------------------------------------------------------------------------------------------------
U32 = 2.0 ** -23               # one fp32 ulp, relative (an upper bound for round-to-nearest and the approximate intrinsics)
LOGF_ABS = 2.0 ** -20          # __logf on [1, 10]: 2^-21.41 absolute on [0.5, 2], 3 ulps above
FTZ = 2.0 ** -126              # --use_fast_math flushes fp32 results (and bf16 conversions) below this to zero


def cmp_bound(name: str, got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> List[Result]:
    """Elementwise |got - ref| <= bound, reported as the largest ratio (a zero bound demands equality)."""
    d = (got.to(F64) - ref.to(F64)).abs()
    bound = torch.as_tensor(bound, dtype=F64, device=d.device).expand_as(d)
    ratio = torch.where(d == 0, torch.zeros_like(d), d / bound)       # d / 0 = inf: a zero bound fails on any difference
    return [(name + "[err/bound]", float(ratio.max()) if ratio.numel() else 0.0, 1.0)]


def cmp_bf16_bound(name: str, got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> List[Result]:
    """bf16 outputs of an fp32 value known to lie within ``bound`` of ``ref``: RNE is monotonic, so each output must lie
    in [RNE(ref - bound), RNE(ref + bound)] -- no exceptions, and exactly RNE(ref) wherever that interval holds one bf16
    number.  For values that pass through exp / log, where cancellation (p - 1 of a confident row) can leave the fp32
    value with no correct bits and the one-ulp / 99 % rule of :func:`cmp_bf16` does not describe the kernel."""
    assert got.dtype == torch.bfloat16
    ref, bound = ref.to(F64), torch.as_tensor(bound, dtype=F64, device=ref.device)
    o = _ordered(got)
    lo = _ordered(rne_bf16(ref - bound).to(torch.bfloat16))
    hi = _ordered(rne_bf16(ref + bound).to(torch.bfloat16))
    return [(name + "[outside RNE(ref+-bound)]", float(((o < lo) | (o > hi)).sum()), 0.0)]


def dense10_xent(h: torch.Tensor, w: torch.Tensor, b: torch.Tensor, labels: torch.Tensor) -> Dict[str, torch.Tensor]:
    """float64 reference of ``dense10_xent`` -- h bf16 [B,H], w the fp32 [H,10] arena weights (NOT the bf16 shadow), b
    [10] -- and the kernel's fp32 error bounds of everything that goes through exp / log:

    ``logits`` = h w + b, ``loss_terms`` per row (logsumexp - logit[label]), ``hits`` per row by the FIRST maximum,
    ``dl`` = (softmax - onehot) / B, ``dh`` = dl w^T where h > 0 else 0 (before its bf16 store), ``logit_err`` [B] bounds
    the kernel's fp32 logits (zero error on grid data), ``term_err`` [B] a row's contribution to the loss sum,
    ``dl_err`` [B,10] the kernel's fp32 dl, ``gap`` the top-two logit distance."""
    B, H = h.shape
    h64, w64, b64 = h.to(F64), w.to(F64), b.to(F64)
    lab = labels.long()
    logits = h64 @ w64 + b64
    logit_abs = h64.abs() @ w64.abs() + b64.abs()
    logit_err = fp32_slack(logit_abs, H + 1).max(dim=1).values             # one lane's fma chain, the shuffle tree, + b
    lse = torch.logsumexp(logits, dim=1)
    lg_label = logits.gather(1, lab[:, None])[:, 0]
    mx = logits.max(dim=1).values
    first = (logits == mx[:, None]).to(torch.int8).argmax(dim=1)
    p = torch.softmax(logits, dim=1)
    y = F.one_hot(lab, 10).to(F64)
    # __expf(x), x = logit - max <= 0: at most 2 + 1.173 |x| ulps; the subtraction adds |x| ulps more
    x = (logits - mx[:, None]).abs()
    e_c = (2.0 + 2.5 * x) * U32
    # relative error of s = sum exp(x_c) (s >= 1; each flushed exp loses less than 2^-126)
    e_s = (p * e_c).sum(dim=1) + 10 * U32 + 10 * FTZ
    L = logit_err[:, None]
    # softmax moves by at most 2 p_c L when every logit moves by L; p * (1 / s), the rcp, - onehot, * (1/B); an exp or a
    # product below 2^-126 is flushed to zero
    dl_err = (p * (e_c + e_s[:, None] + 2 * L + 3 * U32) + U32 * (p - y).abs()) / B + 2 * U32 * ((p - y).abs() / B) \
        + 2 * FTZ
    term = lse - lg_label
    term_err = (e_s + LOGF_ABS + 2 * logit_err + U32 * ((lg_label - mx).abs() + 3 * term.abs())) / B
    dl = (p - y) / B
    on = h64 > 0
    dh = torch.where(on, dl @ w64.t(), torch.zeros_like(h64))
    return dict(logits=logits, logit_abs=logit_abs, logit_err=logit_err, loss_terms=term, term_err=term_err,
                hits=(first == lab), dl=dl, dl_err=dl_err, dh=dh, on=on, gap=_top2_gap(logits))


def relu_bwd_colsum(dh: torch.Tensor, h: Optional[torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(dpre, column sums, column sums of |dpre|), float64: dpre = dh where h > 0, else 0 (dh itself when h is None)."""
    d = dh.to(F64)
    if h is not None:
        d = torch.where(h.to(F64) > 0, d, torch.zeros_like(d))
    return d, d.sum(0), d.abs().sum(0)


def mlp_hidden(src: torch.Tensor, w16: torch.Tensor, b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(relu(src w16 + b) before its bf16 store, sum of |terms|): one hidden layer, src / w16 the bf16 operands."""
    s, w = src.to(F64), w16.to(F64)
    return torch.clamp(s @ w + b.to(F64), min=0.0), s.abs() @ w.abs() + b.to(F64).abs()


def mlp_dgrad(dh: torch.Tensor, w16: torch.Tensor, h: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(d pre-activation of the layer below, before its bf16 store and with the ReLU mask of ``h``, sum of |terms|):
    dh [B,out] times the bf16 shadow w16 [in,out] transposed."""
    d, w = dh.to(F64), w16.to(F64)
    on = h.to(F64) > 0
    z = torch.zeros(1, dtype=F64, device=d.device)
    return torch.where(on, d @ w.t(), z), torch.where(on, d.abs() @ w.abs().t(), z)


def mlp_step_f64(p: Dict[str, torch.Tensor], pb: Dict[str, torch.Tensor], images: torch.Tensor, labels: torch.Tensor,
                 n_layers: int) -> Dict[str, object]:
    """Float64 MLP step with the engine's storage roundings: the input through RNE to bf16, hidden layers on the bf16
    shadow ``pb`` with bias and ReLU and a bf16 store, the output layer on the fp32 weights ``p``, data gradients on the
    shadow with a bf16 store and then the mask, weight / bias gradients from those stored operands."""
    B = images.shape[0]
    src = rne_bf16(images.reshape(B, -1))
    hs = []
    for i in range(1, n_layers):
        src = rne_bf16(mlp_hidden(src, pb["fc%d_weights" % i], p["fc%d_biases" % i])[0])
        hs.append(src)
    out = dense10_xent(src, p["fc%d_weights" % n_layers], p["fc%d_biases" % n_layers], labels)
    g = {"fc%d_weights" % n_layers: src.t() @ rne_bf16(out["dl"]), "fc%d_biases" % n_layers: out["dl"].sum(0)}
    d = rne_bf16(out["dh"])
    for i in range(n_layers - 1, 0, -1):
        below = hs[i - 2] if i > 1 else rne_bf16(images.reshape(B, -1))
        g["fc%d_biases" % i] = d.sum(0)
        g["fc%d_weights" % i] = below.t() @ d
        if i > 1:
            d = rne_bf16(mlp_dgrad(d, pb["fc%d_weights" % i], hs[i - 2])[0])
    out.update(h=hs, grads=g, loss=out["loss_terms"].mean(), acc=out["hits"].to(F64).mean())
    return out
