"""The MLP kernel checks (ops/selfcheck.py, ops/refs.py) separate right from subtly wrong: each MLP kernel emulated on the
CPU in fp32 -- summing in another order than the float64 reference, rounding where the kernel stores bf16 -- passes on
both data kinds, and every seeded fault fails on the data kind that targets it.  CPU only."""
import pytest
import torch

from distributedmnist_b200.ops import refs as R
from distributedmnist_b200.ops import selfcheck as S

BF = torch.bfloat16
CTAS = 3            # emulated grid of dense10_xent: 3 CTAs x 8 warps, so rows 24.. are a warp's second row


def _passes(results):
    return all(e <= t for (_, e, t) in results)


# ---- dense10_xent ------------------------------------------------------------------------------------------------------
def _dense10_emulated(h, w, b, labels, train, g_b0, la0, fault=None):
    B, H = h.shape
    hf = h.float()
    wf = w.to(BF).float() if fault == "w_bf16" else w.float()
    acc = torch.zeros(B, 10)
    for lane in reversed(range(32)):         # lane partial sums (j = lane mod 32), added lane by lane
        acc += hf[:, lane::32] @ wf[lane::32]
    logits = acc + b.float()
    rows = torch.ones(B, dtype=torch.bool)
    if fault == "skip_wrap_row":
        rows[8 * min((B + 7) // 8, CTAS)] = False
    m = logits.max(dim=1).values
    eq = logits == m[:, None]
    idx = torch.arange(10).expand(B, 10)
    arg = torch.where(eq, idx, 10 if fault != "last_max" else -1)
    arg = arg.max(dim=1).values if fault == "last_max" else arg.min(dim=1).values
    inv = torch.tensor(1.0 / B, dtype=torch.float32)
    p = torch.exp(logits - m[:, None])
    s = p.sum(dim=1)
    lab = labels.long()
    term = (torch.log(s) - (logits.gather(1, lab[:, None])[:, 0] - m)) * inv
    hit = (arg == lab).float() * inv
    o = dict(dh=torch.full((B, H), S.SENTINEL, dtype=BF), dl_pad=torch.full((B, S.XN_PAD), S.SENTINEL, dtype=BF),
             g_b=g_b0.clone(), la=la0.clone(), logits=torch.full((B, 10), S.SENTINEL))
    o["logits"][rows] = logits[rows]
    o["la"][0] += term[rows].flip(0).sum()
    o["la"][1] += hit[rows].flip(0).sum()
    if not train:
        return o
    dl = (p / s[:, None] - torch.nn.functional.one_hot(lab, 10).float()) * inv
    dh = dl @ wf.t()
    if fault != "no_dh_mask":
        dh = torch.where(hf > 0, dh, torch.zeros_like(dh))
    o["dh"][rows] = dh[rows].to(BF)
    o["dl_pad"][rows, :10] = dl[rows].to(BF)
    if fault != "dl_pad_stale":
        o["dl_pad"][rows, 10:16] = 0.0
    o["g_b"] += (dl.to(BF).float() if fault == "g_b_from_bf16" else dl)[rows].flip(0).sum(0)
    return o


def _dense10_results(kind, fault=None, train=True, B=40, H=64, seed=0):
    g = S._gen(seed)
    h, w, b, labels = S._dense10_data(kind, g, B, H)
    g_b0 = S._randint(g, (10,), -16, 16, 64)
    la0 = torch.tensor([0.5, 0.25])
    o = _dense10_emulated(h, w, b, labels, train, g_b0, la0, fault)
    return S._dense10_results("dense10_xent.%s" % kind, kind, o, h, w, b, labels, g_b0, la0, train, 1.0 / 512)


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("kind", ["grid", "rand"])
def test_emulated_correct_dense10_xent_passes(kind, train):
    for B in (1, 9, 40, 64):
        res = _dense10_results(kind, train=train, B=B)
        assert _passes(res), res


def test_dense10_grid_data_ties_decide_the_accuracy():
    g = S._gen(0)
    h, w, b, labels = S._dense10_data("grid", g, 40, 64)
    ref = R.dense10_xent(h, w, b, labels)
    assert int(((ref["gap"] == 0) & (labels == 3)).sum()) > int(((ref["gap"] == 0) & (labels == 7)).sum())
    assert float(ref["logits"].abs().max()) > 64       # the rows near +-80


# (fault, data kind that must catch it)
DENSE10_FAULTS = [("w_bf16", "rand"), ("last_max", "grid"), ("dl_pad_stale", "grid"), ("no_dh_mask", "grid"),
                  ("g_b_from_bf16", "rand"), ("skip_wrap_row", "grid")]


@pytest.mark.parametrize("fault,kind", DENSE10_FAULTS)
def test_seeded_dense10_xent_fault_fails(fault, kind):
    res = _dense10_results(kind, fault)
    assert not _passes(res), "fault %s passed on %s data: %s" % (fault, kind, res)


def test_bf16_bound_rule():
    ref = torch.linspace(-3, 3, 1001, dtype=torch.float64)
    good = R.rne_bf16(ref).to(BF)
    assert _passes(R.cmp_bf16_bound("x", good, ref, torch.zeros_like(ref)))
    one_off = good.view(torch.int16).clone()
    one_off[600] += 1
    assert not _passes(R.cmp_bf16_bound("x", one_off.view(BF), ref, 2.0 ** -12 * ref.abs()))
    # a bound reaching the next rounding boundary admits the neighbour, and nothing further
    wide = 2.0 ** -7 * ref.abs()
    assert _passes(R.cmp_bf16_bound("x", one_off.view(BF), ref, wide))
    one_off[600] += 2
    assert not _passes(R.cmp_bf16_bound("x", one_off.view(BF), ref, wide))


# ---- relu_bwd_colsum ---------------------------------------------------------------------------------------------------
def _colsum_emulated(dh, h, mode, g0, fault=None):
    """The kernel's slabs (256 rows each, at most 64), 8 row lanes per slab; slabs land in reverse order."""
    B, H = dh.shape
    slabs = min((B + 255) // 256, 64)
    rows = (B + slabs - 1) // slabs
    d = dh.float()
    if mode != "none":
        d = torch.where(h.float() > 0, d, torch.zeros_like(d))
    out = None if mode == "none" else (dh.clone() if mode == "inplace" else torch.full_like(dh, S.SENTINEL))
    g = g0.clone()
    for s in reversed(range(slabs)):
        r0, r1 = s * rows, min(B, (s + 1) * rows)
        if fault == "drop_last_row" and r1 - r0 != rows:
            r1 -= 1
        part = torch.zeros(H)
        for lane in range(8):
            part += d[r0 + lane:r1:8].sum(0)
        g += part
        if out is not None:
            out[r0:r1] = d[r0:r1].to(BF)
    return out, g


def _colsum_results(kind, mode, fault=None, B=16385, H=6, seed=1):
    g = S._gen(seed)
    dh, h = S._colsum_data(kind, g, B, H)
    g0 = S._randint(g, (H,), -16, 16, 64)
    d, gb = _colsum_emulated(dh, h, mode, g0, fault)
    return S._colsum_results("relu_bwd_colsum.%s.%s" % (kind, mode), kind, dh, h, mode, d, gb, g0)


@pytest.mark.parametrize("mode", ["inplace", "out", "none"])
@pytest.mark.parametrize("kind", ["grid", "rand"])
def test_emulated_correct_relu_bwd_colsum_passes(kind, mode):
    for B in (1, 257, 16385):
        res = _colsum_results(kind, mode, B=B)
        assert _passes(res), res


def test_colsum_edge_values_are_masked_as_the_kernel_must():
    """+0 and -0 are masked, the smallest normal bf16 is kept: a kernel testing h >= 0 (or h != 0) fails."""
    g = S._gen(2)
    dh, h = S._colsum_data("grid", g, 16, 8)
    assert h.view(-1)[1].view(torch.int16) == -32768            # a real -0
    d, gb = _colsum_emulated(dh, h, "out", torch.zeros(8))
    assert _passes(S._colsum_results("c", "grid", dh, h, "out", d, gb, torch.zeros(8)))
    wrong = torch.where(h.float() >= 0, dh.float(), torch.zeros(16, 8)).to(BF)
    assert not _passes(S._colsum_results("c", "grid", dh, h, "out", wrong, gb, torch.zeros(8)))


@pytest.mark.parametrize("mode", ["inplace", "out"])
def test_seeded_colsum_uneven_slab_fault_fails(mode):
    res = _colsum_results("grid", mode, "drop_last_row")
    assert not _passes(res), res


# ---- hidden-layer data gradient (the wgmma GEMM into dh, then relu_bwd_colsum in place) --------------------------------
def _dgrad_results(kind, fault=None, B=48, H=64, seed=3):
    g = S._gen(seed)
    if kind == "grid":
        dh_in, w = R.grid(g, (B, H), -8, 8, 64).to(BF), R.grid(g, (H, H), -8, 8, 64)
    else:
        dh_in, w = (torch.randn(B, H, generator=g) * 0.01).to(BF), torch.randn(H, H, generator=g) * 0.05
    h = torch.randn(B, H, generator=g).to(BF)
    w16 = w.to(BF)
    used = w if fault == "fp32_weights" else w16.float()
    out = torch.zeros(B, H)
    for k in reversed(range(H)):           # another order than the reference
        out += dh_in.float()[:, k:k + 1] * used[:, k][None, :]
    out = out.to(BF)
    out, gb = _colsum_emulated(out, h, "inplace", torch.zeros(H))
    return S._dgrad_results("dgrad.%s" % kind, dh_in, w16, h, out, gb, torch.zeros(1))


@pytest.mark.parametrize("kind", ["grid", "rand"])
def test_emulated_correct_dgrad_passes(kind):
    res = _dgrad_results(kind)
    assert _passes(res), res


def test_seeded_dgrad_on_fp32_weights_fails():
    res = _dgrad_results("rand", "fp32_weights")
    assert not _passes(res), res


# ---- the float64 MLP step ----------------------------------------------------------------------------------------------
def test_float64_step_matches_autograd_on_rounded_operands():
    """mlp_step_f64's gradients are those of the loss of a model whose hidden operands are the bf16 roundings it applies
    (checked against autograd on those rounded tensors, output layer in fp32 weights)."""
    from distributedmnist_b200.models import get_model
    spec, _ = get_model("mlp3", 64)
    flat = spec.init_flat(5).double()
    p = spec.views(flat)
    pb = {k: R.rne_bf16(v) for k, v in p.items()}
    g = S._gen(4)
    x, y = torch.rand(16, 784, generator=g) - 0.5, torch.randint(0, 10, (16,), generator=g)
    out = R.mlp_step_f64(p, pb, x, y, 3)
    h1, h2 = out["h"]
    w3 = p["fc3_weights"].clone().requires_grad_(True)
    b3 = p["fc3_biases"].clone().requires_grad_(True)
    loss = torch.nn.functional.cross_entropy(h2 @ w3 + b3, y)
    loss.backward()
    assert torch.allclose(out["loss"], loss.detach(), rtol=1e-12)
    # the stored dl is rounded to bf16 before the weight gradient GEMM: agreement to bf16 precision
    assert torch.allclose(out["grads"]["fc3_weights"], w3.grad, rtol=2 ** -7, atol=2 ** -7 * float(w3.grad.abs().max()))
    assert torch.allclose(out["grads"]["fc3_biases"], b3.grad, rtol=1e-12, atol=0)
    assert out["grads"]["fc1_weights"].shape == (784, 64) and bool(torch.isfinite(out["grads"]["fc1_weights"]).all())
