"""The comparison rule of the kernel checks (ops/refs.py) separates right from subtly wrong: an emulated correct kernel --
fp32 accumulation in another order, then the kernel's storage rounding -- passes on both data kinds, and every seeded
fault fails on the data kind that targets it.  CPU only, B = 2."""
import pytest
import torch

from distributedmnist_b200.ops import refs as R
from distributedmnist_b200.ops import selfcheck as S

B = 2


def _passes(results):
    return all(e <= t for (_, e, t) in results)


# ---- emulated kernels (fp32 on the CPU) ----------------------------------------------------------------------------------
def _conv2_fwd_emulated(a1, w, bias, fault=None):
    """conv2_fwd: fp32 accumulation tap by tap (not the reference's order), max-pool / bias / ReLU epilogue, bf16 store."""
    x = a1.float().permute(0, 3, 1, 2)
    xp = torch.nn.functional.pad(x, (2, 2, 2, 2))
    z = torch.zeros(x.shape[0], 64, 14, 14)
    for tap in reversed(range(25)):
        if fault == "drop_tap" and tap == 7:
            continue
        kh, kw = divmod(tap, 5)
        z += torch.einsum("bchw,co->bohw", xp[:, :, kh:kh + 14, kw:kw + 14], w[kh, kw].float())
    win = R.windows(z.permute(0, 2, 3, 1))
    mx = win[..., 0].clone()
    idx = torch.zeros(mx.shape, dtype=torch.long)
    for p in range(1, 4):
        take = win[..., p] >= mx if fault == "last_max" else win[..., p] > mx
        mx = torch.where(take, win[..., p], mx)
        idx = torch.where(take, torch.full_like(idx, p), idx)
    pre = mx + bias.float() * (2 if fault == "bias_twice" else 1)
    act = pre >= 0 if fault == "relu_ge" else pre > 0
    out = torch.where(act, pre, torch.zeros_like(pre)).to(torch.bfloat16)
    return out, R.encode(idx, act)


def _conv2_fwd_results(kind, fault=None, seed=0):
    a1, w, b = S._conv2_data(kind, S._gen(seed), B)
    out, code = _conv2_fwd_emulated(a1, w, b, fault)
    z, za = R.conv5x5(a1, w), R.conv5x5(a1.abs(), w.abs())
    return S._pool_results("conv2_fwd.%s" % kind, kind, out, code, z, za, b, 800)


def _conv2_wgrad_emulated(a1, dy, splits=2, fault=None, stale=None):
    """conv2_wgrad: per-tile fp32 partials (tile = half of an image's columns), tiles summed per split in tile order,
    splits summed in split order."""
    tiles = []
    for t in range(2 * a1.shape[0]):
        img, half = divmod(t, 2)
        d = torch.zeros_like(dy[img:img + 1].float())
        d[:, :, 8 * half:8 * half + 8] = dy[img:img + 1, :, 8 * half:8 * half + 8].float()
        tiles.append(torch.nn.grad.conv2d_weight(a1[img:img + 1].float().permute(0, 3, 1, 2), (64, 32, 5, 5),
                                                 d.permute(0, 3, 1, 2), padding=2).permute(2, 3, 1, 0))
    n = len(tiles)
    parts = []
    for s in range(splits):
        acc = torch.zeros(5, 5, 32, 64)
        for t in range(n * s // splits, n * (s + 1) // splits):
            if fault == "drop_tile" and s == 1 and t == n * s // splits:
                continue
            acc += tiles[t]
        if fault == "bf16_partial":
            acc = acc.to(torch.bfloat16).float()
        parts.append(acc)
    if fault == "stale_slot":
        parts[1] = stale
    if fault == "split_twice":
        parts.append(parts[0])
    total = torch.zeros(5, 5, 32, 64)
    for p in parts:
        total += p
    return total


def _conv2_wgrad_results(kind, fault=None, seed=3):
    g = S._gen(seed)
    if kind == "rand":
        a1, dy = S._bf(torch.rand(B, 14, 14, 32, generator=g)), S._bf(torch.randn(B, 14, 14, 64, generator=g) * 0.1)
    else:
        a1, dy = S._bf(R.grid(g, (B, 14, 14, 32), 0, 3)), S._bf(R.grid(g, (B, 14, 14, 64), -3, 3))
        R.assert_exact_grid(R.conv5x5_wgrad(a1.abs(), dy.abs()), 1.0, "conv2_wgrad")
    stale = None
    if fault == "stale_slot":     # the slot of split 1 still holds a partial sum of an earlier launch on other data
        g2 = S._gen(seed + 1)
        stale = _conv2_wgrad_emulated(S._bf(R.grid(g2, (B, 14, 14, 32), 0, 3)), S._bf(R.grid(g2, (B, 14, 14, 64), -3, 3)), 1)
    gw = _conv2_wgrad_emulated(a1, dy, 2, fault, stale)
    return R.compare("conv2_wgrad.%s" % kind, kind, gw, R.conv5x5_wgrad(a1, dy))


@pytest.mark.parametrize("kind", ["grid", "rand", "edges"])
def test_emulated_correct_conv2_fwd_passes(kind):
    res = _conv2_fwd_results(kind)
    assert _passes(res), res


@pytest.mark.parametrize("kind", ["grid", "rand"])
def test_emulated_correct_conv2_wgrad_passes(kind):
    res = _conv2_wgrad_results(kind)
    assert _passes(res), res


# (fault, data kind that must catch it)
FWD_FAULTS = [("drop_tap", "grid"), ("last_max", "edges"), ("relu_ge", "edges"), ("bias_twice", "grid")]
WGRAD_FAULTS = [("drop_tile", "grid"), ("split_twice", "grid"), ("stale_slot", "grid"), ("bf16_partial", "rand")]


@pytest.mark.parametrize("fault,kind", FWD_FAULTS)
def test_seeded_forward_fault_fails(fault, kind):
    res = _conv2_fwd_results(kind, fault)
    assert not _passes(res), "fault %s passed on %s data: %s" % (fault, kind, res)


@pytest.mark.parametrize("fault,kind", WGRAD_FAULTS)
def test_seeded_weight_gradient_fault_fails(fault, kind):
    res = _conv2_wgrad_results(kind, fault)
    assert not _passes(res), "fault %s passed on %s data: %s" % (fault, kind, res)


def _bump(t, idx, ulps):
    """``t`` with the elements at ``idx`` moved by ``ulps`` bf16 ulps"""
    t = t.clone()
    t.view(torch.int16)[idx] += ulps
    return t


@pytest.mark.parametrize("kind", ["grid", "rand"])
def test_references_in_row_chunks_give_the_whole_batch_results(kind, monkeypatch):
    """Large batches evaluate the float64 references S.REF_ROWS rows at a time.  On 7 rows in chunks of 3, 3 and 1,
    with outputs wrong in a few elements of several chunks, every result equals the one on the whole batch."""
    n, bf = 7, torch.bfloat16
    g = S._gen(11)
    a1, w, b = S._conv2_data(kind, g, n)
    p2 = R.pool_fwd(R.conv5x5(a1, w), b)
    out2 = _bump(p2["out"].float().to(bf), ([0, 4, 6], 3, 2, 5), 2)
    code2 = p2["code"].clone()
    code2[[1, 5], 0, 0, 0] ^= 4
    dy = S._bf(R.grid(g, (n, 14, 14, 64), -4, 4)) if kind == "grid" else S._bf(torch.randn(n, 14, 14, 64, generator=g) * 0.1)
    dx = _bump(R.conv5x5_dgrad(dy, w).float().to(bf), ([2, 3, 6], 1, 1, 1), 3)
    gw2 = R.conv5x5_wgrad(a1, dy).float()
    dh, w1 = S._bf(R.grid(g, (n, 512), -1, 1)), S._bf(R.grid(g, (3136, 512), -8, 8, 64))
    c2 = S._codes(g, (n, 3136))
    rdy, rgb = R.fc1_dgrad_unpool(dh, w1, c2)
    dy2 = _bump(rdy.float().to(bf), ([0, 6], 5, 5, 7), 2)
    x, w_1, b_1 = S._conv1_data(kind, g, n)
    p1 = R.pool_fwd(R.conv5x5(x.to(bf)[..., None], w_1.to(bf)), b_1)
    out1 = _bump(p1["out"].float().to(bf), ([3, 6], 7, 7, 0), 2)
    dp, c1 = S._bf(R.grid(g, (n, 14, 14, 32), -4, 4)), S._codes(g, (n, 14, 14, 32))
    gw1, gb1 = (t.float() for t in R.conv1_wgrad(x.to(bf), dp, c1))

    def results():
        return (S.conv2_fwd_results("c2f", kind, a1, w, b, out2, code2) + S.conv2_dgrad_results("c2d", kind, dy, w, dx)
                + S.conv2_wgrad_results("c2w", kind, a1, dy, gw2 + (gw2 == gw2.max()))
                + S.fc1_dgrad_results("f1d", "grid", dh, w1, c2, dy2, rgb.float())
                + S.conv1_fwd_results("c1f", kind, x, w_1, b_1, out1, p1["code"])
                + S.conv1_wgrad_results("c1w", "grid", x, dp, c1, gw1, gb1 + 1))
    whole = results()
    monkeypatch.setattr(S, "REF_ROWS", 3)
    chunked = results()
    assert [r[0] for r in chunked] == [r[0] for r in whole]
    for (name, e, t), (_, e2, t2) in zip(whole, chunked):
        assert e2 == pytest.approx(e, rel=1e-9, abs=1e-15) and t2 == t, name
    assert sum(e > t for (_, e, t) in whole) >= 7, whole


def test_bf16_rule_one_ulp_and_exact_fraction():
    ref = torch.linspace(-3, 3, 1000, dtype=torch.float64)
    good = R.rne_bf16(ref).to(torch.bfloat16)
    assert _passes(R.cmp_bf16("x", good, ref))
    # two ulps off in one element
    bad2 = good.view(torch.int16).clone()
    bad2[600] += 2
    assert not _passes(R.cmp_bf16("x", bad2.view(torch.bfloat16), ref))
    # truncation instead of RNE: one ulp off in about half the elements
    trunc = (ref.float().view(torch.int32) & ~0xFFFF).view(torch.float32).to(torch.bfloat16)
    assert not _passes(R.cmp_bf16("x", trunc, ref))


def test_grid_premise_is_enforced():
    with pytest.raises(AssertionError):
        R.assert_exact_grid(torch.tensor([2.0 ** 24]), 1.0, "too large")
    assert R.assert_exact_grid(torch.tensor([2.0 ** 24 - 1]), 1.0, "fits") < 2 ** 24


def _l2_loss(v):
    """TF's ``tf.nn.l2_loss``: sum(v^2) / 2."""
    return (v * v).sum() / 2


# the reference model's regulariser (src/mnist.py, commented out there): l2_loss of these four, conv layers not decayed
REFERENCE_REGULARISED = {"lenet": ("fc1_weights", "fc1_biases", "fc2_weights", "fc2_biases")}


@pytest.mark.parametrize("model", ["lenet", "mlp2", "mlp3"])
@pytest.mark.parametrize("lam", [5e-4, 0.0123, 2.0 ** -4])
def test_weight_decay_terms_are_the_gradient_of_the_regulariser(model, lam):
    """R and every decayed variable's gradient term against torch.autograd of lambda * sum l2_loss(v) in float64 (lambda
    as its fp32 value), over the whole arena: a variable the helper leaves out, or one it decays that the objective does
    not, fails here, as does sum v^2 in place of sum v^2 / 2."""
    import numpy as np
    from distributedmnist_b200.models import get_model
    spec = get_model(model, 64)[0]
    g = torch.Generator().manual_seed(3)
    flat = (spec.init_flat(7).double() + 0.01 * torch.randn(spec.arena_numel, generator=g, dtype=torch.float64)) \
        * spec.valid_mask()
    names = REFERENCE_REGULARISED.get(model, tuple(q.name for q in spec.params))     # the MLPs: every layer is fc
    x = flat.clone().requires_grad_(True)
    v = spec.views(x)
    lam32 = float(np.float32(lam))
    obj = lam32 * sum(_l2_loss(v[n]) for n in names)
    (grad,) = torch.autograd.grad(obj, x)
    r, terms = R.weight_decay_terms(spec, flat, lam)
    obj = float(obj.detach())
    assert abs(float(r) * lam32 - obj) <= 1e-13 * obj
    want = spec.views(grad)
    assert set(terms) == set(names)
    for q in spec.params:
        if q.name in terms:
            assert torch.allclose(terms[q.name], want[q.name], rtol=1e-15, atol=0), q.name
        else:
            assert not want[q.name].any(), q.name          # not decayed: the objective's gradient is zero there
    if model == "lenet":
        assert not any(n.startswith("conv") for n in terms)


def test_first_max_tie_break():
    win = torch.tensor([[1.0, 3.0, 3.0, 2.0], [5.0, 5.0, 5.0, 5.0], [0.0, 0.0, 0.0, 1.0]], dtype=torch.float64)
    _, idx = R.first_max(win)
    assert idx.tolist() == [1, 0, 3]
