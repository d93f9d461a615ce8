"""wgmma GEMM vs a plain PyTorch fp32 reference of the same op (SURVEY §4 item 2)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(a, b, a_major, b_major):
    A = a.float().t() if a_major == "mn" else a.float()
    Bm = b.float() if b_major == "mn" else b.float().t()
    return A @ Bm


CASES = [
    # (M, N, K) incl. partial tiles and K not a multiple of 64
    (128, 128, 64), (256, 512, 3136), (256, 3136, 512), (3136, 512, 256), (200, 72, 784), (128, 64, 100 * 8),
]


@pytest.mark.parametrize("a_major", ["k", "mn"])
@pytest.mark.parametrize("b_major", ["k", "mn"])
@pytest.mark.parametrize("bn", [64, 128])
def test_gemm_all_majors(a_major, b_major, bn):
    from distributedmnist_b200.ops.gemm import gemm_bf16
    torch.manual_seed(0)
    for (M, N, K) in CASES:
        a = (torch.randn((K, M) if a_major == "mn" else (M, K), device="cuda") * 0.5).to(torch.bfloat16)
        b = (torch.randn((K, N) if b_major == "mn" else (N, K), device="cuda") * 0.5).to(torch.bfloat16)
        out = gemm_bf16(a, b, a_major, b_major, bn=bn)
        ref = _ref(a, b, a_major, b_major)
        err = (out - ref).abs().max().item()
        tol = 2e-3 * (K ** 0.5) + 1e-3
        assert err < tol, "M=%d N=%d K=%d majors=%s/%s bn=%d: max err %g (tol %g)" % (M, N, K, a_major, b_major, bn, err, tol)


def test_gemm_split_k_atomic_and_bf16_out():
    from distributedmnist_b200.ops.gemm import gemm_bf16
    torch.manual_seed(1)
    a = (torch.randn(256, 3136, device="cuda") * 0.3).to(torch.bfloat16)
    w = (torch.randn(3136, 512, device="cuda") * 0.1).to(torch.bfloat16)
    ref = a.float() @ w.float()
    out = gemm_bf16(a, w, "k", "mn", splits=16)
    assert (out - ref).abs().max().item() < 0.05
    out16 = gemm_bf16(a, w, "k", "mn", out_dtype=torch.bfloat16)
    assert (out16.float() - ref).abs().max().item() < 0.25


# ---- float64 references (ops/refs.py): exact on grid data, precision bounds on continuous data --------------------------
def _grid_or_rand(kind, shape, g, lo, hi, denom, scale):
    from distributedmnist_b200.ops import refs as R
    t = R.grid(g, shape, lo, hi, denom) if kind == "grid" else torch.randn(shape, generator=g) * scale
    return t.to(torch.bfloat16).cuda()


def _check(results):
    bad = [(n, e, t) for (n, e, t) in results if not e <= t]
    assert not bad, "failed: %s\nall: %s" % (bad, results)


def _gemm_case(kind, M, N, K, a_mn, b_mn, epi, bn, seed, splits=1, ldo=None, with_bias=False):
    from distributedmnist_b200.ops import gemm as G
    from distributedmnist_b200.ops import refs as R
    g = torch.Generator().manual_seed(seed)
    a = _grid_or_rand(kind, (K, M) if a_mn else (M, K), g, -4, 4, 1, 0.5)
    b = _grid_or_rand(kind, (K, N) if b_mn else (N, K), g, -8, 8, 64, 0.1)
    bias = (R.grid(g, (N,), -16, 16, 64) if kind == "grid" else torch.randn(N, generator=g) * 0.1).cuda()
    A = a.double().t() if a_mn else a.double()
    Bm = b.double() if b_mn else b.double().t()
    ref, ra = A @ Bm, A.abs() @ Bm.abs()
    if with_bias:
        ref = torch.clamp(ref + bias.double(), min=0.0)
    if kind == "grid":
        R.assert_exact_grid(ra + bias.double().abs(), 1.0 / 64, "gemm")
    ldo = ldo or N
    dt = torch.float32 if epi in (G.EPI_STORE_F32, G.EPI_ATOMIC_F32) else torch.bfloat16
    out = torch.full((M, ldo), 7.0, device="cuda").to(dt)
    if epi == G.EPI_ATOMIC_F32:
        out.zero_()
    G.gemm_bf16_raw(a, b, out, M, N, K, a.stride(0), b.stride(0), ldo, a_mn, b_mn, epi, splits=splits, bn=bn,
                    bias=bias if with_bias else None)
    tag = "M%d N%d K%d epi%d bn%d %s" % (M, N, K, epi, bn, kind)
    return R.compare(tag, kind, out[:, :N], ref, R.fp32_slack(ra, K) + 2.0 ** -23 * ref.abs())


@pytest.mark.parametrize("kind", ["grid", "rand"])
@pytest.mark.parametrize("epi", [0, 2, 3])
def test_gemm_bn256_epilogues_vs_float64(kind, epi):
    """bn=256: the MLP default when the hidden width is a multiple of 256; epilogue 3 = bias + ReLU -> bf16."""
    for (M, N, K, a_mn, b_mn) in [(256, 1024, 784, False, True), (200, 512, 1024, False, False),
                                  (784, 1024, 256, True, True)]:
        _check(_gemm_case(kind, M, N, K, a_mn, b_mn, epi, 256, seed=K + epi, with_bias=epi == 3))


@pytest.mark.parametrize("kind", ["grid", "rand"])
@pytest.mark.parametrize("bn", [64, 128])
def test_gemm_bias_relu_epilogue_vs_float64(kind, bn):
    _check(_gemm_case(kind, 300, 192, 784, False, True, 3, bn, seed=bn, with_bias=True))


@pytest.mark.parametrize("kind", ["grid", "rand"])
def test_gemm_n10_ldo10_output_layer_wgrad(kind):
    """The MLP's last-layer weight gradient: dW[H,10] = h^T (MN-major) * dl (MN-major, 64-wide zero-padded rows), ldo 10."""
    from distributedmnist_b200.ops import gemm as G
    from distributedmnist_b200.ops import refs as R
    g = torch.Generator().manual_seed(10)
    for B, H in [(256, 256), (96, 128), (1000, 1024)]:
        h = _grid_or_rand(kind, (B, H), g, 0, 4, 1, 1.0)
        dl = torch.zeros(B, 64, dtype=torch.bfloat16, device="cuda")
        dl[:, :10] = _grid_or_rand(kind, (B, 10), g, -32, 32, 64, 0.1)
        out = torch.full((H, 10), 7.0, device="cuda")
        G.gemm_bf16_raw(h, dl, out, H, 10, B, H, 64, 10, True, True, G.EPI_STORE_F32, bn=64)
        ref = h.double().t() @ dl.double()[:, :10]
        if kind == "grid":
            R.assert_exact_grid(h.double().abs().t() @ dl.double().abs()[:, :10], 1.0 / 64, "n10")
        _check(R.compare("N10 B%d H%d %s" % (B, H, kind), kind, out, ref))


@pytest.mark.parametrize("kind", ["grid", "rand"])
@pytest.mark.parametrize("M,N,K,a_mn,b_mn,epi", [
    (4096, 4096, 8192, True, True, 0),      # hidden weight gradient h^T dh: K = batch, both operands MN-major
    (8192, 4096, 4096, False, False, 2),    # data gradient dh W^T: K-major / K-major, bf16 store
    (784, 4096, 8192, True, True, 0),       # fc1 weight gradient x^T dh: M = 784, a partial M tile
])
def test_gemm_mlp_batch_8192_shapes(kind, M, N, K, a_mn, b_mn, epi):
    """The GEMMs of the 3-layer MLP step at batch 8192, width 4096 (bn = 256) that no other test runs, in full."""
    _check(_gemm_case(kind, M, N, K, a_mn, b_mn, epi, 256, seed=M + K + epi))


@pytest.mark.parametrize("kind", ["grid", "rand"])
def test_gemm_lenet_shapes_at_batch_256(kind):
    """Every GEMM the LeNet engine issues at B=256: fc1 forward (strided split-K, checked per split by check_fc1_fwd),
    fc1 weight gradient fp32 / bf16, and the unfused fc1 data gradient."""
    from distributedmnist_b200.ops import selfcheck
    res = selfcheck.check_fc1_fwd(B=256, seed=31, kinds=(kind,)) + selfcheck.check_fc1_wgrad(B=256, seed=32, kinds=(kind,))
    res += _gemm_case(kind, 256, 3136, 512, False, False, 2, 64, seed=33)
    _check(res)


@pytest.mark.parametrize("kind", ["grid", "rand"])
def test_gemm_strided_split_k_as_fc1_fwd(kind):
    from distributedmnist_b200.ops import gemm as G
    from distributedmnist_b200.ops import refs as R
    g = torch.Generator().manual_seed(34)
    M, N, K, S = 129, 512, 3136, 7
    a = _grid_or_rand(kind, (M, K), g, 0, 2, 1, 0.5)
    w = _grid_or_rand(kind, (K, N), g, -8, 8, 64, 0.05)
    part = torch.full((S, M, N), 7.0, device="cuda")
    G.gemm_bf16_raw(a, w, part, M, N, K, K, N, N, False, True, G.EPI_STORE_F32, splits=S, bn=64, split_stride=part.stride(0))
    res = []
    for z in range(S):
        k0, k1 = 64 * (49 * z // S), 64 * (49 * (z + 1) // S)
        res += R.compare("split%d %s" % (z, kind), kind, part[z], a[:, k0:k1].double() @ w[k0:k1].double())
    _check(res)


def test_gemm_mlp_bench_shape_sampled():
    """M=8192, N=K=4096 with bias+ReLU at bn=256 (the MLP bench layer), compared on 96 random rows x 96 random columns."""
    from distributedmnist_b200.ops import gemm as G
    from distributedmnist_b200.ops import refs as R
    g = torch.Generator().manual_seed(35)
    M, N, K = 8192, 4096, 4096
    for kind in ("grid", "rand"):
        a = _grid_or_rand(kind, (M, K), g, 0, 2, 1, 0.5)
        w = _grid_or_rand(kind, (K, N), g, -8, 8, 64, 0.02)
        bias = (R.grid(g, (N,), -16, 16, 64) if kind == "grid" else torch.randn(N, generator=g) * 0.1).cuda()
        out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        G.gemm_bf16_raw(a, w, out, M, N, K, K, N, N, False, True, G.EPI_BIAS_RELU_BF16, bn=256, bias=bias)
        rows, cols = torch.randperm(M, generator=g)[:96].cuda(), torch.randperm(N, generator=g)[:96].cuda()
        A, W = a[rows].double(), w[:, cols].double()
        ref = torch.clamp(A @ W + bias[cols].double(), min=0.0)
        ra = A.abs() @ W.abs()
        if kind == "grid":
            R.assert_exact_grid(ra + 1.0, 1.0 / 64, "mlp bench")
        _check(R.compare("mlp %s" % kind, kind, out[rows][:, cols], ref, R.fp32_slack(ra, K) + 2.0 ** -23 * ref.abs()))
