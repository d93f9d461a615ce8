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
