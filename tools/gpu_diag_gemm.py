"""GPU diagnostic: run every GEMM layout combination and print error structure (rows / columns with large errors point
at a wrong shared-memory descriptor or swizzle).  Also writes results/gemm_diag.txt."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from distributedmnist_b200.ops.gemm import gemm_bf16  # noqa: E402


def main():
    os.makedirs("results", exist_ok=True)
    lines = []
    torch.manual_seed(0)
    for a_major in ("k", "mn"):
        for b_major in ("k", "mn"):
            for bn in (64, 128, 256):
                for (M, N, K) in [(128, 128, 64), (128, 128, 256), (256, 256, 128), (200, 72, 784)]:
                    a = (torch.randn((K, M) if a_major == "mn" else (M, K), device="cuda") * 0.5).to(torch.bfloat16)
                    b = (torch.randn((K, N) if b_major == "mn" else (N, K), device="cuda") * 0.5).to(torch.bfloat16)
                    try:
                        out = gemm_bf16(a, b, a_major, b_major, bn=bn)
                        torch.cuda.synchronize()
                    except Exception as e:  # noqa: BLE001
                        lines.append("A=%s B=%s bn=%d %s EXC %r" % (a_major, b_major, bn, (M, N, K), e))
                        continue
                    A = a.float().t() if a_major == "mn" else a.float()
                    Bm = b.float() if b_major == "mn" else b.float().t()
                    ref = A @ Bm
                    err = (out - ref).abs()
                    bad = err > 0.05 * (K ** 0.5)
                    rows_bad = bad.any(1).nonzero().flatten().tolist()
                    cols_bad = bad.any(0).nonzero().flatten().tolist()
                    lines.append("A=%s B=%s bn=%d %s maxerr=%.4g bad=%d rows_bad[:8]=%s cols_bad[:8]=%s nan=%d" % (
                        a_major, b_major, bn, (M, N, K), err.max().item(), int(bad.sum()), rows_bad[:8], cols_bad[:8],
                        int(torch.isnan(out).sum())))
    txt = "\n".join(lines)
    print(txt)
    open("results/gemm_diag.txt", "w").write(txt + "\n")


if __name__ == "__main__":
    main()
