"""wgmma GEMM (csrc/gemm_tc.cu) -- Python entry points.

``gemm_bf16(a, b, a_major, b_major)`` multiplies without ever materialising a
transpose: ``a_major="k"`` means ``a`` is ``[M, K]`` row-major, ``"mn"`` means it is
stored ``[K, M]``; likewise ``b`` is ``[N, K]`` (``"k"``) or ``[K, N]`` (``"mn"``).
"""
from __future__ import annotations

from typing import Optional

import torch

from .lib import load, stream_ptr

EPI_STORE_F32, EPI_ATOMIC_F32, EPI_STORE_BF16, EPI_BIAS_RELU_BF16 = 0, 1, 2, 3


def gemm_bf16_raw(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor, M: int, N: int, K: int, lda: int, ldb: int,
                  ldo: int, a_mn: bool, b_mn: bool, epi: int, splits: int = 1, bn: int = 128,
                  split_stride: int = 0, bias: Optional[torch.Tensor] = None,
                  stream: Optional[torch.cuda.Stream] = None) -> None:
    load().dm_gemm_bf16(a, b, out, M, N, K, lda, ldb, ldo, int(a_mn), int(b_mn), epi, splits, bn, split_stride, bias,
                        stream_ptr(stream))


def gemm_bf16(a: torch.Tensor, b: torch.Tensor, a_major: str = "k", b_major: str = "mn",
              out: Optional[torch.Tensor] = None, out_dtype: torch.dtype = torch.float32, splits: int = 1,
              bn: int = 128) -> torch.Tensor:
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.is_cuda and b.is_cuda
    assert a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1
    a_mn, b_mn = a_major == "mn", b_major == "mn"
    M, K = (a.shape[1], a.shape[0]) if a_mn else (a.shape[0], a.shape[1])
    N, Kb = (b.shape[1], b.shape[0]) if b_mn else (b.shape[0], b.shape[1])
    assert K == Kb, (a.shape, b.shape, a_major, b_major)
    if out is None:
        out = (torch.zeros if splits > 1 else torch.empty)((M, N), dtype=out_dtype, device=a.device)
    if splits > 1:
        epi = EPI_ATOMIC_F32
        assert out.dtype == torch.float32
    else:
        epi = EPI_STORE_F32 if out.dtype == torch.float32 else EPI_STORE_BF16
    gemm_bf16_raw(a, b, out, M, N, K, a.stride(0), b.stride(0), out.stride(0), a_mn, b_mn, epi, splits, bn)
    return out
