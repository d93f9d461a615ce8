"""The MLP step kernels (csrc/mlp_simt.cu and the input conversion) vs their float64 references (ops/refs.py) at the
shapes the MLP configurations run -- up to the 3-layer MLP at batch 8192, width 4096 -- on exact-grid data (bitwise
where the inputs allow) and continuous data (derived fp32 bounds), plus the whole CudaMlpEngine step checked stage by
stage and its inference path."""
import pytest

pytestmark = pytest.mark.gpu


def _run(fn, **kw):
    from distributedmnist_b200.ops import selfcheck
    results = getattr(selfcheck, fn)(**kw)
    bad = [(n, e, t) for (n, e, t) in results if not e <= t]
    assert not bad, "failed: %s\nall: %s" % (bad, results)


def _num_sms():
    from distributedmnist_b200.ops.lib import load
    return int(load().dm_num_sms())


# 64 .. 5120: the widest output layer whose [H][11] fp32 weights fit in shared memory (225 280 bytes)
DENSE_H = [64, 192, 1024, 4096, 5120]


@pytest.mark.parametrize("train", [0, 1])
@pytest.mark.parametrize("H", DENSE_H)
def test_dense10_xent(H, train):
    """B = 1, 7 / 8 / 9 around one CTA's eight warps, 1000, one full grid-stride pass (8 rows per CTA, one CTA per SM),
    one row past it (a warp carries its bias-gradient partial into a second row), and the 8192 of the configuration."""
    sms = _num_sms()
    for B in [1, 7, 8, 9, 1000, 8 * sms, 8 * sms + 1, 8192]:
        _run("check_dense10_xent", B=B, H=H, train=bool(train), seed=1000 * train + H + B)


@pytest.mark.parametrize("H", [2, 62, 64, 66, 4096])
@pytest.mark.parametrize("B", [1, 255, 256, 257, 8192, 16385, 40000])
def test_relu_bwd_colsum(B, H):
    """In place, out of place and unmasked.  256 rows per slab up to 64 slabs: 8192 rows = 32 slabs; 16 385 and 40 000
    hit the cap (slabs of 257 and 625 rows, the last one short at 16 385)."""
    _run("check_relu_bwd_colsum", B=B, H=H, seed=B + H)


def test_relu_bwd_colsum_raises_on_odd_width():
    import torch
    from distributedmnist_b200.ops.lib import KernelLibraryError, load, stream_ptr
    dh = torch.zeros(4, 4, dtype=torch.bfloat16, device="cuda")
    g = torch.zeros(4, device="cuda")
    with pytest.raises(KernelLibraryError, match=r"code -1\b"):
        load().dm_relu_bwd_colsum(dh, None, None, g, 4, 3, stream_ptr())


@pytest.mark.parametrize("B", [1, 3, 1001, 8191])
def test_f32_to_bf16_round_to_nearest_even(B):
    _run("check_f32_to_bf16", B=B, seed=B)


# (model, B, H): the configuration, the flag defaults (batch 128, width 1024), the evaluator's batch, partial tiles with
# 128-wide GEMM tiles (192 is not a multiple of 256), and a single row
STEP_SHAPES = [("mlp3", 8192, 4096), ("mlp2", 128, 1024), ("mlp3", 128, 1024), ("mlp3", 1000, 1024), ("mlp3", 96, 192),
               ("mlp2", 1, 64)]


@pytest.mark.parametrize("model,B,H", STEP_SHAPES)
def test_mlp_step_stage_by_stage(model, B, H):
    _run("check_mlp_step", model=model, B=B, hidden=H, seed=B + H)


def test_mlp_evaluate_matches_float64_forward():
    _run("check_mlp_evaluate")


def test_mlp_hidden_width_limit():
    """5120 is the widest output layer dense10_xent takes; the next multiple of 64 is refused when the engine is built,
    not at its first launch."""
    import torch
    from distributedmnist_b200.ops import selfcheck
    eng = selfcheck._mlp_engine("mlp2", 8, 5120, 1)
    assert eng.hidden == 5120
    del eng
    torch.cuda.empty_cache()
    with pytest.raises(ValueError, match="--mlp_hidden"):
        selfcheck._mlp_engine("mlp2", 8, 5184, 1)
