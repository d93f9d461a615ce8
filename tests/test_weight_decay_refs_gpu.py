"""The L2 weight-decay kernels (``--weight_decay``) against float64 references at the engine's batch sizes: the decayed
epilogues of the fc1 weight-gradient GEMM (fp32 arena and bf16 wire) and of fc2_wgrad, bit for bit on exact-grid data and
elementwise on continuous data; every CTA's W^2 partial and R; weight_decay_loss alone against an emulation of its
summation order; the evaluation pass with the decay armed; and one forward/backward against autograd of CE + lambda R."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# 1, an M-tile boundary (128 / 129), the bench batch 256, the evaluator's 1000 and the largest configured batch 1024
BATCHES = [1, 37, 128, 129, 256, 1000, 1024]


def _run(fn, **kw):
    from distributedmnist_b200.ops import selfcheck
    results = getattr(selfcheck, fn)(**kw)
    bad = [(n, e, t) for (n, e, t) in results if not e <= t]
    assert not bad, "failed: %s\nall: %s" % (bad, results)
    return results


@pytest.mark.parametrize("B", BATCHES)
def test_fc1_wgrad_decay(B):
    """K = B: the K-tail tiles at 1, 37 and 129; M = 3136 leaves the last row tile half empty."""
    _run("check_fc1_wgrad_decay", B=B, seed=1800 + B)


@pytest.mark.parametrize("B", BATCHES)
def test_fc2_wgrad_decay(B):
    """More than 256 rows (1000, 1024) take fc2_wgrad's multi-tile row loop; g_b2 and its square belong to CTA 0."""
    _run("check_fc2_wgrad_decay", B=B, seed=1900 + B)


@pytest.mark.parametrize("B", [1, 129, 1024])
def test_decay_workspace_second_launch_overwrites_the_first(B):
    _run("check_weight_decay_workspace", B=B, seed=2000 + B)


@pytest.mark.parametrize("n", [1, 31, 32, 33, 164])
def test_weight_decay_loss_matches_its_emulation(n):
    """164 = 100 fc1 CTAs + 64 fc2_wgrad CTAs, the engine's count."""
    _run("check_weight_decay_loss", n=n, seed=2100 + n)


def test_weight_decay_loss_refuses_bad_arguments():
    """n < 1 and null pointers are refused by the launcher before anything is launched."""
    from distributedmnist_b200.ops.lib import KernelLibraryError, load, stream_ptr
    lib = load()
    part = torch.full((4,), 3.0, dtype=torch.float64, device="cuda")
    la = torch.tensor([1.5, 0.5], device="cuda")
    for args in ((part, 0, 0.1, la), (part, -3, 0.1, la), (None, 3, 0.1, la), (part, 3, 0.1, None)):
        with pytest.raises(KernelLibraryError):
            lib.dm_weight_decay_loss(*args, stream_ptr())
    torch.cuda.synchronize()
    assert part.tolist() == [3.0] * 4 and la.tolist() == [1.5, 0.5]


def test_evaluation_pass_is_unchanged_by_the_decay():
    """The README and arm_weight_decay: the evaluation pass scores cross entropy, with or without the decay armed."""
    from distributedmnist_b200.ops import selfcheck as S
    eng, _ = S._engine(256, 2200)
    g = torch.Generator().manual_seed(2201)
    x = S.mnist_like(g, 3000)
    y = torch.randint(0, 10, (3000,), generator=g)
    eng.arm_eval(x, y)
    runs = []
    for lam in (0.0, 0.0123, 0.25):
        eng.arm_weight_decay(lam)
        rec = eng.run_eval()
        step, _t0, _t1, examples, correct, loss_sum = rec
        runs.append((step, examples, correct, np.float64(loss_sum).tobytes()))
    assert runs[0][1] == 3000 and runs[1:] == [runs[0]] * 2, runs


def test_end_to_end_decayed_gradients():
    """lambda = 0.25: the decay term is a larger share of each fc gradient than its FP32_GRAD_TOLS."""
    res = _run("check_end_to_end", B=256, seed=2300, lam=0.25)
    assert sum(1 for n, _, _ in res if n.startswith("e2e.decay_share_vs_tol.")) == 4
