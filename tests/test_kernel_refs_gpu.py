"""Every kernel of the default LeNet step vs its float64 reference (ops/refs.py) at the engine's batch sizes, on exact-grid
data (bitwise) and continuous data (precision bounds), plus the split structures, stale workspaces and pooling edge
cases where a reduction or an epilogue would go subtly wrong."""
import pytest

pytestmark = pytest.mark.gpu

# 1, an M-tile boundary (128 / 129), the bench batch 256, the evaluator's 1000 and the largest configured batch 1024
BATCHES = [1, 37, 128, 129, 256, 1000, 1024]


def _run(fn, **kw):
    from distributedmnist_b200.ops import selfcheck
    results = getattr(selfcheck, fn)(**kw)
    bad = [(n, e, t) for (n, e, t) in results if not e <= t]
    assert not bad, "failed: %s\nall: %s" % (bad, results)


def _stale(B):
    """a batch of a different size, run first so the workspace holds stale partial sums"""
    return 1024 if B < 1024 else 256


@pytest.mark.parametrize("B", BATCHES)
def test_conv1_fwd_tc(B):
    _run("check_conv1_fwd_tc", B=B, seed=100 + B)


@pytest.mark.parametrize("B", BATCHES)
def test_conv1_wgrad_tc(B):
    _run("check_conv1_wgrad", B=B, seed=200 + B, stale_B=_stale(B))


@pytest.mark.parametrize("B", BATCHES)
def test_conv2_fwd(B):
    _run("check_conv2_fwd", B=B, seed=300 + B)


@pytest.mark.parametrize("B", BATCHES)
def test_conv2_dgrad(B):
    _run("check_conv2_dgrad", B=B, seed=400 + B)


@pytest.mark.parametrize("B", BATCHES)
def test_conv2_wgrad(B):
    _run("check_conv2_wgrad", B=B, seed=500 + B, stale_B=_stale(B))


@pytest.mark.parametrize("B", BATCHES)
def test_fc1_fwd_split_k_then_fc2_fwd_bwd(B):
    _run("check_fc1_fwd", B=B, seed=600 + B)


def test_fc1_fwd_inference_path():
    _run("check_fc1_fwd", B=1000, seed=650, train=False)


@pytest.mark.parametrize("B", [1, 256, 1024])
def test_fc2_fwd_bwd_after_stale_launch(B):
    _run("check_fc2_loss", B=B, seed=660 + B, stale_B=_stale(B))


@pytest.mark.parametrize("keep_prob,probe", [(0.25, -1), (0.25, 0), (0.25, 1), (0.8, -1), (0.8, 0), (0.8, 1), (1.0, -1)])
def test_fc2_dropout_threshold_edges(keep_prob, probe):
    """One element hashed exactly to threshold - 1 / threshold / threshold + 1 (at keep 1.0 the threshold is 2^24, one
    past every hash value).  0.8: fp32 rounds it up, so the kernel's threshold is one above floor(0.8 * 2^24)."""
    _run("check_fc2_loss", B=64, seed=670, keep_prob=keep_prob, probe=probe)


@pytest.mark.parametrize("B", BATCHES)
def test_fc2_wgrad(B):
    _run("check_fc2_wgrad", B=B, seed=700 + B)


@pytest.mark.parametrize("B", BATCHES)
def test_fc1_wgrad_f32_and_bf16(B):
    _run("check_fc1_wgrad", B=B, seed=800 + B)


@pytest.mark.parametrize("B", BATCHES)
def test_fc1_dgrad_unpool(B):
    _run("check_fc1_dgrad_unpool", B=B, seed=900 + B, stale_B=_stale(B))


@pytest.mark.parametrize("ctas,B", [(8, 256), (27, 257)])
def test_weight_gradient_split_structure(ctas, B):
    """8 CTAs: conv2_wgrad runs ONE split walking all 2B tiles (the 4-stage ring wraps 128 times); 27: three conv2 splits
    of uneven length and 27 uneven conv1 slices."""
    from distributedmnist_b200.ops.lib import load
    lib = load()
    if lib.dm_num_sms() < ctas:
        pytest.skip("device has fewer than %d SMs" % ctas)
    prev = lib.dm_get_max_ctas()
    try:
        assert lib.dm_set_max_ctas(ctas) == ctas
        _run("check_conv2_wgrad", B=B, seed=1000 + ctas, stale_B=64)
        _run("check_conv1_wgrad", B=B, seed=1100 + ctas, stale_B=64)
    finally:
        lib.dm_set_max_ctas(prev)              # whatever was in force before (0: the default)


@pytest.mark.parametrize("B", [2, 129])
def test_pool_ties_exact_zeros_and_negative_windows(B):
    _run("check_conv1_fwd_tc", B=B, seed=1200 + B, kinds=("edges",))
    _run("check_conv2_fwd", B=B, seed=1300 + B, kinds=("edges",))


def test_end_to_end_gradients_on_mnist_like_images():
    _run("check_end_to_end", B=256, seed=1400, images="mnist")


def test_evaluate_matches_float64_forward():
    _run("check_evaluate")
