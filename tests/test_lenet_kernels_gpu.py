"""sm_90a LeNet kernels vs float64 references (ops/refs.py) and the engine-level checks (SURVEY §4 item 2)."""
import pytest

pytestmark = pytest.mark.gpu


def _run(fn, **kw):
    from distributedmnist_b200.ops import selfcheck
    results = getattr(selfcheck, fn)(**kw)
    bad = [(n, e, t) for (n, e, t) in results if not e <= t]
    assert not bad, "failed: %s\nall: %s" % (bad, results)


def test_conv1_fwd_tcgen05_software_im2col():
    _run("check_conv1_fwd_tc")
    _run("check_conv1_fwd_tc", B=3, seed=9)        # one partial tile
    _run("check_conv1_fwd_tc", B=150, seed=19)     # 230 tiles > one CTA per SM: persistent loop over the two-stage operand ring


def test_conv1_wgrad_tcgen05():
    _run("check_conv1_wgrad")
    _run("check_conv1_wgrad", B=150, seed=20)


def test_conv2_fwd_tcgen05_implicit_gemm():
    _run("check_conv2_fwd")
    _run("check_conv2_fwd", B=75, seed=10)     # 150 tiles > one CTA per SM: persistent loop over the TMA stage ring


def test_conv2_dgrad_tcgen05():
    _run("check_conv2_dgrad")
    _run("check_conv2_dgrad", B=75, seed=11)


def test_conv2_wgrad_tcgen05_split_pixels():
    _run("check_conv2_wgrad")
    _run("check_conv2_wgrad", B=5, seed=12)    # fewer pixel tiles than CTAs


def test_fc2_softmax_xent_fwd_bwd():
    _run("check_fc2_loss")
    _run("check_fc2_loss", B=13, seed=13)


def test_fc1_dgrad_with_fused_unpool_epilogue():
    _run("check_fc1_dgrad_unpool")
    _run("check_fc1_dgrad_unpool", B=37, seed=15)   # partial M tile: rows beyond the batch contribute nothing


def test_end_to_end_gradients_match_autograd():
    _run("check_end_to_end")
    _run("check_end_to_end", B=256, seed=14)   # the benchmark batch size


def test_bucketed_bf16_wire_step_matches_single_kernel_step():
    _run("check_bucketed_step_matches_single_kernel")
    _run("check_bucketed_step_matches_single_kernel", B=256, steps=4, seed=32)


def test_bucketed_mlp_step_matches_single_kernel_step():
    _run("check_bucketed_mlp_step_matches_single_kernel")


def test_training_under_cuda_graph_reduces_loss():
    _run("check_training_reduces_loss")


def test_mlp_engines_match_autograd():
    _run("check_mlp_end_to_end")                       # 3-layer, batch 256
    _run("check_mlp2_end_to_end")                      # 2-layer, batch 96 (partial tiles everywhere)
