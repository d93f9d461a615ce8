"""The conv2 forward and data-gradient kernels write every element of their outputs and nothing past the end.

Their tiles run over the batch's real pixels (32 pooled pixels / 128 pixels) and the last tile of most batches is
partial, so a tile-to-pixel mistake shows up as an element left unwritten or a write past the batch.  The outputs start
out as NaN (codes 0xFF) at the head of a longer poisoned allocation; the numeric checks run as in
test_kernel_refs_gpu.py, at the same batches."""
import pytest

from test_kernel_refs_gpu import BATCHES

pytestmark = pytest.mark.gpu

GUARD = 4096                      # poisoned elements past the end of each output


def _run(fn, **kw):
    from distributedmnist_b200.ops import selfcheck
    results = getattr(selfcheck, fn)(**kw)
    bad = [(n, e, t) for (n, e, t) in results if not e <= t]
    assert not bad, "failed: %s\nall: %s" % (bad, results)


@pytest.mark.parametrize("B", BATCHES)
def test_conv2_fwd_writes_every_output_and_nothing_past_it(B):
    _run("check_conv2_fwd", B=B, seed=1500 + B, guard=GUARD)


@pytest.mark.parametrize("B", BATCHES)
def test_conv2_dgrad_writes_every_output_and_nothing_past_it(B):
    _run("check_conv2_dgrad", B=B, seed=1600 + B, guard=GUARD)
