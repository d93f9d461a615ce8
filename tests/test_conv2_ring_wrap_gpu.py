"""conv2 forward and data-gradient kernels over many tiles per CTA.

B = 600 is 1200 pixel tiles, at least 9 per persistent CTA on a 132-SM H100: the 4-stage (forward) and 3-stage
(data-gradient) TMA patch rings wrap several times, and every CTA runs its pipelined tap loop back to back over
tiles.  A phase or buffer-index mistake there shows up only past the first wrap, which the smaller batches of
test_lenet_kernels_gpu.py never reach."""
import pytest

pytestmark = pytest.mark.gpu


def _run(fn, **kw):
    from distributedmnist_b200.ops import selfcheck
    results = getattr(selfcheck, fn)(**kw)
    bad = [(n, e, t) for (n, e, t) in results if not e <= t]
    assert not bad, "failed: %s\nall: %s" % (bad, results)


def test_conv2_fwd_many_tiles_per_cta():
    _run("check_conv2_fwd", B=600, seed=40)


def test_conv2_dgrad_many_tiles_per_cta():
    _run("check_conv2_dgrad", B=600, seed=41)
