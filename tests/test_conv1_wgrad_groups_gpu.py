"""The conv1 weight gradient adds its per-CTA partial sums in groups of ceil(sqrt(grid)) consecutive CTAs, then the
groups in order.  13 CTAs make groups of 4, 4, 4 and 1: a last group of a single CTA, which the grids of
test_kernel_refs_gpu.py do not produce."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("ctas,B", [(13, 256)])
def test_conv1_wgrad_last_group_of_one(ctas, B):
    from distributedmnist_b200.ops import selfcheck
    from distributedmnist_b200.ops.lib import load
    lib = load()
    if lib.dm_num_sms() < ctas:
        pytest.skip("device has fewer than %d SMs" % ctas)
    prev = lib.dm_get_max_ctas()
    try:
        assert lib.dm_set_max_ctas(ctas) == ctas
        results = selfcheck.check_conv1_wgrad(B=B, seed=1300 + ctas, stale_B=64)
        bad = [(n, e, t) for (n, e, t) in results if not e <= t]
        assert not bad, "failed: %s\nall: %s" % (bad, results)
    finally:
        lib.dm_set_max_ctas(prev)              # whatever was in force before (0: the default)
