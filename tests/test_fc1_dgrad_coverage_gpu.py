"""fc1_dgrad_unpool writes every element of dy2 and nothing past the end of the batch.

The epilogue stages each 128-row tile's un-pooled gradient in shared memory and stores it a row per warp instruction,
so a row-to-address mistake shows up as an element left unwritten or a write into the rows after the batch.  dy2 starts
out as NaN at the head of a longer poisoned allocation; the numeric checks of test_kernel_refs_gpu.py run at the same
batches."""
import pytest
import torch

from test_kernel_refs_gpu import BATCHES

pytestmark = pytest.mark.gpu

GUARD_ROWS = 3                    # poisoned batch rows past the end of dy2


@pytest.mark.parametrize("B", BATCHES)
def test_fc1_dgrad_unpool_writes_every_output_and_nothing_past_it(B):
    from distributedmnist_b200.ops.lib import load, stream_ptr
    g = torch.Generator().manual_seed(2100 + B)
    dh = (torch.randn(B, 512, generator=g) * 0.1).to(torch.bfloat16).cuda()
    w1 = (torch.randn(3136, 512, generator=g) * 0.05).to(torch.bfloat16).cuda()
    code = (torch.randint(0, 4, (B, 3136), generator=g) | (torch.randint(0, 2, (B, 3136), generator=g) << 2)).to(torch.uint8).cuda()
    buf = torch.full((B + GUARD_ROWS, 14, 14, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    gb = torch.zeros(64, device="cuda")
    load().dm_fc1_dgrad_unpool(dh, w1, code, buf, gb, B, stream_ptr())
    torch.cuda.synchronize()
    assert not torch.isnan(buf[:B]).any(), "%d elements of dy2 left unwritten" % int(torch.isnan(buf[:B]).sum())
    assert torch.isnan(buf[B:]).all(), "%d elements written past the batch" % int((~torch.isnan(buf[B:])).sum())
    assert torch.isfinite(gb).all()
