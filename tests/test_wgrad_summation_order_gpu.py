"""pnx_wgrad sums every dW element in an order fixed by the shape alone: the rows of each K split in order, then the
splits in order.  A 64-channel X runs a different kernel variant (both consumer warpgroups over half of the columns each)
than a 128-channel X, but the two have the same split plan, so the 64-channel result equals the first 64 rows of the
128-channel one bit for bit."""
import pytest
import torch

from pillarnext_b200 import ops

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cy,taps,shuffle", [(64, 9, False), (128, 9, False), (256, 9, False), (384, 9, False), (64, 4, True),
                                             (64, 1, False), (128, 1, False)])
def test_wgrad_64_channel_x_matches_the_full_block(cy, taps, shuffle):
    torch.manual_seed(cy + taps)
    B, H, W = 2, 72, 72
    if shuffle:
        M, ry, geo = B * H * W, 4 * B * H * W, (H, W, 2 * H, 2 * W, 2, 2, 1, 0)
    else:
        M, ry, geo = B * H * W, B * H * W, (H, W, H, W, 3, 1, 1, 1) if taps == 9 else None
    X = torch.randn(M, 128, device="cuda").bfloat16()
    Y = torch.randn(ry, cy, device="cuda").bfloat16()
    assert ops.wgrad_splits(64, cy, taps, M, ops.sm_count()) == ops.wgrad_splits(128, cy, taps, M, ops.sm_count())
    full = torch.zeros(taps, 128, cy, device="cuda")
    ops.wgrad(X, 128, Y, cy, M, taps, full, dense=geo, shuffle=shuffle)
    x64 = X[:, :64].contiguous()
    part = torch.zeros(taps, 64, cy, device="cuda")
    ops.wgrad(x64, 64, Y, cy, M, taps, part, dense=geo, shuffle=shuffle)
    assert torch.equal(part, full[:, :64])
    ref = torch.zeros_like(full)
    ops.wgrad(X, 128, Y, cy, M, taps, ref, dense=geo, shuffle=shuffle)
    assert torch.equal(ref, full)
