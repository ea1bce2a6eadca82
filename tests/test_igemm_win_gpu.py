"""TMA-window 3x3 convolution (pnx_conv3x3_win: im2col folded into 4-D TMA loads, horizontally shifted wgmma
descriptors) vs torch fp32 conv2d on the same bf16 operands (tolerance: accumulation order + bf16 output rounding)."""
import pytest
import torch
import torch.nn.functional as F

from pillarnext_b200 import ops

pytestmark = pytest.mark.gpu


def run(B, H, W, Cin, Cout, bn, base_off, bias=True, relu=True):
    torch.manual_seed(H * W + Cin + Cout)
    x = torch.randn(B, Cin, H, W, device="cuda").bfloat16()
    w = (torch.randn(Cout, Cin, 3, 3, device="cuda") * 0.05).bfloat16()
    b = torch.randn(Cout, device="cuda") if bias else None
    ref = F.conv2d(x.float(), w.float(), b, padding=1)
    if relu:
        ref = F.relu(ref)
    rows = x.permute(0, 2, 3, 1).contiguous().view(-1, Cin)
    wp = w.permute(2, 3, 0, 1).contiguous().view(9, Cout, Cin)
    out = torch.full((B * H * W, Cout), float("nan"), dtype=torch.bfloat16, device="cuda")
    stats = torch.zeros(2 * Cout, dtype=torch.float64, device="cuda")
    ops.conv3x3_win(rows, B, H, W, wp, Cin, Cout, out, bias=b, stats=stats, relu=relu, block_n=bn, base_off=base_off)
    got = out.view(B, H, W, Cout).permute(0, 3, 1, 2).float()
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item()
    s = out.double()
    stats_ok = torch.allclose(stats[:Cout], s.sum(0), rtol=1e-5, atol=1e-2) and torch.allclose(stats[Cout:], (s * s).sum(0), rtol=1e-5, atol=1e-2)
    return err / scale, stats_ok


def test_descriptor_base_offset_convention():
    """Exactly one wgmma descriptor base-offset convention reproduces the shifted windows; it must be the library default."""
    e1, _ = run(1, 6, 200, 64, 64, 64, 1)
    e0, _ = run(1, 6, 200, 64, 64, 64, 0)
    print("rel err with base_offset=(start>>7)&7: %.3g ; with base_offset=0: %.3g" % (e1, e0))
    good = 1 if e1 < 1.2e-2 else (0 if e0 < 1.2e-2 else None)
    assert good is not None, (e1, e0)
    assert good == ops.WIN_BASE_OFF, "flip ops.WIN_BASE_OFF to %d" % good


@pytest.mark.parametrize("B,H,W,Cin,Cout,bn", [(2, 9, 336, 64, 384, 192), (1, 5, 130, 384, 64, 64), (2, 7, 128, 128, 128, 128),
                                               (1, 12, 40, 256, 64, 64), (1, 3, 257, 64, 192, 192),
                                               # Cin = 64 with block_n <= 128: weights-stationary variant
                                               (2, 9, 336, 64, 384, 128), (1, 3, 257, 64, 128, 64)])
def test_conv3x3_win(B, H, W, Cin, Cout, bn):
    err, stats_ok = run(B, H, W, Cin, Cout, bn, None)
    assert err < 1.2e-2, err
    assert stats_ok
