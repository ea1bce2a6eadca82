"""wgmma gather implicit-GEMM vs a plain torch fp32 reference on the SAME bf16-rounded operands
(fp32 accumulate): tolerance 2e-3 relative to the output scale (accumulation order only) plus the
final bf16 rounding (2^-8 relative) when the output is bf16."""
import pytest
import torch
import torch.nn.functional as F

from pillarnext_b200 import ops

pytestmark = pytest.mark.gpu


def _grid_cases(cases, skip=()):
    """Each case as it was (same id, the device's SM count as grid budget) and again with a budget of one SM (id + "-1sm"):
    one CTA per column block then walks every tile, carrying its smem ring and epilogue handoff from tile to tile.  Cases
    with fewer than 3 tiles (`skip`) gain nothing from it."""
    out = []
    for c in cases:
        cid = "-".join(str(v) for v in c)
        out.append(pytest.param(*c, None, id=cid))
        if c not in skip:
            out.append(pytest.param(*c, 1, id=cid + "-1sm"))
    return out


def _use_sms(monkeypatch, sms, tiles, n_blocks):
    """Grid budget `sms` (None: the device's) for the launches that follow; with one SM, assert that a CTA gets >= 3 tiles."""
    if sms is None:
        return
    monkeypatch.setattr(ops, "sm_count", lambda: sms)
    gx = max(1, min(sms // n_blocks, tiles))
    assert -(-tiles // gx) >= 3, "tiles per CTA: %d tiles on %d CTAs" % (tiles, gx)


def _close(out, ref, bf16_out):
    scale = ref.abs().max().item() + 1e-6
    tol = (2e-3 + (8e-3 if bf16_out else 0)) * scale
    err = (out.float() - ref).abs().max().item()
    assert err <= tol, "max abs err %g > tol %g (scale %g)" % (err, tol, scale)


@pytest.mark.parametrize("M,K,N,bn,sms", _grid_cases([(128, 64, 64, 64), (1000, 128, 256, 256), (333, 256, 128, 128),
                                                      (5000, 64, 384, 192), (257, 64, 16, 16), (4096, 256, 32, 32),
                                                      (20000, 256, 256, 256)], skip=[(128, 64, 64, 64)]))
def test_plain_gemm(M, K, N, bn, sms, monkeypatch):
    _use_sms(monkeypatch, sms, -(-M // 128), N // bn)
    torch.manual_seed(M + K + N)
    A = torch.randn(M, K, device="cuda").bfloat16()
    W = (torch.randn(1, N, K, device="cuda") * 0.1).bfloat16()
    bias = torch.randn(N, device="cuda")
    ref = A.float() @ W[0].float().t()
    out = torch.empty(M, N, dtype=torch.float32, device="cuda")
    ops.igemm(A, M, W, 1, K, N, out, block_n=bn)
    _close(out, ref, False)
    out2 = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    stats = torch.zeros(2 * N, dtype=torch.float64, device="cuda")
    ops.igemm(A, M, W, 1, K, N, out2, bias=bias, relu=True, stats=stats, block_n=bn)
    ref2 = F.relu(ref + bias)
    _close(out2, ref2, True)
    s = out2.double()
    assert torch.allclose(stats[:N], s.sum(0), rtol=1e-6, atol=1e-3)
    assert torch.allclose(stats[N:], (s * s).sum(0), rtol=1e-6, atol=1e-3)


@pytest.mark.parametrize("M,Min,C,N,sms", _grid_cases([(3000, 2500, 64, 64), (1500, 4000, 128, 256), (700, 700, 256, 256)]))
def test_table_gather(M, Min, C, N, sms, monkeypatch):
    _use_sms(monkeypatch, sms, -(-M // 128), N // ops.pick_block_n(N))
    torch.manual_seed(M)
    A = torch.randn(Min, C, device="cuda").bfloat16()
    W = (torch.randn(9, N, C, device="cuda") * 0.05).bfloat16()
    nbr = torch.randint(-Min // 2, Min, (M, 9), device="cuda", dtype=torch.int32).clamp(min=-1)
    ref = torch.zeros(M, N, device="cuda")
    for t in range(9):
        idx = nbr[:, t].long()
        rows = torch.where((idx >= 0).unsqueeze(1), A[idx.clamp(min=0)].float(), torch.zeros(1, device="cuda"))
        ref += rows @ W[t].float().t()
    out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    ops.igemm(A, M, W, 9, C, N, out, nbr=nbr)
    _close(out, ref, True)


@pytest.mark.parametrize("B,H,W_,Cin,Cout,k,stride,dil,sms", _grid_cases(
    [(2, 24, 24, 64, 64, 3, 1, 1), (1, 40, 36, 256, 256, 3, 1, 6), (1, 21, 33, 128, 256, 3, 2, 1), (2, 16, 16, 256, 256, 1, 1, 1),
     (1, 48, 48, 64, 384, 3, 1, 1), (1, 50, 50, 256, 64, 3, 1, 18)], skip=[(1, 21, 33, 128, 256, 3, 2, 1)]))
def test_dense_conv(B, H, W_, Cin, Cout, k, stride, dil, sms, monkeypatch):
    Ho_, Wo_ = (H + 2 * dil * (k // 2) - dil * (k - 1) - 1) // stride + 1, (W_ + 2 * dil * (k // 2) - dil * (k - 1) - 1) // stride + 1
    _use_sms(monkeypatch, sms, -(-B * Ho_ * Wo_ // 128), Cout // ops.pick_block_n(Cout))
    torch.manual_seed(H * W_ + Cin)
    x = torch.randn(B, Cin, H, W_, device="cuda").bfloat16()
    w = (torch.randn(Cout, Cin, k, k, device="cuda") * 0.05).bfloat16()
    pad = dil * (k // 2)
    ref = F.conv2d(x.float(), w.float(), stride=stride, padding=pad, dilation=dil)
    Ho, Wo = ref.shape[2], ref.shape[3]
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().view(-1, Cin)
    wp = w.permute(2, 3, 0, 1).contiguous().view(k * k, Cout, Cin)
    out = torch.empty(B * Ho * Wo, Cout, dtype=torch.bfloat16, device="cuda")
    ops.igemm(x_nhwc, B * Ho * Wo, wp, k * k, Cin, Cout, out, dense=(Ho, Wo, H, W_, k, stride, dil, pad))
    _close(out.view(B, Ho, Wo, Cout).permute(0, 3, 1, 2), ref, True)


def test_conv_transpose_shuffle():
    _conv_transpose_shuffle()


def test_conv_transpose_shuffle_1sm(monkeypatch):
    _conv_transpose_shuffle(monkeypatch)


def _conv_transpose_shuffle(monkeypatch=None):
    torch.manual_seed(5)
    B, H, W_, C = 2, 12, 20, 64
    if monkeypatch is not None:
        _use_sms(monkeypatch, 1, -(-B * H * W_ // 128), 4 * C // ops.pick_block_n(4 * C))
    x = torch.randn(B, C, H, W_, device="cuda").bfloat16()
    w = (torch.randn(C, C, 2, 2, device="cuda") * 0.1).bfloat16()           # [Cin, Cout, kh, kw]
    ref = F.conv_transpose2d(x.float(), w.float(), stride=2)
    wp = w.permute(2, 3, 1, 0).contiguous().view(1, 4 * C, C)               # n = (dy*2+dx)*64 + co
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().view(-1, C)
    out = torch.empty(B * 2 * H * 2 * W_, C, dtype=torch.bfloat16, device="cuda")
    stats = torch.zeros(2 * C, dtype=torch.float64, device="cuda")
    ops.igemm(x_nhwc, B * H * W_, wp, 1, C, 4 * C, out, ldc=C, dense=(H, W_, H, W_, 1, 1, 1, 0), shuffle=True, stats=stats, stats_mod=C)
    got = out.view(B, 2 * H, 2 * W_, C).permute(0, 3, 1, 2)
    _close(got, ref, True)
    s = out.double()
    assert torch.allclose(stats[:C], s.sum(0), rtol=1e-6, atol=1e-3)
