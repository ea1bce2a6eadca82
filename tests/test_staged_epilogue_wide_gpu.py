"""The store warpgroup of igemm at BN = 256 (bf16, with and without the fused BatchNorm-backward gate) and with fp32 output
(F = 2, BN <= 128): bias, ReLU, addends, statistics, row masking of a partial last tile, guard columns and rows past M.
Each case runs at the device's grid budget and at one SM, where one CTA per column block walks >= 3 tiles.  Results are
checked against an fp64 reference and, bit for bit, against another block width (BN = 128 for the bf16 cases, the
in-register BN = 256 epilogue for fp32): the per-element sums and the statistic slots do not depend on the block width."""
import types

import pytest
import torch
import torch.nn.functional as F

from pillarnext_b200 import ops

pytestmark = pytest.mark.gpu

SENTINEL = 7.0     # exact in bf16 and fp32
GUARD = 16         # guard columns on each side of the slot (keeps the slot 16-byte aligned)
SMS = [pytest.param(None, id="grid"), pytest.param(1, id="1sm")]


def _slot(M, N, dtype):
    buf = torch.full((M + 100, GUARD + N + GUARD), SENTINEL, dtype=dtype, device="cuda")
    return buf, buf[:M, GUARD:GUARD + N]


def _check_sentinel(buf, M, N):
    assert (buf[:, :GUARD] == SENTINEL).all(), "left guard columns overwritten"
    assert (buf[:, GUARD + N:] == SENTINEL).all(), "right guard columns overwritten"
    assert (buf[M:] == SENTINEL).all(), "rows past M overwritten"


def _use_sms(monkeypatch, sms, M, n_blocks):
    if sms is None:
        return
    monkeypatch.setattr(ops, "sm_count", lambda: sms)
    tiles = -(-M // 128)
    gx = max(1, min(sms // n_blocks, tiles))
    assert M % 128 and -(-tiles // gx) >= 3, "partial last tile and >= 3 tiles per CTA: %d rows on %d CTAs" % (M, gx)


def _close(out, ref, rel):
    scale = ref.abs().max().item() + 1e-6
    err = (out.double() - ref).abs().max().item()
    assert err <= rel * scale, "max abs err %g (scale %g)" % (err, scale)


def _stats_match(got, vals):
    v = vals.double()
    C = v.shape[1]
    for g, want, mag in ((got[:C], v.sum(0), v.abs().sum(0)), (got[C:], (v * v).sum(0), (v * v).sum(0))):
        tol = 1e-5 * mag.max().item() + 1e-6
        assert (g - want).abs().max().item() <= tol, "statistics differ by %g (tol %g)" % ((g - want).abs().max().item(), tol)


def _conv3x3(B, H, W_, Cin, Cout, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, Cin, H, W_, device="cuda", generator=g).bfloat16()
    w = (torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) * 0.05).bfloat16()
    ref = F.conv2d(x.double(), w.double(), padding=1).permute(0, 2, 3, 1).reshape(-1, Cout)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().view(-1, Cin)
    wp = w.permute(2, 3, 0, 1).contiguous().view(9, Cout, Cin)
    return x_nhwc, wp, ref, g


@pytest.mark.parametrize("sms", SMS)
def test_bn256_bias_relu_addend_stats(sms, monkeypatch):
    B, H, W_, Cin, Cout = 1, 13, 23, 128, 512     # 299 rows: 3 tiles, the last partial; 2 column blocks
    M = B * H * W_
    _use_sms(monkeypatch, sms, M, Cout // 256)
    x, wp, ref, g = _conv3x3(B, H, W_, Cin, Cout, 256)
    bias = torch.randn(Cout, device="cuda", generator=g) * 0.1
    addend = torch.randn(M, Cout + 8, device="cuda", generator=g).bfloat16()[:, 4:4 + Cout]
    want = torch.relu(ref + bias.double() + addend.double())
    outs = {}
    for bn in (256, 128):
        buf, out = _slot(M, Cout, torch.bfloat16)
        stats = torch.zeros(2 * Cout, dtype=torch.float64, device="cuda")
        ops.igemm(x, M, wp, 9, Cin, Cout, out, dense=(H, W_, H, W_, 3, 1, 1, 1), bias=bias, relu=True, stats=stats,
                  addend=addend, block_n=bn)
        _check_sentinel(buf, M, Cout)
        _close(out, want, 1e-2)
        _stats_match(stats, out)
        outs[bn] = (out.clone(), stats)
    assert torch.equal(outs[256][0], outs[128][0]), "BN = 256 and BN = 128 outputs differ"
    if sms == 1:   # one CTA per column block: each channel's statistics are one fp64 add of the same fp32 slot sums
        assert torch.equal(outs[256][1], outs[128][1]), "BN = 256 and BN = 128 statistics differ"


@pytest.mark.parametrize("sms", SMS)
def test_bn256_bnr_gate(sms, monkeypatch):
    M, Min, Cin, Cout = 1000, 900, 128, 512
    _use_sms(monkeypatch, sms, M, Cout // 256)
    g = torch.Generator(device="cuda").manual_seed(512)
    A = torch.randn(Min, Cin, device="cuda", generator=g).bfloat16()
    W = (torch.randn(9, Cout, Cin, device="cuda", generator=g) * 0.05).bfloat16()
    nbr = torch.randint(-Min // 3, Min, (M, 9), device="cuda", dtype=torch.int32, generator=g).clamp(min=-1)
    plain = torch.empty(M, Cout, dtype=torch.bfloat16, device="cuda")
    ops.igemm(A, M, W, 9, Cin, Cout, plain, nbr=nbr, block_n=256)
    Ad = torch.cat([A.double(), torch.zeros(1, Cin, dtype=torch.float64, device="cuda")])
    rows = torch.where(nbr < 0, torch.full_like(nbr, Min), nbr).long()
    ref = torch.einsum("mtc,tnc->mn", Ad[rows], W.double())
    _close(plain, ref, 1e-2)

    raw = torch.randn(M, Cout, device="cuda", generator=g).bfloat16()
    scale = torch.rand(Cout, device="cuda", generator=g) + 0.5
    shift = torch.randn(Cout, device="cuda", generator=g) * 0.5
    mean = torch.randn(Cout, device="cuda", generator=g) * 0.1
    invstd = torch.rand(Cout, device="cuda", generator=g) + 0.5
    outs = {}
    for bn in (256, 128):
        bnr = types.SimpleNamespace(raw=raw, scale=scale, shift=shift, mean=mean, invstd=invstd, C=Cout,
                                    red=torch.zeros(2 * Cout, dtype=torch.float64, device="cuda"))
        buf, out = _slot(M, Cout, torch.bfloat16)
        ops.igemm(A, M, W, 9, Cin, Cout, out, nbr=nbr, block_n=bn, bnr=bnr)
        _check_sentinel(buf, M, Cout)
        gate = raw.double() * scale.double() + shift.double() > 0
        gated = torch.where(gate, plain, torch.zeros_like(plain))
        assert torch.equal(out, gated), "gated output differs"
        gd = gated.double()
        xhat = (raw.double() - mean.double()) * invstd.double()
        for got, exp, mag in ((bnr.red[:Cout], gd.sum(0), gd.abs().sum(0)),
                              (bnr.red[Cout:], (gd * xhat).sum(0), (gd * xhat).abs().sum(0))):
            tol = 1e-5 * mag.max().item() + 1e-6
            assert (got - exp).abs().max().item() <= tol, "bnr sums differ by %g" % (got - exp).abs().max().item()
        outs[bn] = bnr.red
    if sms == 1:
        assert torch.equal(outs[256], outs[128]), "BN = 256 and BN = 128 reduce sums differ"


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("with_addend", [False, True], ids=["plain", "addend_f32"])
def test_fp32_output(with_addend, sms, monkeypatch):
    B, H, W_, Cin, Cout = 2, 11, 19, 128, 256     # 418 rows: 4 tiles, the last partial; 2 column blocks at BN = 128
    M = B * H * W_
    _use_sms(monkeypatch, sms, M, Cout // 128)
    x, wp, ref, g = _conv3x3(B, H, W_, Cin, Cout, 128 + with_addend)
    bias = torch.randn(Cout, device="cuda", generator=g) * 0.1
    addend = torch.randn(M, Cout + 8, device="cuda", generator=g)[:, 4:4 + Cout] if with_addend else None
    want = ref + bias.double() + (addend.double() if with_addend else 0)
    outs = {}
    for bn in (128, 256):     # staged fp32 drain; in-register fp32 epilogue
        buf, out = _slot(M, Cout, torch.float32)
        stats = torch.zeros(2 * Cout, dtype=torch.float64, device="cuda")
        ops.igemm(x, M, wp, 9, Cin, Cout, out, dense=(H, W_, H, W_, 3, 1, 1, 1), bias=bias, stats=stats, addend=addend,
                  block_n=bn)
        _check_sentinel(buf, M, Cout)
        _close(out, want, 1e-4)
        _stats_match(stats, out)
        outs[bn] = out.clone()
    assert torch.equal(outs[128], outs[256]), "staged and in-register fp32 outputs differ"
