"""The store warps of the implicit-GEMM epilogue (igemm, igemm_win): row masking of the last partial tile, column slots
inside a wider output buffer, the pixel-shuffle store and the fused BatchNorm-backward gate.  Guard columns and the
rows past M hold a sentinel that must survive; the epilogue's statistics must equal fp64 sums over the stored bf16
values (fp32 summation tolerance)."""
import types

import pytest
import torch
import torch.nn.functional as F

from pillarnext_b200 import ops

pytestmark = pytest.mark.gpu

SENTINEL = 7.0     # exact in bf16
GUARD = 16         # guard columns on each side of the slot (keeps the slot 16-byte aligned)


def _slot_buffer(M, N):
    """[M + 100, GUARD + N + GUARD] bf16 of SENTINEL; returns (buffer, the [M, N] slot view, ldc = row pitch)."""
    buf = torch.full((M + 100, GUARD + N + GUARD), SENTINEL, dtype=torch.bfloat16, device="cuda")
    return buf, buf[:M, GUARD:GUARD + N]


def _grid_cases(cases):
    """Each case as it was (same id, the device's SM count as grid budget) and again with a budget of one SM (id + "-1sm"):
    one CTA per column block then walks every tile, so the store warpgroup's staged / sfree handoff, its pass parity and the
    per-CTA statistics carry over from tile to tile."""
    out = []
    for c in (cases if isinstance(cases[0], tuple) else [(c,) for c in cases]):
        cid = "-".join(str(v) for v in c)
        out.append(pytest.param(*c, None, id=cid))
        out.append(pytest.param(*c, 1, id=cid + "-1sm"))
    return out


def _use_sms(monkeypatch, sms, tiles, n_blocks):
    """Grid budget `sms` (None: the device's) for the launches that follow; with one SM, assert that a CTA gets >= 3 tiles."""
    if sms is None:
        return
    monkeypatch.setattr(ops, "sm_count", lambda: sms)
    gx = max(1, min(sms // n_blocks, tiles))
    assert -(-tiles // gx) >= 3, "tiles per CTA: %d tiles on %d CTAs" % (tiles, gx)


def _check_sentinel(buf, M, N):
    assert (buf[:, :GUARD] == SENTINEL).all(), "left guard columns overwritten"
    assert (buf[:, GUARD + N:] == SENTINEL).all(), "right guard columns overwritten"
    assert (buf[M:] == SENTINEL).all(), "rows past M overwritten"


def _close(out, ref):
    scale = ref.abs().max().item() + 1e-6
    err = (out.float() - ref).abs().max().item()
    assert err <= 1e-2 * scale, "max abs err %g (scale %g)" % (err, scale)


def _stats_match(got, vals):
    """got: [2C] fp64 sums / sums of squares from the epilogue; vals: [rows, C] stored values."""
    v = vals.double()
    C = v.shape[1]
    for g, want, mag in ((got[:C], v.sum(0), v.abs().sum(0)), (got[C:], (v * v).sum(0), (v * v).sum(0))):
        tol = 1e-5 * mag.max().item() + 1e-6
        assert (g - want).abs().max().item() <= tol, "statistics differ by %g (tol %g)" % ((g - want).abs().max().item(), tol)


def _bnr(M, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    raw = torch.randn(M, C, device="cuda", generator=g).bfloat16()
    scale = torch.rand(C, device="cuda", generator=g) + 0.5
    shift = torch.randn(C, device="cuda", generator=g) * 0.5
    mean = torch.randn(C, device="cuda", generator=g) * 0.1
    invstd = torch.rand(C, device="cuda", generator=g) + 0.5
    red = torch.zeros(2 * C, dtype=torch.float64, device="cuda")
    return types.SimpleNamespace(raw=raw, scale=scale, shift=shift, mean=mean, invstd=invstd, C=C, red=red)


def _check_bnr(bnr, plain, gated):
    """gated = bf16(gate ? plain : 0), red = (sum g, sum g * xhat); the gate's sign is exact in fp64."""
    raw = bnr.raw.double()
    gate = raw * bnr.scale.double() + bnr.shift.double() > 0
    want = torch.where(gate, plain, torch.zeros_like(plain))
    assert torch.equal(gated, want), "gated output differs"
    g = want.double()
    xhat = (raw - bnr.mean.double()) * bnr.invstd.double()
    C = bnr.C
    for got, exp, mag in ((bnr.red[:C], g.sum(0), g.abs().sum(0)), (bnr.red[C:], (g * xhat).sum(0), (g * xhat).abs().sum(0))):
        tol = 1e-5 * mag.max().item() + 1e-6
        assert (got - exp).abs().max().item() <= tol, "bnr sums differ by %g (tol %g)" % ((got - exp).abs().max().item(), tol)


# ------------------------------------------------------------------------------------------------- igemm
# igemm stages its epilogue for BN <= 192; the BN = 256 sets run the in-register epilogue (a regression check of that path,
# not coverage of the store warps).
@pytest.mark.parametrize("B,H,W_,Cin,Cout,bn,sms", _grid_cases([(1, 9, 37, 64, 64, 64), (2, 7, 29, 128, 128, 128),
                                                                (1, 11, 31, 64, 384, 192), (1, 13, 23, 256, 256, 256),
                                                                (1, 5, 53, 64, 32, 32)]))
def test_igemm_slot_tail_stats(B, H, W_, Cin, Cout, bn, sms, monkeypatch):
    _use_sms(monkeypatch, sms, -(-B * H * W_ // 128), Cout // bn)
    torch.manual_seed(Cout + W_)
    x = torch.randn(B, Cin, H, W_, device="cuda").bfloat16()
    w = (torch.randn(Cout, Cin, 3, 3, device="cuda") * 0.05).bfloat16()
    bias = torch.randn(Cout, device="cuda") * 0.1
    ref = F.relu(F.conv2d(x.float(), w.float(), padding=1) + bias.view(1, -1, 1, 1)).permute(0, 2, 3, 1).reshape(-1, Cout)
    M = B * H * W_
    assert M % 128
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().view(-1, Cin)
    wp = w.permute(2, 3, 0, 1).contiguous().view(9, Cout, Cin)
    buf, out = _slot_buffer(M, Cout)
    stats = torch.zeros(2 * Cout, dtype=torch.float64, device="cuda")
    ops.igemm(x_nhwc, M, wp, 9, Cin, Cout, out, dense=(H, W_, H, W_, 3, 1, 1, 1), bias=bias, relu=True, stats=stats, block_n=bn)
    _check_sentinel(buf, M, Cout)
    _close(out, ref)
    _stats_match(stats, out)


@pytest.mark.parametrize("bn,sms", _grid_cases([16, 64, 128, 256]))   # store warps for 16 / 64 / 128; 256: in-register epilogue
def test_igemm_shuffle_stats(bn, sms, monkeypatch):
    torch.manual_seed(11)
    B, H, W_, C = 2, 9, 23, 64          # 414 input pixels: the last tile is partial
    _use_sms(monkeypatch, sms, -(-B * H * W_ // 128), 4 * C // bn)
    x = torch.randn(B, C, H, W_, device="cuda").bfloat16()
    w = (torch.randn(C, C, 2, 2, device="cuda") * 0.1).bfloat16()
    ref = F.conv_transpose2d(x.float(), w.float(), stride=2).permute(0, 2, 3, 1).reshape(-1, C)
    wp = w.permute(2, 3, 1, 0).contiguous().view(1, 4 * C, C)
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().view(-1, C)
    Mo = B * 2 * H * 2 * W_
    buf, out = _slot_buffer(Mo, C)
    stats = torch.zeros(2 * C, dtype=torch.float64, device="cuda")
    ops.igemm(x_nhwc, B * H * W_, wp, 1, C, 4 * C, out, dense=(H, W_, H, W_, 1, 1, 1, 0), shuffle=True, stats=stats, stats_mod=C,
              block_n=bn)
    _check_sentinel(buf, Mo, C)
    _close(out, ref)
    _stats_match(stats, out)


@pytest.mark.parametrize("Cout,bn,sms", _grid_cases([(64, 64), (128, 128), (192, 192), (256, 256)]))   # 256: in-register epilogue
def test_igemm_bnr_gate(Cout, bn, sms, monkeypatch):
    torch.manual_seed(Cout)
    M, Min, Cin = 1000, 900, 128
    _use_sms(monkeypatch, sms, -(-M // 128), Cout // bn)
    A = torch.randn(Min, Cin, device="cuda").bfloat16()
    W = (torch.randn(9, Cout, Cin, device="cuda") * 0.05).bfloat16()
    nbr = torch.randint(-Min // 3, Min, (M, 9), device="cuda", dtype=torch.int32).clamp(min=-1)
    plain = torch.empty(M, Cout, dtype=torch.bfloat16, device="cuda")
    ops.igemm(A, M, W, 9, Cin, Cout, plain, nbr=nbr, block_n=bn)
    bnr = _bnr(M, Cout, Cout)
    buf, out = _slot_buffer(M, Cout)
    ops.igemm(A, M, W, 9, Cin, Cout, out, nbr=nbr, block_n=bn, bnr=bnr)
    _check_sentinel(buf, M, Cout)
    _check_bnr(bnr, plain, out)


# ------------------------------------------------------------------------------------------------- igemm_win
@pytest.mark.parametrize("B,H,W_,Cin,Cout,bn,sms", _grid_cases([(1, 5, 200, 64, 64, 64), (2, 3, 150, 64, 128, 128),
                                                                (1, 4, 140, 128, 128, 128), (1, 3, 130, 128, 192, 192),
                                                                (1, 6, 90, 256, 64, 64)]))
def test_win_slot_tail_stats(B, H, W_, Cin, Cout, bn, sms, monkeypatch):
    _use_sms(monkeypatch, sms, B * H * -(-W_ // 128), Cout // bn)
    torch.manual_seed(Cout + W_ + Cin)
    x = torch.randn(B, Cin, H, W_, device="cuda").bfloat16()
    w = (torch.randn(Cout, Cin, 3, 3, device="cuda") * 0.05).bfloat16()
    bias = torch.randn(Cout, device="cuda") * 0.1
    ref = F.relu(F.conv2d(x.float(), w.float(), padding=1) + bias.view(1, -1, 1, 1)).permute(0, 2, 3, 1).reshape(-1, Cout)
    M = B * H * W_
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().view(-1, Cin)
    wp = w.permute(2, 3, 0, 1).contiguous().view(9, Cout, Cin)
    buf, out = _slot_buffer(M, Cout)
    stats = torch.zeros(2 * Cout, dtype=torch.float64, device="cuda")
    ops.conv3x3_win(x_nhwc, B, H, W_, wp, Cin, Cout, out, bias=bias, stats=stats, relu=True, block_n=bn)
    _check_sentinel(buf, M, Cout)
    _close(out, ref)
    _stats_match(stats, out)


@pytest.mark.parametrize("Cin,Cout,bn,sms", _grid_cases([(64, 128, 128), (128, 64, 64)]))
def test_win_bnr_gate(Cin, Cout, bn, sms, monkeypatch):
    torch.manual_seed(Cin + Cout)
    B, H, W_ = 1, 5, 170
    _use_sms(monkeypatch, sms, B * H * -(-W_ // 128), Cout // bn)
    M = B * H * W_
    x = torch.randn(M, Cin, device="cuda").bfloat16()
    wp = (torch.randn(9, Cout, Cin, device="cuda") * 0.05).bfloat16()
    plain = torch.empty(M, Cout, dtype=torch.bfloat16, device="cuda")
    ops.conv3x3_win(x, B, H, W_, wp, Cin, Cout, plain, block_n=bn)
    bnr = _bnr(M, Cout, Cin + Cout)
    buf, out = _slot_buffer(M, Cout)
    ops.conv3x3_win(x, B, H, W_, wp, Cin, Cout, out, block_n=bn, bnr=bnr)
    _check_sentinel(buf, M, Cout)
    _check_bnr(bnr, plain, out)
