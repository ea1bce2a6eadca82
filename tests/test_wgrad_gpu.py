"""wgmma weight-gradient GEMM (MN-major operands) and the row-wise BatchNorm kernels vs torch fp32
autograd on the same bf16-rounded operands.  Tolerance: 3e-3 of the result scale (fp32 accumulation
order + fp32 atomics); BN backward additionally carries bf16 rounding of dx (2^-8 relative)."""
import pytest
import torch
import torch.nn.functional as F

from pillarnext_b200 import ops

pytestmark = pytest.mark.gpu


def _close(out, ref, extra=0.0):
    scale = ref.abs().max().item() + 1e-6
    err = (out.float() - ref).abs().max().item()
    assert err <= (3e-3 + extra) * scale, "max abs err %g (scale %g)" % (err, scale)


def _split_cases(cases):
    """Each case as it was (same id, the device's SM count sizes the K splits) and again with a budget of one SM (id +
    "-1sm": one split, or two, of many rows each) and of 4096 SMs (id + "-4096sm": the most splits the rows allow)."""
    out = []
    for c in cases:
        cid = "-".join(str(v) for v in c)
        out += [pytest.param(*c, None, id=cid), pytest.param(*c, 1, id=cid + "-1sm"), pytest.param(*c, 4096, id=cid + "-4096sm")]
    return out


def _use_sms(monkeypatch, sms, cx, cy, taps, M):
    """Grid budget `sms` (None: the device's) for the wgrad launches that follow, and the split count it must give."""
    if sms is None:
        return
    monkeypatch.setattr(ops, "sm_count", lambda: sms)
    splits = ops.wgrad_splits(cx, cy, taps, M, ops.sm_count())
    if sms == 1:
        assert splits <= 2, "%d K splits with one SM" % splits
    else:
        assert splits * 1024 >= M, "%d K splits of %d rows: not the most the rows allow" % (splits, M)


@pytest.mark.parametrize("M,Min,Cx,Cy,sms", _split_cases([(5000, 4000, 64, 64), (20000, 20000, 256, 256), (3000, 3000, 128, 64),
                                                           (7777, 9000, 384, 64), (700, 900, 256, 128), (100, 100, 256, 1536),
                                                           (6000, 5000, 64, 384), (4100, 4100, 128, 192)]))
def test_wgrad_table(M, Min, Cx, Cy, sms, monkeypatch):
    """X = dOut (direct, M rows), Y = In (gathered through a random neighbour table with holes)."""
    torch.manual_seed(M + Cx)
    T = 9
    _use_sms(monkeypatch, sms, Cx, Cy, T, M)
    nbr = torch.randint(-Min // 3, Min, (M, T), device="cuda", dtype=torch.int32).clamp(min=-1)
    X = torch.randn(M, Cx, device="cuda").bfloat16()
    Y = torch.randn(Min, Cy, device="cuda").bfloat16()
    ref = torch.zeros(T, Cx, Cy, device="cuda")
    for t in range(T):
        idx = nbr[:, t].long()
        yg = torch.where((idx >= 0).unsqueeze(1), Y[idx.clamp(min=0)].float(), torch.zeros(1, device="cuda"))
        ref[t] = X.float().t() @ yg
    dW = torch.zeros(T, Cx, Cy, device="cuda")
    ops.wgrad(X, Cx, Y, Cy, M, T, dW, nbr=nbr)
    _close(dW, ref)
    # no gather, single tap (1x1 convolutions)
    Y1 = torch.randn(M, Cy, device="cuda").bfloat16()
    d1 = torch.zeros(1, Cx, Cy, device="cuda")
    ops.wgrad(X, Cx, Y1, Cy, M, 1, d1)
    _close(d1[0], X.float().t() @ Y1.float())


@pytest.mark.parametrize("B,H,W_,Cin,Cout,k,stride,dil,sms", _split_cases([(2, 24, 24, 64, 64, 3, 1, 1), (1, 40, 36, 256, 256, 3, 1, 6),
                                                                        (1, 21, 33, 128, 256, 3, 2, 1), (2, 16, 16, 256, 256, 1, 1, 1)]))
def test_wgrad_dense_conv(B, H, W_, Cin, Cout, k, stride, dil, sms, monkeypatch):
    Ho_, Wo_ = (H + 2 * dil * (k // 2) - dil * (k - 1) - 1) // stride + 1, (W_ + 2 * dil * (k // 2) - dil * (k - 1) - 1) // stride + 1
    _use_sms(monkeypatch, sms, Cout, Cin, k * k, B * Ho_ * Wo_)
    torch.manual_seed(H + Cin)
    x = torch.randn(B, Cin, H, W_, device="cuda").bfloat16()
    w = torch.zeros(Cout, Cin, k, k, device="cuda", requires_grad=True)
    pad = dil * (k // 2)
    y = F.conv2d(x.float(), w, stride=stride, padding=pad, dilation=dil)
    dy = torch.randn_like(y).bfloat16()
    y.backward(dy.float())
    Ho, Wo = y.shape[2], y.shape[3]
    M = B * Ho * Wo
    x_rows = x.permute(0, 2, 3, 1).contiguous().view(-1, Cin)
    dy_rows = dy.permute(0, 2, 3, 1).contiguous().view(-1, Cout)
    dW = torch.zeros(k * k, Cout, Cin, device="cuda")
    ops.wgrad(dy_rows, Cout, x_rows, Cin, M, k * k, dW, dense=(Ho, Wo, H, W_, k, stride, dil, pad) if k > 1 else None)
    got = dW.view(k, k, Cout, Cin).permute(2, 3, 0, 1)
    _close(got, w.grad)


@pytest.mark.parametrize("sms", [1, 4096])
def test_wgrad_conv_transpose_grid(sms, monkeypatch):
    _use_sms(monkeypatch, sms, 64, 64, 4, 2 * 12 * 20)
    test_wgrad_conv_transpose()


def test_wgrad_conv_transpose():
    torch.manual_seed(3)
    B, H, W_, C = 2, 12, 20, 64
    x = torch.randn(B, C, H, W_, device="cuda").bfloat16()
    w = torch.zeros(C, C, 2, 2, device="cuda", requires_grad=True)
    y = F.conv_transpose2d(x.float(), w, stride=2)
    dy = torch.randn_like(y).bfloat16()
    y.backward(dy.float())
    x_rows = x.permute(0, 2, 3, 1).contiguous().view(-1, C)
    dy_rows = dy.permute(0, 2, 3, 1).contiguous().view(-1, C)
    dW = torch.zeros(4, C, C, device="cuda")                      # [q, ci, co]
    ops.wgrad(x_rows, C, dy_rows, C, B * H * W_, 4, dW, dense=(H, W_, 2 * H, 2 * W_, 2, 2, 1, 0), shuffle=True)
    got = dW.view(2, 2, C, C).permute(2, 3, 0, 1)                 # [ci, co, dy, dx]
    _close(got, w.grad)


@pytest.mark.parametrize("M,C,relu,with_res", [(5000, 64, True, False), (3001, 256, True, True), (777, 128, False, True), (4000, 384, True, False)])
def test_bn_rows(M, C, relu, with_res):
    torch.manual_seed(M)
    x = (torch.randn(M, C, device="cuda") * 2 + 0.5).bfloat16()
    res = torch.randn(M, C, device="cuda").bfloat16() if with_res else None
    gamma = (torch.rand(C, device="cuda") + 0.5).requires_grad_()
    beta = (torch.randn(C, device="cuda") * 0.1).requires_grad_()
    xf = x.float().requires_grad_()
    rf = res.float().requires_grad_() if with_res else None
    mean = xf.mean(0)
    var = xf.var(0, unbiased=False)
    yref = (xf - mean) / torch.sqrt(var + 1e-3) * gamma + beta
    if with_res:
        yref = yref + rf
    if relu:
        yref = F.relu(yref)
    # forward through the kernels: stats (fp64) -> finalize -> apply
    stats = torch.cat([x.double().sum(0), (x.double() ** 2).sum(0)])
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    sc, sh, mu, istd = ops.bn_finalize(stats, C, None, M, gamma.detach(), beta.detach(), 1e-3, 0.01, rm, rv)
    y = torch.empty(M, C, dtype=torch.bfloat16, device="cuda")
    ops.bn_apply(x, M, C, sc, sh, y, res=res, relu=relu)
    _close(y, yref.detach(), extra=8e-3)
    assert torch.allclose(rm, 0.01 * mean.detach(), atol=1e-5)
    assert torch.allclose(rv, 0.99 + 0.01 * xf.detach().var(0, unbiased=True), atol=1e-4)
    # backward; use the kernel's own y for the relu mask so both sides see the same mask
    dy = torch.randn(M, C, device="cuda").bfloat16()
    mask = (y.float() > 0) if relu else torch.ones_like(yref, dtype=torch.bool)
    pre = (xf - mean) / torch.sqrt(var + 1e-3) * gamma + beta
    pre.backward(torch.where(mask, dy.float(), torch.zeros(1, device="cuda")))
    dx = torch.empty(M, C, dtype=torch.bfloat16, device="cuda")
    dres = torch.empty(M, C, dtype=torch.bfloat16, device="cuda") if with_res else None
    red = ops.bn_bwd(dy, y, x, M, C, mu, istd, gamma.detach(), M, relu, dx, dres=dres)
    _close(dx, xf.grad, extra=8e-3)
    _close(red[:C].float(), beta.grad)
    _close(red[C:].float(), gamma.grad)
    if with_res:
        assert torch.equal(dres.float(), torch.where(mask, dy.float(), torch.zeros(1, device="cuda")))
    else:
        # mask recomputed from x (y not read): identical result
        dx2 = torch.empty_like(dx)
        red2 = ops.bn_bwd(dy, None, x, M, C, mu, istd, gamma.detach(), M, relu, dx2, affine=(sc, sh))
        assert torch.equal(dx2, dx) and torch.allclose(red2, red)


def test_add_relu_roundtrip():
    a = torch.randn(1000, 256, device="cuda").bfloat16()
    b = torch.randn(1000, 256, device="cuda").bfloat16()
    y = torch.empty_like(a)
    ops.add_relu(a, b, 1000, 256, y)
    assert torch.equal(y, F.relu(a.float() + b.float()).bfloat16())
    dy = torch.randn(1000, 256, device="cuda").bfloat16()
    g = torch.empty_like(a)
    ops.relu_bwd(dy, y, 1000, 256, g)
    assert torch.equal(g.float(), torch.where(y.float() > 0, dy.float(), torch.zeros(1, device="cuda")))
    ops.add_rows(g, b, 1000, 256)


def test_wgrad_deterministic_partials_are_bitwise_reproducible():
    """pnx_wgrad with a `partials` buffer: per-split slabs + ordered reduction instead of fp32 red.global.add -- equal to
    the atomic path within accumulation-order noise, and bit-identical between two launches (the atomic path is not)."""
    from pillarnext_b200 import ops
    torch.manual_seed(5)
    B, H, W, cx, cy = 2, 96, 96, 128, 64
    M = B * H * W
    X = torch.randn(M, cx, device="cuda").bfloat16()
    Y = torch.randn(M, cy, device="cuda").bfloat16()
    geo = (H, W, H, W, 3, 1, 1, 1)

    def run():
        dW = torch.zeros(9, cx, cy, device="cuda")
        ops.wgrad(X, cx, Y, cy, M, 9, dW, dense=geo)
        return dW

    ref = run()
    prev = ops.set_deterministic(True)
    try:
        assert ops.wgrad_splits(cx, cy, 9, M, ops.sm_count()) > 1, "the case must exercise several K splits"
        a, b = run(), run()
        acc = torch.ones(9, cx, cy, device="cuda")          # accumulates into dW like the atomic path
        ops.wgrad(X, cx, Y, cy, M, 9, acc, dense=geo)
    finally:
        ops.set_deterministic(prev)
    assert torch.equal(a, b)
    assert ((a - ref).norm() / ref.norm()).item() < 1e-5
    assert ((acc - 1.0 - a).abs().max() / a.abs().max()).item() < 1e-5
