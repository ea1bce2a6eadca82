"""Window producer of pnx_wgrad: dense 3x3 stride-1 dilation-1 'same' weight gradients read their Y operand (the layer
input) as one TMA window per image-row chunk and kernel row instead of one gathered copy per tap.  Checked against an
fp64 torch reference on the same bf16 inputs, bit for bit against the gather path on the same shape, and in the
deterministic and split (multi-segment) modes."""
import pytest
import torch
import torch.nn.functional as F

from pillarnext_b200 import ops

pytestmark = pytest.mark.gpu


def _ref(X, Y, B, H, W):
    """fp64 dW[r*3+s, x, y] = sum over pixels of X[p, x] * Y[p shifted by (r-1, s-1), y] (zero outside the image)."""
    cx, cy = X.shape[1], Y.shape[1]
    Xd = X.double().view(B * H * W, cx)
    Yp = F.pad(Y.double().view(B, H, W, cy), (0, 0, 1, 1, 1, 1))
    out = torch.empty(9, cx, cy, dtype=torch.float64, device=X.device)
    for r in range(3):
        for s in range(3):
            out[3 * r + s] = Xd.t() @ Yp[:, r:r + H, s:s + W].reshape(-1, cy)
    return out


def _close(got, ref, tol=2e-5):
    scale = ref.abs().max().item()
    err = (got.double() - ref).abs().max().item()
    assert err <= tol * scale, "max abs err %g (scale %g)" % (err, scale)


def _run(X, Y, B, H, W, cx=None, cy=None):
    cx, cy = cx or X.shape[1], cy or Y.shape[1]
    dW = torch.zeros(9, cx, cy, device="cuda")
    ops.wgrad(X, cx, Y, cy, B * H * W, 9, dW, dense=(H, W, H, W, 3, 1, 1, 1))
    return dW


def _split_cases(cases):
    """Each case as it was (same id, the device's SM count sizes the K splits) and again with a budget of one SM (id +
    "-1sm": one split, or two, of many rows each) and of 4096 SMs (id + "-4096sm": the most splits the rows allow)."""
    out = []
    for c in cases:
        cid = "-".join(str(v) for v in c)
        out += [pytest.param(*c, None, id=cid), pytest.param(*c, 1, id=cid + "-1sm"), pytest.param(*c, 4096, id=cid + "-4096sm")]
    return out


@pytest.mark.parametrize("B,H,W,cx,cy,sms", _split_cases([
    (1, 24, 336, 384, 64),     # the head's 64 -> 384 convolution at its 336-pixel width (chunk 112, no padding)
    (2, 20, 176, 128, 64),     # 176: not a multiple of the chunk (96)
    (1, 9, 101, 128, 128),     # odd width: not a multiple of 16, the gather path runs
    (3, 1, 208, 256, 64),      # H = 1: every window row above and below is padding
    (2, 12, 80, 128, 256),
    (2, 12, 80, 64, 64),       # 64-channel X: each consumer warpgroup takes two shifts of the window
    (1, 10, 144, 64, 192),
]))
def test_window_wgrad_matches_fp64(B, H, W, cx, cy, sms, monkeypatch):
    if sms is not None:
        monkeypatch.setattr(ops, "sm_count", lambda: sms)
        splits, M = ops.wgrad_splits(cx, cy, 9, B * H * W, sms), B * H * W
        assert (splits <= 2) if sms == 1 else (splits * 1024 >= M), "%d K splits of %d rows with %d SMs" % (splits, M, sms)
    torch.manual_seed(B * 1000 + H + W + cx + cy)
    X = torch.randn(B * H * W, cx, device="cuda").bfloat16()
    Y = torch.randn(B * H * W, cy, device="cuda").bfloat16()
    _close(_run(X, Y, B, H, W), _ref(X, Y, B, H, W))


def test_window_path_is_the_one_that_runs():
    """The head shape launches the window instantiation (Y = 64, three taps per kernel row, 7 k-steps = 112 pixels)."""
    from torch.profiler import ProfilerActivity, profile
    B, H, W = 1, 4, 336
    X = torch.randn(B * H * W, 384, device="cuda").bfloat16()
    Y = torch.randn(B * H * W, 64, device="cuda").bfloat16()
    _run(X, Y, B, H, W)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        _run(X, Y, B, H, W)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "wgrad_kernel" in e.name]
    assert any("wgrad_kernel<64, 3, false, 7>" in n for n in names), names


@pytest.mark.parametrize("B,H,W,cx,cy,deterministic", [
    (2, 16, 112, 128, 64, False),
    (2, 30, 336, 384, 64, True),   # several K splits, their boundaries inside image rows
    (2, 12, 176, 64, 128, True),   # 64-channel X; rows end in a partial chunk
])
def test_window_and_gather_paths_agree_bit_for_bit(B, H, W, cx, cy, deterministic):
    """The same dense convolution through a neighbour table (gather path) and through its geometry (window path): both
    run the same K splits and the same 16-row k-steps in the same order, so dW is the same bit for bit."""
    torch.manual_seed(7 + W + cx)
    M = B * H * W
    X = torch.randn(M, cx, device="cuda").bfloat16()
    Y = torch.randn(M, cy, device="cuda").bfloat16()
    b, y, x = torch.meshgrid(torch.arange(B), torch.arange(H), torch.arange(W), indexing="ij")
    cols = []
    for r in range(3):
        for s in range(3):
            yi, xi = y + r - 1, x + s - 1
            ok = (yi >= 0) & (yi < H) & (xi >= 0) & (xi < W)
            cols.append(torch.where(ok, (b * H + yi) * W + xi, torch.full_like(yi, -1)).reshape(-1))
    nbr = torch.stack(cols, 1).int().cuda().contiguous()
    prev = ops.set_deterministic(deterministic)
    try:
        gather = torch.zeros(9, cx, cy, device="cuda")
        ops.wgrad(X, cx, Y, cy, M, 9, gather, nbr=nbr)
        window = _run(X, Y, B, H, W)
    finally:
        ops.set_deterministic(prev)
    if deterministic:
        assert ops.wgrad_splits(cx, cy, 9, M, ops.sm_count()) > 1
    _close(window, _ref(X, Y, B, H, W))
    assert torch.equal(window, gather)


def test_window_deterministic_mode():
    torch.manual_seed(11)
    B, H, W, cx, cy = 2, 40, 336, 384, 64
    X = torch.randn(B * H * W, cx, device="cuda").bfloat16()
    Y = torch.randn(B * H * W, cy, device="cuda").bfloat16()
    prev = ops.set_deterministic(True)
    try:
        a, b = _run(X, Y, B, H, W), _run(X, Y, B, H, W)
    finally:
        ops.set_deterministic(prev)
    assert torch.equal(a, b)
    _close(a, _ref(X, Y, B, H, W))


def test_window_split_mode_segments():
    """fp32-grade split operands: one window launch per (X piece, Y piece) segment, all accumulating into one dW, equal
    to the fp64 weight gradient of the fp32 values the pieces represent."""
    torch.manual_seed(13)
    B, H, W, cx, cy = 1, 12, 336, 128, 64
    M = B * H * W
    xf = torch.randn(M, cx, device="cuda")
    yf = torch.randn(M, cy, device="cuda")
    X, Y = ops.rows_split(xf), ops.rows_split(yf)
    dW = torch.zeros(9, cx, cy, device="cuda")
    ops.wgrad_split(X, cx, cx, Y, cy, cy, M, 9, dW, dense=(H, W, H, W, 3, 1, 1, 1))
    assert len(ops.split_segments()) > 1
    _close(dW, _ref(xf, yf, B, H, W), tol=1e-4)
