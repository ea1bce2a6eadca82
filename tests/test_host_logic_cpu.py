"""Host-side (Python) logic of the ops layer that needs no GPU: operand splitting, eligibility rules, config helpers."""
import torch

from pillarnext_b200 import ops


def test_wgrad_splits_channel_counts_the_kernel_does_not_tile(monkeypatch):
    """448 = 7 sibling heads x 64: the weight-gradient kernel tiles X in 128-channel blocks (or one 64 block), the
    wrapper issues 384 + 64 column slices of the SAME row matrix and accumulates each into its rows of dW."""
    calls = []

    class FakeLib:
        def pnx_wgrad(self, X, ldx, xc, Y, ldy, y_rows, yc, gathered, M, taps, nbr, *rest):
            dW_ptr = rest[9]   # ..., shuffle, dW, partials, sm_count, stream
            calls.append(dict(x_off=X, ldx=ldx, xc=xc, yc=yc, taps=taps, dW=dW_ptr))
            return 0

        def pnx_wgrad_splits(self, xc, yc, taps, M, sm_count):
            return 2

    monkeypatch.setattr(ops, "lib", lambda: FakeLib())
    monkeypatch.setattr(ops, "ptr", lambda t: None if t is None else t.data_ptr())
    monkeypatch.setattr(ops, "stream", lambda: 0)
    monkeypatch.setattr(ops, "sm_count", lambda: 148)
    X = torch.zeros(10, 448, dtype=torch.bfloat16)
    Y = torch.zeros(10, 192, dtype=torch.bfloat16)
    dW = torch.ones(9, 448, 192)
    out = ops.wgrad(X, 448, Y, 192, 10, 9, dW, dense=(4, 4, 4, 4, 3, 1, 1, 1))
    assert out is dW and torch.equal(dW, torch.ones_like(dW))                 # parts were zero: dW untouched
    assert [(c["xc"], c["ldx"], c["x_off"] - X.data_ptr(), c["taps"]) for c in calls] == [(384, 448, 0, 9), (64, 448, 768, 9)]
    assert all(c["dW"] != dW.data_ptr() for c in calls)                       # each part accumulates into its own buffer
    calls.clear()
    ops.wgrad(X[:, :384], 384, Y, 192, 10, 9, torch.zeros(9, 384, 192), dense=(4, 4, 4, 4, 3, 1, 1, 1))
    assert len(calls) == 1 and calls[0]["xc"] == 384                          # supported widths go straight through


def test_window_conv_eligibility():
    d = lambda H, W, k=3, s=1, dil=1, pad=1: (H, W, H, W, k, s, dil, pad)
    assert ops.win_eligible(d(336, 336), 384, 64)            # head conv at nuScenes resolution (3 x 128-pixel tiles)
    assert ops.win_eligible(d(376, 376), 64, 64)             # Waymo-bench head
    assert not ops.win_eligible(d(168, 168), 256, 256)       # 168 -> 2 tiles of 128 wastes 34 %: gather engine instead
    assert not ops.win_eligible(d(336, 336, dil=6, pad=6), 256, 256)
    assert not ops.win_eligible(d(336, 336, s=2), 64, 64)
    assert not ops.win_eligible(None, 64, 64)
    assert not ops.win_eligible(d(336, 336), 64, 64, out_fp32=True)


def test_pack_descriptors_reproduce_the_torch_packing():
    """functional.WLayout.gather_desc (the 4-D gather-copy descriptors pnx_pack_weights executes on the GPU) against the
    per-weight torch packing, emulated here with numpy strides: every layout / flip combination, odd shapes included."""
    import numpy as np
    from pillarnext_b200 import functional as Fn
    g = torch.Generator().manual_seed(1)
    cases = [("dense", (20, 12, 3, 3)), ("dense", (10, 64, 1, 1)), ("sp", (24, 3, 3, 8)), ("convT", (16, 12, 2, 2))]
    for kind, shape in cases:
        w = torch.randn(*shape, generator=g)
        lay = Fn.WLayout(kind)
        flat = w.numpy().reshape(-1)
        for which, flip in (("fwd", False), ("dgrad", False), ("dgrad", True)):
            if kind == "convT" and flip:
                continue
            dims, strides, base = lay.gather_desc(tuple(shape), which, flip)
            idx = base + sum(np.arange(d).reshape([-1 if i == j else 1 for j in range(4)]) * s
                             for i, (d, s) in enumerate(zip(dims, strides)))
            got = torch.tensor(flat[idx.reshape(-1)]).to(torch.bfloat16)
            want = lay.pack_fwd(w) if which == "fwd" else lay.pack_dgrad(w, flip)
            assert got.numel() == want.numel() and torch.equal(got, want.reshape(-1)), (kind, which, flip)


def test_frame_tiled_voxelizer_host_plan():
    """Host-side planning of pnx_voxelize_frames (no GPU needed): slices per frame from the shared-memory budget, geometries
    whose frame is not a whole number of 32-word blocks are refused, scratch size grows with the batch."""
    from pillarnext_b200 import _lib
    L = _lib.lib()
    assert L.pnx_voxelize_frames_supported(6, 1344, 1344) == 12        # nuScenes: 226 KB bitmap per frame -> 2 slices
    assert L.pnx_voxelize_frames_supported(3, 1504, 1504) == 6         # Waymo: 283 KB -> 2 slices
    assert L.pnx_voxelize_frames_supported(2, 128, 128) == 2           # tiny grid: one slice per frame
    assert L.pnx_voxelize_frames_supported(2, 40, 40) == 0             # 40 x 2 words: not whole 32-word blocks
    assert L.pnx_voxelize_frames_supported(0, 128, 128) == 0
    assert L.pnx_voxelize_frames_scratch(8) > L.pnx_voxelize_frames_scratch(2) > 0
    # deterministic weight gradients: the split count is a pure function of the shape
    assert L.pnx_wgrad_splits(384, 64, 9, 677376, 148) == L.pnx_wgrad_splits(384, 64, 9, 677376, 148) >= 1
    assert L.pnx_wgrad_splits(384, 64, 9, 0, 148) == 0
    assert L.pnx_set_deterministic(1) == 0 and L.pnx_set_deterministic(0) == 1
