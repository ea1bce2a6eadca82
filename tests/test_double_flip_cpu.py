"""Double-flip test-time augmentation, CPU only.

* the oracle's undo transforms (oracle/flip_oracle.py) invert the reference's own box mirroring (box_np_ops.flip, frozen
  in tests/golden/ref_flip.npz by oracle/make_golden_flip.py) for boxes encoded the way the head is trained;
* four copies that are exact mirrors of one map give the single-pass oracle detections;
* the product's flip-merging decode, compiled for the host (pnx_det_decode_flip4_host), matches the oracle pixel by pixel;
* the double-flip preconditions and the `+model.post_processing.double_flip=True` override.
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import flip_oracle as FO
from oracle import predict_oracle as P
from oracle.predict_fixtures import fake_preds, test_cfg as _test_cfg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
OSF, VS, PC = 4, 0.5, 32.0                       # symmetric 128 x 128 grid of 0.5 m pillars -> 32 x 32 head maps
HW = int(2 * PC / (OSF * VS))


def encode(box):
    """One box as the head is trained to output it (assign.py:101-105): pixel (py, px) and its 10 raw channels."""
    u, v = (box[0] + PC) / (OSF * VS), (box[1] + PC) / (OSF * VS)
    px, py = int(math.floor(u)), int(math.floor(v))
    ch = dict(reg=[u - px, v - py], height=[box[2]], dim=list(np.log(box[3:6])), vel=[box[6], box[7]],
              rot=[math.sin(box[8]), math.cos(box[8])])
    return py, px, ch


@pytest.mark.parametrize("name,flip_y,flip_x", [("flip_x", True, False), ("flip_y", False, True), ("flip_xy", True, True)])
def test_undo_inverts_reference_flip(name, flip_y, flip_x):
    """The reference mirrors a box (flip(axis='x'): y mirror, flip(axis='y'): x mirror); the mirrored box, encoded on its
    pixel and mapped back by the undo, decodes to the original box: reg offset, (sin, cos) and (vx, vy) round-trip."""
    gold = np.load(os.path.join(GOLDEN, "ref_flip.npz"))
    for box, mirrored in zip(gold["boxes"], gold[name]):
        assert (mirrored[0] == -box[0]) == flip_x and (mirrored[1] == -box[1]) == flip_y
        py, px, ch = encode(mirrored)
        pd = {k: torch.zeros(1, len(v), HW, HW, dtype=torch.float64) for k, v in ch.items()}
        pd["hm"] = torch.zeros(1, 1, HW, HW, dtype=torch.float64)
        for k, v in ch.items():
            pd[k][0, :, py, px] = torch.tensor(v, dtype=torch.float64)
        back = FO.undo_flip(pd, flip_y, flip_x)
        oy, ox, _ = encode(box)
        assert (oy, ox) == ((HW - 1 - py) if flip_y else py, (HW - 1 - px) if flip_x else px)
        boxes, _, _ = P.decode(back, OSF, [VS, VS], [-PC, -PC])
        got = boxes[0, oy * HW + ox].numpy()
        np.testing.assert_allclose(got[:8], box[:8], atol=1e-9)
        assert abs(math.remainder(got[8] - box[8], 2 * math.pi)) < 1e-9, (got[8], box[8])


def test_exact_mirror_copies_give_single_pass_detections():
    cfg = _test_cfg()
    tasks = [["car"], ["truck", "construction_vehicle"]]
    preds = [fake_preds(2, 24, 20, len(t), 40 + i) for i, t in enumerate(tasks)]
    want = P.predict(preds, [1, 2], cfg, [[0.0], [0.0, 0.0]], tokens=["a", "b"])
    got = FO.predict_double_flip([FO.mirror_copies(pd) for pd in preds], [1, 2], cfg, [[0.0], [0.0, 0.0]], tokens=["a", "b"])
    for g, w in zip(got, want):
        assert g["token"] == w["token"] and w["scores"].numel() > 5
        assert torch.equal(g["label_preds"], w["label_preds"])
        assert torch.allclose(g["scores"], w["scores"], atol=1e-6)
        assert torch.allclose(g["box3d_lidar"], w["box3d_lidar"], atol=1e-5)


def rows_with_iou(pd, with_iou):
    """Head dict -> channels-last rows [B*H*W, 16]; returns (rows, offs)."""
    B, _, H, W = pd["hm"].shape
    cols = dict(reg=0, height=2, dim=3, rot=6, vel=8)
    cols.update(dict(iou=10, hm=11) if with_iou else dict(hm=10))
    out = torch.zeros(B * H * W, 16)
    for k, o in cols.items():
        v = pd[k].permute(0, 2, 3, 1).reshape(B * H * W, -1)
        out[:, o:o + v.shape[1]] = v
    return out.contiguous(), [cols["reg"], cols["height"], cols["dim"], cols["rot"], cols["vel"], cols["hm"],
                              cols.get("iou", -1)]


@pytest.mark.parametrize("with_iou,rect_v", [(False, [0.0, 0.0]), (True, [0.71, 0.65])])
def test_host_compiled_flip_decode_matches_oracle(with_iou, rect_v):
    from pillarnext_b200 import ops
    cfg = _test_cfg()
    B, H, W, C = 2, 12, 10, 2
    pd = fake_preds(4 * B, H, W, C, 23)                         # four unrelated copies: every merge term matters
    if with_iou:
        pd["iou"] = torch.randn(4 * B, 1, H, W, generator=torch.Generator().manual_seed(4)) * 0.8
    pd["reg"][0, :, 0, 0] = torch.tensor([-900.0, 0.3])       # merged pixel (0, 0, 0) is pushed out of range
    out, offs = rows_with_iou(pd, with_iou)
    boxes, hm, iou = FO.decode_double_flip(pd, 4, cfg["voxel_size"], cfg["pc_range"])
    scores, labels = hm.max(-1)
    pcr = torch.tensor(cfg["post_center_limit_range"])
    keep = (scores > cfg["score_threshold"]) & (boxes[..., :3] >= pcr[:3]).all(-1) & (boxes[..., :3] <= pcr[3:]).all(-1)
    rect = torch.tensor(rect_v)[labels]
    scores = torch.pow(scores, 1 - rect) * torch.pow(torch.clamp(iou, 0, 1), rect)
    kept, b9, sc, lb = ops.det_decode_host(out.numpy(), B, H, W, C, offs, 4.0, [0.075, 0.075], [-50.4, -50.4],
                                           cfg["score_threshold"], cfg["post_center_limit_range"], rect_v, double_flip=True)
    n_kept = 0
    for m in range(B * H * W):
        b, i = divmod(m, H * W)
        assert kept[m] == bool(keep[b, i]), (m, kept[m])
        if kept[m]:
            n_kept += 1
            assert lb[m] == int(labels[b, i])
            assert abs(float(sc[m]) - float(scores[b, i])) < 2e-6
            assert torch.allclose(torch.from_numpy(b9[m]), boxes[b, i], atol=1e-5, rtol=1e-6)
    assert 20 < n_kept < B * H * W and not keep[0, 0]


def test_double_flip_preconditions():
    from pillarnext_b200 import modules
    head = modules.CenterHead.__new__(modules.CenterHead)
    cfg = dict(pc_range=[-32.0, -32.0, -5.0, 32.0, 32.0, 3.0], voxel_size=[0.5, 0.5, 8.0], out_size_factor=[4])
    raws = [dict(B=8, H=32, W=32)]
    head._check_double_flip(raws, cfg)                                        # symmetric grid, maps of grid / 4
    with pytest.raises(ValueError, match="mirror-symmetric"):
        head._check_double_flip(raws, dict(cfg, pc_range=[-32.0, -30.0, -5.0, 32.0, 34.0, 3.0]))
    with pytest.raises(ValueError, match="grid / out_size_factor"):
        head._check_double_flip([dict(B=8, H=32, W=30)], cfg)
    with pytest.raises(ValueError, match="4 mirrored copies"):
        head._check_double_flip([dict(B=6, H=32, W=32)], cfg)
    with pytest.raises(ValueError, match="6-value pc_range"):
        head._check_double_flip(raws, dict(cfg, pc_range=[-32.0, -32.0]))


def test_double_flip_config_override():
    from pillarnext_b200 import hydra_lite, modules
    d = os.path.join(ROOT, "configs", "experiments")
    base = hydra_lite.main(d, "synth_det_pp18_aspp", [])
    cfg = hydra_lite.main(d, "synth_det_pp18_aspp", ["+model.post_processing.double_flip=True"])
    assert modules._cfg_get(base.model.post_processing, "double_flip", False) is False
    assert modules._cfg_get(cfg.model.post_processing, "double_flip", False) is True
