"""Oracle pinning for row F1 (decode + rotated NMS), CPU only.

* oracle.predict_oracle.iou_bev  vs  the reference's own iou3d_cpu.cpp (its output on seeded boxes is stored in
  tests/golden/ref_live.npz by oracle/make_golden_live.py);
* oracle.predict_oracle.predict  vs  the reference's own CenterHead.predict run on CPU with its CUDA-only nms_gpu call
  replaced by the oracle's greedy rotated NMS (outputs stored in tests/golden/ref_predict.npz);
* closed-form IoU cases and NMS invariants that need neither.
"""
import math
import os

import numpy as np
import pytest
import torch

from oracle import predict_oracle as P
from oracle.predict_fixtures import fake_preds as _fake_preds, test_cfg as _test_cfg, to_rows

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def rand_boxes(n, seed, spread=6.0):
    g = torch.Generator().manual_seed(seed)
    xy = (torch.rand(n, 2, generator=g) - 0.5) * spread
    z = torch.rand(n, 1, generator=g)
    dims = torch.rand(n, 3, generator=g) * 3 + 0.5
    yaw = (torch.rand(n, 1, generator=g) - 0.5) * 2 * math.pi
    return torch.cat([xy, z, dims, yaw], 1).float()


def test_iou_closed_form():
    a = np.array([0, 0, 0, 4, 2, 1, 0], dtype=np.float32)
    b = np.array([1, 0, 0, 4, 2, 1, 0], dtype=np.float32)
    assert abs(float(P.iou_bev(a, b)) - 0.6) < 1e-6                       # 6 / (8 + 8 - 6)
    assert abs(float(P.iou_bev(a, a)) - 1.0) < 1e-6
    c = np.array([10, 10, 0, 1, 1, 1, 0.3], dtype=np.float32)
    assert float(P.iou_bev(a, c)) == 0.0
    sq = np.array([0, 0, 0, 2, 2, 1, 0], dtype=np.float32)
    sq45 = np.array([0, 0, 0, 2, 2, 1, math.pi / 4], dtype=np.float32)
    inter = 8 * (math.sqrt(2) - 1)                                         # regular octagon
    assert abs(float(P.iou_bev(sq, sq45)) - inter / (8 - inter)) < 1e-4


def test_iou_matches_reference_extension():
    """tests/golden/ref_live.npz holds the reference's boxes_iou_bev_cpu (iou3d_cpu.cpp) on these boxes."""
    a, b = rand_boxes(24, 1), rand_boxes(24, 2)
    want = torch.from_numpy(np.load(os.path.join(GOLDEN, "ref_live.npz"))["iou_bev"])
    got = torch.tensor([[float(P.iou_bev(x.numpy(), y.numpy())) for y in b] for x in a])
    assert (want > 0.05).sum() > 20                                        # the sample does overlap
    assert (got - want).abs().max().item() < 2e-5, (got - want).abs().max().item()


def test_nms_invariants():
    boxes = rand_boxes(60, 5, spread=5.0).numpy()
    keep = P.nms_rotated(boxes, 0.2)
    assert keep[0] == 0 and keep == sorted(keep)
    for i, a in enumerate(keep):                                            # kept boxes do not suppress each other
        for b in keep[i + 1:]:
            assert float(P.iou_bev(boxes[a], boxes[b])) <= 0.2
    for j in set(range(60)) - set(keep):                                    # every dropped box has a kept suppressor before it
        assert any(k < j and float(P.iou_bev(boxes[k], boxes[j])) > 0.2 for k in keep)
    assert P.nms_rotated(boxes, 1.1) == list(range(60))


def test_predict_matches_reference_predict():
    """tests/golden/ref_predict.npz holds the reference's CenterHead.predict on these inputs (oracle/make_golden_predict.py)."""
    gold = np.load(os.path.join(GOLDEN, "ref_predict.npz"))
    tasks = [["car"], ["truck", "construction_vehicle"]]
    cfg = _test_cfg()
    preds = [_fake_preds(2, 24, 20, len(t), 10 + i) for i, t in enumerate(tasks)]
    want = [dict(token=tok, **{k: torch.from_numpy(gold["%s_%d" % (k, i)]) for k in ("box3d_lidar", "scores", "label_preds")})
            for i, tok in enumerate(["a", "b"])]
    got = P.predict(preds, [len(t) for t in tasks], cfg, [[0.0], [0.0, 0.0]], tokens=["a", "b"])
    assert len(got) == len(want) == 2
    for g, w in zip(got, want):
        assert g["token"] == w["token"]
        assert g["box3d_lidar"].shape == w["box3d_lidar"].shape and w["box3d_lidar"].shape[0] > 5
        assert torch.equal(g["label_preds"], w["label_preds"])
        assert torch.allclose(g["scores"], w["scores"], atol=1e-6)
        assert torch.allclose(g["box3d_lidar"], w["box3d_lidar"], atol=1e-5)


# ---------------------------------------------------------------------- product math compiled for the host (no GPU needed)


def test_host_compiled_decode_and_iou_match_oracle():
    from pillarnext_b200 import ops
    cfg = _test_cfg()
    pd = _fake_preds(2, 12, 10, 2, 3)
    pd["reg"][0, :, 0, 0] = torch.tensor([-900.0, 0.3])                  # pushed outside post_center_limit_range
    out = to_rows(pd)
    boxes, hm, iou = P.decode(pd, 4, cfg["voxel_size"], cfg["pc_range"])
    scores, labels = hm.max(-1)
    pcr = torch.tensor(cfg["post_center_limit_range"])
    keep = (scores > cfg["score_threshold"]) & (boxes[..., :3] >= pcr[:3]).all(-1) & (boxes[..., :3] <= pcr[3:]).all(-1)
    kept, b9, sc, lb = ops.det_decode_host(out.numpy(), 2, 12, 10, 2, [0, 2, 3, 6, 8, 10, -1], 4.0, [0.075, 0.075],
                                           [-50.4, -50.4], cfg["score_threshold"], cfg["post_center_limit_range"], [0.0] * 8)
    n_kept = 0
    for m in range(out.shape[0]):
        b, i = divmod(m, 120)
        assert kept[m] == bool(keep[b, i]), (m, kept[m])
        if kept[m]:
            n_kept += 1
            assert lb[m] == int(labels[b, i])
            assert abs(float(sc[m]) - float(scores[b, i])) < 1e-6
            assert torch.allclose(torch.from_numpy(b9[m]), boxes[b, i], atol=1e-5, rtol=1e-6)
    assert 20 < n_kept < out.shape[0] and not keep[0, 0]
    bx = rand_boxes(40, 8).numpy()
    got = ops.det_iou_bev_host(bx[0::2], bx[1::2])
    for i in range(0, 40, 2):
        assert abs(float(got[i // 2]) - float(P.iou_bev(bx[i], bx[i + 1]))) < 2e-6


def test_host_compiled_iou_equals_reference_extension_bit_for_bit():
    """The product's rotated IoU compiled for the host equals the reference's iou3d_cpu.cpp (golden) to the bit on every
    pair: the same statements in the same order, down to the corners rounded as x - dx / 2 before the rotation."""
    from pillarnext_b200 import ops
    a, b = rand_boxes(24, 1).numpy(), rand_boxes(24, 2).numpy()
    want = np.load(os.path.join(GOLDEN, "ref_live.npz"))["iou_bev"]
    got = ops.det_iou_bev_host(np.repeat(a, 24, 0), np.tile(b, (24, 1))).reshape(24, 24)
    assert (want > 0).sum() > 200
    assert np.array_equal(got.view(np.int32), want.view(np.int32)), "%d of 576 pairs differ" % int(
        (got.view(np.int32) != want.view(np.int32)).sum())


def test_oracle_predict_matches_golden_reference_outputs():
    """Runs anywhere: tests/golden/ref_predict.npz holds the reference's own predict outputs (oracle/make_golden_predict.py)."""
    from oracle.make_golden_predict import SEEDS, SHAPE, TASKS
    path = os.path.join(GOLDEN, "ref_predict.npz")
    gold = np.load(path)
    preds = [_fake_preds(*SHAPE, len(t), SEEDS[i]) for i, t in enumerate(TASKS)]
    got = P.predict(preds, [len(t) for t in TASKS], _test_cfg(), [[0.0], [0.0, 0.0]], tokens=["a", "b"])
    for i, g in enumerate(got):
        assert gold["box3d_lidar_%d" % i].shape[0] > 5
        assert np.array_equal(g["label_preds"].numpy(), gold["label_preds_%d" % i])
        assert np.allclose(g["scores"].numpy(), gold["scores_%d" % i], atol=1e-6)
        assert np.allclose(g["box3d_lidar"].numpy(), gold["box3d_lidar_%d" % i], atol=1e-5)


def test_host_compiled_decode_with_rectifier_and_iou_head():
    """Waymo-style task: `iou` head present and rectifier != 0 (waymo_det_pp18_aspp_iou_car_sp.yaml: [[0.68],[0.71,0.65]]);
    nuScenes uses rectifier 0.5 without an iou head (score -> sqrt(score))."""
    from pillarnext_b200 import ops
    cfg = _test_cfg()
    for with_iou, rect_v in ((True, [0.71, 0.65]), (False, [0.5, 0.5])):
        pd = _fake_preds(1, 10, 12, 2, 17)
        g = torch.Generator().manual_seed(3)
        if with_iou:
            pd["iou"] = torch.randn(1, 1, 10, 12, generator=g) * 0.8          # raw head output in [-inf, inf] -> clamp((x+1)/2)
        B, H, W = 1, 10, 12
        cols = dict(reg=0, height=2, dim=3, rot=6, vel=8)
        cols.update(dict(iou=10, hm=11) if with_iou else dict(hm=10))
        out = torch.zeros(B * H * W, 16)
        for k, o in cols.items():
            v = pd[k].permute(0, 2, 3, 1).reshape(B * H * W, -1)
            out[:, o:o + v.shape[1]] = v
        boxes, hm, iou = P.decode(pd, 4, cfg["voxel_size"], cfg["pc_range"])
        want = P.post_processing(boxes, hm, iou, rect_v, cfg["score_threshold"], cfg["post_center_limit_range"],
                                 [1.1, 1.1], 10000, 10000)[0]            # threshold > 1: NMS keeps everything
        kept, b9, sc, lb = ops.det_decode_host(out.numpy(), B, H, W, 2, [0, 2, 3, 6, 8, cols["hm"], cols.get("iou", -1)],
                                               4.0, [0.075, 0.075], [-50.4, -50.4], cfg["score_threshold"],
                                               cfg["post_center_limit_range"], rect_v)
        got = [(int(lb[m]), float(sc[m]), b9[m].tolist()) for m in range(out.shape[0]) if kept[m]]
        assert len(got) == want["scores"].numel() > 10
        # same multiset of detections (several candidates can tie at score 0 when the clamped iou is 0: order by box too)
        key = lambda t: (t[0], -round(t[1], 5), round(t[2][0], 3), round(t[2][1], 3))
        got.sort(key=key)
        ref = sorted(zip(want["label_preds"].tolist(), want["scores"].tolist(), want["box3d_lidar"].tolist()), key=key)
        assert [t[0] for t in got] == [t[0] for t in ref]
        assert torch.allclose(torch.tensor([t[1] for t in got]), torch.tensor([t[1] for t in ref]), atol=2e-6)
        assert torch.allclose(torch.tensor([t[2] for t in got]), torch.tensor([t[2] for t in ref]), atol=1e-5, rtol=1e-6)


def test_iou_head_loss_oracle_matches_reference_loss():
    """Waymo-style head (extra `iou` head, with_reg_iou): the reference's own CenterHead.loss on CPU, with only the
    CUDA-only boxes_aligned_iou3d_gpu swapped for the oracle's aligned IoU (stored in tests/golden/ref_live.npz by
    oracle/make_golden_live.py, which builds the same inputs), against the oracle's center_loss(with_iou)."""
    from oracle import pillarnext_oracle as O
    from pillarnext_b200 import synth
    gold = np.load(os.path.join(GOLDEN, "ref_live.npz"))
    tasks = [["vehicle"], ["pedestrian", "cyclist"]]
    cfg = synth.tiny_config(64, tasks)
    heads = dict(reg=[2, 2], height=[1, 2], dim=[3, 2], rot=[2, 2], vel=[2, 2], iou=[1, 2])
    ex = synth.make_batch([3, 4], 1500, cfg, n_boxes=12, sweeps=1)
    H = W = 64 // 8 * 2
    g = torch.Generator().manual_seed(5)
    preds = []
    for t, names in enumerate(tasks):
        pd = {k: torch.randn(2, c, H, W, generator=g) * 0.5 for k, (c, _) in heads.items()}
        pd["hm"] = torch.randn(2, len(names), H, W, generator=g) - 2.0
        preds.append(pd)
    want = float(gold["iou_head_loss"][0])
    got, logs = O.center_loss(ex, preds, 1.0, cfg["code_weights"], True, cfg["voxel_size"], cfg["pc_range"], [4, 4],
                              with_iou=True)
    assert abs(float(got) - want) < 1e-5 * max(1.0, abs(want))
    for t in range(2):
        assert float(ex["mask"][t].sum()) > 0
        assert abs(float(logs[t]["iou_loss"]) - float(gold["iou_head_iou_loss"][t])) < 1e-6
        assert 0.0 < float(logs[t]["iou_loss"]) < 2.0
