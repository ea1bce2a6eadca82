"""Double-flip test-time augmentation on the GPU: point expansion, the flip-merging decode + NMS against the CPU oracle
(oracle/flip_oracle.py, pinned by tests/test_double_flip_cpu.py), mirror equivariance of the whole eval forward, and
TTA detection quality of a briefly trained model against the oracle's TTA forward."""
import math
import os
import sys

import pytest
import torch

from oracle import flip_oracle as FO
from oracle import pillarnext_oracle as O
from oracle import predict_oracle as P
from oracle.predict_fixtures import fake_preds as _fake_preds, test_cfg as _test_cfg
from pillarnext_b200 import functional as Fn
from pillarnext_b200 import hydra_lite, modules, ops, scenes, synth
from pillarnext_b200.trainer import example_to_device
from test_double_flip_cpu import rows_with_iou
from test_predict_gpu import clustered_preds, screen

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_flip4_points_bit_exact():
    g = torch.Generator().manual_seed(3)
    pts = torch.cat([torch.randint(0, 3, (5001, 1), generator=g).float(), torch.randn(5001, 5, generator=g) * 20], 1)
    got = ops.flip4_points(pts.cuda()).cpu()
    want = torch.cat([torch.stack([pts[:, 0] * 4 + k, -pts[:, 1] if k & 2 else pts[:, 1], -pts[:, 2] if k & 1 else pts[:, 2],
                                   pts[:, 3], pts[:, 4], pts[:, 5]], 1) for k in range(4)])
    assert torch.equal(got, want)
    assert torch.equal(got, FO.flip4_points(pts))
    assert ops.flip4_points(torch.zeros(0, 6, device="cuda")).shape == (0, 6)


def flip_run_and_compare(pd4, C, thr, cfg, pre_max, post_max, with_iou=False, rect=None, label_offset=0):
    """det_postprocess(double_flip=True) on a [4B]-frame head output against the oracle's merge + post-processing."""
    B4, _, H, W = pd4["hm"].shape
    B = B4 // 4
    rect = rect or [0.0] * C
    boxes, hm, iou = FO.decode_double_flip(pd4, 4, cfg["voxel_size"], cfg["pc_range"])
    want = P.post_processing(boxes, hm, iou, rect, cfg["score_threshold"], cfg["post_center_limit_range"], thr, pre_max,
                             post_max)
    sc, lb = hm.max(-1)
    for b in range(B):                                      # the comparison is only meaningful away from the threshold
        for c in range(C):
            m = (sc[b] > cfg["score_threshold"]) & (lb[b] == c)
            assert screen(boxes[b][m][:, [0, 1, 2, 3, 4, 5, 8]], thr[c]), "test input sits on the NMS threshold: change the seed"
            assert sc[b][m].unique().numel() == int(m.sum()), "tied scores: change the seed"
    out, offs = rows_with_iou(pd4, with_iou)
    det_box, det_score, det_label, cnt = ops.det_postprocess(
        out.cuda(), B, H, W, C, offs, 4, cfg["voxel_size"], cfg["pc_range"], cfg["score_threshold"],
        cfg["post_center_limit_range"], rect, thr, pre_max, post_max, label_offset=label_offset, double_flip=True)
    cnt = cnt.cpu().tolist()
    total = 0
    for b in range(B):
        gb = torch.cat([det_box[b * C + c, :cnt[b * C + c]] for c in range(C)]).cpu()
        gs = torch.cat([det_score[b * C + c, :cnt[b * C + c]] for c in range(C)]).cpu()
        gl = torch.cat([det_label[b * C + c, :cnt[b * C + c]] for c in range(C)]).cpu()
        w = want[b]
        assert gb.shape == w["box3d_lidar"].shape, (gb.shape, w["box3d_lidar"].shape)
        assert torch.equal(gl, w["label_preds"] + label_offset)
        assert torch.allclose(gs, w["scores"], atol=2e-6)
        assert torch.allclose(gb, w["box3d_lidar"], atol=1e-5, rtol=1e-6)
        total += gb.shape[0]
    return total


def clustered4(B, H, W, C, seed):
    """Four copies per frame: the mirror images of one clustered map plus independent noise, so the merge matters."""
    pd = clustered_preds(B, H, W, C, seed)
    pd4 = FO.mirror_copies(pd)
    g = torch.Generator().manual_seed(seed + 1)
    return {k: v + torch.randn(v.shape, generator=g) * 0.3 for k, v in pd4.items()}


def test_flip_postprocess_matches_oracle():
    cfg = _test_cfg()
    n = flip_run_and_compare(clustered4(2, 24, 20, 2, 21), 2, [0.2, 0.2], cfg, 1000, 83, label_offset=1)
    assert n > 10
    n_cut = flip_run_and_compare(clustered4(2, 24, 20, 2, 21), 2, [0.2, 0.2], cfg, 40, 2)
    assert n_cut == 2 * 2 * 2
    n = flip_run_and_compare(_fake_preds(8, 17, 33, 1, 14), 1, [0.2], cfg, 1000, 83)     # four unrelated copies
    assert n > 20


def test_flip_postprocess_waymo_iou_head_and_rectifier():
    cfg = _test_cfg()
    pd4 = clustered4(2, 24, 20, 2, 39)
    pd4["iou"] = torch.randn(8, 1, 24, 20, generator=torch.Generator().manual_seed(9)) * 0.3 + 0.5     # no ties at iou 0
    n = flip_run_and_compare(pd4, 2, [0.2, 0.2], cfg, 4096, 500, with_iou=True, rect=[0.71, 0.65])
    assert n > 10


# ------------------------------------------------------------------ end to end: mirror equivariance of the eval forward
def _tiny_model():
    tasks = [["car"], ["truck", "construction_vehicle"]]
    cfg = synth.tiny_config(128, tasks)
    torch.manual_seed(1)
    model = modules.build_pillarnext_b(cfg).cuda().eval()
    with torch.no_grad():
        for task in model.head.tasks:                       # spread the heat-map logits so a few hundred pass
            task.hm[3].bias.fill_(-1.5)
            task.hm[3].weight.mul_(6.0)
    model.post_processing = dict(post_center_limit_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], score_threshold=0.1,
                                 out_size_factor=[4, 4], voxel_size=cfg["voxel_size"], pc_range=cfg["pc_range"],
                                 nms=dict(nms_iou_threshold=[[0.2], [0.2, 0.2]], nms_pre_max_size=64,
                                          nms_post_max_size=20), double_flip=True)
    return model, cfg


def _merged_scores(model, points):
    """Per task, the merged score map [C, H, W] the flip decode sees, from the model's own 4-copy head output."""
    preds = model._forward(dict(points=ops.flip4_points(points), token=["f"]), copies=4)
    pcpu = [{k: v.detach().float().cpu() for k, v in pd.items()} for pd in preds]
    return pcpu, [FO.merge_double_flip(pd)[1][0] for pd in pcpu]


@pytest.mark.parametrize("axis", ["y", "x"])
def test_double_flip_mirror_equivariance(axis):
    model, cfg = _tiny_model()
    model.reader.frame_sorted = False
    ex = synth.make_batch([5], 3000, cfg, n_boxes=10, sweeps=10)
    pts = ex["points"].cuda().float()
    mir = pts.clone()
    col = 2 if axis == "y" else 1
    mir[:, col] = -mir[:, col]
    with torch.no_grad():
        p_f, s_f = _merged_scores(model, pts)
        p_m, s_m = _merged_scores(model, mir)
    # each copy's head map must not depend on its batch slot: copy k of F' is copy k ^ (1 or 2) of F, computed from the
    # same points in another slot
    swap = 1 if axis == "y" else 2
    for a, b in zip(p_f, p_m):
        for k in a:
            for c in range(4):
                assert torch.equal(a[k][c], b[k][c ^ swap]), "head output is not slot-independent (%s, copy %d)" % (k, c)
    dim = 1 if axis == "y" else 2                                   # [C, H, W]: rows are y, columns x
    for a, b in zip(s_f, s_m):
        assert torch.equal(a, torch.flip(b, [dim])), "merged score map is not bit-identically equivariant"
    with torch.no_grad():
        d_f = model(dict(points=pts, token=["f"]))["f"]
        d_m = model(dict(points=mir, token=["f"]))["f"]
    assert d_f["scores"].numel() > 5 and d_f["scores"].numel() == d_m["scores"].numel()
    # mirror F's detections and match them to F''s as sets (by label and score, then the nearest centre)
    bf = d_f["box3d_lidar"].clone()
    if axis == "y":
        bf[:, 1], bf[:, 7], bf[:, 8] = -bf[:, 1], -bf[:, 7], -bf[:, 8]
    else:
        bf[:, 0], bf[:, 6], bf[:, 8] = -bf[:, 0], -bf[:, 6], math.pi - bf[:, 8]
    bm = d_m["box3d_lidar"]
    used = set()
    for i in range(bf.shape[0]):
        cand = [j for j in range(bm.shape[0]) if j not in used and int(d_m["label_preds"][j]) == int(d_f["label_preds"][i])
                and float(d_m["scores"][j]) == float(d_f["scores"][i])]
        assert cand, "detection %d of F has no mirror image in F'" % i
        j = min(cand, key=lambda j: float((bm[j, :2] - bf[i, :2]).norm()))
        used.add(j)
        assert (bm[j, :8] - bf[i, :8]).abs().max().item() < 1e-4, (bm[j], bf[i])
        assert abs(math.remainder(float(bm[j, 8] - bf[i, 8]), 2 * math.pi)) < 1e-5, (bm[j, 8], bf[i, 8])


def test_double_flip_unset_leaves_eval_unchanged():
    """double_flip False (or absent) is the single-pass path: same detections as without the key."""
    model, cfg = _tiny_model()
    ex = synth.make_batch([0, 1], 3000, cfg, n_boxes=10, sweeps=10)
    exg = dict(points=ex["points"].cuda(), token=["a", "b"])
    with torch.no_grad():
        model.post_processing["double_flip"] = False
        d0 = model(exg)
        del model.post_processing["double_flip"]
        d1 = model(exg)
    for t in ("a", "b"):
        for k in ("box3d_lidar", "scores", "label_preds"):
            assert torch.equal(d0[t][k], d1[t][k])


# ------------------------------------------------------------------ TTA detection quality of a briefly trained model
def test_double_flip_map_against_oracle(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import train as train_tool
    work = str(tmp_path)
    overrides = ["trainer.max_epochs=6", "data.train_dataset.n_frames=640", "data.val_dataset.n_frames=12",
                 "dataloader.train.num_workers=0", "dataloader.val.num_workers=0", "dataloader.train.batch_size=4"]
    tr = train_tool.main(["--config-name", "synth_det_pp18_aspp", "--work-dir", work] + overrides)
    cfg = hydra_lite.main(os.path.join(ROOT, "configs", "experiments"), "synth_det_pp18_aspp", overrides)
    val = hydra_lite.instantiate(cfg.data.val_dataset)
    model = tr.model.eval()
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items()}
    head, pp = cfg.model.head, cfg.model.post_processing
    ocfg = dict(voxel_size=list(cfg.model.reader.voxel_size), pc_range=list(cfg.model.reader.pc_range), strides=[1, 2, 2, 2],
                tasks=[list(t) for t in head.tasks], common_heads={k: tuple(v) for k, v in head.common_heads.items()})
    tcfg = dict(post_center_limit_range=list(pp.post_center_limit_range), score_threshold=pp.score_threshold,
                out_size_factor=list(pp.out_size_factor), voxel_size=list(pp.voxel_size)[:2], pc_range=list(pp.pc_range)[:2],
                nms=dict(nms_iou_threshold=[list(t) for t in pp.nms.nms_iou_threshold], nms_pre_max_size=pp.nms.nms_pre_max_size,
                         nms_post_max_size=pp.nms.nms_post_max_size))
    batches = [scenes.collate([val[i] for i in range(i0, min(len(val), i0 + 4))]) for i0 in range(0, len(val), 4)]
    oracle = {}
    with torch.no_grad():
        for ex in batches:
            preds = O.detector_forward(FO.flip4_points(ex["points"]), sd, ocfg, 4 * len(ex["token"]), train=False)
            for o in FO.predict_double_flip([{k: v.contiguous() for k, v in pd.items()} for pd in preds],
                                            [len(t) for t in head.tasks], tcfg, [list(r) for r in head.rectifier],
                                            tokens=ex["token"]):
                oracle[o["token"]] = o
    m_oracle = val.evaluation(oracle)["mAP"]

    def product_map(double_flip):
        model.post_processing = dict(pp, double_flip=double_flip)
        dets = {}
        with torch.no_grad():
            for ex in batches:
                dets.update(model(example_to_device(ex, torch.device("cuda"))))
        assert sorted(dets) == sorted(oracle)
        return val.evaluation(dets)["mAP"]

    with Fn.precision("split"):
        m_split, m_split_single = product_map(True), product_map(False)
    m_bf16, m_bf16_single = product_map(True), product_map(False)
    msg = ("double-flip mAP on %d held-out scenes: oracle TTA (fp32 CPU) %.3f | product fp32-grade TTA %.3f (single pass "
           "%.3f) | product bf16 TTA %.3f (single pass %.3f)" % (len(val), m_oracle, m_split, m_split_single, m_bf16,
                                                                 m_bf16_single))
    print(msg)                                      # reported with `pytest -s` (or -rP)
    assert m_oracle > 5.0, "the detector did not learn the synthetic task: " + msg
    assert abs(m_split - m_oracle) <= 0.1, msg
    assert abs(m_bf16 - m_oracle) <= 1.5, msg
