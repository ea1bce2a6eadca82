"""Row F1 on the GPU: decode + rotated NMS kernels (through the C-ABI) against the CPU oracle (oracle/predict_oracle.py,
itself pinned to the reference's predict and iou3d_cpu.cpp by tests/test_predict_cpu.py).

Scores/boxes are fp32 on both sides (tolerance 1e-5: expf/atan2f implementations differ in the last ulp); the kept SETS
must be identical -- the inputs are screened so that no candidate pair sits within 1e-4 of the IoU threshold, where
a last-ulp difference could legitimately flip a suppression decision."""
import numpy as np
import pytest
import torch

from oracle import predict_oracle as P
from pillarnext_b200 import modules, ops, synth
from oracle.predict_fixtures import fake_preds as _fake_preds, test_cfg as _test_cfg, to_rows

pytestmark = pytest.mark.gpu
OFFS7 = [0, 2, 3, 6, 8, 10, -1]


def clustered_preds(B, H, W, classes, seed, n=160):
    """Many confident peaks in a small window with large boxes: heavy mutual overlap, long suppression chains."""
    g = torch.Generator().manual_seed(seed)
    pd = _fake_preds(B, H, W, classes, seed)
    pd["hm"].fill_(-6.0)
    pd["dim"] = torch.randn(B, 3, H, W, generator=g) * 0.25 + 0.9
    for b in range(B):
        ys = torch.randint(4, 14, (n,), generator=g)
        xs = torch.randint(3, 13, (n,), generator=g)
        cs = torch.randint(0, classes, (n,), generator=g)
        pd["hm"][b, cs, ys, xs] = torch.randn(n, generator=g) * 1.5 + 1.0
    return pd


def screen(boxes7, thr, margin=1e-4):
    """True when no pair of candidate boxes has an IoU within `margin` of the threshold (host-compiled product IoU)."""
    b = boxes7.numpy()
    i, j = np.triu_indices(len(b), 1)
    return not (np.abs(ops.det_iou_bev_host(b[i], b[j]).astype(np.float64) - thr) < margin).any()


def run_and_compare(pd, C, t, cfg, pre_max, post_max, label_offset=0):
    B, _, H, W = pd["hm"].shape
    boxes, hm, iou = P.decode(pd, cfg["out_size_factor"][t], cfg["voxel_size"], cfg["pc_range"])
    thr = cfg["nms"]["nms_iou_threshold"][t]
    want = P.post_processing(boxes, hm, iou, [0.0] * C, cfg["score_threshold"], cfg["post_center_limit_range"], thr,
                             pre_max, post_max)
    sc, lb = hm.max(-1)
    for b in range(B):                                      # the comparison is only meaningful away from the threshold
        for c in range(C):
            m = (sc[b] > cfg["score_threshold"]) & (lb[b] == c)
            assert screen(boxes[b][m][:, [0, 1, 2, 3, 4, 5, 8]], thr[c]), "test input sits on the NMS threshold: change the seed"
            assert sc[b][m].unique().numel() == int(m.sum()), "tied scores: change the seed"
    out = to_rows(pd).cuda()
    det_box, det_score, det_label, cnt = ops.det_postprocess(
        out, B, H, W, C, OFFS7, cfg["out_size_factor"][t], cfg["voxel_size"], cfg["pc_range"], cfg["score_threshold"],
        cfg["post_center_limit_range"], [0.0] * C, thr, pre_max, post_max, label_offset=label_offset)
    cnt = cnt.cpu().tolist()
    total = 0
    for b in range(B):
        gb = torch.cat([det_box[b * C + c, :cnt[b * C + c]] for c in range(C)]).cpu()
        gs = torch.cat([det_score[b * C + c, :cnt[b * C + c]] for c in range(C)]).cpu()
        gl = torch.cat([det_label[b * C + c, :cnt[b * C + c]] for c in range(C)]).cpu()
        w = want[b]
        assert gb.shape == w["box3d_lidar"].shape, (gb.shape, w["box3d_lidar"].shape)
        assert torch.equal(gl, w["label_preds"] + label_offset)
        assert torch.allclose(gs, w["scores"], atol=1e-6)
        assert torch.allclose(gb, w["box3d_lidar"], atol=1e-5, rtol=1e-6)
        total += gb.shape[0]
    return total


def test_postprocess_sparse_peaks():
    cfg = _test_cfg()
    n = run_and_compare(_fake_preds(2, 24, 20, 2, 11), 2, 1, cfg, 1000, 83, label_offset=1)
    assert n > 20
    n = run_and_compare(_fake_preds(3, 17, 33, 1, 12), 1, 0, cfg, 1000, 83)
    assert n > 20


def test_postprocess_heavy_overlap_and_truncation():
    cfg = _test_cfg()
    n_all = run_and_compare(clustered_preds(2, 24, 20, 2, 21), 2, 1, cfg, 1000, 83)
    n_cut = run_and_compare(clustered_preds(2, 24, 20, 2, 21), 2, 1, cfg, 40, 2)       # pre_max / post_max truncation
    assert n_cut == 2 * 2 * 2 and n_all > n_cut


def test_detector_eval_forward_matches_oracle_predict():
    """model.eval(); model(example) -> {token: detections}: the det3d eval contract (single_stage.py:47-59), checked
    against the oracle's predict applied to the model's own head outputs."""
    tasks = [["car"], ["truck", "construction_vehicle"]]
    cfg = synth.tiny_config(128, tasks)
    torch.manual_seed(1)
    model = modules.build_pillarnext_b(cfg).cuda().eval()
    with torch.no_grad():
        for t, task in enumerate(model.head.tasks):                       # spread the heat-map logits so a few hundred pass
            task.hm[3].bias.fill_(-1.5)
            task.hm[3].weight.mul_(6.0)
    tcfg = dict(post_center_limit_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], score_threshold=0.1,
                out_size_factor=[4, 4], voxel_size=cfg["voxel_size"][:2], pc_range=cfg["pc_range"][:2],
                nms=dict(nms_iou_threshold=[[0.2], [0.2, 0.2]], nms_pre_max_size=32, nms_post_max_size=10))
    model.post_processing = tcfg
    ex = synth.make_batch([0, 1], 3000, cfg, n_boxes=10, sweeps=10)
    exg = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in ex.items() if k in ("points", "token")}
    exg["token"] = ["f0", "f1"]
    with torch.no_grad():
        preds = model._forward(exg)
        dets = model(exg)
    pcpu = [{k: v.detach().float().cpu().contiguous() for k, v in pd.items()} for pd in preds]
    for t, pd in enumerate(pcpu):                     # kept sets are only comparable away from the IoU threshold
        boxes, hm, _ = P.decode(pd, 4, tcfg["voxel_size"], tcfg["pc_range"])
        sc, lb = hm.max(-1)
        for b in range(2):
            for c in range(hm.shape[-1]):
                m = (sc[b] > 0.1) & (lb[b] == c)
                top = sc[b][m].sort(descending=True)[1][:32]
                if not screen(boxes[b][m][top][:, [0, 1, 2, 3, 4, 5, 8]], 0.2, margin=1e-5) or \
                        sc[b][m][top].unique().numel() != top.numel():
                    pytest.skip("model output sits on the NMS threshold / has tied scores for this seed")
    want = P.predict(pcpu, [1, 2], tcfg, [[0.0], [0.0, 0.0]], tokens=["f0", "f1"])
    assert sorted(dets.keys()) == ["f0", "f1"]
    for w in want:
        g = dets[w["token"]]
        assert not g["box3d_lidar"].is_cuda
        assert g["box3d_lidar"].shape == w["box3d_lidar"].shape and w["box3d_lidar"].shape[0] > 3
        assert torch.equal(g["label_preds"], w["label_preds"])
        assert torch.allclose(g["scores"], w["scores"], atol=1e-6)
        assert torch.allclose(g["box3d_lidar"], w["box3d_lidar"], atol=1e-5, rtol=1e-6)


def test_postprocess_waymo_pre_max_4096():
    """The reference's Waymo configs use nms_pre_max_size 4096 (configs/experiments/waymo_det_pp18_aspp_iou_car_sp.yaml
    post_processing): 4096 candidates of one class in one frame go through the mask + on-GPU sweep (removed-set words
    spread over lanes x 4 slots) and must match the oracle's greedy NMS.  post_max = 4096 so the sweep walks the whole
    candidate list (about 200 suppressions happen past candidate 2048).  The CPU side prefilters pairs by centre distance
    (disjoint boxes have IoU exactly 0) before the exact oracle IoU; the seed keeps every evaluated pair 1e-4 away from
    the threshold."""
    import numpy as np
    cfg = _test_cfg()
    B, H, W, C = 1, 96, 96, 1
    g = torch.Generator().manual_seed(77)
    pd = _fake_preds(B, H, W, C, 31)
    n = H * W
    pd["hm"] = torch.linspace(-2.0, 3.0, n)[torch.randperm(n, generator=g)].view(B, C, H, W)      # distinct scores
    pd["dim"] = torch.randn(B, 3, H, W, generator=g) * 0.3 - 1.3                                    # ~0.3 m boxes on 0.3 m cells
    boxes, hm, iou = P.decode(pd, cfg["out_size_factor"][0], cfg["voxel_size"], cfg["pc_range"])
    thr = 0.25
    sc = hm[0, :, 0]
    pcr = torch.tensor(cfg["post_center_limit_range"])
    m = (sc > cfg["score_threshold"]) & (boxes[0][:, :3] >= pcr[:3]).all(1) & (boxes[0][:, :3] <= pcr[3:]).all(1)
    assert int(m.sum()) > 4096, int(m.sum())
    order = sc[m].sort(descending=True)[1][:4096]
    assert sc[m][order].unique().numel() == 4096, "tied scores: change the seed"
    b7 = boxes[0][m][order][:, [0, 1, 2, 3, 4, 5, 8]].contiguous().numpy().astype(np.float32)
    rad = 0.5 * np.sqrt(b7[:, 3] ** 2 + b7[:, 4] ** 2)
    removed = np.zeros(len(b7), dtype=bool)
    keep, late = [], 0
    for i in range(len(b7)):
        if removed[i]:
            continue
        keep.append(i)
        d = np.hypot(b7[i + 1:, 0] - b7[i, 0], b7[i + 1:, 1] - b7[i, 1])
        for j in np.nonzero((d < rad[i + 1:] + rad[i]) & ~removed[i + 1:])[0] + i + 1:
            v = float(P.iou_bev(b7[i], b7[j]))
            assert abs(v - thr) > 1e-4, "test input sits on the NMS threshold: change the seed"
            if v > thr:
                removed[j] = True
                late += int(j > 2048)
    assert late > 50 and 3000 < len(keep) < 4096          # suppressions past word 32 of the removed-set
    out = to_rows(pd).cuda()
    det_box, det_score, det_label, cnt = ops.det_postprocess(
        out, B, H, W, C, OFFS7, cfg["out_size_factor"][0], cfg["voxel_size"], cfg["pc_range"], cfg["score_threshold"],
        cfg["post_center_limit_range"], [0.0], [thr], 4096, 4096)
    assert int(cnt[0]) == len(keep), (int(cnt[0]), len(keep))
    sel = torch.tensor(keep)
    assert torch.allclose(det_box[0, :len(keep)].cpu(), boxes[0][m][order][sel], atol=1e-5, rtol=1e-6)
    assert torch.allclose(det_score[0, :len(keep)].cpu(), sc[m][order][sel], atol=1e-6)
