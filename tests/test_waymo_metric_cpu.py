"""Waymo-style AP / APH (pillarnext_b200/evaluate_waymo.py) without a GPU: closed-form cases through the sequential
oracle (oracle/waymo_metric_oracle.py) and through the product's host path (the pnx_eval_*_host twins of
csrc/det_eval.cu + the same numpy curve code), and the host twins against the oracle on crowded seeded scenes."""
import math
import os

import numpy as np
import pytest

from oracle import gts_oracle, waymo_fixtures
from oracle import waymo_metric_oracle as O
from pillarnext_b200 import evaluate_waymo as EW

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def box_points(box, n):
    """n points strictly inside box (x, y, z, dx, dy, dz, yaw), on a fixed pattern."""
    u = (np.arange(n) + 0.5) / max(n, 1) - 0.5
    loc = np.stack([u * 0.8 * box[3], np.roll(u, 1) * 0.8 * box[4], np.roll(u, 2) * 0.8 * box[5]], 1)
    c, s = math.cos(box[6]), math.sin(box[6])
    return np.stack([loc[:, 0] * c - loc[:, 1] * s + box[0], loc[:, 0] * s + loc[:, 1] * c + box[1], loc[:, 2] + box[2]],
                    1).astype(np.float32)


def frame(boxes, names, npts):
    boxes = np.asarray(boxes, np.float32).reshape(-1, 7)
    pts = [box_points(b, k) for b, k in zip(boxes, npts)] + [np.array([[200.0, 200.0, 0.0]], np.float32)]
    return {"boxes": boxes, "names": list(names), "points": np.concatenate(pts)}


def dets(boxes, scores, labels):
    b = np.asarray(boxes, np.float32).reshape(-1, 7)
    b9 = np.zeros((len(b), 9), np.float32)
    b9[:, :6], b9[:, 8] = b[:, :6], b[:, 6]
    return {"box3d_lidar": b9, "scores": np.asarray(scores, np.float32), "label_preds": np.asarray(labels, np.int64)}


def host_metrics(gts, detections, classes, iou_thresholds=None):
    pk = EW.pack(gts, detections, classes, iou_thresholds)
    counts, match, _, heading = EW.run_host(pk)
    return EW.score(pk, counts, match, heading, classes)


def both(gts, detections, classes, iou_thresholds=None):
    return O.waymo_metrics(gts, detections, classes, iou_thresholds), host_metrics(gts, detections, classes, iou_thresholds)


CAR = [0.0, 0.0, 0.85, 4.0, 2.0, 1.7, 0.3]
CAR2 = [10.0, 5.0, 0.85, 4.2, 2.0, 1.6, -1.0]
PED = [5.0, -5.0, 0.9, 0.8, 0.8, 1.8, 0.0]
CLS = ["vehicle", "pedestrian"]


def test_perfect_detections():
    gts = {"a": frame([CAR, PED], ["vehicle", "pedestrian"], [20, 12]), "b": frame([CAR2], ["vehicle"], [30])}
    d = {"a": dets([CAR, PED], [0.9, 0.8], [0, 1]), "b": dets([CAR2], [0.7], [0])}
    for r in both(gts, d, CLS):
        for k in ("mAP_L1", "mAPH_L1", "mAP_L2", "mAPH_L2"):
            assert abs(r[k] - 100.0) < 1e-9, (k, r)
        assert r["per_class"]["vehicle"]["n_gt_L1"] == 2 and r["per_class"]["pedestrian"]["n_gt_L2"] == 1


@pytest.mark.parametrize("dyaw,aph", [(math.pi, 0.0), (math.pi / 2, 50.0)])
def test_heading_error(dyaw, aph):
    sq = [0.0, 0.0, 0.9, 0.8, 0.8, 1.8, 0.2]                    # square footprint: IoU 1 under a quarter turn
    turned = list(sq)
    turned[6] += dyaw
    gts = {"a": frame([sq], ["pedestrian"], [20])}
    for r in both(gts, {"a": dets([turned], [0.9], [0])}, ["pedestrian"]):
        assert abs(r["mAP_L2"] - 100.0) < 1e-9 and abs(r["mAP_L1"] - 100.0) < 1e-9
        assert abs(r["mAPH_L2"] - aph) < 1e-4 and abs(r["mAPH_L1"] - aph) < 1e-4


def test_iou_just_under_threshold_is_one_fp_and_one_fn():
    s = 4.0 * 0.301 / 1.699                                     # IoU (4 - s) / (4 + s) = 0.699 (same size, shifted in x)
    box = [0.0, 0.0, 0.85, 4.0, 2.0, 1.7, 0.0]
    shifted = [s, 0.0, 0.85, 4.0, 2.0, 1.7, 0.0]
    gts = {"a": frame([box], ["vehicle"], [20])}
    d = {"a": dets([shifted], [0.9], [0])}
    pk = EW.pack(gts, d, ["vehicle"])
    _, match, iou, _ = EW.run_host(pk)
    assert match.tolist() == [-1] and 0.69 < iou[0] < 0.7
    for r in both(gts, d, ["vehicle"]):
        assert r["mAP_L2"] == 0.0 and r["per_class"]["vehicle"]["n_gt_L2"] == 1


def test_duplicate_detection_is_one_tp_and_one_fp():
    gts = {"a": frame([CAR], ["vehicle"], [20])}
    d = {"a": dets([CAR, CAR], [0.6, 0.9], [0, 0])}
    pk = EW.pack(gts, d, ["vehicle"])
    _, match, _, _ = EW.run_host(pk)
    assert match.tolist() == [-1, 0]                            # the higher score takes the box
    cheap = {"a": dets([CAR2, CAR], [0.9, 0.6], [0, 0])}        # an FP ranked first halves the precision of the TP
    for r in both(gts, d, ["vehicle"]):
        assert abs(r["mAP_L2"] - 100.0) < 1e-9
    for r in both(gts, cheap, ["vehicle"]):
        assert abs(r["mAP_L2"] - 50.0) < 1e-9


def test_level_2_box_is_ignored_at_level_1():
    gts = {"a": frame([CAR, CAR2], ["vehicle", "vehicle"], [20, 3])}
    d = {"a": dets([CAR2, CAR], [0.9, 0.5], [0, 0])}
    for r in both(gts, d, ["vehicle"]):
        pc = r["per_class"]["vehicle"]
        assert (pc["n_gt_L1"], pc["n_gt_L2"]) == (1, 2)
        assert abs(pc["AP_L1"] - 100.0) < 1e-9 and abs(pc["AP_L2"] - 100.0) < 1e-9


def test_zero_point_box_is_ignored():
    gts = {"a": frame([CAR, CAR2], ["vehicle", "vehicle"], [20, 0])}
    d = {"a": dets([CAR2, CAR], [0.9, 0.5], [0, 0])}
    for r in both(gts, d, ["vehicle"]):
        pc = r["per_class"]["vehicle"]
        assert (pc["n_gt_L1"], pc["n_gt_L2"]) == (1, 1)
        assert abs(pc["AP_L1"] - 100.0) < 1e-9 and abs(pc["AP_L2"] - 100.0) < 1e-9


def test_no_detections_scores_zero():
    gts = {"a": frame([CAR], ["vehicle"], [20])}
    for r in both(gts, {}, ["vehicle"]):
        assert r["mAP_L1"] == 0.0 and r["mAPH_L2"] == 0.0


def test_class_without_ground_truth_is_nan_and_left_out():
    gts = {"a": frame([CAR], ["vehicle"], [20])}
    d = {"a": dets([CAR, PED], [0.9, 0.95], [0, 1])}
    for r in both(gts, d, CLS):
        assert math.isnan(r["per_class"]["pedestrian"]["AP_L2"]) and math.isnan(r["per_class"]["pedestrian"]["APH_L1"])
        assert abs(r["mAP_L2"] - 100.0) < 1e-9


def test_unknown_class_needs_a_threshold():
    gts = {"a": frame([CAR], ["sign"], [20])}
    d = {"a": dets([CAR], [0.9], [0])}
    for fn in (O.waymo_metrics, host_metrics):
        with pytest.raises(ValueError):
            fn(gts, d, ["sign"])
    for r in both(gts, d, ["sign"], {"sign": 0.6}):
        assert abs(r["mAP_L2"] - 100.0) < 1e-9


def test_host_twins_match_the_oracle_on_crowded_scenes():
    gts, det, classes = waymo_fixtures.make_frames(11, 3, n_points=4000, n_labels=(14, 10, 4), fp_per_class=(10, 8, 4),
                                                   extent=6.0)
    pk = EW.pack(gts, det, classes)
    counts, match, iou, _ = EW.run_host(pk)
    from det3d.datasets.pipelines.sample_ops import libm_trig
    n_match = 0
    off = 0
    thr = EW.class_thresholds(classes)
    for f, t in enumerate(gts):
        g, d = gts[t], det[t]
        want_counts = gts_oracle.points_in_boxes(g["points"][:, :3], g["boxes"], libm_trig(g["boxes"][:, 8])).sum(0)
        assert np.array_equal(counts[f, :len(g["boxes"])], want_counts)
        k = len(d["scores"])
        wm, wi = O.match_frame(g["boxes"], g["names"], d["box3d_lidar"], d["scores"], d["label_preds"], classes, thr)
        assert np.array_equal(match[off:off + k], wm)
        np.testing.assert_allclose(iou[off:off + k], wi, rtol=1e-5, atol=1e-7)
        n_match += int((wm >= 0).sum())
        off += k
    assert n_match > 20 and (counts > 0).sum() > 20 and ((counts >= 1) & (counts <= 5)).sum() > 0
    r_o, r_h = O.waymo_metrics(gts, det, classes), EW.score(pk, counts, match, EW.run_host(pk)[3], classes)
    for k in ("mAP_L1", "mAP_L2"):
        assert abs(r_o[k] - r_h[k]) < 1e-9
    for k in ("mAPH_L1", "mAPH_L2"):
        assert abs(r_o[k] - r_h[k]) < 1e-6


def test_waymo_experiment_composes():
    from pillarnext_b200 import hydra_lite
    cfg = hydra_lite.main(os.path.join(ROOT, "configs", "experiments"), "synth_det_pp18_aspp_waymo", [])
    assert [list(t) for t in cfg.model.head.tasks] == [["vehicle"], ["pedestrian", "cyclist"]]
    assert list(cfg.model.head.common_heads.iou) == [1, 2]
    assert [list(r) for r in cfg.model.head.rectifier] == [[0.68], [0.71, 0.65]]
    assert [list(r) for r in cfg.model.post_processing.nms.nms_iou_threshold] == [[0.7], [0.2, 0.25]]
    val = hydra_lite.instantiate(cfg.data.val_dataset)
    assert val.metric == "waymo" and val.class_names == ["vehicle", "pedestrian", "cyclist"]
    gt = val.ground_truth()
    assert all(g["points"].shape[1] == 5 for g in gt.values())
    train = hydra_lite.instantiate(cfg.data.train_dataset)
    assert train.metric == "nuscenes"
