"""nuScenes detection score (pillarnext_b200/evaluate_nuscenes.py) without a GPU: closed-form cases through the sequential
oracle (oracle/nds_oracle.py) and through the product's host path (the pnx_eval_*_host twins of csrc/det_eval.cu + the
same numpy filters and curves), and the host path against the oracle on seeded nuScenes-shaped frames."""
import math

import numpy as np
import pytest

from oracle import nds_fixtures
from oracle import nds_oracle as O
from pillarnext_b200 import evaluate_nuscenes as EN


def box(x, y, size=(4.0, 2.0, 1.5), vel=(0.0, 0.0), yaw=0.3):
    return [x, y, 0.75, *size, *vel, yaw]


def frame(boxes, names, npts=None, **extra):
    b = np.asarray(boxes, np.float32).reshape(-1, 9)
    g = {"boxes": b, "names": list(names), "num_points": np.full(len(b), 10) if npts is None else np.asarray(npts)}
    g.update(extra)
    return g


def dets(boxes, scores, labels):
    return {"box3d_lidar": np.asarray(boxes, np.float32).reshape(-1, 9), "scores": np.asarray(scores, np.float32),
            "label_preds": np.asarray(labels, np.int64)}


def host_metrics(gts, detections, classes, class_range=None):
    pk = EN.pack(gts, detections, classes, class_range)
    counts, match = EN.run_host(pk)
    return EN.score(pk, counts, match)


def both(gts, detections, classes, class_range=None):
    return O.nuscenes_metrics(gts, detections, classes, class_range), host_metrics(gts, detections, classes, class_range)


def host_match(gts, detections, classes):
    pk = EN.pack(gts, detections, classes)
    return EN.run_host(pk)[1]


def test_one_true_positive_at_30_cm():
    gts = {"a": frame([box(10.0, 0.0)], ["car"])}
    d = {"a": dets([box(10.0, 0.3)], [0.9], [0])}
    for r in both(gts, d, ["car"]):
        pc = r["per_class"]["car"]
        assert abs(pc["ATE"] - 0.3) < 1e-6 and pc["ASE"] < 1e-12 and pc["AOE"] == 0 and pc["AVE"] == 0 and pc["AAE"] == 0
        assert abs(pc["AP"] - 100.0) < 1e-9 and pc["n_gt"] == 1
        assert abs(r["NDS"] - 100.0 * (5 + 0.7 + 4) / 10) < 1e-5


def test_scale_error_is_one_minus_the_aligned_volume_iou():
    gts = {"a": frame([box(10.0, 0.0, size=(4.0, 2.0, 1.5))], ["car"])}
    d = {"a": dets([box(10.0, 0.0, size=(5.0, 1.5, 1.5))], [0.9], [0])}
    inter = 4.0 * 1.5 * 1.5
    want = 1.0 - inter / (4.0 * 2.0 * 1.5 + 5.0 * 1.5 * 1.5 - inter)
    for r in both(gts, d, ["car"]):
        assert abs(r["per_class"]["car"]["ASE"] - want) < 1e-12


@pytest.mark.parametrize("name,want", [("car", math.pi), ("barrier", 0.0)])
def test_yaw_off_by_pi(name, want):
    gts = {"a": frame([box(10.0, 0.0, yaw=0.3)], [name])}
    d = {"a": dets([box(10.0, 0.0, yaw=0.3 + math.pi)], [0.9], [0])}
    for r in both(gts, d, [name]):
        assert abs(r["per_class"][name]["AOE"] - want) < 1e-6


def test_traffic_cone_and_barrier_nan_rules():
    classes = ["car", "barrier", "traffic_cone"]
    gts = {"a": frame([box(10.0, 0.0), box(0.0, 10.0), box(-10.0, 0.0)], classes)}
    d = {"a": dets([box(10.0, 0.0), box(0.0, 10.0), box(-10.0, 0.0)], [0.9, 0.8, 0.7], [0, 1, 2])}
    for r in both(gts, d, classes):
        cone, bar = r["per_class"]["traffic_cone"], r["per_class"]["barrier"]
        assert math.isnan(cone["AAE"]) and math.isnan(cone["AVE"]) and math.isnan(cone["AOE"])
        assert not math.isnan(cone["ATE"]) and not math.isnan(cone["ASE"])
        assert math.isnan(bar["AAE"]) and math.isnan(bar["AVE"]) and bar["AOE"] == 0.0
        assert r["mAAE"] == 0.0 and r["mAOE"] == 0.0 and abs(r["NDS"] - 100.0) < 1e-9


def test_class_without_ground_truth_counts_as_zero():
    gts = {"a": frame([box(10.0, 0.0)], ["car"])}
    d = {"a": dets([box(10.0, 0.0), box(0.0, 5.0)], [0.9, 0.8], [0, 1])}
    for r in both(gts, d, ["car", "pedestrian"]):
        ped = r["per_class"]["pedestrian"]
        assert ped["n_gt"] == 0 and ped["AP"] == 0.0
        assert all(ped[k] == 1.0 for k in ("ATE", "ASE", "AOE", "AVE", "AAE"))
        assert abs(r["mAP"] - 50.0) < 1e-9 and all(r[k] == 0.5 for k in ("mATE", "mASE", "mAOE", "mAVE", "mAAE"))
        assert abs(r["NDS"] - 50.0) < 1e-9


def test_detection_exactly_2_m_away_is_a_false_positive_at_2_m_only():
    gts = {"a": frame([box(10.0, 0.0)], ["car"])}
    d = {"a": dets([box(12.0, 0.0)], [0.9], [0])}
    assert host_match(gts, d, ["car"])[:, 0].tolist() == [-1, -1, -1, 0]
    for r in both(gts, d, ["car"]):
        pc = r["per_class"]["car"]
        assert (pc["AP@0.5"], pc["AP@1.0"], pc["AP@2.0"]) == (0.0, 0.0, 0.0) and abs(pc["AP@4.0"] - 100.0) < 1e-9
        assert abs(pc["AP"] - 25.0) < 1e-9 and pc["ATE"] == 1.0                # no TP at 2 m: the errors are 1


def test_range_limit_is_strict():
    gts = {"a": frame([box(50.0, 0.0), box(0.0, -49.875), box(18.0, 24.0)], ["car", "car", "pedestrian"])}
    d = {"a": dets([box(50.0, 0.0), box(0.0, -49.875), box(18.0, 24.0)], [0.9, 0.8, 0.7], [0, 0, 1])}
    for r in both(gts, d, ["car", "pedestrian"]):
        assert r["per_class"]["car"]["n_gt"] == 1 and abs(r["per_class"]["car"]["AP"] - 100.0) < 1e-9
        assert r["per_class"]["pedestrian"]["n_gt"] == 1
    for r in both(gts, d, ["car", "pedestrian"], {"pedestrian": 30.0}):   # 30 m from the origin: out
        assert r["per_class"]["pedestrian"]["n_gt"] == 0
    cone = {"a": frame([box(30.0, 0.0)], ["traffic_cone"])}
    for r in both(cone, {"a": dets([box(29.75, 0.0)], [0.9], [0])}, ["traffic_cone"]):
        assert r["per_class"]["traffic_cone"]["n_gt"] == 0


def test_unknown_class_needs_a_range():
    """A class outside the nuScenes ten has no attribute: every attr_err is NaN, so its AAE is the all-NaN 1."""
    gts = {"a": frame([box(10.0, 0.0)], ["sign"])}
    d = {"a": dets([box(10.0, 0.0)], [0.9], [0])}
    for fn in (O.nuscenes_metrics, host_metrics):
        with pytest.raises(ValueError):
            fn(gts, d, ["sign"])
    for r in both(gts, d, ["sign"], {"sign": 20.0}):
        assert abs(r["per_class"]["sign"]["AP"] - 100.0) < 1e-9 and r["per_class"]["sign"]["AAE"] == 1.0


def box_points(b, n):
    """n points within 0.3 m of the centre of box b (yaw 0, at least 0.6 m on every side)."""
    u = np.linspace(-0.3, 0.3, n)
    return np.stack([b[0] + u, b[1] - u, b[2] + 0.5 * u], 1).astype(np.float32)


def test_detection_near_a_zero_point_box_is_a_false_positive():
    b0, b1 = box(10.0, 0.0, yaw=0.0), box(20.0, 0.0, yaw=0.0)
    pts = np.concatenate([box_points(b1, 7), np.array([[100.0, 100.0, 0.0]], np.float32)])
    gts = {"a": frame([b0, b1], ["car", "car"]) | {"points": pts}}
    del gts["a"]["num_points"]
    d = {"a": dets([b0, b1], [0.9, 0.5], [0, 0])}
    pk = EN.pack(gts, d, ["car"])
    counts, match = EN.run_host(pk)
    assert counts[0, :2].tolist() == [0, 7] and match[:, 0].tolist() == [-1] * 4 and match[:, 1].tolist() == [1] * 4
    # curve: FP then TP -> precision 0, 1/2 at recall 0, 1; P(r) = r / 2
    p = np.arange(101) / 200.0
    want = 100.0 * np.mean(np.maximum(p[11:] - 0.1, 0)) / 0.9
    for r in both(gts, d, ["car"]):
        assert r["per_class"]["car"]["n_gt"] == 1 and abs(r["per_class"]["car"]["AP"] - want) < 1e-9


def test_score_tie_visits_the_later_detection_first():
    gts = {"a": frame([box(10.0, 0.0)], ["car"])}
    d = {"a": dets([box(10.5, 0.0), box(10.0, 0.25)], [0.8, 0.8], [0, 0])}
    assert host_match(gts, d, ["car"])[2].tolist() == [-1, 0]
    for r in both(gts, d, ["car"]):
        assert r["per_class"]["car"]["ATE"] == 0.25
    # across frames: position follows the order of the frames in `detections`
    gts2 = {"a": frame([box(10.0, 0.0)], ["car"]), "b": frame([box(10.0, 0.0)], ["car"])}
    d2 = {"b": dets([box(10.5, 0.0)], [0.8], [0]), "a": dets([box(10.0, 0.25)], [0.8], [0])}
    # at 0.5 m: TP then FP at recall 0.5, so precision 1 below recall 0.5 and 1/2 at it (the last point of a repeated x)
    for r in both(gts2, d2, ["car"]):
        assert abs(r["per_class"]["car"]["AP@0.5"] - 100.0 * (39 * 0.9 + 0.4) / 90 / 0.9) < 1e-9
    pk = EN.pack(gts2, d2, ["car"])
    assert pk["det_frames"][pk["visit"]].tolist() == [0, 1]    # frame "a" came second in `detections`: visited first


def test_distance_tie_goes_to_the_lower_box_index():
    same = (4.0, 2.0, 1.5)
    other = (4.5, 2.0, 1.5)
    for boxes in ([box(10.0, 0.0, size=same), box(12.0, 0.0, size=other)],
                  [box(12.0, 0.0, size=same), box(10.0, 0.0, size=other)]):
        gts = {"a": frame(boxes, ["car", "car"])}
        d = {"a": dets([box(11.0, 0.0, size=same)], [0.9], [0])}
        assert host_match(gts, d, ["car"])[:, 0].tolist() == [-1, -1, 0, 0]
        for r in both(gts, d, ["car"]):
            assert r["per_class"]["car"]["ASE"] < 1e-12 and r["per_class"]["car"]["ATE"] == 1.0


def test_all_nan_velocity_errors_give_ones():
    gts = {"a": frame([box(10.0, 0.0, vel=(float("nan"), 0.0))], ["car"])}
    d = {"a": dets([box(10.0, 0.0, vel=(1.0, 0.0))], [0.9], [0])}
    for r in both(gts, d, ["car"]):
        assert r["per_class"]["car"]["AVE"] == 1.0 and r["per_class"]["car"]["ATE"] == 0.0


def test_recall_below_11_percent_gives_error_one():
    gts = {"a": frame([box(10.0 + 3 * k, 0.0) for k in range(10)], ["car"] * 10)}
    d = {"a": dets([box(10.0, 0.3)], [0.9], [0])}
    for r in both(gts, d, ["car"]):
        pc = r["per_class"]["car"]
        assert pc["ATE"] == 1.0 and pc["AP"] == 0.0 and pc["AP@4.0"] == 0.0


def test_more_than_500_detections_raise():
    gts = {"a": frame([box(10.0, 0.0)], ["car"])}
    d = {"a": dets([box(100.0, 0.0)] * 501, np.full(501, 0.5), np.zeros(501))}    # all out of range: raises first
    for fn in (O.nuscenes_metrics, host_metrics):
        with pytest.raises(ValueError):
            fn(gts, d, ["car"])
    d = {"a": dets([box(100.0, 0.0)] * 500, np.full(500, 0.5), np.zeros(500))}
    for r in both(gts, d, ["car"]):
        assert r["mAP"] == 0.0


def test_missing_inputs_raise():
    with pytest.raises(ValueError):
        host_metrics({"a": {"boxes": np.zeros((1, 9), np.float32), "names": ["car"]}}, {}, ["car"])
    with pytest.raises(ValueError):
        host_metrics({"a": frame([box(10.0, 0.0)], ["car"])}, {"b": dets([box(10.0, 0.0)], [0.9], [0])}, ["car"])


ATTR_TABLE = {   # class: (at 0.1 m/s, at 0.3 m/s)
    "car": ("vehicle.parked", "vehicle.moving"), "truck": ("vehicle.parked", "vehicle.moving"),
    "trailer": ("vehicle.parked", "vehicle.moving"), "construction_vehicle": ("vehicle.parked", "vehicle.moving"),
    "bus": ("vehicle.parked", "vehicle.moving"), "bicycle": ("cycle.without_rider", "cycle.with_rider"),
    "motorcycle": ("cycle.without_rider", "cycle.with_rider"), "pedestrian": ("pedestrian.standing", "pedestrian.moving"),
    "barrier": ("cycle.with_rider", "cycle.with_rider"), "traffic_cone": ("cycle.with_rider", "cycle.with_rider"),
}


def test_attribute_derivation_for_every_class():
    classes = list(ATTR_TABLE)
    vocab = EN._Vocab()
    name_of = {v: k for k, v in vocab.codes.items()}
    for i, speed in enumerate((0.1, 0.3)):
        vel = np.array([[speed * 0.6, speed * 0.8]] * len(classes), np.float32)
        got = EN.derive_attributes(np.arange(len(classes)), vel, classes, vocab)
        for c, name in enumerate(classes):
            assert name_of[int(got[c])] == ATTR_TABLE[name][i], (name, speed)
            assert O.attribute(name, float(vel[c, 0]), float(vel[c, 1])) == ATTR_TABLE[name][i], (name, speed)
    # through the metric: a pedestrian labelled "pedestrian.moving" detected standing still is an attribute error
    gts = {"a": frame([box(5.0, 0.0, size=(0.7, 0.7, 1.8))], ["pedestrian"], attributes=["pedestrian.moving"])}
    for vel, aae in (((0.1, 0.0), 1.0), ((0.3, 0.0), 0.0)):
        d = {"a": dets([box(5.0, 0.0, size=(0.7, 0.7, 1.8), vel=vel)], [0.9], [0])}
        for r in both(gts, d, ["pedestrian"]):
            assert r["per_class"]["pedestrian"]["AAE"] == aae


def test_nds_formula_on_hand_set_errors():
    nan = float("nan")
    per_class = {"a": dict(AP=60.0, ATE=0.5, ASE=0.2, AOE=1.5, AVE=nan, AAE=0.1),
                 "b": dict(AP=40.0, ATE=nan, ASE=0.4, AOE=0.5, AVE=nan, AAE=0.3),
                 "c": dict(AP=20.0, ATE=1.5, ASE=0.0, AOE=1.0, AVE=nan, AAE=nan)}
    r = EN.summarize(per_class)
    assert abs(r["mAP"] - 40.0) < 1e-12
    assert abs(r["mATE"] - 1.0) < 1e-12 and abs(r["mASE"] - 0.2) < 1e-12 and abs(r["mAOE"] - 1.0) < 1e-12
    assert math.isnan(r["mAVE"]) and abs(r["mAAE"] - 0.2) < 1e-12
    # 5 x 0.4 + (1 - 1) + (1 - 0.2) + 0 + 0 (NaN) + (1 - 0.2), over 10
    assert abs(r["NDS"] - 100.0 * (2.0 + 0.8 + 0.8) / 10) < 1e-9


def assert_close(got, want, tol=1e-9):
    for k, v in want.items():
        if k == "per_class":
            for name, pc in v.items():
                assert_close(got[k][name], pc, tol)
            continue
        g = got[k]
        assert (math.isnan(v) and math.isnan(g)) or abs(g - v) <= tol, (k, g, v)


@pytest.mark.parametrize("kw", [dict(n_points=4000, extent=55.0), dict(n_points=None, with_attributes=True),
                                dict(n_points=3000, extent=10.0, n_labels=60), dict(n_points=None, tie_scores=False)])
def test_host_path_equals_the_oracle_on_fixture_frames(kw):
    gts, det, classes = nds_fixtures.make_frames(7, 4, fp_per_frame=80, **kw)
    want = O.nuscenes_metrics(gts, det, classes)
    pk = EN.pack(gts, det, classes)
    counts, match = EN.run_host(pk, point_budget=5000)
    got = EN.score(pk, counts, match)
    assert_close(got, want)
    assert (match[0] >= 0).sum() > 20 and (match[3] >= 0).sum() > (match[0] >= 0).sum()
    assert 5 < got["mAP"] < 95 and 5 < got["NDS"] < 95


def test_nds_experiment_composes():
    import os
    from pillarnext_b200 import hydra_lite
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = hydra_lite.main(os.path.join(root, "configs", "experiments"), "synth_det_pp18_aspp_nds", [])
    tasks = [list(t) for t in cfg.model.head.tasks]
    assert tasks == [["car"], ["truck", "construction_vehicle"], ["bus", "trailer"], ["barrier"], ["motorcycle", "bicycle"],
                     ["pedestrian", "traffic_cone"]]
    assert list(cfg.model.head.strides) == [2] * 6 and list(cfg.model.post_processing.out_size_factor) == [4] * 6
    assert [len(r) for r in cfg.model.head.rectifier] == [len(t) for t in tasks]
    assert [len(r) for r in cfg.model.post_processing.nms.nms_iou_threshold] == [len(t) for t in tasks]
    # at most 50 boxes per class leave the NMS: ten classes never exceed the 500-box cap
    assert cfg.model.post_processing.nms.nms_post_max_size * sum(len(t) for t in tasks) <= EN.MAX_BOXES_PER_SAMPLE
    val = hydra_lite.instantiate(cfg.data.val_dataset)
    assert val.metric == "nds" and val.class_names == [n for t in tasks for n in t]
    assert sorted(val.class_names) == sorted(EN.CLASS_RANGE)
    gt = val.ground_truth()
    assert all(g["points"].shape[1] == 5 for g in gt.values())
    assert hydra_lite.instantiate(cfg.data.train_dataset).metric == "nuscenes"
