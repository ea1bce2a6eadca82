"""nuScenes tracking metric (evaluate_nuscenes_tracking) through the host twins of pnx_eval_pairs_center and
pnx_eval_mot_center, against the sequential oracle (oracle/nusc_track_oracle.py): hand-built cases for each rule, and
seeded nuScenes-shaped scenes."""
import json
import math
import os

import numpy as np
import pytest

from oracle import nusc_track_fixtures as NF
from oracle import nusc_track_oracle as O
from pillarnext_b200 import evaluate_nuscenes_tracking as ENT
from pillarnext_b200 import ops

NAMES = ["car", "truck", "bus", "barrier"]


def scene(frames, name="scene", t0=0):
    """frames: [(boxes [(x, y, id, class)], dets [(x, y, score, tracking id, class)])] -> (gts, tracks)."""
    gts, tracks = {}, {}
    for f, (boxes, dets) in enumerate(frames):
        tok = "%s_%d" % (name, f)
        b = np.zeros((len(boxes), 9), np.float32)
        b[:, 3:6] = (4.0, 2.0, 1.5)
        b[:, :2] = [(x, y) for x, y, *_ in boxes] if boxes else np.zeros((0, 2))
        gts[tok] = dict(boxes=b, names=[c for *_, c in boxes], ids=[i for _, _, i, _ in boxes],
                        num_points=np.full(len(boxes), 10, np.int64), sequence=name, timestamp=t0 + 500000 * f)
        d = np.zeros((len(dets), 9), np.float32)
        d[:, 3:6] = (4.0, 2.0, 1.5)
        d[:, :2] = [(x, y) for x, y, *_ in dets] if dets else np.zeros((0, 2))
        tracks[tok] = dict(box3d_lidar=d, scores=np.array([s for _, _, s, _, _ in dets], np.float32),
                           label_preds=np.array([NAMES.index(c) for *_, c in dets], np.int64),
                           tracking_id=np.array([i for _, _, _, i, _ in dets], np.int64))
    return gts, tracks


def lowest_cutoff_counts(gts, tracks, name="car"):
    """Product counts (TP, IDS, FRAG, sum d) of `name` at its lowest reached cutoff, over all scenes."""
    pk = ENT.pack(gts, tracks, NAMES)
    res = ENT.run_host(pk, gts)
    c = pk["tracking_names"].index(name)
    n = res["counts"].sum(0)[c, 0]
    return int(n[0]), int(n[1]), int(n[2]), float(res["dist"].sum(0)[c, 0])


def same(a, b, tol=1e-9):
    if isinstance(a, dict):
        assert set(a) == set(b), (sorted(a), sorted(b))
        for k in a:
            same(a[k], b[k], tol)
        return
    if isinstance(a, float) and math.isnan(a):
        assert isinstance(b, float) and math.isnan(b), (a, b)
    elif isinstance(a, float) or isinstance(b, float):
        assert abs(a - b) <= tol, (a, b)
    else:
        assert a == b, (a, b)


def both(gts, tracks):
    got = ENT.nuscenes_tracking_metrics(gts, tracks, NAMES, host=True)
    same(got, O.tracking_metrics(gts, tracks, NAMES))
    return got


def test_carry_over_keeps_the_old_match_although_a_closer_detection_exists():
    gts, tracks = scene([([(0, 0, "a", "car")], [(0.5, 0, 0.95, 7, "car")]),
                         ([(0, 0, "a", "car")], [(1.5, 0, 0.9, 7, "car"), (0.1, 0, 0.92, 8, "car")])])
    both(gts, tracks)
    assert lowest_cutoff_counts(gts, tracks) == (2, 0, 0, 2.0)
    # without the carry-over the closer detection would take the box: one identity switch
    assert O.run(O.load(gts, tracks, NAMES)[1], "car", 0.9, ("no_carry_over",))[3] == 1


def test_an_identity_switch():
    gts, tracks = scene([([(0, 0, "a", "car")], [(0.5, 0, 0.9, 1, "car")]),
                         ([(0, 0, "a", "car")], [(0.5, 0, 0.9, 2, "car")]),
                         ([(0, 0, "a", "car")], [(0.5, 0, 0.9, 2, "car")])])
    m = both(gts, tracks)
    assert lowest_cutoff_counts(gts, tracks)[:3] == (3, 1, 0)
    assert m["per_class"]["car"]["IDS"] == 1 and m["IDS"] == 1


def test_a_fragmentation():
    gts, tracks = scene([([(0, 0, "a", "car")], [(0.5, 0, 0.9, 1, "car")]),
                         ([(0, 0, "a", "car")], []),
                         ([(0, 0, "a", "car")], []),
                         ([(0, 0, "a", "car")], [(0.5, 0, 0.9, 1, "car")]),
                         ([(9, 9, "b", "car")], [(9, 9, 0.9, 3, "car")])])   # b's first match is no fragmentation
    m = both(gts, tracks)
    assert lowest_cutoff_counts(gts, tracks)[:3] == (3, 0, 1)
    assert m["per_class"]["car"]["FRAG"] == 1 and m["per_class"]["car"]["FN"] == 2


def test_the_pair_boundary_is_strictly_below_two_metres():
    below = float(np.nextafter(np.float32(2.0), np.float32(0.0)))
    gts, tracks = scene([([(0, 0, "a", "car")], [(2.0, 0, 0.9, 1, "car")]),
                         ([(0, 0, "a", "car")], [(below, 0, 0.9, 1, "car")]),
                         ([(10, 0, "b", "car")], [(10, 2.0, 0.9, 2, "car")])])
    both(gts, tracks)
    assert lowest_cutoff_counts(gts, tracks) == (1, 0, 0, below)
    pk = ENT.pack(gts, tracks, NAMES)
    start, e_det, e_box, e_dist = ops.eval_pairs_center_host(pk["det_boxes"], pk["order"], pk["seg_start"],
                                                             pk["seg_count"], pk["gt_boxes"], pk["gt_classes"], pk["C"],
                                                             ENT.PAIR_DIST)
    assert len(e_det) == 1 and e_dist[0] == np.float32(below)


def test_score_and_distance_ties_follow_the_tie_rule():
    # equal scores and distances: the lower-index detection (tracking id 5) takes the box, so id 6 later switches
    gts, tracks = scene([([(0, 0, "a", "car")], [(1, 0, 0.5, 5, "car"), (-1, 0, 0.5, 6, "car")]),
                         ([(0, 0, "a", "car")], [(1, 0, 0.5, 6, "car")])])
    both(gts, tracks)
    assert lowest_cutoff_counts(gts, tracks)[:2] == (2, 1)
    # one detection equidistant from two boxes takes the lower box index, and the other detection the remaining box
    gts, tracks = scene([([(0, 0, "a", "car"), (2, 0, "b", "car")], [(1, 0, 0.9, 1, "car"), (2.5, 0, 0.8, 2, "car")])])
    both(gts, tracks)
    assert lowest_cutoff_counts(gts, tracks) == (2, 0, 0, 1.5)


def test_cardinality_comes_before_distance():
    # two matches (sum 3.8 m) beat the single closest match
    gts, tracks = cardinality_case()
    both(gts, tracks)
    tp, _, _, d = lowest_cutoff_counts(gts, tracks)
    assert tp == 2 and abs(d - 3.8) < 1e-6
    frames = O.load(gts, tracks, NAMES)[1]
    assert O.run(frames, "car", 0.8, ("not_cardinality_first",))[0] == 1


def test_unreached_recalls_count_zero_and_two_metres():
    gts, tracks = scene([([(0, 0, "a", "car"), (10, 0, "b", "car"), (20, 0, "c", "car"), (30, 0, "d", "car")],
                          [(0.5, 0, 0.9, 1, "car")])])
    m = both(gts, tracks)["per_class"]["car"]
    r = ENT.RECALLS[np.ceil(ENT.RECALLS * 4) <= 1]
    assert len(r) == 7
    motar = np.maximum(0.0, 1.0 - (3 - (1 - r) * 4) / (r * 4))
    assert abs(m["AMOTA"] - motar.sum() / 40) < 1e-12
    assert abs(m["AMOTP"] - (7 * 0.5 + 33 * 2.0) / 40) < 1e-12
    assert m["recall"] == 0.25 and m["FN"] == 3 and m["FP"] == 0


def test_classes_without_ground_truth_or_detections():
    gts, tracks = scene([([(0, 0, "a", "car"), (10, 0, "t", "truck")], [(0.5, 0, 0.9, 1, "car"), (30, 0, 0.9, 2, "bus")])])
    m = both(gts, tracks)
    bus, truck = m["per_class"]["bus"], m["per_class"]["truck"]
    assert bus["n_gt"] == 0 and all(math.isnan(v) for k, v in bus.items() if k != "n_gt")
    assert truck["AMOTA"] == 0.0 and truck["AMOTP"] == 2.0 and truck["FN"] == 1
    assert m["FN"] == 1 and abs(m["AMOTA"] - (m["per_class"]["car"]["AMOTA"] + 0.0) / 2) < 1e-12


def test_untracked_classes_are_ignored():
    base = [([(0, 0, "a", "car")], [(0.5, 0, 0.9, 1, "car")]), ([(0, 0, "a", "car")], [(0.5, 0, 0.9, 1, "car")])]
    extra = [(b + [(5, 5, "x", "barrier")], d + [(5, 5, 0.99, 9, "barrier"), (0.2, 0, 0.95, 4, "barrier")])
             for b, d in base]
    plain = ENT.nuscenes_tracking_metrics(*scene(base), NAMES, host=True)
    mixed = both(*scene(extra))
    assert "barrier" not in mixed["per_class"]
    same(plain, mixed, tol=0.0)


def test_bad_inputs_raise():
    gts, tracks = scene([([(0, 0, "a", "car")], [(0.5, 0, 0.9, 1, "car")])])
    with pytest.raises(ValueError, match="ids"):
        ENT.nuscenes_tracking_metrics({t: {k: v for k, v in g.items() if k != "ids"} for t, g in gts.items()}, tracks,
                                      NAMES, host=True)
    with pytest.raises(ValueError, match="without ground truth"):
        ENT.nuscenes_tracking_metrics(gts, dict(tracks, other=next(iter(tracks.values()))), NAMES, host=True)
    with pytest.raises(ValueError, match="no tracking class"):
        ENT.nuscenes_tracking_metrics(gts, {}, ["barrier"], host=True)


def seeded(seed):
    dets, _, gts = NF.nusc_val_shaped(seed, n_scenes=3, n_frames=8, max_dup=30, max_fp=10)
    return gts, ENT.track_and_score(gts, dets, NF.CLASSES, host=True)[0]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_host_twins_equal_the_oracle_on_seeded_scenes(seed):
    gts, tracks = seeded(seed)
    got = ENT.nuscenes_tracking_metrics(gts, tracks, NF.CLASSES, host=True)
    want = O.tracking_metrics(gts, tracks, NF.CLASSES)
    same(got, want)
    assert set(got["per_class"]) == set(ENT.tracking_classes(NF.CLASSES))
    assert got["IDS"] > 0 and got["FRAG"] > 0 and got["FP"] > 0 and got["FN"] > 0


def cardinality_case():
    """Detection 1 is 0.1 m from box a and 1.9 m from box b, detection 2 pairs box a only (1.9 m)."""
    return scene([([(0, 0, "a", "car"), (2.0, 0, "b", "car")], [(0.1, 0, 0.9, 1, "car"), (-1.9, 0, 0.8, 2, "car")])])


@pytest.mark.parametrize("defect", O.DEFECTS)
def test_each_oracle_defect_changes_the_result(defect):
    # the seeded scenes rarely hold a detection between two close boxes at a reached cutoff: the cardinality rule is
    # shown on the hand-built case
    if defect == "not_cardinality_first":
        gts, tracks, names = *cardinality_case(), NAMES
    else:
        gts, tracks = seeded(0)
        names = NF.CLASSES
    got = ENT.nuscenes_tracking_metrics(gts, tracks, names, host=True)
    same(got, O.tracking_metrics(gts, tracks, names))
    with pytest.raises(AssertionError):
        same(got, O.tracking_metrics(gts, tracks, names, defects=(defect,)))


def test_track_and_score_hands_only_tracking_classes_to_the_tracker():
    dets, _, gts = NF.nusc_val_shaped(3, n_scenes=2, n_frames=4, max_dup=5, max_fp=5)
    tracks, _ = ENT.track_and_score(gts, dets, NF.CLASSES, host=True)
    for t, d in tracks.items():
        names = {NF.CLASSES[int(c)] for c in d["label_preds"]}
        assert names <= set(ENT.TRACKING_NAMES)
        assert len(d["tracking_id"]) == sum(NF.CLASSES[int(c)] in ENT.TRACKING_NAMES for c in dets[t]["label_preds"])


NUSC_TASKS = [["car"], ["truck", "construction_vehicle"], ["bus", "trailer"], ["barrier"], ["motorcycle", "bicycle"],
              ["pedestrian", "traffic_cone"]]
SEEDS = [3, 4, 5, 6]


def nusc_tracking_tree(root):
    """oracle/reader_fixtures.write_nusc's tree of four frames plus the devkit's sample table: frames 3, 4 in scene
    "sA", 5, 6 in "sB", 0.5 s apart (the scenes are unrelated make_scene draws, so few tracks continue).  -> (the dataset's class names, infos, detections: each labelled box, with its
    class, moved 0.1 m)."""
    from oracle import reader_fixtures as RF
    cfg = dict(tasks=NUSC_TASKS, pc_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], voxel_size=[0.1, 0.1, 8],
               intensity_max=255.0, xy_extent=50.4, z_range=[-5.0, 3.0])
    infos, _ = RF.write_nusc(root, SEEDS, cfg, n_points=2000, n_boxes=12, nsweeps=1)
    os.makedirs(os.path.join(root, "v1.0-trainval"))
    samples = [{"token": "scene_%d" % s, "scene_token": "sA" if s < 5 else "sB",
                "timestamp": 1533000000000000 + 500000 * ((s - 3) % 2), "prev": "", "next": ""} for s in SEEDS]
    with open(os.path.join(root, "v1.0-trainval", "sample.json"), "w") as f:
        json.dump(samples, f)
    names = [n for t in NUSC_TASKS for n in t]
    dets = {}
    for info in infos:
        b = np.asarray(info["gt_boxes"], np.float32).copy()
        b[:, 0] += 0.1
        dets[info["token"]] = dict(box3d_lidar=b, scores=np.linspace(0.9, 0.3, len(b)).astype(np.float32),
                                   label_preds=np.array([names.index(n) for n in info["gt_names"]], np.int64))
    return names, infos, dets


def test_tracking_json_round_trips_on_the_reader_fixture(tmp_path):
    from det3d.datasets.nuscenes import NuScenesDataset
    from det3d.datasets.nuscenes.nusc import lidar_to_global
    root = str(tmp_path)
    names, infos, dets = nusc_tracking_tree(root)
    info_name = "infos_train_10sweeps_withvelo_filterZero.pkl"
    ds = NuScenesDataset(info_name, root, nsweeps=1, class_names=NUSC_TASKS, tracking=True)
    frames = ds.frames(list(dets))
    assert frames["scene_4"]["sequence"] == "sA" and frames["scene_4"]["timestamp"] == 1533000000500000
    path = tmp_path / "out_tracking.json"
    tracks = ds.write_tracks(dets, path, host=True)
    out = json.load(open(path))
    assert out["meta"] == {"use_camera": False, "use_lidar": True, "use_radar": False, "use_map": False,
                           "use_external": False}
    n_tracked = 0
    for info in infos:
        t = info["token"]
        T = lidar_to_global(info)
        annos = out["results"][t]
        d = tracks[t]
        assert len(annos) == len(d["tracking_id"])
        for a, b, lab, i, s in zip(annos, d["box3d_lidar"], d["label_preds"], d["tracking_id"], d["scores"]):
            assert set(a) == {"sample_token", "translation", "size", "rotation", "velocity", "tracking_id",
                              "tracking_name", "tracking_score"}
            assert a["sample_token"] == t and a["tracking_id"] == str(int(i)) and a["tracking_score"] == float(s)
            assert a["tracking_name"] == names[int(lab)] and a["tracking_name"] in ENT.TRACKING_NAMES
            back = np.linalg.solve(T[:3, :3], np.array(a["translation"]) - T[:3, 3])
            np.testing.assert_allclose(back, np.asarray(b[:3], np.float64), atol=1e-6)
            assert a["size"] == [float(b[4]), float(b[3]), float(b[5])]
            n_tracked += 1
        want = sum(names[int(c)] in ENT.TRACKING_NAMES for c in dets[t]["label_preds"])
        assert len(annos) == want
    assert n_tracked > 0


def test_synthetic_sequence_interval_and_nds_tracking_metric():
    from pillarnext_b200 import scenes
    cfg = dict(tasks=NUSC_TASKS, pc_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], voxel_size=[0.1, 0.1, 8],
               intensity_max=255.0, xy_extent=50.4, z_range=[-5.0, 3.0])
    base = scenes.SyntheticSceneDataset(cfg, 4, seed0=40, n_points=1500, metric="nds", sequence_length=2)
    same_ = scenes.SyntheticSceneDataset(cfg, 4, seed0=40, n_points=1500, metric="nds", sequence_length=2,
                                         sequence_interval=0.1)
    half = scenes.SyntheticSceneDataset(cfg, 4, seed0=40, n_points=1500, metric="nds_tracking", sequence_length=2,
                                        sequence_interval=0.5)
    g0, g1, g5 = base.ground_truth(), same_.ground_truth(), half.ground_truth()
    assert list(g0) == list(g1)                      # the default 0.1 s leaves every frame and token as it was
    for t in g0:
        np.testing.assert_array_equal(g0[t]["points"], g1[t]["points"])
        np.testing.assert_array_equal(g0[t]["boxes"], g1[t]["boxes"])
    toks = list(g5)
    assert toks[1] == "seq40-1000500000" and g5[toks[1]]["timestamp"] - g5[toks[0]]["timestamp"] == 500000
    a, b = g5[toks[0]], g5[toks[1]]
    T = b["pose"]
    np.testing.assert_allclose(b["boxes"][:, :2].astype(np.float64) @ T[:2, :2].T + T[:2, 3],
                               a["boxes"][:, :2] + 0.5 * a["boxes"][:, 6:8], atol=1e-4)
    with pytest.raises(ValueError, match="nds_tracking"):
        scenes.SyntheticSceneDataset(cfg, 4, metric="nds_tracking")
    with pytest.raises(ValueError, match="sequence_interval"):
        scenes.SyntheticSceneDataset(cfg, 4, sequence_length=2, sequence_interval=0.0)
