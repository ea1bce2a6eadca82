"""The greedy velocity tracker (track.py) and the CLEAR-MOT metric (evaluate_waymo_tracking.py) through their host
twins, CPU only: hand-built sequences with known answers, the host twins against oracle/track_oracle.py on seeded
random sequences, and WaymoDataset(tracking=True) on an info tree of oracle/reader_fixtures.py."""
import numpy as np
import pytest

from oracle import track_fixtures as TF
from oracle import track_oracle as O
from pillarnext_b200 import evaluate_waymo_tracking as EWT
from pillarnext_b200 import track as TR

CLASSES = ["vehicle", "pedestrian", "cyclist"]
DIMS = [(4.5, 2.0, 1.6), (0.8, 0.8, 1.8), (1.8, 0.7, 1.6)]


def random_sequences(seed, n_seq=3, n_frames=6, n_obj=6, fp=2):
    """(detections, frames, gts) of n_seq sequences: objects of random class moving at constant global velocity, seen
    by an ego whose pose turns and drives; each object labelled with probability 0.9 (0, 3 or 50 points) and detected
    with probability 0.85 (noisy centre and velocity, the velocity in the sensor frame), plus fp random detections per
    frame.  Timestamps are 0.1 s apart with jitter."""
    g = np.random.default_rng(seed)
    dets, frames, gts = {}, {}, {}
    for s in range(n_seq):
        objs = []
        for _ in range(n_obj):
            c = int(g.integers(0, 3))
            objs.append((c, g.uniform(-40, 40, 2), g.normal(0, 5, 2) * (c == 0) + g.normal(0, 1, 2), g.uniform(-3, 3)))
        yaw0, t0 = g.uniform(-np.pi, np.pi), int(g.integers(10 ** 15, 2 * 10 ** 15))
        for f in range(n_frames):
            ts = t0 + 100000 * f + int(g.integers(-500, 500))
            tok = "ctx%d-%d" % (s, ts)
            a = yaw0 + 0.01 * f
            T = np.eye(4)
            T[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
            T[:3, 3] = [100 + 1.0 * f, -50, 0.2]
            Ti = np.linalg.inv(T)
            b, names, ids, npts, db, ds, dl = [], [], [], [], [], [], []
            for o, (c, p0, v, yaw) in enumerate(objs):
                pl, vl = Ti[:2, :2] @ (p0 + v * 0.1 * f) + Ti[:2, 3], Ti[:2, :2] @ v
                box = [pl[0], pl[1], 0.0, *DIMS[c], vl[0], vl[1], yaw]
                if g.uniform() < 0.9:
                    b.append(box)
                    names.append(CLASSES[c])
                    ids.append("o%d" % o)
                    npts.append(int(g.choice([0, 3, 50])))
                if g.uniform() < 0.85:
                    n = list(box)
                    n[0] += g.normal(0, 0.15)
                    n[1] += g.normal(0, 0.15)
                    n[6] += g.normal(0, 0.3)
                    n[7] += g.normal(0, 0.3)
                    db.append(n)
                    ds.append(float(g.choice([0.3, 0.5, g.uniform()])))
                    dl.append(c)
            for _ in range(fp):
                db.append([*g.uniform(-40, 40, 2), 0.0, 2.0, 2.0, 1.5, 0.0, 0.0, 0.0])
                ds.append(g.uniform())
                dl.append(int(g.integers(0, 3)))
            frames[tok] = dict(sequence="ctx%d" % s, timestamp=ts, pose=T)
            dets[tok] = dict(box3d_lidar=np.array(db, np.float32).reshape(-1, 9), scores=np.array(ds, np.float32),
                             label_preds=np.array(dl, np.int64))
            gts[tok] = dict(boxes=np.array(b, np.float32).reshape(-1, 9), names=names, ids=ids,
                            num_points=np.array(npts, np.int64), sequence="ctx%d" % s, timestamp=ts)
    return dets, frames, gts


def frames_of(n, seq="s", dt=100000):
    return {"%s-%d" % (seq, 1000000 + dt * f): dict(sequence=seq, timestamp=1000000 + dt * f, pose=np.eye(4))
            for f in range(n)}


def det(rows, label=0):
    """rows of (x, y, vx, vy, score) -> one frame's detections of class `label` (a 4.5 x 2 x 1.6 box at yaw 0)."""
    b = np.array([[x, y, 0.0, 4.5, 2.0, 1.6, vx, vy, 0.0] for x, y, vx, vy, _ in rows], np.float32).reshape(-1, 9)
    return dict(box3d_lidar=b, scores=np.array([r[4] for r in rows], np.float32),
                label_preds=np.full(len(rows), label, np.int64))


def ids_both(dets, frames, **kw):
    """tracking ids from the host twin, checked equal to the oracle's; token -> list."""
    got = TR.track(dets, frames, CLASSES, host=True, **kw)
    want = O.track(dets, frames, CLASSES, **kw)
    for t in dets:
        np.testing.assert_array_equal(got[t]["tracking_id"], want[t], err_msg=t)
    return {t: got[t]["tracking_id"].tolist() for t in dets}


def test_birth_coast_death_and_revival_as_a_new_id():
    frames = frames_of(11)
    toks = list(frames)
    dets = {t: det([]) for t in toks}
    # a car moving at 10 m/s: seen in frames 0-1, missed 2-4 (3 misses, coasting), seen again in 5 (same track), missed
    # 6-9 (4 misses > max_age 3: dropped), seen in 10 (a new track)
    for f in (0, 1, 5, 10):
        dets[toks[f]] = det([(1.0 * f, 0.0, 10.0, 0.0, 0.9)])
    ids = ids_both(dets, frames, max_age=3)
    assert [ids[toks[f]] for f in (0, 1, 5, 10)] == [[0], [0], [0], [1]]
    # a static car that does not move with the detection's velocity claim is lost to the distance gate
    dets2 = {toks[0]: det([(0.0, 0.0, 0.0, 0.0, 0.9)]), toks[1]: det([(2.5, 0.0, 0.0, 0.0, 0.9)])}
    assert ids_both(dets2, frames) == {toks[0]: [0], toks[1]: [1]}


def test_ties_in_score_and_distance_and_min_score():
    frames = frames_of(2)
    t0, t1 = list(frames)
    # two tracks at x = -1 and x = +1 (ids 0, 1); in frame 1 one detection at x = 0 is equally far from both: the older
    # track (id 0) takes it; two detections of equal score at the same place: the lower index is visited first
    dets = {t0: det([(-1.0, 0.0, 0, 0, 0.8), (1.0, 0.0, 0, 0, 0.8)]),
            t1: det([(0.0, 0.0, 0, 0, 0.5), (0.0, 0.0, 0, 0, 0.5), (20.0, 0.0, 0, 0, 0.05)])}
    ids = ids_both(dets, frames, min_score=0.1)
    assert ids[t0] == [0, 1]
    assert ids[t1] == [0, 1, -1]                          # index 0 takes id 0 (tie to the older), index 1 id 1


def test_ids_are_consecutive_per_sequence_in_birth_order_over_classes():
    frames = dict(frames_of(2, "a"), **frames_of(2, "b"))
    ta, tb = [t for t in frames if t.startswith("a")], [t for t in frames if t.startswith("b")]
    mixed = det([(0, 0, 0, 0, 0.9), (30, 0, 0, 0, 0.8)])
    mixed["label_preds"] = np.array([1, 0], np.int64)     # a pedestrian first by index, a vehicle second
    dets = {ta[0]: mixed, ta[1]: det([(50, 0, 0, 0, 0.9)]), tb[0]: det([(0, 0, 0, 0, 0.9)])}
    ids = ids_both(dets, frames)
    assert ids[ta[0]] == [1, 0]                           # frame 0: the vehicle (class 0) is born before the pedestrian
    assert ids[ta[1]] == [2] and ids[tb[0]] == [0]


def gt_frame(rows, seq, ts):
    """rows of (x, y, id, num_points) -> one frame's vehicle ground truth."""
    b = np.array([[x, y, 0.0, 4.5, 2.0, 1.6, 0.0, 0.0, 0.0] for x, y, _, _ in rows], np.float32).reshape(-1, 9)
    return dict(boxes=b, names=["vehicle"] * len(rows), ids=[r[2] for r in rows],
                num_points=np.array([r[3] for r in rows], np.int64), sequence=seq, timestamp=ts)


def tracked(rows):
    """rows of (x, y, score, tracking id) -> one frame's tracked vehicle detections."""
    d = det([(x, y, 0, 0, s) for x, y, s, _ in rows])
    d["tracking_id"] = np.array([r[3] for r in rows], np.int64)
    return d


def mot_both(gts, tracks):
    got = EWT.waymo_tracking_metrics(gts, tracks, CLASSES, num_score_cutoffs=1, host=True)
    want = O.tracking_metrics(gts, tracks, CLASSES, num_score_cutoffs=1)
    assert_metrics_close(got, want, 1e-12)
    return got["per_class"]["vehicle"]


def assert_metrics_close(got, want, tol):
    for k in ("mMOTA_L1", "mMOTP_L1", "mMOTA_L2", "mMOTP_L2"):
        assert np.isclose(got[k], want[k], atol=tol, equal_nan=True), (k, got[k], want[k])
    for name, res in want["per_class"].items():
        for k, v in res.items():
            assert np.isclose(got["per_class"][name][k], v, atol=tol, equal_nan=True), (name, k, got["per_class"][name][k], v)


def test_a_crossing_counts_exactly_one_mismatch():
    gts = {"s-1": gt_frame([(0, 0, "A", 50), (10, 0, "B", 50)], "s", 1),
           "s-2": gt_frame([(0, 0, "A", 50), (10, 0, "B", 50)], "s", 2)}
    # frame 2: B's track (id 1) lands on A, B is missed
    tracks = {"s-1": tracked([(0, 0, 0.9, 0), (10, 0, 0.9, 1)]), "s-2": tracked([(0.1, 0, 0.9, 1)])}
    r = mot_both(gts, tracks)
    assert r["n_gt_L1"] == 4 and r["mismatch_L1"] == 0.25 and r["miss_L1"] == 0.25 and r["fp_L1"] == 0.0
    assert r["MOTA_L1"] == 0.5


def test_carry_over_wins_over_a_higher_iou_newcomer():
    gts = {"s-1": gt_frame([(0, 0, "A", 50)], "s", 1), "s-2": gt_frame([(0, 0, "A", 50)], "s", 2)}
    # frame 2: the old track is 0.4 m off (IoU ~0.82), a new track 0.05 m off (IoU ~0.98): the old id is kept
    tracks = {"s-1": tracked([(0, 0, 0.9, 0)]), "s-2": tracked([(0.05, 0, 0.95, 7), (0.4, 0, 0.6, 0)])}
    r = mot_both(gts, tracks)
    assert r["mismatch_L1"] == 0.0 and r["fp_L1"] == 0.5 and r["miss_L1"] == 0.0
    iou_kept = 1 - 2 * r["MOTP_L1"]                       # frame 1's pair is exact: MOTP = (0 + (1 - IoU)) / 2
    assert abs(iou_kept - 4.1 / 4.9) < 1e-5


def test_a_level_2_box_is_ignored_at_level_1():
    gts = {"s-1": gt_frame([(0, 0, "A", 50), (10, 0, "B", 3), (20, 0, "C", 0)], "s", 1)}
    tracks = {"s-1": tracked([(0, 0, 0.9, 0), (10, 0, 0.9, 1), (20, 0, 0.9, 2)])}
    r = mot_both(gts, tracks)
    assert (r["n_gt_L1"], r["n_gt_L2"]) == (1, 2)
    assert r["MOTA_L1"] == 1.0 and r["fp_L1"] == 0.0      # the matches to B (L2) and C (0 points) are not FPs
    assert r["MOTA_L2"] == 1.0


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_host_twins_equal_the_oracle_on_random_sequences(seed):
    dets, frames, gts = random_sequences(seed)
    tracks = TR.track(dets, frames, CLASSES, host=True, min_score=0.2, max_age=2)
    want = O.track(dets, frames, CLASSES, min_score=0.2, max_age=2)
    for t in dets:
        np.testing.assert_array_equal(tracks[t]["tracking_id"], want[t])
    got = EWT.waymo_tracking_metrics(gts, tracks, CLASSES, num_score_cutoffs=5, host=True)
    assert_metrics_close(got, O.tracking_metrics(gts, tracks, CLASSES, num_score_cutoffs=5), 1e-12)


def test_bad_inputs_raise():
    frames = frames_of(2)
    t0 = list(frames)[0]
    with pytest.raises(ValueError, match="max_dist"):
        TR.track({t0: det([])}, frames, ["truck"], host=True)
    with pytest.raises(ValueError, match="without a frame"):
        TR.track({"x-1": det([])}, frames, CLASSES, host=True)
    dup = {"s-1": dict(sequence="s", timestamp=5, pose=np.eye(4)), "s-2": dict(sequence="s", timestamp=5, pose=np.eye(4))}
    with pytest.raises(ValueError, match="two frames"):
        TR.track({}, dup, CLASSES, host=True)
    gts = {"s-1": gt_frame([(0, 0, "A", 50)], "s", 1)}
    del gts["s-1"]["ids"]
    with pytest.raises(ValueError, match="ids"):
        EWT.waymo_tracking_metrics(gts, {}, CLASSES, host=True)


def waymo_tracking_tree(root):
    """oracle/track_fixtures.write_waymo_sequences: two sequences of four frames in which the objects persist and move."""
    cfg = dict(tasks=[["vehicle"], ["pedestrian", "cyclist"]], pc_range=[-76.8, -76.8, -5.0, 76.8, 76.8, 3.0],
               voxel_size=[0.075, 0.075, 8], intensity_max=255.0, xy_extent=76.8, z_range=[-5.0, 3.0])
    return TF.write_waymo_sequences(root, [3, 4], cfg, length=4)


def test_waymo_dataset_ground_truth_and_tracking(tmp_path):
    from det3d.datasets.waymo.waymo import WaymoDataset
    root = str(tmp_path)
    infos = waymo_tracking_tree(root)
    off = WaymoDataset("waymo_infos_val.pkl", root, nsweeps=1)
    on = WaymoDataset("waymo_infos_val.pkl", root, nsweeps=1, tracking=True)
    g_off, g_on = off.ground_truth(), on.ground_truth()
    assert set(next(iter(g_off.values()))) == {"boxes", "names", "num_points"}
    for info in infos:
        g = g_on[info["token"]]
        assert g["sequence"] == info["token"].split("-")[0] and g["timestamp"] == int(info["token"].split("-")[1])
        assert g["ids"] == [o["id"] for o in info["objects"]]
        np.testing.assert_array_equal(g["pose"], info["pose"])
    # every object detected where it is, with its velocity: one track per object, no miss, FP or mismatch
    dets = {}
    for info in infos:
        objs = info["objects"]
        dets[info["token"]] = dict(box3d_lidar=np.array([o["box"] for o in objs], np.float32).reshape(-1, 9),
                                   scores=np.linspace(0.9, 0.5, len(objs)).astype(np.float32),
                                   label_preds=np.array([CLASSES.index(o["label"]) for o in objs], np.int64))
    tracks = TR.track(dets, g_on, CLASSES, host=True)
    for info in infos[1:4]:
        np.testing.assert_array_equal(tracks[info["token"]]["tracking_id"], tracks[infos[0]["token"]]["tracking_id"])
    got = EWT.waymo_tracking_metrics(g_on, tracks, CLASSES, host=True)
    assert_metrics_close(got, O.tracking_metrics(g_on, tracks, CLASSES), 1e-12)
    for name, r in got["per_class"].items():
        if r["n_gt_L2"]:
            assert r["MOTA_L2"] == 1.0 and r["mismatch_L2"] == 0.0 and r["MOTP_L2"] < 1e-5, (name, r)
    # the ids of two objects swapped from the third frame of the first sequence on: one mismatch each, once
    swapped = {t: dict(d) for t, d in tracks.items()}
    for info in infos[2:4]:
        tid = swapped[info["token"]]["tracking_id"].copy()
        tid[[0, 1]] = tid[[1, 0]]
        swapped[info["token"]]["tracking_id"] = tid
    got = EWT.waymo_tracking_metrics(g_on, swapped, CLASSES, host=True)
    want = O.tracking_metrics(g_on, swapped, CLASSES)
    assert_metrics_close(got, want, 1e-12)
    c0, c1 = infos[0]["objects"][0]["label"], infos[0]["objects"][1]["label"]
    n_mism = sum(got["per_class"][c]["mismatch_L2"] * got["per_class"][c]["n_gt_L2"] for c in {c0, c1})
    assert round(n_mism) == 2


def test_synthetic_sequences(tmp_path):
    from pillarnext_b200 import scenes
    cfg = dict(tasks=[["vehicle"], ["pedestrian", "cyclist"]], pc_range=[-76.8, -76.8, -5.0, 76.8, 76.8, 3.0],
               voxel_size=[0.075, 0.075, 8], intensity_max=255.0, xy_extent=76.8, z_range=[-5.0, 3.0])
    one = scenes.SyntheticSceneDataset(cfg, 3, seed0=40, n_points=2000, metric="waymo")
    for i in range(3):                                    # sequence_length 1: the frames of make_scene, as before
        pts, boxes, names = scenes.make_scene(40 + i, cfg, 2000, 12)
        assert one[i]["token"] == "scene_%d" % (40 + i)
        np.testing.assert_array_equal(one[i]["points"], pts)
        np.testing.assert_array_equal(one[i]["gt_boxes_raw"], boxes)
    seq = scenes.SyntheticSceneDataset(cfg, 8, seed0=40, n_points=2000, metric="waymo_tracking", sequence_length=4)
    gts = seq.ground_truth()
    toks = list(gts)
    assert toks[0] == "seq40-1000000000" and toks[5] == "seq44-1000100000" and seq[5]["token"] == toks[5]
    np.testing.assert_array_equal(seq[0]["points"], scenes.make_scene(40, cfg, 2000, 12)[0])
    # each object's global centre (the first frame's sensor frame) moves by its velocity label, 0.1 s per frame
    g0 = gts[toks[0]]
    for k in range(1, 4):
        g = gts[toks[k]]
        T, b = g["pose"], g["boxes"].astype(np.float64)
        assert g["ids"] == g0["ids"] and g["sequence"] == "seq40" and g["timestamp"] == 1000000000 + 100000 * k
        np.testing.assert_allclose(b[:, :2] @ T[:2, :2].T + T[:2, 3], g0["boxes"][:, :2] + 0.1 * k * g0["boxes"][:, 6:8],
                                   atol=1e-4)
        np.testing.assert_allclose(b[:, 6:8] @ T[:2, :2].T, g0["boxes"][:, 6:8], atol=1e-5)
    with pytest.raises(ValueError, match="sequence_length"):
        scenes.SyntheticSceneDataset(cfg, 8, nsweeps=3, sequence_length=4)
