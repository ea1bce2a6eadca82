"""The nuScenes and Waymo info-file readers (det3d.datasets: BaseDataset, NuScenesDataset, WaymoDataset, AssignLabel,
loader), CPU only, on the seeded trees of oracle/reader_fixtures.py.

* the reference's data nodes (shaped as its nusc_det / waymo_det configs compose them) instantiate this package's
  classes, and the import lines of the reference's tools/train.py and tools/test.py resolve;
* against tests/golden/ref_readers.npz (oracle/make_golden_readers.py: the reference's own readers, sampler,
  augmentation, AssignLabel and create_groundtruth_database on the same seeded trees): the reader records plus the host
  twins (accumulate_sweeps_host, gt_sample_host, global_aug_host) reproduce the reference's points and boxes to the bit
  for nuScenes with 10 sweeps, the sampler and the augmentation, for Waymo with 3 sweeps and drop_frames 0.5 and for
  Waymo with 1 sweep; the CBGS order; the 10-sweep nuScenes and the thinned Waymo databases (dbinfos and SHA-256 of
  every file); the reference's composed experiments instantiate these classes through tools/train.py's config path;
* waymo_metrics with "num_points" decides LEVEL_2 by the label's count, not the geometric one (against the oracle);
* scenes written to disk and read back give collated batches byte-identical to SyntheticSceneDataset + scenes.collate
  for the same seeds: nuScenes with 10 sweeps, the sampler and the augmentation; Waymo with 3 sweeps and drop_frames
  0.5; Waymo with 1 sweep.  Self-checks: a swapped no-label-zone sign, one sweep too few and a ring column left in
  each break the equality;
* CBGS draws the reference's np.random.choice;
* tools/create_gt_database.py --dataset NUSC / WAYMO writes the reference's records: objects cut from the accumulated
  frame with the numpy restatement of points_in_rbbox, Waymo's thinning;
* the nuScenes results JSON follows the devkit's quaternion path (Box.rotate / translate with the pose quaternions)
  within 1e-9, with the reference's names and attributes."""
import json
import os
import pickle
import sys

import numpy as np
import pytest
import torch

from oracle import reader_fixtures as RF
from oracle.gts_oracle import points_in_boxes
from pillarnext_b200 import hydra_lite, ops, scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NUSC_TASKS = [["car"], ["truck", "construction_vehicle"], ["bus", "trailer"], ["barrier"], ["motorcycle", "bicycle"],
              ["pedestrian", "traffic_cone"]]
WAYMO_TASKS = [["vehicle"], ["pedestrian", "cyclist"]]
AUG = {"rotation": {"_target_": "det3d.datasets.pipelines.augmentation.Rotation", "rotation": [-0.785, 0.785]},
       "scaling": {"_target_": "det3d.datasets.pipelines.augmentation.Scaling", "scale": [0.9, 1.1]},
       "translation": {"_target_": "det3d.datasets.pipelines.augmentation.Translation", "noise": 0.5},
       "flip": {"_target_": "det3d.datasets.pipelines.augmentation.Flip", "flip_prob": [0.5, 0.5]}}


def scene_cfg(tasks, half):
    return dict(tasks=tasks, pc_range=[-half, -half, -5.0, half, half, 3.0], voxel_size=[0.075, 0.075, 8],
                intensity_max=255.0, xy_extent=half, z_range=[-5.0, 3.0])


def centermap(tasks, half):
    return {"_target_": "det3d.datasets.pipelines.assign.AssignLabel", "gaussian_overlap": 0.1, "max_objs": 500,
            "min_radius": 2, "tasks": tasks, "pc_range": [-half, -half, -5.0, half, half, 3.0],
            "voxel_size": [0.075, 0.075, 8], "out_size_factor": [4] * len(tasks)}


def sampler_node(root, dbinfo, groups):
    return {"_target_": "det3d.datasets.pipelines.sample_ops.DataBaseSamplerV2", "_partial_": True, "root_path": root,
            "dbinfo_path": dbinfo, "groups": [groups],
            "db_prepor": {"filter_by_num": {"_target_": "det3d.datasets.pipelines.sample_ops.DBFilterByMinNumPoint",
                                            "min_gt_point_dict": {k: 5 for k in groups}}},
            "rate": 1.0, "gt_drop_percentage": 0, "gt_drop_max_keep_points": -1, "point_dim": 5}


def nusc_node(root, info, sampler=None, aug=None, label=True, **kw):
    node = {"_target_": "det3d.datasets.nuscenes.NuScenesDataset", "nsweeps": 10, "root_path": root, "info_path": info,
            "class_names": NUSC_TASKS, "loading_pipelines": ["load_pointcloud", "load_box3d"]}
    if label:
        node["prepare_label"] = {"centermap": centermap(NUSC_TASKS, 50.4)}
    if sampler:
        node["sampler"] = sampler
    if aug:
        node["augmentation"] = aug
    node.update(kw)
    return node


def waymo_node(root, info, nsweeps, drop_frames, label=True):
    node = {"_target_": "det3d.datasets.waymo.waymo.WaymoDataset", "nsweeps": nsweeps, "root_path": root,
            "info_path": info, "drop_frames": drop_frames, "loading_pipelines": ["load_pointcloud", "load_box3d"]}
    if label:
        node["prepare_label"] = {"centermap": centermap(WAYMO_TASKS, 76.8)}
    return node


def batches(ds, n, bs, seed):
    """Collated batches of frames 0 .. n - 1 with np.random seeded first (the draws of a single-process loader)."""
    np.random.seed(seed + 1)
    frames = [ds[i] for i in range(n)]
    return [scenes.collate(frames[i:i + bs]) for i in range(0, n, bs)]


def build(node, seed):
    np.random.seed(seed)                          # the sampler shuffles its class lists when it is built
    return hydra_lite.instantiate(node)


def assert_same_batches(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert sorted(g) == sorted(w)
        for k in w:
            if isinstance(w[k], torch.Tensor):
                assert g[k].dtype == w[k].dtype and g[k].shape == w[k].shape, k
                assert g[k].numpy().tobytes() == w[k].numpy().tobytes(), k
            else:
                assert g[k] == w[k], k


def same_batches(got, want):
    try:
        assert_same_batches(got, want)
    except AssertionError:
        return False
    return True


# ---------------------------------------------------------------------- trees
SEEDS = [3, 4, 5, 6]


@pytest.fixture(scope="module")
def nusc_tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("nusc"))
    cfg = scene_cfg(NUSC_TASKS, 50.4)
    infos, poses = RF.write_nusc(root, SEEDS, cfg, n_points=3000, n_boxes=14)
    import create_gt_database as tool
    tool.create_reader_database("NUSC", root, "infos_train_10sweeps_withvelo_filterZero.pkl", nsweeps=10, host=True)
    return root, cfg, infos, poses


@pytest.fixture(scope="module")
def waymo_tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("waymo"))
    cfg = scene_cfg(WAYMO_TASKS, 76.8)
    RF.write_waymo(root, SEEDS, cfg, n_points=3000, n_boxes=10, identity_pose=True)
    return root, cfg


@pytest.fixture(autouse=True, scope="module")
def _tools_on_path():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    yield
    sys.path.remove(os.path.join(ROOT, "tools"))


# ---------------------------------------------------------------------- drop-in
def test_reference_entry_point_imports_resolve():
    from det3d.datasets.loader.build_loader import build_dataloader           # tools/train.py:2
    from det3d.datasets.loader.collate import collate
    assert collate is scenes.collate and callable(build_dataloader)
    for target in ("det3d.datasets.nuscenes.NuScenesDataset", "det3d.datasets.waymo.waymo.WaymoDataset",
                   "det3d.datasets.pipelines.assign.AssignLabel"):
        mod, _, name = target.rpartition(".")
        assert isinstance(getattr(__import__(mod, fromlist=[name]), name), type)


def test_reference_data_nodes_instantiate_our_classes(nusc_tree, waymo_tree):
    from det3d.datasets.nuscenes import NuScenesDataset
    from det3d.datasets.waymo.waymo import WaymoDataset
    root = nusc_tree[0]
    train = build(nusc_node(root, "infos_train_10sweeps_withvelo_filterZero.pkl",
                            sampler_node(root, "dbinfos_train_10sweeps_withvelo.pkl", {"car": 2, "pedestrian": 2}), AUG,
                            resampling=True), 0)
    assert isinstance(train, NuScenesDataset) and train.sampler is not None and len(train.augmentations) == 4
    val = build({"_target_": "det3d.datasets.nuscenes.NuScenesDataset", "nsweeps": 10, "root_path": root,
                 "info_path": "infos_train_10sweeps_withvelo_filterZero.pkl", "class_names": NUSC_TASKS,
                 "loading_pipelines": ["load_pointcloud"]}, 0)
    rec = val[0]
    assert "annotations" not in rec and rec["gt_boxes_raw"].shape == (0, 9) and len(rec["sweeps"]["counts"]) == 9
    w = build(waymo_node(waymo_tree[0], "waymo_infos_train.pkl", 3, 0.5), 0)
    assert isinstance(w, WaymoDataset) and len(w) == len(SEEDS)


def test_assign_label_refuses_values_the_gpu_does_not_use():
    from det3d.datasets.pipelines.assign import AssignLabel
    node = centermap(NUSC_TASKS, 50.4)
    for key, bad in (("gaussian_overlap", 0.2), ("max_objs", 300), ("min_radius", 1)):
        with pytest.raises(ValueError, match="label assignment"):
            hydra_lite.instantiate(dict(node, **{key: bad}))
    a = hydra_lite.instantiate(node)
    assert isinstance(a, AssignLabel)
    res = a({"annotations": {"gt_boxes": np.ones((3, 9)), "gt_names": np.array(["bus", "ignore", "car"])}})
    assert res["gt_classes"].tolist() == [3, 10, 0] and res["gt_boxes_raw"].dtype == np.float32


# ---------------------------------------------------------------------- records = synthetic records
def synthetic(cfg, n_points, n_boxes, **kw):
    return scenes.SyntheticSceneDataset(cfg, len(SEEDS), seed0=SEEDS[0], n_points=n_points, n_boxes=n_boxes, **kw)


def test_nusc_batches_equal_the_synthetic_ones(nusc_tree):
    root, cfg, _, _ = nusc_tree
    smp = sampler_node(root, "dbinfos_train_10sweeps_withvelo.pkl", {"car": 6, "pedestrian": 5, "barrier": 4})
    got = batches(build(nusc_node(root, "infos_train_10sweeps_withvelo_filterZero.pkl", smp, AUG), 7), 4, 2, 7)
    np.random.seed(7)
    syn = synthetic(cfg, 3000, 14, augmentation=AUG, sampler=smp, root_path=root, nsweeps=10, min_distance=1.0)
    want = batches(syn, 4, 2, 7)
    assert want[0]["gts_classes"].ge(0).sum() > 0 and want[0]["sweep_points"].shape[0] > 0
    assert_same_batches(got, want)


@pytest.mark.parametrize("nsweeps,drop", [(3, 0.5), (1, 0.0)])
def test_waymo_batches_equal_the_synthetic_ones(waymo_tree, nsweeps, drop):
    root, cfg = waymo_tree
    got = batches(build(waymo_node(root, "waymo_infos_train.pkl", nsweeps, drop), 5), 4, 2, 5)
    syn = synthetic(cfg, 3000, 10, nsweeps=nsweeps, drop_frames=drop, min_distance=0.0)
    want = batches(syn, 4, 2, 5)
    assert ("sweep_points" in want[0]) == (nsweeps > 1)
    assert_same_batches(got, want)
    if nsweeps > 1:
        lens = np.concatenate([np.diff(b["sweep_offsets"].numpy()) for b in want])
        assert (lens == 0).any() and (lens > 0).any()                 # drop_frames dropped some sweeps, kept others


def test_self_checks_see_a_swapped_nlz_sign_a_missing_sweep_and_a_ring_column(waymo_tree, nusc_tree, monkeypatch):
    from det3d.datasets.nuscenes.nusc import NuScenesDataset
    from det3d.datasets.waymo.waymo import WaymoDataset
    root, cfg = waymo_tree
    want = batches(synthetic(cfg, 3000, 10, nsweeps=3, drop_frames=0.0, min_distance=0.0), 4, 2, 5)
    node = waymo_node(root, "waymo_infos_train.pkl", 3, 0.0)
    assert same_batches(batches(build(node, 5), 4, 2, 5), want)
    read = WaymoDataset.read_file

    def wrong_sign(self, path, timestamp=0):
        p = np.fromfile(os.path.join(self._root_path, path), dtype=np.float32).reshape(-1, 6)
        p = p[p[:, -1] == 1, :4]
        return np.concatenate([p, np.full((len(p), 1), np.float32(timestamp))], 1)
    monkeypatch.setattr(WaymoDataset, "read_file", wrong_sign)
    assert not same_batches(batches(build(node, 5), 4, 2, 5), want)
    monkeypatch.setattr(WaymoDataset, "read_file", read)
    assert not same_batches(batches(build(dict(node, nsweeps=2), 5), 4, 2, 5), want)
    nroot, ncfg, _, _ = nusc_tree
    nwant = batches(synthetic(ncfg, 3000, 14, nsweeps=10, min_distance=1.0), 4, 2, 9)
    nnode = nusc_node(nroot, "infos_train_10sweeps_withvelo_filterZero.pkl")
    assert same_batches(batches(build(nnode, 9), 4, 2, 9), nwant)
    monkeypatch.setattr(NuScenesDataset, "read_file", lambda self, path, num_point_feature=4: np.fromfile(
        os.path.join(self._root_path, path), dtype=np.float32).reshape(-1, 5)[:, [0, 1, 2, 4]])
    assert not same_batches(batches(build(nnode, 9), 4, 2, 9), nwant)


# ---------------------------------------------------------------------- CBGS
def test_cbgs_draws_np_random_choice_per_class(nusc_tree):
    root = nusc_tree[0]
    with open(os.path.join(root, "infos_train_10sweeps_withvelo_filterZero.pkl"), "rb") as fh:
        infos = pickle.load(fh)
    names = [n for t in NUSC_TASKS for n in t]
    present = sorted({n for i in infos for n in i["gt_names"]}, key=names.index)
    tasks = [[n] for n in present]
    np.random.seed(21)
    ds = hydra_lite.instantiate(nusc_node(root, "infos_train_10sweeps_withvelo_filterZero.pkl", label=False,
                                          class_names=tasks, resampling=True))
    # the reference's loop, with the infos' tokens for the dicts it draws
    np.random.seed(21)
    per = {n: [i["token"] for i in infos if n in set(i["gt_names"])] for n in present}
    total = sum(len(v) for v in per.values())
    want = []
    for n in present:
        k = int(len(per[n]) * ((1.0 / len(present)) / (len(per[n]) / total)))
        want += list(np.random.choice(np.array(per[n], dtype=object), k))
    assert [i["token"] for i in ds.infos] == want and len(want) > len(infos)


# ---------------------------------------------------------------------- ground-truth database
@pytest.mark.parametrize("dataset", ["NUSC", "WAYMO"])
def test_create_gt_database_writes_the_reference_records(nusc_tree, tmp_path, dataset):
    import create_gt_database as tool
    if dataset == "NUSC":
        root, info, nsweeps = nusc_tree[0], "infos_train_10sweeps_withvelo_filterZero.pkl", 10
    else:
        root, info, nsweeps = str(tmp_path), "waymo_infos_train.pkl", 3
        RF.write_waymo(root, list(range(20, 28)), scene_cfg(WAYMO_TASKS, 76.8), n_points=2000, n_boxes=10)
    dbinfos = tool.create_reader_database(dataset, root, info, nsweeps=nsweeps, host=True,
                                         db_path=os.path.join(str(tmp_path), "db"),
                                         dbinfo_path=os.path.join(str(tmp_path), "dbinfos.pkl"))
    with open(os.path.join(str(tmp_path), "dbinfos.pkl"), "rb") as fh:
        assert pickle.load(fh).keys() == dbinfos.keys()
    node = (nusc_node if dataset == "NUSC" else lambda r, i, label: waymo_node(r, i, 3, 0.0, label))(root, info,
                                                                                                    label=False)
    ds = hydra_lite.instantiate(dict(node, create_database=True))
    from det3d.datasets.pipelines.sample_ops import libm_trig
    group, seen = 0, {}
    for index in range(len(ds)):
        rec = ds[index]
        pts = tool.frame_points(rec, host=True)
        boxes, names = rec["annotations"]["gt_boxes"], rec["annotations"]["gt_names"]
        if dataset == "WAYMO":
            keep = ~(((index % 4 != 0) & (names == "vehicle")) | ((index % 2 != 0) & (names == "pedestrian")))
            boxes, names = boxes[keep], names[keep]
        inside = points_in_boxes(pts, boxes, libm_trig(boxes[:, 8]))
        for i, name in enumerate(names):
            rec_i = dbinfos[name][seen.get(name, 0)]
            seen[name] = seen.get(name, 0) + 1
            want = pts[inside[:, i]].copy()
            want[:, :3] -= boxes[i, :3]
            got = np.fromfile(os.path.join(str(tmp_path), "db", name, "%s_%s_%d.bin" % (rec["token"], name, i)),
                              dtype=np.float32).reshape(-1, 5)
            assert got.tobytes() == want.tobytes()
            assert rec_i["path"] == os.path.join("db", name, "%s_%s_%d.bin" % (rec["token"], name, i))
            assert rec_i["image_idx"] == rec["token"] and rec_i["gt_idx"] == i and rec_i["group_id"] == group
            assert rec_i["num_points_in_gt"] == len(want) and rec_i["box3d_lidar"].tobytes() == boxes[i].tobytes()
            assert rec_i["difficulty"] == 0 and isinstance(rec_i["difficulty"], np.int32)
            group += 1
    assert seen == {k: len(v) for k, v in dbinfos.items()} and group > 0


def test_host_twin_cuts_objects_like_the_numpy_restatement(nusc_tree):
    """points_in_rbbox on the host twin equals the numpy restatement on an accumulated 10-sweep frame."""
    import create_gt_database as tool
    from det3d.datasets.pipelines.sample_ops import libm_trig
    root = nusc_tree[0]
    ds = hydra_lite.instantiate(dict(nusc_node(root, "infos_train_10sweeps_withvelo_filterZero.pkl", label=False),
                                     create_database=True))
    rec = ds[0]
    pts, boxes = tool.frame_points(rec, host=True), rec["annotations"]["gt_boxes"]
    assert len(pts) > 9 * 2000
    assert np.array_equal(tool.points_in_rbbox(pts, boxes), points_in_boxes(pts, boxes, libm_trig(boxes[:, 8])))


# ---------------------------------------------------------------------- nuScenes results JSON
def _qmul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def test_nusc_results_json_follows_the_devkit_quaternion_path(nusc_tree, tmp_path):
    from pillarnext_b200.evaluate_nuscenes import DEFAULT_ATTRIBUTE
    root, _, infos, poses = nusc_tree
    ds = hydra_lite.instantiate(nusc_node(root, "infos_train_10sweeps_withvelo_filterZero.pkl", label=False))
    g = np.random.default_rng(5)
    dets = {}
    for info in infos:
        k = 7
        b = np.concatenate([g.uniform(-40, 40, (k, 2)), g.uniform(-2, 1, (k, 1)), g.uniform(0.5, 5, (k, 3)),
                            g.normal(0, 1, (k, 2)), g.uniform(-np.pi, np.pi, (k, 1))], 1).astype(np.float32)
        b[:3, 6:8] *= 0.05                                                    # some below the 0.2 m/s attribute speed
        dets[info["token"]] = {"box3d_lidar": torch.tensor(b), "scores": torch.tensor(g.uniform(0, 1, k), dtype=torch.float32),
                               "label_preds": torch.tensor(np.arange(k) % 10)}
    assert ds.evaluation(dets, str(tmp_path), testset=True) is None
    with open(os.path.join(str(tmp_path), "infos_train_10sweeps_withvelo_filterZero.json")) as fh:
        out = json.load(fh)
    assert out["meta"]["use_lidar"] and not out["meta"]["use_camera"]
    names = [n for t in NUSC_TASKS for n in t]
    for token, det in dets.items():
        (qc, tc), (qp, tp) = poses[token]
        Rc, Rp = RF.quat_matrix(qc), RF.quat_matrix(qp)
        rows = out["results"][token]
        assert len(rows) == len(det["scores"])
        for row, b, s, l in zip(rows, det["box3d_lidar"].double().numpy(), det["scores"].numpy(), det["label_preds"].numpy()):
            # Box(center, wlh = (dy, dx, dz), Quaternion(axis=z, radians=yaw), velocity (vx, vy, 0)), rotated and
            # translated by the sensor pose, then by the ego pose
            q = _qmul(qp, _qmul(qc, np.array([np.cos(b[8] / 2), 0.0, 0.0, np.sin(b[8] / 2)])))
            q = -q if q[0] < 0 else q
            c = Rp @ (Rc @ b[:3] + tc) + tp
            v = Rp @ (Rc @ np.array([b[6], b[7], 0.0]))
            np.testing.assert_allclose(row["translation"], c, rtol=0, atol=1e-9)
            np.testing.assert_allclose(row["rotation"], q, rtol=0, atol=1e-9)
            np.testing.assert_allclose(row["velocity"], v[:2], rtol=0, atol=1e-9)
            assert row["size"] == [float(np.float32(b[4])), float(np.float32(b[3])), float(np.float32(b[5]))]
            name = names[int(l)]
            assert row["detection_name"] == name and row["detection_score"] == float(s) and row["sample_token"] == token
            speed = np.hypot(v[0], v[1])
            if speed > 0.2:
                want = {"car": "vehicle.moving", "construction_vehicle": "vehicle.moving", "bus": "vehicle.moving",
                        "truck": "vehicle.moving", "trailer": "vehicle.moving", "bicycle": "cycle.with_rider",
                        "motorcycle": "cycle.with_rider"}.get(name)
            else:
                want = {"pedestrian": "pedestrian.standing", "bus": "vehicle.parked"}.get(name)
            assert row["attribute_name"] == (want or DEFAULT_ATTRIBUTE[name])


# ---------------------------------------------------------------------- the reference's goldens
from oracle import make_golden_readers as MGR  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden", "ref_readers.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


@pytest.fixture(scope="module")
def gold_trees(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("gold"))
    paths = {name: os.path.join(root, name) for name in MGR.TREES}
    for name, path in paths.items():
        MGR.write_tree(name, path)
    return paths


def assert_db_equals_golden(dbinfos, root, db_dir, gold, key):
    recs, boxes, sha = MGR.db_record(dbinfos, root, db_dir)
    assert json.loads(recs) == json.loads(str(gold[key + "_dbinfos"]))
    assert boxes.tobytes() == gold[key + "_boxes"].tobytes()
    assert json.loads(sha) == json.loads(str(gold[key + "_sha256"]))


def reader(node_kw, label_kw=None):
    node = dict(node_kw, loading_pipelines=["load_pointcloud", "load_box3d"], create_database=True)
    if label_kw is not None:
        node["prepare_label"] = {"centermap": dict(label_kw, _target_="det3d.datasets.pipelines.assign.AssignLabel")}
    return node


def gold_frames(gold, case, n):
    return [(gold["%s_%d_points" % (case, i)], gold["%s_%d_boxes" % (case, i)], list(gold["%s_%d_names" % (case, i)]))
            for i in range(n)]


def check_frames(points, count, boxes, classes, class_names, want):
    """points [n, 6] of a host-twin chain (rows past count ignored), boxes [B, M, 9], classes [B, M] vs the golden."""
    p = points[:count]
    for f, (wp, wb, wn) in enumerate(want):
        got = np.ascontiguousarray(p[p[:, 0] == f, 1:])
        assert got.tobytes() == np.ascontiguousarray(wp).tobytes(), f
        real = classes[f] >= 0
        assert boxes[f][real].tobytes() == np.ascontiguousarray(wb).tobytes(), f
        assert [class_names[c] if c < len(class_names) else None for c in classes[f][real]] == wn


def test_nusc_reader_and_database_reproduce_the_reference(gold, gold_trees):
    import create_gt_database as tool
    root = gold_trees["nusc"]
    dbinfos = tool.create_reader_database("NUSC", root, MGR.NUSC_INFO, nsweeps=10, host=True)
    assert_db_equals_golden(dbinfos, root, "gt_database_10sweeps_withvelo", gold, "ndb")
    smp = sampler_node(root, "dbinfos_train_10sweeps_withvelo.pkl", MGR.NUSC_GROUPS)
    node = reader(dict(nusc_node(root, MGR.NUSC_INFO, smp, AUG, label=False)), MGR.label_args(NUSC_TASKS, 50.4))
    ds = build(node, MGR.SEED)
    np.random.seed(MGR.SEED + 1)
    b = scenes.collate([ds[i] for i in range(len(ds))])
    assert b["gts_classes"].ge(0).any() and len(b["sweep_points"]) > 0
    pts, _ = ops.accumulate_sweeps_host(b["points"].numpy(), b["point_offsets"].numpy(), b["sweep_points"].numpy(),
                                        b["sweep_offsets"].numpy(), b["sweep_transforms"].numpy(), b["sweep_min_distance"])
    pts, boxes, classes, accepted, count = ops.gt_sample_host(
        pts, b["gt_boxes_raw"].numpy(), b["gt_classes"].numpy(), b["gt_trig"].numpy(), b["gts_boxes"].numpy(),
        b["gts_classes"].numpy(), b["gts_trig"].numpy(), b["gts_points"].numpy(), b["gts_offsets"].numpy())
    assert accepted.any()
    pts, boxes = ops.global_aug_host(pts, boxes, b["aug"].numpy())
    names = [n for t in NUSC_TASKS for n in t]
    check_frames(pts, count, boxes, classes, names, gold_frames(gold, "nusc", len(ds)))


@pytest.mark.parametrize("case,nsweeps,drop", [("waymo", 3, 0.5), ("f1", 1, 0.0)])
def test_waymo_reader_reproduces_the_reference(gold, gold_trees, case, nsweeps, drop):
    root = gold_trees["waymo"]
    node = reader(waymo_node(root, MGR.WAYMO_INFO, nsweeps, drop, label=False), MGR.label_args(WAYMO_TASKS, 76.8))
    ds = build(node, MGR.SEED)
    np.random.seed(MGR.SEED + 1)
    b = scenes.collate([ds[i] for i in range(len(ds))])
    if nsweeps > 1:
        lens = np.diff(b["sweep_offsets"].numpy())
        assert (lens == 0).any() and (lens > 0).any()                  # drop_frames dropped some sweeps, kept others
        pts, count = ops.accumulate_sweeps_host(b["points"].numpy(), b["point_offsets"].numpy(), b["sweep_points"].numpy(),
                                                b["sweep_offsets"].numpy(), b["sweep_transforms"].numpy(), 0.0)
    else:
        assert "sweep_points" not in b
        pts, count = b["points"].numpy(), len(b["points"])
    names = [n for t in WAYMO_TASKS for n in t]
    want = gold_frames(gold, case, len(ds))
    assert sum(len(w[1]) for w in want) < sum(len(i["objects"]) for i in ds.infos)   # 0-point objects dropped
    check_frames(pts, count, b["gt_boxes_raw"].numpy(), b["gt_classes"].numpy(), names, want)


def test_cbgs_order_is_the_reference(gold, gold_trees):
    node = nusc_node(gold_trees["nusc"], MGR.NUSC_INFO, label=False, class_names=[[str(n)] for n in gold["cbgs_classes"]],
                     resampling=True)
    np.random.seed(MGR.SEED)
    ds = hydra_lite.instantiate(node)
    assert [i["token"] for i in ds.infos] == list(gold["cbgs_tokens"]) and len(ds) > len(MGR.TREES["nusc"]["seeds"])


def test_waymo_database_with_its_thinning_is_the_reference(gold, gold_trees):
    import create_gt_database as tool
    root = gold_trees["wdb"]
    dbinfos = tool.create_reader_database("WAYMO", root, MGR.WAYMO_INFO, nsweeps=1, host=True)
    assert_db_equals_golden(dbinfos, root, "gt_database_1sweeps_withvelo", gold, "wdb")


def write_experiment(gold, name, config_dir):
    """The reference's composed experiment as one yaml file, the way tools/train.py --config-path reads it."""
    import yaml
    os.makedirs(config_dir, exist_ok=True)
    with open(os.path.join(config_dir, name + ".yaml"), "w") as fh:
        yaml.safe_dump(json.loads(str(gold["cfg_" + name])), fh)


def test_reference_composed_experiments_instantiate_our_classes(gold, gold_trees, tmp_path):
    import shutil
    from det3d.datasets.nuscenes import NuScenesDataset
    from det3d.datasets.pipelines.assign import AssignLabel
    from det3d.datasets.waymo.waymo import WaymoDataset
    root = gold_trees["nusc"]
    import create_gt_database as tool
    tool.create_reader_database("NUSC", root, MGR.NUSC_INFO, nsweeps=10, host=True)
    shutil.copy(os.path.join(root, MGR.NUSC_INFO), os.path.join(root, "infos_val_10sweeps_withvelo_filterZero.pkl"))
    cdir = str(tmp_path)
    for name in ("nusc_det_pp18_aspp_iou_sp", "waymo_det_pp18_aspp_iou_car_sp"):
        write_experiment(gold, name, cdir)
    cfg = hydra_lite.main(cdir, "nusc_det_pp18_aspp_iou_sp", ["data.train_dataset.root_path=" + root])
    assert cfg.data.train_dataset._target_ == "det3d.datasets.nuscenes.NuScenesDataset"
    np.random.seed(0)
    train, val = hydra_lite.instantiate(cfg.data.train_dataset), hydra_lite.instantiate(cfg.data.val_dataset)
    assert isinstance(train, NuScenesDataset) and isinstance(val, NuScenesDataset)
    assert isinstance(train.prepare_label["centermap"], AssignLabel) and train.sampler is not None
    assert len(train) > len(val) and train.nsweeps == 10                # CBGS resampling: True
    rec = train[0]
    assert rec["gt_boxes_raw"].shape[1] == 9 and "gts" in rec and len(rec["aug"]) == 4
    assert val[0]["gt_boxes_raw"].shape == (0, 9)
    w = hydra_lite.main(cdir, "waymo_det_pp18_aspp_iou_car_sp", [])
    assert w.data.train_dataset._target_ == "det3d.datasets.waymo.waymo.WaymoDataset"
    node = {k: v for k, v in dict(w.data.train_dataset).items() if k != "sampler"}
    node["root_path"] = gold_trees["waymo"]
    assert isinstance(hydra_lite.instantiate(node), WaymoDataset)


def test_waymo_level_2_follows_the_label_point_count(monkeypatch):
    """The same frames scored with "num_points" labels and with the oracle counting points whose counts equal those
    labels; a box with many points but a 3-point label is LEVEL_2."""
    from oracle import waymo_metric_oracle as WO
    from pillarnext_b200 import evaluate_waymo as EW
    g = np.random.default_rng(2)
    gts, dets, labels = {}, {}, []
    for f in range(3):
        boxes = np.array([[x, 0.0, 0.85, 4.0, 2.0, 1.7, 0.0, 0.0, 0.0] for x in (0.0, 10.0, 20.0, 30.0)], np.float32)
        pts = np.concatenate([b[:3] + g.uniform(-0.5, 0.5, (40, 3)) for b in boxes]).astype(np.float32)
        lab = np.array([3, 40, 2, 0][f:] + [3, 40, 2, 0][:f], np.int64)
        gts["f%d" % f] = {"boxes": boxes, "names": ["vehicle"] * 4, "points": pts}
        labels.append(lab)
        d = boxes + g.normal(0, 0.05, boxes.shape).astype(np.float32)
        dets["f%d" % f] = {"box3d_lidar": d, "scores": g.uniform(0.2, 1, 4).astype(np.float32),
                           "label_preds": np.zeros(4, np.int64)}
    labelled = {t: {"boxes": v["boxes"], "names": v["names"], "num_points": labels[i]} for i, (t, v) in enumerate(gts.items())}
    pk = EW.pack(labelled, dets, ["vehicle"])
    counts, match, _, heading = EW.run_host(pk)
    assert (counts == 0).all()                                        # no points given: nothing counted geometrically
    got = EW.score(pk, EW.known_counts(pk, counts), match, heading, ["vehicle"])
    it = iter(labels)

    def label_counts(points, boxes, trig):
        lab = next(it)
        mask = np.zeros((int(lab.max()), len(boxes)), bool)
        for j, n in enumerate(lab):
            mask[:n, j] = True
        return mask
    monkeypatch.setattr(WO.gts_oracle, "points_in_boxes", label_counts)
    want = WO.waymo_metrics(gts, dets, ["vehicle"])
    for k in ("mAP_L1", "mAPH_L1", "mAP_L2", "mAPH_L2"):
        assert abs(got[k] - want[k]) < 1e-6, k                     # APH: fp32 heading accuracy vs the oracle's
    assert got["per_class"]["vehicle"]["n_gt_L1"] == 3 and got["per_class"]["vehicle"]["n_gt_L2"] == 9
    geometric = EW.score(pk, np.full_like(counts, 40), match, heading, ["vehicle"])
    assert geometric["per_class"]["vehicle"]["n_gt_L1"] == 12
