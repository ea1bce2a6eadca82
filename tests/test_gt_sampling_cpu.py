"""Ground-truth database sampling, CPU only.

* the drop-in sampler (det3d/datasets/pipelines/sample_ops.py), seeded like the reference, draws the reference's
  candidates, frame after frame (tests/golden/ref_gts.npz, frozen by oracle/make_golden_gts.py);
* the product's selection and paste compiled for the host (pnx_gt_sample_host) reproduce the reference's output bit
  for bit -- points, boxes, classes -- and put frame index B on the unused tail rows; so does the numpy oracle;
* the reference experiments' sampler nodes instantiate the drop-in classes; unsupported options raise;
* tools/create_gt_database.py writes the reference's record fields, and its point test is the reference's;
* dataset and collate: test mode refuses a sampler, no gts_* keys without one, packed candidates with one.
"""
import json
import os
import pickle
import sys

import numpy as np
import pytest
import torch

from det3d.datasets.pipelines import sample_ops as SO
from oracle import gts_oracle
from pillarnext_b200 import hydra_lite, modules, scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
EXPERIMENTS = os.path.join(ROOT, "configs", "experiments")
sys.path.insert(0, os.path.join(ROOT, "tools"))


def golden():
    return np.load(os.path.join(GOLDEN, "ref_gts.npz"))


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


@pytest.fixture
def np_random_state():
    state = np.random.get_state()
    yield
    np.random.set_state(state)


def write_golden_db(g, root):
    """The golden's gt database as files under `root`; returns the dbinfos path."""
    infos = {}
    off = np.concatenate([[0], np.cumsum(g["db_counts"])])
    for k, (name, path) in enumerate(zip(g["db_names"], g["db_paths"])):
        os.makedirs(os.path.join(root, os.path.dirname(str(path))), exist_ok=True)
        g["db_points"][off[k]:off[k + 1]].astype(np.float32).tofile(os.path.join(root, str(path)))
        infos.setdefault(str(name), []).append({"name": str(name), "path": str(path), "image_idx": "golden", "gt_idx": k,
                                                "box3d_lidar": g["db_boxes"][k].copy(), "num_points_in_gt": int(g["db_counts"][k]),
                                                "difficulty": 0, "group_id": k})
    with open(os.path.join(root, "dbinfos_train_1sweeps_withvelo.pkl"), "wb") as fh:
        pickle.dump(infos, fh)
    return "dbinfos_train_1sweeps_withvelo.pkl"


def golden_batch(g):
    """The golden scenes and their drawn candidates as collated arrays (the inputs of pnx_gt_sample)."""
    classes = json.loads(str(g["classes"]))
    names = json.loads(str(g["names"]))
    B, M = g["boxes"].shape[:2]
    S = g["draws"].shape[1]
    cls = np.full((B, M), -1, np.int32)
    for f, n in enumerate(names):
        cls[f, :len(n)] = [classes.index(x) for x in n]
    cb = np.zeros((B, S, 9), np.float32)
    cb[:, :, 3:6] = 1
    cc = np.full((B, S), -1, np.int32)
    counts = np.zeros((B, S), np.int64)
    db_off = np.concatenate([[0], np.cumsum(g["db_counts"])])
    cpts = []
    for f in range(B):
        for s, k in enumerate(g["draws"][f]):
            if k < 0:
                continue
            cb[f, s], cc[f, s], counts[f, s] = g["db_boxes"][k], classes.index(str(g["db_names"][k])), g["db_counts"][k]
            cpts.append(g["db_points"][db_off[k]:db_off[k + 1]])
    off = np.concatenate([[0], np.cumsum(counts.reshape(-1))]).astype(np.int32)
    return dict(points=g["points"], boxes=g["boxes"], classes=cls, trig=g["scene_trig"], cboxes=cb, cclasses=cc,
                ctrig=g["cand_trig"], cpoints=np.concatenate(cpts).astype(np.float32), coffsets=off)


def golden_expected(g):
    classes = json.loads(str(g["classes"]))
    out_names = json.loads(str(g["out_names"]))
    ob = g["out_boxes"]
    oc = np.full(ob.shape[:2], -1, np.int32)
    for f, n in enumerate(out_names):
        oc[f, :len(n)] = [classes.index(x) for x in n]
    return g["out_points"], ob, oc


def host_gts(points, boxes, classes, trig, cboxes, cclasses, ctrig, cpoints, coffsets):
    from pillarnext_b200 import ops
    f, i = (lambda a: np.asarray(a, np.float32)), (lambda a: np.asarray(a, np.int32))
    return ops.gt_sample_host(f(points), f(boxes), i(classes), f(trig), f(cboxes), i(cclasses), f(ctrig), f(cpoints),
                              i(coffsets))


def test_dropin_sampler_draws_the_reference_candidates(tmp_path, np_random_state):
    g = golden()
    dbinfo = write_golden_db(g, str(tmp_path))
    path_index = {str(p): k for k, p in enumerate(g["db_paths"])}
    min_points = json.loads(str(g["min_points"]))
    np.random.seed(int(g["seed"]))
    sampler = SO.DataBaseSamplerV2(root_path=str(tmp_path), dbinfo_path=dbinfo, groups=json.loads(str(g["groups"])),
                                   db_prepor={"filter_by_num": SO.DBFilterByMinNumPoint(dict(min_points))}, rate=1.0,
                                   gt_drop_percentage=0, gt_drop_max_keep_points=-1, point_dim=5)
    log = []
    orig = SO.BatchSampler.sample
    names = json.loads(str(g["names"]))
    try:
        SO.BatchSampler.sample = lambda self, num: (lambda r: (log.extend(path_index[i["path"]] for i in r), r)[1])(orig(self, num))
        for f, n in enumerate(names):
            log.clear()
            rec = sampler.sample_all(g["boxes"][f, :len(n)], np.array(n))
            want = [int(k) for k in g["draws"][f] if k >= 0]
            assert log == want, (f, log, want)
            assert rec is not None and len(rec["gt_boxes"]) == len(want)
            assert np.array_equal(bits(rec["gt_boxes"]), bits(g["db_boxes"][want]))
            assert list(rec["gt_names"]) == [str(g["db_names"][k]) for k in want]
            db_off = np.concatenate([[0], np.cumsum(g["db_counts"])])
            assert np.array_equal(rec["points"], np.concatenate([g["db_points"][db_off[k]:db_off[k + 1]] for k in want]))
            assert rec["num_points"].tolist() == [int(g["db_counts"][k]) for k in want]
            # the trig pairs: numpy's vectorised fp32 pair and libm's cosf / sinf, of exactly these boxes
            assert np.array_equal(rec["trig"][:, :2], SO.numpy_trig(rec["gt_boxes"]))
            assert np.array_equal(bits(rec["trig"][:, 2:]), bits(g["cand_trig"][f, :len(want), 2:]))
    finally:
        SO.BatchSampler.sample = orig
    assert np.random.random_sample() == g["next_draw"]            # same state afterwards: nothing extra drawn
    car = [k for k, nm in enumerate(g["db_names"]) if nm == "car"]
    assert sum(g["db_counts"][car] >= 5) == 12 and len(car) == 14  # the filter drops two cars


def test_host_twin_reproduces_the_reference_bit_for_bit():
    g = golden()
    batch = golden_batch(g)
    keep = {k: v.copy() for k, v in batch.items()}
    p, b, c, acc, count = host_gts(**batch)
    want_p, want_b, want_c = golden_expected(g)
    assert count == len(want_p)
    assert np.array_equal(bits(p[:count]), bits(want_p))
    assert np.array_equal(bits(b), bits(want_b)) and np.array_equal(c, want_c)
    B = g["boxes"].shape[0]
    assert np.all(p[count:, 0] == B) and np.all(p[count:, 1:] == 0)
    assert all(np.array_equal(keep[k], batch[k]) for k in batch)
    assert acc.sum() == (want_c >= 0).sum() - (batch["classes"] >= 0).sum()


def test_goldens_cover_the_quirks():
    g = golden()
    batch = golden_batch(g)
    _, _, _, acc, _ = host_gts(**batch)
    draws, names = g["draws"], json.loads(str(g["names"]))
    trucks = {k: i for i, k in enumerate(np.flatnonzero(g["db_names"] == "truck"))}   # A, B, C, D in database order
    for f in (0, 4, 5, 6, 7):
        slot = {trucks[k]: s for s, k in enumerate(draws[f]) if k in trucks}
        first, later = sorted((slot[0], slot[1]))
        assert not acc[f, first] and acc[f, later]                 # rejected only by a later candidate of its class
        assert acc[f, slot[2]] and not acc[f, slot[3]]             # touching: accepted; containing a scene box: rejected
    assert len(names[1]) == 0 and acc[1].sum() > 0                 # a frame without scene boxes
    assert (draws[2] >= 0).sum() > 0 and acc[2].sum() == 0         # every candidate rejected
    assert all(str(g["db_names"][k]) != "car" for k in draws[3] if k >= 0)   # nothing to sample for car
    # the ties: scene points exactly on truck C's faces are removed, those one ulp outside are kept
    C = g["db_boxes"][list(trucks)[2]]
    out = g["out_points"]
    on_face = np.array([[47, 20, 0], [53, 20.5, 1], [50, 18.75, -1], [51, 21.25, 0.5], [49, 19, 1.5]], np.float32)
    for q in on_face:
        assert not np.any(np.all(out[:, 1:4] == q, 1) & (out[:, 0] == 0))
        assert np.any(np.all(g["points"][:, 1:4] == q, 1) & (g["points"][:, 0] == 0))
    outside = np.array([np.nextafter(np.float32(47), np.float32(0)), 20, 0], np.float32)
    assert np.any(np.all(out[:, 1:4] == outside, 1) & (out[:, 0] == 0)) and C[8] == 0


def test_oracle_reproduces_the_reference_bit_for_bit():
    g = golden()
    p, b, c, _ = gts_oracle.apply(**golden_batch(g))
    want_p, want_b, want_c = golden_expected(g)
    assert np.array_equal(bits(p), bits(want_p)) and np.array_equal(bits(b), bits(want_b)) and np.array_equal(c, want_c)


def test_point_test_is_the_reference_points_in_rbbox():
    import create_gt_database as tool
    g = golden()
    got = tool.points_in_rbbox(g["points"][:, 1:], g["db_boxes"])
    assert np.array_equal(got, g["inside"]) and g["inside"].sum() > 50


def test_reference_sampler_nodes_instantiate_the_dropin_classes(tmp_path):
    with open(os.path.join(GOLDEN, "ref_gts_configs.json")) as fh:
        nodes = json.load(fh)
    assert sorted(nodes) == ["nusc_det_pp18_aspp_iou_sp", "nusc_det_voxel18_aspp_iou_sp", "waymo_det_pp18_aspp_iou_car_sp",
                             "waymo_det_pp18_aspp_iou_car_sp_f1"]
    for name, node in nodes.items():
        classes = [k for grp in node["groups"] for k in grp]
        infos = {c: [{"name": c, "path": "x.bin", "image_idx": 0, "gt_idx": i, "box3d_lidar": np.zeros(9, np.float32),
                      "num_points_in_gt": 3 + 2 * i, "difficulty": 0, "group_id": i} for i in range(4)] for c in classes}
        with open(tmp_path / node["dbinfo_path"], "wb") as fh:
            pickle.dump(infos, fh)
        part = hydra_lite.instantiate(dict(node, root_path=str(tmp_path)))
        sampler = part()
        assert isinstance(sampler, SO.DataBaseSamplerV2), name
        assert sampler._sample_classes == classes and sampler._rate == 1.0 and sampler._point_dim == 5
        assert node["db_prepor"]["filter_by_num"]["min_gt_point_dict"] == {c: 5 for c in classes}
        assert all(len(sampler.db_infos[c]) == 3 for c in classes)          # 3, 5, 7 points >= 5 kept; 3 dropped
        assert set(sampler._sampler_dict) == set(classes)


def test_unsupported_sampler_options_raise(tmp_path):
    info = {"name": "car", "path": "x.bin", "image_idx": 0, "gt_idx": 0, "box3d_lidar": np.zeros(9, np.float32),
            "num_points_in_gt": 9, "difficulty": 0, "group_id": 0}
    kw = dict(root_path=str(tmp_path), dbinfo_path="db.pkl", groups=[{"car": 2}], db_prepor=None, rate=1.0,
              gt_drop_percentage=0, gt_drop_max_keep_points=-1, point_dim=5)
    for extra, kws, match in [({}, dict(gt_drop_percentage=0.2), "gt_drop_percentage"),
                              ({"rot_transform": 0.1}, {}, "rot_transform"),
                              ({"box3d_lidar": np.zeros(9)}, {}, "float32"),
                              ({}, dict(groups=[{"car": 2}, {"car": 3}]), "twice")]:
        with open(tmp_path / "db.pkl", "wb") as fh:
            pickle.dump({"car": [dict(info, **extra)]}, fh)
        with pytest.raises(ValueError, match=match):
            SO.DataBaseSamplerV2(**dict(kw, **kws))


def test_batch_sampler_wraps_as_the_reference_does(np_random_state):
    np.random.seed(0)
    bs = SO.BatchSampler(list(range(5)))
    first = list(bs._indices)
    assert bs.sample(3) == first[:3]
    assert bs.sample(2) == first[3:] and bs._idx == 0             # exact fit: the rest, then a reshuffle
    second = list(bs._indices)
    assert bs.sample(4) == second[:4] and bs.sample(3) == second[4:]   # short rest


def _gts_db(tmp_path, n_frames=24):
    import create_gt_database as tool
    cfg = hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp_gts", ["data.train_dataset.root_path=%s" % tmp_path,
                                                                    "data.train_dataset.n_frames=%d" % n_frames])
    node = {k: v for k, v in dict(cfg.data.train_dataset).items() if k not in ("sampler", "augmentation")}
    infos = tool.create_groundtruth_database(hydra_lite.instantiate(node), str(tmp_path))
    return cfg, infos


def test_create_gt_database_writes_the_reference_records(tmp_path):
    import create_gt_database as tool
    cfg, infos = _gts_db(tmp_path, 3)
    with open(tmp_path / "dbinfos_train_1sweeps_withvelo.pkl", "rb") as fh:
        assert pickle.load(fh).keys() == infos.keys()
    recs = [r for v in infos.values() for r in v]
    assert len(recs) > 20 and sorted({r["group_id"] for r in recs}) == list(range(len(recs)))
    for r in recs:
        assert set(r) == {"name", "path", "image_idx", "gt_idx", "box3d_lidar", "num_points_in_gt", "difficulty", "group_id"}
        assert r["path"] == os.path.join("gt_database_1sweeps_withvelo", r["name"], "%s_%s_%d.bin" % (r["image_idx"], r["name"], r["gt_idx"]))
        assert r["box3d_lidar"].dtype == np.float32 and r["box3d_lidar"].shape == (9,)
        pts = np.fromfile(str(tmp_path / r["path"]), dtype=np.float32).reshape(-1, 5)
        assert len(pts) == r["num_points_in_gt"]
    # the cut of one frame equals the oracle's restatement of points_in_rbbox, relative to the box centres
    r = infos["car"][0]
    seed = int(r["image_idx"].split("_")[1])
    pts, boxes, names = scenes.make_scene(seed, cfg.data.train_dataset.cfg, cfg.data.train_dataset.n_points, cfg.data.train_dataset.n_boxes)
    inside = gts_oracle.points_in_boxes(pts, boxes, SO.libm_trig(boxes[:, -1]))
    assert np.array_equal(tool.points_in_rbbox(pts, boxes), inside)
    want = pts[inside[:, r["gt_idx"]]]
    want[:, :3] -= boxes[r["gt_idx"], :3]
    assert np.array_equal(np.fromfile(str(tmp_path / r["path"]), dtype=np.float32).reshape(-1, 5), want)


def test_test_mode_dataset_with_sampler_raises():
    cfg = hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp_gts", [])
    node = dict(cfg.data.val_dataset, sampler=cfg.data.train_dataset.sampler)
    with pytest.raises(ValueError, match="test_mode"):
        hydra_lite.instantiate(node)


def test_collate_without_sampler_is_unchanged():
    cfg = hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp", ["data.train_dataset.n_frames=2"])
    ds = hydra_lite.instantiate(cfg.data.train_dataset)
    assert ds.sampler is None
    ex = scenes.collate([ds[0], ds[1]])
    assert sorted(ex) == ["gt_boxes_raw", "gt_classes", "points", "token"] and "gts" not in ds[0]


def test_sampled_dataset_and_collate(tmp_path, np_random_state):
    cfg, _ = _gts_db(tmp_path)
    ds = hydra_lite.instantiate(cfg.data.train_dataset)
    plain = hydra_lite.instantiate(hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp", []).data.train_dataset)
    np.random.seed(4)
    items = [ds[i] for i in range(3)]
    for i, it in enumerate(items):
        ref = plain[i]
        assert np.array_equal(it["points"], ref["points"]) and np.array_equal(it["gt_boxes_raw"], ref["gt_boxes_raw"])
        g = it["gts"]
        assert len(g["classes"]) > 0 and g["trig"].shape == (len(g["classes"]), 4) and len(it["aug"]) == 4
        assert np.array_equal(g["scene_trig"], SO.numpy_trig(it["gt_boxes_raw"]))
    ex = scenes.collate(items)
    S = max(len(it["gts"]["classes"]) for it in items)
    M = ex["gt_boxes_raw"].shape[1]
    assert tuple(ex["gts_boxes"].shape) == (3, S, 9) and ex["gts_classes"].dtype == torch.int32
    assert tuple(ex["gts_trig"].shape) == (3, S, 4) and tuple(ex["gt_trig"].shape) == (3, M, 2)
    off = ex["gts_offsets"].numpy()
    assert off.dtype == np.int32 and len(off) == 3 * S + 1 and off[-1] == len(ex["gts_points"])
    for i, it in enumerate(items):
        k = len(it["gts"]["classes"])
        assert np.array_equal(ex["gts_classes"][i, :k].numpy(), it["gts"]["classes"]) and (ex["gts_classes"][i, k:] == -1).all()
        assert np.array_equal(ex["gts_points"][off[i * S]:off[i * S + k]].numpy(), it["gts"]["points"])
    # the candidates of one frame stay in class-call order (runs of equal class ids, in group order)
    order = [0, 1, 2]                                           # car, truck, pedestrian: the group order of the config
    for it in items:
        c = it["gts"]["classes"].tolist()
        assert c == sorted(c, key=order.index)
    with pytest.raises(ValueError, match="every frame"):
        scenes.collate([items[0], plain[0]])
    p, b, cl, acc = gts_oracle.apply(ex["points"].numpy(), ex["gt_boxes_raw"].numpy(), ex["gt_classes"].numpy(),
                                     ex["gt_trig"].numpy(), ex["gts_boxes"].numpy(), ex["gts_classes"].numpy(),
                                     ex["gts_trig"].numpy(), ex["gts_points"].numpy(), ex["gts_offsets"].numpy())
    h = host_gts(ex["points"].numpy(), ex["gt_boxes_raw"].numpy(), ex["gt_classes"].numpy(), ex["gt_trig"].numpy(),
                 ex["gts_boxes"].numpy(), ex["gts_classes"].numpy(), ex["gts_trig"].numpy(), ex["gts_points"].numpy(),
                 ex["gts_offsets"].numpy())
    assert acc.sum() > 0 and np.array_equal(h[3].astype(bool), acc) and h[4] == len(p)
    assert np.array_equal(bits(h[0][:h[4]]), bits(p)) and np.array_equal(bits(h[1]), bits(b)) and np.array_equal(h[2], cl)


def test_sampling_after_label_assignment_is_an_error():
    with pytest.raises(ValueError, match="assigned labels"):
        modules.SingleStageDetector.gt_sample(None, {"hm": [], "gts_boxes": torch.zeros(1, 1, 9)})
