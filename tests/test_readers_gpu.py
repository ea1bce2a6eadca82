"""The info-file readers on the GPU.

* ops.points_in_boxes (pnx_points_in_boxes) equals its host twin to the bit on a 10 x 26.5k-point accumulated frame
  with 60 boxes, with points exactly on box faces and z bounds and NaN rows;
* three bf16 training steps fed by NuScenesDataset (10 sweeps, the sampler, the augmentation) or WaymoDataset (3 sweeps,
  drop_frames 0.5) equal the steps fed by SyntheticSceneDataset for the same seeds: loss, logged terms and the updated
  parameters and buffers; validation detections are identical;
* WaymoDataset.evaluation equals waymo_metrics with the points counted in the frames (the fixture's num_points are the
  counts);
* tools/create_gt_database.py cuts the same database on the GPU as on the host twins;
* the label targets the GPU builds from WaymoDataset's records equal the reference AssignLabel's
  (tests/golden/ref_readers.npz);
* tools/train.py trains one epoch of the reference's composed nuScenes experiment with root_path at a fixture tree
  (10 sweeps, CBGS, the 10-sweep database through the sampler, the augmentation), and tools/test.py reloads the
  checkpoint and writes the devkit's results JSON."""
import os
import pickle
import sys

import numpy as np
import pytest
import torch

from oracle import reader_fixtures as RF
from oracle import sweeps_oracle as O
from pillarnext_b200 import functional as Fn
from pillarnext_b200 import hydra_lite, ops, scenes
from pillarnext_b200.trainer import example_to_device

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXPERIMENTS = os.path.join(ROOT, "configs", "experiments")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from test_readers_cpu import AUG, batches, build, sampler_node, synthetic  # noqa: E402

SEEDS = [3, 4, 5, 6]


def test_points_in_boxes_matches_the_host_twin_bit_for_bit():
    from det3d.datasets.pipelines.sample_ops import libm_trig
    a = O.random_operands(10, 10, 26500, seed=4)
    pts, count = ops.accumulate_sweeps_host(*[a[k] for k in ("points", "point_offsets", "sweep_points", "sweep_offsets",
                                                              "transforms")], 1.0)
    pts = np.ascontiguousarray(pts[:count, 1:])                       # one frame of 10 x 26.5k points, 5 columns
    g = np.random.default_rng(8)
    m = 60
    boxes = np.concatenate([g.uniform(-30, 30, (m, 2)), g.uniform(-2, 1, (m, 1)), g.uniform(0.5, 6, (m, 3)),
                            g.normal(0, 1, (m, 2)), g.uniform(-np.pi, np.pi, (m, 1))], 1).astype(np.float32)
    boxes[:20, 8] = 0.0                                                # axis-aligned: faces land exactly on points
    edge = []
    for b in boxes[:20]:
        for sx, sy, sz in ((0.5, 0.0, 0.0), (-0.5, 0.2, 0.0), (0.1, 0.5, 0.0), (0.0, -0.5, 0.3), (0.2, 0.1, 0.5),
                           (0.0, 0.0, -0.5), (0.5, 0.5, 0.5)):
            edge.append([b[0] + np.float32(sx) * b[3], b[1] + np.float32(sy) * b[4], b[2] + np.float32(sz) * b[5], 1, 0])
    edge = np.array(edge, np.float32)
    nan = np.full((7, 5), np.nan, np.float32)
    nan[1:4, 0] = 1.0
    pts = np.concatenate([pts[: len(pts) // 2], edge, nan, pts[len(pts) // 2:]])
    assert len(pts) > 10 * 26000
    trig = libm_trig(boxes[:, 8])
    want = ops.points_in_boxes_host(pts, boxes, trig)
    got = ops.points_in_boxes(*[torch.from_numpy(x).cuda() for x in (pts, boxes, trig)])
    assert got.dtype == torch.bool and tuple(got.shape) == (len(pts), m)
    got = got.cpu().numpy()
    assert np.array_equal(got, want)
    e0 = len(pts) // 2
    assert want[e0:e0 + len(edge)].any() and not want[e0 + len(edge):e0 + len(edge) + 7].any()
    view = np.zeros((len(pts), 8), np.float32)
    view[:, :5] = pts
    strided = ops.points_in_boxes(torch.from_numpy(view).cuda()[:, :5], *[torch.from_numpy(x).cuda() for x in (boxes, trig)])
    assert np.array_equal(strided.cpu().numpy(), want)
    assert ops.points_in_boxes(*[torch.from_numpy(x).cuda() for x in (pts[:0], boxes, trig)]).shape == (0, m)


# ---------------------------------------------------------------------- training and validation parity
def _cfg(name):
    return hydra_lite.main(EXPERIMENTS, name, ["data.train_dataset.n_frames=%d" % len(SEEDS)])


def _label_node(cfg):
    return {"centermap": {"_target_": "det3d.datasets.pipelines.assign.AssignLabel", "gaussian_overlap": 0.1,
                          "max_objs": 500, "min_radius": 2, "tasks": [list(t) for t in cfg._tasks],
                          "pc_range": list(cfg.model.reader.pc_range), "voxel_size": list(cfg.model.reader.voxel_size),
                          "out_size_factor": [4] * len(cfg._tasks)}}


def _steps(cfg, batches_):
    torch.manual_seed(0)
    model = hydra_lite.instantiate(cfg.model).cuda().train()
    opt = hydra_lite.instantiate(cfg.optimizer, params=model.parameters())
    out = []
    prev = Fn.set_deterministic(True)
    try:
        for b in batches_:
            loss, logs = model(example_to_device(b, torch.device("cuda")))
            opt.zero_grad()
            loss.backward()
            opt.step()
            out.append((loss.detach().clone(), _copy(logs)))
        torch.cuda.synchronize()
    finally:
        Fn.set_deterministic(prev)
    return out, {k: v.detach().clone() for k, v in model.state_dict().items()}, model


def _copy(x):
    if torch.is_tensor(x):
        return x.detach().clone()
    if isinstance(x, dict):
        return {k: _copy(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [_copy(v) for v in x]
    return x


def _same(a, b):
    if torch.is_tensor(a):
        return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(-1).view(torch.uint8), b.view(-1).view(torch.uint8))
    if isinstance(a, dict):
        return sorted(a) == sorted(b) and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def _train_parity(cfg, reader_batches, synth_batches):
    (ra, sa, model), (rb, sb, _) = _steps(cfg, reader_batches), _steps(cfg, synth_batches)
    assert len(ra) == 3 and all(torch.isfinite(l) for l, _ in ra)
    for (la, logs_a), (lb, logs_b) in zip(ra, rb):
        assert _same(la, lb), (la.item(), lb.item())
        assert _same(logs_a, logs_b)
    assert sorted(sa) == sorted(sb) and not [k for k in sa if not _same(sa[k], sb[k])]
    return model


def test_nusc_reader_trains_like_the_synthetic_dataset(tmp_path):
    import create_gt_database as tool
    cfg = _cfg("synth_det_pp18_aspp_nds_sweeps")
    root, scene = str(tmp_path), dict(cfg.data._scene)
    RF.write_nusc(root, SEEDS, scene, n_points=6000, n_boxes=12)
    info = "infos_train_10sweeps_withvelo_filterZero.pkl"
    tool.create_reader_database("NUSC", root, info, nsweeps=10, host=False)
    smp = sampler_node(root, "dbinfos_train_10sweeps_withvelo.pkl", {"car": 6, "pedestrian": 5, "barrier": 4})
    node = {"_target_": "det3d.datasets.nuscenes.NuScenesDataset", "nsweeps": 10, "root_path": root, "info_path": info,
            "class_names": [list(t) for t in cfg._tasks], "loading_pipelines": ["load_pointcloud", "load_box3d"],
            "sampler": smp, "augmentation": AUG, "prepare_label": _label_node(cfg)}
    n = len(SEEDS)
    got = batches(build(node, 7), n, 2, 7) + batches(build(node, 8), 2, 2, 8)
    syn_kw = dict(augmentation=AUG, sampler=smp, root_path=root, nsweeps=10, min_distance=1.0)
    np.random.seed(7)
    want = batches(synthetic(scene, 6000, 12, **syn_kw), n, 2, 7)
    np.random.seed(8)
    want += batches(synthetic(scene, 6000, 12, **syn_kw), 2, 2, 8)
    assert "gts_boxes" in want[0] and "aug" in want[0] and "sweep_points" in want[0]
    model = _train_parity(cfg, got[:3], want[:3])
    # validation on the key frames + sweeps, no labels
    val = dict(node, loading_pipelines=["load_pointcloud"])
    for k in ("sampler", "augmentation", "prepare_label"):
        val.pop(k)
    vb = batches(build(val, 9), n, 2, 9)
    vw = batches(synthetic(scene, 6000, 12, nsweeps=10, min_distance=1.0, test_mode=True), n, 2, 9)
    model.eval()
    for a, b in zip(vb, vw):
        da, db = model(example_to_device(a, torch.device("cuda"))), model(example_to_device(b, torch.device("cuda")))
        assert sorted(da) == sorted(db)
        for t in da:
            assert all(_same(da[t][k], db[t][k]) for k in da[t] if k != "token")


def test_waymo_reader_trains_like_the_synthetic_dataset(tmp_path):
    cfg = _cfg("synth_det_pp18_aspp_waymo")
    root, scene = str(tmp_path), dict(cfg.data._scene)
    RF.write_waymo(root, SEEDS + [7, 8], scene, n_points=6000, n_boxes=12, nsweeps=3, identity_pose=True)
    node = {"_target_": "det3d.datasets.waymo.waymo.WaymoDataset", "nsweeps": 3, "drop_frames": 0.5, "root_path": root,
            "info_path": "waymo_infos_train.pkl", "loading_pipelines": ["load_pointcloud", "load_box3d"],
            "prepare_label": _label_node(cfg)}
    got = batches(build(node, 5), 6, 2, 5)
    want = batches(scenes.SyntheticSceneDataset(scene, 6, seed0=SEEDS[0], n_points=6000, n_boxes=12, nsweeps=3,
                                                drop_frames=0.5, min_distance=0.0), 6, 2, 5)
    _train_parity(cfg, got, want)


def test_waymo_evaluation_equals_waymo_metrics_with_counted_points(tmp_path):
    from pillarnext_b200.evaluate_waymo import waymo_metrics
    cfg = _cfg("synth_det_pp18_aspp_waymo")
    root, scene = str(tmp_path), dict(cfg.data._scene)
    infos = RF.write_waymo(root, SEEDS, scene, n_points=6000, n_boxes=12, nsweeps=1)
    ds = hydra_lite.instantiate({"_target_": "det3d.datasets.waymo.waymo.WaymoDataset", "nsweeps": 1, "root_path": root,
                                 "info_path": "waymo_infos_train.pkl", "loading_pipelines": ["load_pointcloud"],
                                 "tasks": [list(t) for t in cfg._tasks]})
    g = np.random.default_rng(3)
    dets, gts = {}, {}
    names = [n for t in cfg._tasks for n in t]
    for info in infos:
        b = np.array([o["box"] for o in info["objects"]], np.float32)
        d = b + g.normal(0, 0.15, b.shape).astype(np.float32)
        d[:, 3:6] = np.abs(d[:, 3:6])
        dets[info["token"]] = {"box3d_lidar": torch.tensor(d), "scores": torch.tensor(g.uniform(0, 1, len(d)), dtype=torch.float32),
                               "label_preds": torch.tensor([names.index(o["label"]) for o in info["objects"]])}
        gts[info["token"]] = {"boxes": b, "names": [o["label"] for o in info["objects"]],
                              "points": ds.read_file("lidar_point/%s.bin" % info["token"])}
    got = ds.evaluation(dets, str(tmp_path))
    want = waymo_metrics(gts, dets, names)
    assert str(got) == str(want) and want["mAP_L2"] > 0


def test_create_gt_database_on_the_gpu_equals_the_host_twins(tmp_path):
    import create_gt_database as tool
    cfg = _cfg("synth_det_pp18_aspp_nds_sweeps")
    root = str(tmp_path)
    RF.write_nusc(root, SEEDS, dict(cfg.data._scene), n_points=6000, n_boxes=12, nan_velocity=0.3, none_transform=True)
    info = "infos_train_10sweeps_withvelo_filterZero.pkl"
    out = {}
    for host in (True, False):
        d = os.path.join(root, "host" if host else "gpu")
        tool.create_reader_database("NUSC", root, info, nsweeps=10, host=host, db_path=os.path.join(d, "db"),
                                    dbinfo_path=os.path.join(d, "dbinfos.pkl"))
        with open(os.path.join(d, "dbinfos.pkl"), "rb") as fh:
            db = pickle.load(fh)
        files = {}
        for dp, _, fs in os.walk(os.path.join(d, "db")):
            for f in fs:
                with open(os.path.join(dp, f), "rb") as fh:
                    files[os.path.relpath(os.path.join(dp, f), d)] = fh.read()
        out[host] = (db, files)
    (dh, fh_), (dg, fg) = out[True], out[False]
    assert fh_ == fg and len(fh_) > 20
    assert sorted(dh) == sorted(dg)
    for k in dh:
        assert len(dh[k]) == len(dg[k])
        for a, b in zip(dh[k], dg[k]):
            assert sorted(a) == sorted(b)
            assert all(np.asarray(a[f]).tobytes() == np.asarray(b[f]).tobytes() for f in a)


# ---------------------------------------------------------------------- against the reference's goldens
from oracle import make_golden_readers as MGR  # noqa: E402
from test_readers_cpu import gold, gold_trees, reader, waymo_node, write_experiment  # noqa: E402,F401


def test_gpu_targets_equal_the_reference_assign_label(gold, gold_trees):
    tasks = [["vehicle"], ["pedestrian", "cyclist"]]
    lab = MGR.label_args(tasks, 76.8)
    ds = build(reader(waymo_node(gold_trees["waymo"], MGR.WAYMO_INFO, 3, 0.5, label=False), lab), MGR.SEED)
    np.random.seed(MGR.SEED + 1)
    b = scenes.collate([ds[i] for i in range(len(ds))])
    got = ops.assign_labels(b["gt_boxes_raw"].cuda(), b["gt_classes"].cuda(), tasks, lab["voxel_size"], lab["pc_range"],
                            lab["out_size_factor"], max_objs=lab["max_objs"], gaussian_overlap=lab["gaussian_overlap"],
                            min_radius=lab["min_radius"])
    for t in range(len(tasks)):
        for key, tol in (("ind", 0), ("mask", 0), ("cat", 0), ("hm", 1e-6), ("anno_box", 2e-6), ("gt_boxes", 0)):
            w = torch.stack([torch.from_numpy(gold["waymo_%d_%s_%d" % (f, key, t)]) for f in range(len(ds))])
            g = got[key][t].cpu()
            assert g.shape == w.shape and g.dtype == w.dtype, (t, key)
            if tol == 0:
                assert torch.equal(g, w), (t, key)
            else:
                d = torch.where(torch.isnan(g) & torch.isnan(w), torch.zeros_like(g), (g - w).abs())
                assert not torch.isnan(d).any() and d.max().item() <= tol, (t, key, d.max().item())
        assert int(got["mask"][t].sum()) > 0


def test_train_and_test_entry_points_on_the_reference_nusc_experiment(gold, gold_trees, tmp_path):
    import importlib.util
    import json
    import shutil
    import create_gt_database as tool
    import train as train_tool
    root = gold_trees["nusc"]
    tool.create_reader_database("NUSC", root, MGR.NUSC_INFO, nsweeps=10, host=False)
    shutil.copy(os.path.join(root, MGR.NUSC_INFO), os.path.join(root, "infos_val_10sweeps_withvelo_filterZero.pkl"))
    cdir, work = str(tmp_path / "configs"), str(tmp_path / "work")
    write_experiment(gold, "nusc_det_pp18_aspp_iou_sp", cdir)
    args = ["--config-path", cdir, "--config-name", "nusc_det_pp18_aspp_iou_sp", "--work-dir", work]
    overrides = ["data.train_dataset.root_path=" + root, "trainer.max_epochs=1", "dataloader.train.num_workers=0",
                 "dataloader.val.num_workers=0", "dataloader.train.batch_size=2", "dataloader.val.batch_size=2"]
    np.random.seed(0)
    tr = train_tool.main(args + overrides)
    assert tr.epoch == 1 and os.path.exists(os.path.join(work, "epoch_1.pth"))
    spec = importlib.util.spec_from_file_location("pnx_tools_test", os.path.join(ROOT, "tools", "test.py"))
    test_tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(test_tool)
    results = os.path.join(work, "infos_val_10sweeps_withvelo_filterZero.json")
    os.remove(results)                                     # written by the training run's validation epoch
    res = test_tool.main(args + overrides + ["+load_from=" + os.path.join(work, "epoch_1.pth")])
    assert res is not None and "NDS" in str(res)
    with open(results) as fh:
        out = json.load(fh)
    tokens = {"scene_%d" % s for s in MGR.TREES["nusc"]["seeds"]}
    assert set(out["results"]) == tokens and out["meta"]["use_lidar"]
    for rows in out["results"].values():
        for r in rows:
            assert len(r["rotation"]) == 4 and len(r["translation"]) == 3 and r["detection_name"] and r["attribute_name"]
