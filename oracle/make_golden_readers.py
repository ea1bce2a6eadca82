"""Freeze the reference's OWN info-file readers into tests/golden/ref_readers.npz (TEST INFRASTRUCTURE; run where the
reference tree is present).

The reference's NuScenesDataset, WaymoDataset, AssignLabel, DataBaseSamplerV2, global augmentation transforms and
tools/create_gt_database.py run on the seeded trees of oracle/reader_fixtures.py, written to a temporary root; the
packages they import but these paths never use are stubbed in sys.modules (the pattern of make_golden_sweeps.py).
Cases (trees: TREES below):
  nusc   10 sweeps (one stored with transform_matrix None), NaN velocities; the reference's 10-sweep database is built
         first (its dbinfos and per-file SHA-256 are frozen), then __getitem__ with that sampler, the four augmentation
         transforms and AssignLabel, create_database=True, np.random.seed(SEED) before the dataset is built and
         SEED + 1 before the frames are read: per frame the final points and annotations
  waymo  3 sweeps, drop_frames 0.5, random poses: the points after load_pointcloud, the annotations (0-point objects
         dropped) and AssignLabel's targets (hm, anno_box, ind, mask, cat, gt_boxes per task)
  f1     the same tree with nsweeps 1: points and annotations
  cbgs   NuScenesDataset(resampling=True) on the nusc tree under np.random.seed(SEED): the info token order
  wdb    the reference's single-sweep Waymo database of an 8-frame tree (the every-4th / every-2nd-frame thinning)
  cfg    the reference's nusc_det_pp18_aspp_iou_sp and waymo_det_pp18_aspp_iou_car_sp experiments composed by
         pillarnext_b200.hydra_lite (unresolved, JSON): the data nodes and the whole experiment tools/train.py reads
Stored keys: <case>_<frame>_points / _boxes / _names, waymo_<frame>_<target>_<task>, <db>_dbinfos (JSON: every
record without its box, in dbinfos order), <db>_boxes [R, 9], <db>_sha256 (JSON: relative path -> digest),
cbgs_tokens, cbgs_classes, cfg_<experiment> (JSON).

    python -m oracle.make_golden_readers
"""
import contextlib
import hashlib
import importlib
import importlib.util
import json
import os
import sys
import tempfile

import numpy as np

from oracle import make_golden_sweeps as MGS
from oracle import reader_fixtures as RF
from oracle import reference_loader
from pillarnext_b200 import hydra_lite

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SEED = 31
NUSC_TASKS = [["car"], ["truck", "construction_vehicle"], ["bus", "trailer"], ["barrier"], ["motorcycle", "bicycle"],
              ["pedestrian", "traffic_cone"]]
WAYMO_TASKS = [["vehicle"], ["pedestrian", "cyclist"]]
# the fixture trees: writer keyword arguments shared by this script and tests/test_readers_cpu.py
TREES = {
    "nusc": dict(seeds=[11, 12, 13], n_points=400, n_boxes=10, nsweeps=10, nan_velocity=0.3, none_transform=True,
                 half=50.4),
    "waymo": dict(seeds=[21, 22, 23], n_points=900, n_boxes=10, nsweeps=3, empty_objects=2, half=76.8),
    "wdb": dict(seeds=list(range(31, 39)), n_points=500, n_boxes=8, nsweeps=1, half=76.8),
}
NUSC_GROUPS = {"car": 3, "pedestrian": 3, "barrier": 2, "bicycle": 2}
LABEL = dict(gaussian_overlap=0.1, max_objs=500, min_radius=2, voxel_size=[0.32, 0.32, 8])
NUSC_INFO = "infos_train_10sweeps_withvelo_filterZero.pkl"
WAYMO_INFO = "waymo_infos_train.pkl"


def scene_cfg(tasks, half):
    return dict(tasks=tasks, pc_range=[-half, -half, -5.0, half, half, 3.0], voxel_size=[0.075, 0.075, 8],
                intensity_max=255.0, xy_extent=half, z_range=[-5.0, 3.0])


def write_tree(name, root):
    t = dict(TREES[name])
    seeds, half = t.pop("seeds"), t.pop("half")
    if name == "nusc":
        return RF.write_nusc(root, seeds, scene_cfg(NUSC_TASKS, half), **t)
    return RF.write_waymo(root, seeds, scene_cfg(WAYMO_TASKS, half), **t)


def label_args(tasks, half):
    return dict(LABEL, tasks=tasks, pc_range=[-half, -half, -5.0, half, half, 3.0], out_size_factor=[4] * len(tasks))


def db_record(dbinfos, root, db_dir):
    """(JSON of the records without boxes, boxes [R, 9] fp32, JSON of path -> SHA-256) of a database."""
    recs, boxes = [], []
    for name, infos in dbinfos.items():
        for r in infos:
            recs.append({k: (v.item() if hasattr(v, "item") else v) for k, v in r.items() if k != "box3d_lidar"})
            recs[-1]["difficulty_dtype"] = str(np.asarray(r["difficulty"]).dtype)
            boxes.append(np.asarray(r["box3d_lidar"], np.float32))
    sha = {}
    for dp, _, fs in os.walk(os.path.join(root, db_dir)):
        for f in fs:
            with open(os.path.join(dp, f), "rb") as fh:
                sha[os.path.relpath(os.path.join(dp, f), root)] = hashlib.sha256(fh.read()).hexdigest()
    return json.dumps(recs), np.stack(boxes), json.dumps(sha, sort_keys=True)


@contextlib.contextmanager
def reference():
    """The reference's det3d in sys.modules (this repo's set aside), its tools/create_gt_database.py as a module."""
    saved = {k: v for k, v in sys.modules.items() if k == "det3d" or k.startswith("det3d.") or k in MGS.STUBS}
    for k in saved:
        del sys.modules[k]
    for k in MGS.STUBS:
        sys.modules[k] = MGS._Stub(k)
    sys.path.insert(0, reference_loader.REF_ROOT)
    try:
        importlib.import_module("det3d")
        spec = importlib.util.spec_from_file_location(
            "ref_create_gt_database", os.path.join(reference_loader.REF_ROOT, "tools", "create_gt_database.py"))
        tool = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(tool)
        tool.tqdm = iter                          # the progress bar (stubbed) only wraps the frame loop
        yield dict(nusc=importlib.import_module("det3d.datasets.nuscenes.nusc").NuScenesDataset,
                   waymo=importlib.import_module("det3d.datasets.waymo.waymo").WaymoDataset,
                   assign=importlib.import_module("det3d.datasets.pipelines.assign").AssignLabel,
                   sample_ops=importlib.import_module("det3d.datasets.pipelines.sample_ops"),
                   aug=importlib.import_module("det3d.datasets.pipelines.augmentation"), tool=tool)
    finally:
        sys.path.remove(reference_loader.REF_ROOT)
        for k in [k for k in sys.modules if k == "det3d" or k.startswith("det3d.") or k in MGS.STUBS]:
            del sys.modules[k]
        sys.modules.update(saved)


def frames(ds, seed, out, case, targets=False):
    np.random.seed(seed)
    for i in range(len(ds)):
        res = ds[i]
        a = res["annotations"]
        out["%s_%d_points" % (case, i)] = np.asarray(res["points"], np.float32)
        out["%s_%d_boxes" % (case, i)] = np.asarray(a["gt_boxes"], np.float32)
        out["%s_%d_names" % (case, i)] = np.array(a["gt_names"], dtype=str)
        if targets:
            for key in ("hm", "anno_box", "ind", "mask", "cat", "gt_boxes"):
                for t, v in enumerate(res[key]):
                    out["%s_%d_%s_%d" % (case, i, key, t)] = v


def main():
    out = {}
    cfg_dir = os.path.join(reference_loader.REF_ROOT, "configs", "experiments")
    for exp in ("nusc_det_pp18_aspp_iou_sp", "waymo_det_pp18_aspp_iou_car_sp"):
        out["cfg_" + exp] = json.dumps(hydra_lite.compose(cfg_dir, exp))
    with tempfile.TemporaryDirectory() as tmp:
        nroot, wroot, droot = (os.path.join(tmp, n) for n in ("nusc", "waymo", "wdb"))
        write_tree("nusc", nroot)
        write_tree("waymo", wroot)
        write_tree("wdb", droot)
        with reference() as R:
            run(R, out, nroot, wroot, droot)
    path = os.path.join(GOLDEN, "ref_readers.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: %d arrays, %d bytes" % (path, len(out), os.path.getsize(path)))


def run(R, out, nroot, wroot, droot):
    """Every case that runs the reference's code (module docstring)."""
    import pickle
    # nuScenes: the 10-sweep database, then training frames through sampler + augmentation + AssignLabel
    R["tool"].create_groundtruth_database("NUSC", nroot, NUSC_INFO, nsweeps=10)
    with open(os.path.join(nroot, "dbinfos_train_10sweeps_withvelo.pkl"), "rb") as fh:
        dbinfos = pickle.load(fh)
    out["ndb_dbinfos"], out["ndb_boxes"], out["ndb_sha256"] = db_record(dbinfos, nroot, "gt_database_10sweeps_withvelo")
    so = R["sample_ops"]

    def sampler():
        return so.DataBaseSamplerV2(
            root_path=nroot, dbinfo_path="dbinfos_train_10sweeps_withvelo.pkl", groups=[dict(NUSC_GROUPS)],
            db_prepor={"filter_by_num": so.DBFilterByMinNumPoint({k: 5 for k in NUSC_GROUPS})}, rate=1.0,
            gt_drop_percentage=0, gt_drop_max_keep_points=-1, point_dim=5)
    aug = {"rotation": R["aug"].Rotation([-0.785, 0.785]), "scaling": R["aug"].Scaling([0.9, 1.1]),
           "translation": R["aug"].Translation(0.5), "flip": R["aug"].Flip([0.5, 0.5])}
    np.random.seed(SEED)
    ds = R["nusc"](NUSC_INFO, nroot, 10, sampler=sampler, loading_pipelines=["load_pointcloud", "load_box3d"],
                   augmentation=aug, prepare_label={"centermap": R["assign"](**label_args(NUSC_TASKS, 50.4))},
                   class_names=NUSC_TASKS, create_database=True)
    frames(ds, SEED + 1, out, "nusc")
    # Waymo: 3 sweeps with drop_frames, and 1 sweep
    ds = R["waymo"](WAYMO_INFO, wroot, 3, drop_frames=0.5, loading_pipelines=["load_pointcloud", "load_box3d"],
                    prepare_label={"centermap": R["assign"](**label_args(WAYMO_TASKS, 76.8))}, create_database=True)
    frames(ds, SEED + 1, out, "waymo", targets=True)
    ds = R["waymo"](WAYMO_INFO, wroot, 1, loading_pipelines=["load_pointcloud", "load_box3d"], create_database=True)
    frames(ds, SEED + 1, out, "f1")
    # CBGS on the classes the nuScenes tree holds
    ds = R["nusc"](NUSC_INFO, nroot, 10, loading_pipelines=["load_pointcloud"])
    names = [n for t in NUSC_TASKS for n in t]
    present = sorted({n for i in ds.infos for n in i["gt_names"]}, key=names.index)
    np.random.seed(SEED)
    ds = R["nusc"](NUSC_INFO, nroot, 10, class_names=[[n] for n in present], resampling=True)
    out["cbgs_classes"], out["cbgs_tokens"] = np.array(present), np.array([i["token"] for i in ds.infos])
    # Waymo single-sweep database with the thinning
    R["tool"].create_groundtruth_database("WAYMO", droot, WAYMO_INFO, nsweeps=1)
    with open(os.path.join(droot, "dbinfos_train_1sweeps_withvelo.pkl"), "rb") as fh:
        dbinfos = pickle.load(fh)
    out["wdb_dbinfos"], out["wdb_boxes"], out["wdb_sha256"] = db_record(dbinfos, droot, "gt_database_1sweeps_withvelo")


if __name__ == "__main__":
    main()
