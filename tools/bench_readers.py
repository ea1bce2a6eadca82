"""Throughput of the nuScenes and Waymo info-file readers, and of the GPU point test that cuts the ground-truth database.

  * DataLoader frames/s (det3d.datasets.loader.build_dataloader, batch 4) at 0, 4 and 16 workers over seeded fixture
    trees (oracle/reader_fixtures.py) at the scale of the reference's experiments: nuScenes 10 sweeps x 26.5k points
    with the sampler and the augmentation, Waymo 3 sweeps x 180k points with drop_frames 0.5.  The trees are written to
    a temporary directory.
  * tools/create_gt_database.py --dataset NUSC per frame: the GPU path (ops.accumulate_sweeps + ops.points_in_boxes)
    against the host twins.
  * ops.points_in_boxes on one 10 x 26.5k-point frame with 60 boxes (CUDA events) against points_in_boxes_host.
The card name, power limit and SM clocks are printed with the numbers, because every number depends on them.

    python tools/bench_readers.py [--frames 16] [--json out.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import create_gt_database as tool  # noqa: E402
from gemm_shape_table import card  # noqa: E402
from oracle import reader_fixtures as RF  # noqa: E402
from pillarnext_b200 import hydra_lite, ops  # noqa: E402

NUSC_TASKS = [["car"], ["truck", "construction_vehicle"], ["bus", "trailer"], ["barrier"], ["motorcycle", "bicycle"],
              ["pedestrian", "traffic_cone"]]
WAYMO_TASKS = [["vehicle"], ["pedestrian", "cyclist"]]
AUG = {k: dict(v, _target_="det3d.datasets.pipelines.augmentation." + n) for k, n, v in (
    ("rotation", "Rotation", {"rotation": [-0.785, 0.785]}), ("scaling", "Scaling", {"scale": [0.9, 1.1]}),
    ("translation", "Translation", {"noise": 0.5}), ("flip", "Flip", {"flip_prob": [0.5, 0.5]}))}


def scene_cfg(tasks, half):
    return dict(tasks=tasks, pc_range=[-half, -half, -5.0, half, half, 3.0], voxel_size=[0.075, 0.075, 8],
                intensity_max=255.0, xy_extent=half, z_range=[-5.0, 3.0])


def label(tasks, half):
    return {"centermap": {"_target_": "det3d.datasets.pipelines.assign.AssignLabel", "gaussian_overlap": 0.1,
                          "max_objs": 500, "min_radius": 2, "tasks": tasks, "pc_range": [-half, -half, -5.0, half, half, 3.0],
                          "voxel_size": [0.075, 0.075, 8], "out_size_factor": [4] * len(tasks)}}


def loader_rate(node, workers, epochs=2):
    from det3d.datasets.loader.build_loader import build_dataloader
    ds = hydra_lite.instantiate(node)
    dl = build_dataloader(ds, batch_size=4, num_workers=workers, shuffle=True)
    for _ in dl:                                                         # warm-up epoch: worker start, page cache
        pass
    t0, n = time.perf_counter(), 0
    for _ in range(epochs):
        for b in dl:
            n += len(b["token"])
    return n / (time.perf_counter() - t0)


def time_points_in_boxes(pts, boxes, trig, iters=50):
    cu = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (pts, boxes, trig)]
    for _ in range(5):
        ops.points_in_boxes(*cu)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        ops.points_in_boxes(*cu)
    b.record()
    torch.cuda.synchronize()
    gpu_us = 1000 * a.elapsed_time(b) / iters
    t = []
    for _ in range(3):
        t0 = time.perf_counter()
        ops.points_in_boxes_host(pts, boxes, trig)
        t.append(time.perf_counter() - t0)
    return dict(points=len(pts), boxes=len(boxes), gpu_us=gpu_us, host_ms=1000 * float(np.median(t)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16, help="frames per fixture tree")
    ap.add_argument("--workers", default="0,4,16")
    ap.add_argument("--json", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_readers.py needs a CUDA device")
    torch.cuda.set_device(0)
    gpu = card()
    print("card: %s" % gpu)
    seeds = list(range(100, 100 + args.frames))
    out = dict(card=gpu, loader={})
    with tempfile.TemporaryDirectory() as tmp:
        nroot, wroot = os.path.join(tmp, "nusc"), os.path.join(tmp, "waymo")
        RF.write_nusc(nroot, seeds, scene_cfg(NUSC_TASKS, 50.4), n_points=26500, n_boxes=40, nan_velocity=0.1)
        RF.write_waymo(wroot, seeds, scene_cfg(WAYMO_TASKS, 76.8), n_points=180000, n_boxes=60, nsweeps=3)
        info = "infos_train_10sweeps_withvelo_filterZero.pkl"
        db = {}
        for host in (False, True):
            t0 = time.perf_counter()
            tool.create_reader_database("NUSC", nroot, info, nsweeps=10, host=host)
            db["host" if host else "gpu"] = 1000 * (time.perf_counter() - t0) / len(seeds)
        out["gt_database_ms_per_frame"] = db
        print("create_gt_database NUSC, 10 sweeps x 26.5k points, per frame: GPU path %.1f ms, host twins %.1f ms"
              % (db["gpu"], db["host"]))
        smp = {"_target_": "det3d.datasets.pipelines.sample_ops.DataBaseSamplerV2", "_partial_": True, "root_path": nroot,
               "dbinfo_path": "dbinfos_train_10sweeps_withvelo.pkl", "groups": [{"car": 2, "pedestrian": 2, "barrier": 2}],
               "db_prepor": None, "rate": 1.0, "gt_drop_percentage": 0, "gt_drop_max_keep_points": -1, "point_dim": 5}
        nodes = {
            "nusc_10x26.5k": {"_target_": "det3d.datasets.nuscenes.NuScenesDataset", "nsweeps": 10, "root_path": nroot,
                              "info_path": info, "class_names": NUSC_TASKS, "sampler": smp, "augmentation": AUG,
                              "loading_pipelines": ["load_pointcloud", "load_box3d"], "prepare_label": label(NUSC_TASKS, 50.4)},
            "waymo_3x180k": {"_target_": "det3d.datasets.waymo.waymo.WaymoDataset", "nsweeps": 3, "drop_frames": 0.5,
                             "root_path": wroot, "info_path": "waymo_infos_train.pkl", "augmentation": AUG,
                             "loading_pipelines": ["load_pointcloud", "load_box3d"], "prepare_label": label(WAYMO_TASKS, 76.8)}}
        for name, node in nodes.items():
            for w in [int(x) for x in args.workers.split(",")]:
                r = loader_rate(node, w)
                out["loader"]["%s_workers%d" % (name, w)] = r
                print("DataLoader %s, batch 4, %2d workers: %8.1f frames/s" % (name, w, r))
        from det3d.datasets.pipelines.sample_ops import libm_trig
        ds = hydra_lite.instantiate(dict(nodes["nusc_10x26.5k"], sampler=None, augmentation=None, prepare_label=None,
                                         create_database=True))
        rec = ds[0]
        pts = tool.frame_points(rec, host=True)
        g = np.random.default_rng(1)
        gt = rec["annotations"]["gt_boxes"]
        boxes = np.concatenate([gt] * (60 // len(gt) + 1))[:60].copy()      # the frame's boxes, copies moved aside
        boxes[len(gt):, :2] += g.uniform(-5, 5, (60 - len(gt), 2)).astype(np.float32)
        pib = time_points_in_boxes(pts, boxes, libm_trig(boxes[:, 8]))
        out["points_in_boxes"] = pib
        print("ops.points_in_boxes %d points x %d boxes: %.1f us (CUDA events); points_in_boxes_host %.1f ms"
              % (pib["points"], pib["boxes"], pib["gpu_us"], pib["host_ms"]))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
