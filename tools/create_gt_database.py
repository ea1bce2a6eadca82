"""Build a ground-truth database in the reference's layout (tools/create_gt_database.py there):
<data_path>/gt_database_<n>sweeps_withvelo/<class>/<token>_<class>_<i>.bin holds the fp32 points [k, 5] of object i of a
frame, relative to its box centre, and <data_path>/dbinfos_train_<n>sweeps_withvelo.pkl maps each class to its records
(name, path, image_idx, gt_idx, box3d_lidar, num_points_in_gt, difficulty, group_id).  DataBaseSamplerV2
(det3d/datasets/pipelines/sample_ops.py) reads both.

Two sources of frames:
  * the synthetic training scenes of an experiment (single sweep; the default);
  * --dataset NUSC | WAYMO: the info file of a nuScenes or Waymo tree, read by this package's NuScenesDataset /
    WaymoDataset with create_database=True, as the reference does.  Each frame's sweeps are accumulated by
    ops.accumulate_sweeps, and Waymo keeps the reference's thinning: vehicles on every 4th frame, pedestrians on every
    2nd.
The objects are cut by ops.points_in_boxes, the GPU point test that removes scene points during training (--host: its
host twin, pnx_points_in_boxes_host, and the host twin of the accumulation; the synthetic scenes always use the host
twin).  The product has one implementation of the reference's points_in_rbbox.

    python tools/create_gt_database.py --data-path data/synth_gts [--config-name synth_det_pp18_aspp_gts] [--n-frames N]
    python tools/create_gt_database.py --dataset NUSC --data-path data/nuscenes \\
        --info-path infos_train_10sweeps_withvelo_filterZero.pkl --nsweeps 10
"""
import argparse
import os
import pickle
import sys
from pathlib import Path

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def points_in_rbbox(points, boxes, host=True):
    """[n, >= 3] fp32 points x [m, 9] fp32 boxes -> [n, m] bool (box_np_ops.points_in_rbbox, libm cosf / sinf), on
    the host twin or (host=False) on the GPU."""
    from det3d.datasets.pipelines.sample_ops import libm_trig
    from pillarnext_b200 import ops
    boxes = np.asarray(boxes, dtype=np.float32).reshape(-1, 9)
    points = np.asarray(points, dtype=np.float32)
    if host:
        return ops.points_in_boxes_host(points, boxes, libm_trig(boxes[:, -1]))
    import torch
    cu = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (points, boxes, libm_trig(boxes[:, -1]))]
    return ops.points_in_boxes(*cu).cpu().numpy()


def _write_database(frames, db_path, dbinfo_path, used_classes, relative_path, host):
    """frames: (token, points [n, 5] fp32, gt_boxes [m, 9] fp32, names [m], difficulty [m]) -> the dbinfos it wrote."""
    db_path.mkdir(parents=True, exist_ok=True)
    all_db_infos, group_counter = {}, 0
    for token, points, gt_boxes, names, difficulty in frames:
        if gt_boxes.shape[0] == 0:
            continue
        inside = points_in_rbbox(points, gt_boxes, host)
        for i, name in enumerate(names):
            if used_classes is not None and name not in used_classes:
                continue
            filename = f"{token}_{name}_{i}.bin"
            (db_path / name).mkdir(parents=True, exist_ok=True)
            gt_points = points[inside[:, i]]
            gt_points[:, :3] -= gt_boxes[i, :3]
            gt_points.tofile(str(db_path / name / filename))
            info = {"name": name, "path": os.path.join(db_path.stem, name, filename) if relative_path else
                    str(db_path / name / filename), "image_idx": token, "gt_idx": i, "box3d_lidar": gt_boxes[i],
                    "num_points_in_gt": gt_points.shape[0], "difficulty": difficulty[i], "group_id": group_counter}
            group_counter += 1
            all_db_infos.setdefault(name, []).append(info)
    with open(dbinfo_path, "wb") as fh:
        pickle.dump(all_db_infos, fh)
    return all_db_infos


def _paths(data_path, db_path, dbinfo_path, nsweeps):
    root_path = Path(data_path)
    return (Path(db_path) if db_path is not None else root_path / f"gt_database_{nsweeps}sweeps_withvelo",
            Path(dbinfo_path) if dbinfo_path is not None else root_path / f"dbinfos_train_{nsweeps}sweeps_withvelo.pkl")


def create_groundtruth_database(dataset, data_path, used_classes=None, db_path=None, dbinfo_path=None,
                                relative_path=True, nsweeps=1):
    """dataset: a scenes.SyntheticSceneDataset (training seeds).  Returns the dbinfos dict it wrote."""
    if nsweeps != 1:
        raise ValueError("only single-sweep databases are supported for synthetic scenes")
    from pillarnext_b200 import scenes

    def frames():
        for index in range(len(dataset)):
            seed = dataset.seed0 + index
            points, gt_boxes, names = scenes.make_scene(seed, dataset.cfg, dataset.n_points, dataset.n_boxes)
            yield "scene_%d" % seed, points, gt_boxes, names, [0] * len(names)
    return _write_database(frames(), *_paths(data_path, db_path, dbinfo_path, nsweeps), used_classes, relative_path,
                           host=True)


def frame_points(record, host):
    """The accumulated points [n, 5] of one reader record (its key frame and, if any, its sweeps)."""
    from pillarnext_b200 import ops, scenes
    if "sweeps" not in record:
        return np.asarray(record["points"], np.float32)
    b = scenes.collate([record])
    keys = ("points", "point_offsets", "sweep_points", "sweep_offsets", "sweep_transforms")
    if host:
        pts, count = ops.accumulate_sweeps_host(*[b[k].numpy() for k in keys], b["sweep_min_distance"])
    else:
        pts, count = ops.accumulate_sweeps(*[b[k].cuda() for k in keys], b["sweep_min_distance"])
        pts, count = pts.cpu().numpy(), int(count.cpu()[0])
    return np.ascontiguousarray(pts[:count, 1:])


def create_reader_database(dataset_name, data_path, info_path, used_classes=None, db_path=None, dbinfo_path=None,
                           relative_path=True, nsweeps=1, host=False):
    """The reference's create_groundtruth_database for a nuScenes ("NUSC") or Waymo ("WAYMO") info file.  Returns the
    dbinfos dict it wrote."""
    if dataset_name == "NUSC":
        from det3d.datasets.nuscenes import NuScenesDataset as Dataset
    elif dataset_name == "WAYMO":
        from det3d.datasets.waymo.waymo import WaymoDataset as Dataset
    else:
        raise ValueError("dataset_name must be NUSC or WAYMO, got %r" % (dataset_name,))
    dataset = Dataset(info_path=info_path, root_path=data_path, loading_pipelines=["load_pointcloud", "load_box3d"],
                      nsweeps=nsweeps, create_database=True)

    def frames():
        for index in range(len(dataset)):
            res = dataset[index]
            annos = res["annotations"]
            gt_boxes, names = annos["gt_boxes"], annos["gt_names"]
            if dataset_name == "WAYMO":
                if index % 4 != 0:
                    keep = names != "vehicle"
                    gt_boxes, names = gt_boxes[keep], names[keep]
                if index % 2 != 0:
                    keep = names != "pedestrian"
                    gt_boxes, names = gt_boxes[keep], names[keep]
            if gt_boxes.shape[0] == 0:
                continue
            yield (res.get("token", index), frame_points(res, host), gt_boxes, names,
                   np.zeros(gt_boxes.shape[0], dtype=np.int32))
    return _write_database(frames(), *_paths(data_path, db_path, dbinfo_path, nsweeps), used_classes, relative_path,
                           host)


def main(argv=None):
    from pillarnext_b200 import hydra_lite
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--data-path", required=True)
    ap.add_argument("--config-name", default="synth_det_pp18_aspp_gts")
    ap.add_argument("--n-frames", type=int, default=None, help="training frames to cut (default: the experiment's)")
    ap.add_argument("--dataset", choices=["NUSC", "WAYMO"], default=None, help="read an info file instead")
    ap.add_argument("--info-path", default=None, help="the info pickle, relative to --data-path")
    ap.add_argument("--nsweeps", type=int, default=1)
    ap.add_argument("--host", action="store_true", help="accumulate and cut with the host twins instead of the GPU")
    a = ap.parse_args(argv)
    if a.dataset is not None:
        if a.info_path is None:
            ap.error("--dataset needs --info-path")
        infos = create_reader_database(a.dataset, a.data_path, a.info_path, nsweeps=a.nsweeps, host=a.host)
    else:
        cfg = hydra_lite.main(os.path.join(ROOT, "configs", "experiments"), a.config_name, [])
        node = {k: v for k, v in dict(cfg.data.train_dataset).items() if k not in ("sampler", "augmentation")}
        if a.n_frames is not None:
            node["n_frames"] = a.n_frames
        ds = hydra_lite.instantiate(node)
        infos = create_groundtruth_database(ds, a.data_path, nsweeps=a.nsweeps)
    for k, v in infos.items():
        print(f"load {len(v)} {k} database infos")
    return infos


if __name__ == "__main__":
    main()
