"""Build the ground-truth database of the synthetic training scenes, in the reference's layout
(tools/create_gt_database.py there): <data_path>/gt_database_1sweeps_withvelo/<class>/<token>_<class>_<i>.bin holds the
fp32 points [k, 5] of object i of a frame, relative to its box centre, and <data_path>/dbinfos_train_1sweeps_withvelo.pkl
maps each class to its records (name, path, image_idx, gt_idx, box3d_lidar, num_points_in_gt, difficulty, group_id).
DataBaseSamplerV2 (det3d/datasets/pipelines/sample_ops.py) reads both.

The objects are cut with pnx_points_in_boxes_host, the host twin of the GPU point test that removes scene points
during training: the product has one implementation of the reference's points_in_rbbox.

    python tools/create_gt_database.py --data-path data/synth_gts [--config-name synth_det_pp18_aspp_gts] [--n-frames N]
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


def points_in_rbbox(points, boxes):
    """[n, >= 3] fp32 points x [m, 9] fp32 boxes -> [n, m] bool (box_np_ops.points_in_rbbox, libm cosf / sinf)."""
    from det3d.datasets.pipelines.sample_ops import libm_trig
    from pillarnext_b200 import ops
    boxes = np.asarray(boxes, dtype=np.float32).reshape(-1, 9)
    return ops.points_in_boxes_host(np.asarray(points, dtype=np.float32), boxes, libm_trig(boxes[:, -1]))


def create_groundtruth_database(dataset, data_path, used_classes=None, db_path=None, dbinfo_path=None,
                                relative_path=True, nsweeps=1):
    """dataset: a scenes.SyntheticSceneDataset (training seeds).  Returns the dbinfos dict it wrote."""
    if nsweeps != 1:
        raise ValueError("only single-sweep databases are supported")
    root_path = Path(data_path)
    db_path = Path(db_path) if db_path is not None else root_path / f"gt_database_{nsweeps}sweeps_withvelo"
    dbinfo_path = Path(dbinfo_path) if dbinfo_path is not None else root_path / f"dbinfos_train_{nsweeps}sweeps_withvelo.pkl"
    db_path.mkdir(parents=True, exist_ok=True)
    from pillarnext_b200 import scenes
    all_db_infos, group_counter = {}, 0
    for index in range(len(dataset)):
        token = "scene_%d" % (dataset.seed0 + index)
        points, gt_boxes, names = scenes.make_scene(dataset.seed0 + index, dataset.cfg, dataset.n_points, dataset.n_boxes)
        if gt_boxes.shape[0] == 0:
            continue
        inside = points_in_rbbox(points, gt_boxes)
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
                    "num_points_in_gt": gt_points.shape[0], "difficulty": 0, "group_id": group_counter}
            group_counter += 1
            all_db_infos.setdefault(name, []).append(info)
    with open(dbinfo_path, "wb") as fh:
        pickle.dump(all_db_infos, fh)
    return all_db_infos


def main(argv=None):
    from pillarnext_b200 import hydra_lite
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--data-path", required=True)
    ap.add_argument("--config-name", default="synth_det_pp18_aspp_gts")
    ap.add_argument("--n-frames", type=int, default=None, help="training frames to cut (default: the experiment's)")
    a = ap.parse_args(argv)
    cfg = hydra_lite.main(os.path.join(ROOT, "configs", "experiments"), a.config_name, [])
    node = {k: v for k, v in dict(cfg.data.train_dataset).items() if k not in ("sampler", "augmentation")}
    if a.n_frames is not None:
        node["n_frames"] = a.n_frames
    ds = hydra_lite.instantiate(node)
    infos = create_groundtruth_database(ds, a.data_path)
    for k, v in infos.items():
        print(f"load {len(v)} {k} database infos")
    return infos


if __name__ == "__main__":
    main()
