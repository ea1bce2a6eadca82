"""Drop-in for the reference's NuScenesDataset (det3d/datasets/nuscenes/nusc.py): the nuScenes info-file reader.

Constructor arguments, the info format, the .bin layout (5 fp32 columns, the ring index dropped) and the CBGS
resampling with its np.random.choice draws are the reference's.  Difference: load_pointcloud does not transform and
merge the sweeps.  The key frame gets a time column of 0, and every entry of info["sweeps"] (all of them, whatever
nsweeps says, as the reference loops) becomes one sweep of the `sweeps` record: its points as stored with time
float32(time_lag), its transform_matrix (None = NaN, no transform) and the remove_close radius 1.0.  The detector takes
them into the key frame on the GPU (ops.accumulate_sweeps), with the reference's arithmetic.

evaluation() writes the devkit's results JSON, <info name>.json; the boxes go to the global frame through each info's
ref_from_car and car_from_global matrices (the devkit's pose records are not read).  When the infos carry gt_boxes it
also returns evaluate_nuscenes.nuscenes_metrics, with the points counted in the key-frame files."""
import itertools
import json
import os
from pathlib import Path

import numpy as np

from det3d.datasets.base import BaseDataset
from pillarnext_b200.evaluate_nuscenes import (DEFAULT_ATTRIBUTE, MOVING_ATTRIBUTE, MOVING_SPEED, STILL_ATTRIBUTE,
                                               nuscenes_metrics)


def attribute(name, velocity):
    """The attribute nusc.py:152-185 gives a detection of class `name` with BEV velocity (vx, vy)."""
    moving = np.sqrt(velocity[0] ** 2 + velocity[1] ** 2) > MOVING_SPEED
    return (MOVING_ATTRIBUTE if moving else STILL_ATTRIBUTE).get(name) or DEFAULT_ATTRIBUTE[name]


def _quaternion(R):
    """Unit quaternion (w, x, y, z) of a 3x3 rotation, with w >= 0 (Shepperd's method: full precision at any angle)."""
    t = np.trace(R)
    k = int(np.argmax([t, R[0, 0], R[1, 1], R[2, 2]]))
    if k == 0:
        r = np.sqrt(1.0 + t)
        q = [r / 2, (R[2, 1] - R[1, 2]) / (2 * r), (R[0, 2] - R[2, 0]) / (2 * r), (R[1, 0] - R[0, 1]) / (2 * r)]
    else:
        i, j, m = k - 1, k % 3, (k + 1) % 3
        r = np.sqrt(1.0 + R[i, i] - R[j, j] - R[m, m])
        q = [0.0] * 4
        q[0] = (R[m, j] - R[j, m]) / (2 * r)
        q[1 + i], q[1 + j], q[1 + m] = r / 2, (R[j, i] + R[i, j]) / (2 * r), (R[m, i] + R[i, m]) / (2 * r)
    return [float(-v if q[0] < 0 else v) for v in q]


class NuScenesDataset(BaseDataset):
    def __init__(self, info_path, root_path, nsweeps, sampler=None, loading_pipelines=None, augmentation=None,
                 prepare_label=None, class_names=[], resampling=False, evaluations=None, create_database=False,
                 use_gt_sampling=True, version="v1.0-trainval"):
        super().__init__(root_path, info_path, sampler, loading_pipelines, augmentation, prepare_label, evaluations,
                         create_database, use_gt_sampling=use_gt_sampling)
        self.nsweeps = nsweeps
        assert self.nsweeps > 0, "At least input one sweep please!"
        self._class_names = list(itertools.chain(*[t for t in class_names]))
        self.version = version
        if resampling:
            self.cbgs()

    def cbgs(self):
        """Class-balanced resampling of the infos (nusc.py:50-70), with the reference's np.random.choice draws."""
        cls_infos = {name: [] for name in self._class_names}
        for info in self.infos:
            for name in set(info["gt_names"]):
                if name in self._class_names:
                    cls_infos[name].append(info)
        empty = [k for k, v in cls_infos.items() if not v]
        if empty:
            raise ValueError("CBGS needs every class in some info, none has %s" % empty)
        duplicated = sum(len(v) for v in cls_infos.values())
        frac = 1.0 / len(self._class_names)
        out = []
        for infos in cls_infos.values():
            ratio = frac / (len(infos) / duplicated)
            out += [infos[i] for i in np.random.choice(len(infos), int(len(infos) * ratio))]
        self.infos = out

    def read_file(self, path, num_point_feature=4):
        return np.fromfile(os.path.join(self._root_path, path), dtype=np.float32).reshape(-1, 5)[:, :num_point_feature]

    def load_pointcloud(self, res, info):
        key = self.read_file(str(info["lidar_path"]))
        res["points"] = np.concatenate([key, np.zeros((len(key), 1), np.float32)], 1)
        pts, counts, tms = [], [], []
        for sweep in info["sweeps"]:
            p = self.read_file(str(sweep["lidar_path"]))
            pts.append(np.concatenate([p, np.full((len(p), 1), np.float32(sweep["time_lag"]))], 1))
            counts.append(len(p))
            T = sweep["transform_matrix"]
            tms.append(np.full((4, 4), np.nan) if T is None else np.asarray(T, np.float64))
        res["sweeps"] = {"points": np.concatenate(pts, 0) if pts else np.zeros((0, 5), np.float32),
                         "counts": np.array(counts, np.int64), "transforms": np.stack(tms) if tms else np.zeros((0, 4, 4)),
                         "min_distance": 1.0}
        return res

    def ground_truth(self):
        """token -> {"boxes" [M, 9], "names", "points" [N, 4]} of the infos that carry gt_boxes (key-frame points)."""
        gts = {}
        for info in self.infos:
            if "gt_boxes" in info:
                gts[info["token"]] = {"boxes": np.asarray(info["gt_boxes"], np.float32).reshape(-1, 9),
                                      "names": list(info["gt_names"]), "points": self.read_file(str(info["lidar_path"]))}
        return gts

    def evaluation(self, detections, output_dir=None, testset=False):
        infos = {info["token"]: info for info in self.infos}
        results = {}
        for token, det in detections.items():
            info = infos[token]
            # lidar -> global: the inverse of ref_from_global = ref_from_car @ car_from_global
            to_global = np.linalg.inv(np.asarray(info["ref_from_car"]) @ np.asarray(info["car_from_global"]))
            boxes = np.asarray(det["box3d_lidar"], np.float64).reshape(-1, 9)
            scores = np.asarray(det["scores"], np.float64).reshape(-1)
            labels = np.asarray(det["label_preds"]).reshape(-1)
            annos = []
            for b, s, l in zip(boxes, scores, labels):
                name = self._class_names[int(l)]
                yaw = b[8]
                Rl = np.array([[np.cos(yaw), -np.sin(yaw), 0], [np.sin(yaw), np.cos(yaw), 0], [0, 0, 1]])
                velocity = to_global[:3, :3] @ np.array([b[6], b[7], 0.0])
                annos.append({
                    "sample_token": token,
                    "translation": (to_global[:3, :3] @ b[:3] + to_global[:3, 3]).tolist(),
                    "size": [float(b[4]), float(b[3]), float(b[5])],
                    "rotation": _quaternion(to_global[:3, :3] @ Rl),
                    "velocity": velocity[:2].tolist(),
                    "detection_name": name,
                    "detection_score": float(s),
                    "attribute_name": attribute(name, velocity),
                })
            results[token] = annos
        out = {"results": results, "meta": {"use_camera": False, "use_lidar": True, "use_radar": False,
                                             "use_map": False, "use_external": False}}
        name = str(self._info_path).split("/")[-1].split(".")[0]
        with open(Path(output_dir) / (name + ".json"), "w") as f:
            json.dump(out, f)
        gts = self.ground_truth()
        if testset or not gts:
            return None
        return nuscenes_metrics(gts, detections, self._class_names)
