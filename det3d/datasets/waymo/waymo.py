"""Drop-in for the reference's WaymoDataset (det3d/datasets/waymo/waymo.py): the Waymo info-file reader.

Constructor arguments, the info format, the .bin layout (6 fp32 columns: x, y, z, intensity, elongation, no-label-zone
flag; rows with a flag other than -1 dropped), the drop_frames draws and load_box3d (objects without points dropped)
are the reference's.  Difference: load_pointcloud does not transform and merge the sweeps.  With nsweeps > 1 the first
min(nsweeps - 1, len(info["sweeps"])) stored sweeps become the `sweeps` record, each dropped by one np.random.uniform()
draw when drop_frames > 0 (an empty slot), each kept one with its points as stored, time float32(timestamp) and the
transform inv(pose) @ sweep_pose in fp64.  The detector takes them into the key frame on the GPU
(ops.accumulate_sweeps).

evaluation() scores the detections against the infos' objects with evaluate_waymo.waymo_metrics, each box's LEVEL_2
decided by the label's num_points as the Waymo devkit does.  The devkit's protobuf file is not written."""
import os

import numpy as np

from det3d.datasets.base import BaseDataset

# class order of the reference's label_to_type (0 vehicle, 1 pedestrian, otherwise cyclist)
CLASS_NAMES = ["vehicle", "pedestrian", "cyclist"]


class WaymoDataset(BaseDataset):
    def __init__(self, info_path, root_path, nsweeps, drop_frames=0, sampler=None, loading_pipelines=None,
                 augmentation=None, prepare_label=None, tasks=[], evaluations=None, create_database=False,
                 use_gt_sampling=True):
        super().__init__(root_path, info_path, sampler, loading_pipelines, augmentation, prepare_label, evaluations,
                         create_database, use_gt_sampling=use_gt_sampling)
        self.nsweeps = nsweeps
        assert self.nsweeps > 0, "At least input one sweep please!"
        self.drop_frames = drop_frames
        assert 0 <= drop_frames <= 1
        self.tasks = tasks

    def read_file(self, path, timestamp=0):
        points = np.fromfile(os.path.join(self._root_path, path), dtype=np.float32).reshape(-1, 6)
        points = points[points[:, -1] == -1, :4]
        return np.concatenate([points, np.full((len(points), 1), np.float32(timestamp))], 1)

    def load_pointcloud(self, res, info):
        res["points"] = self.read_file("lidar_point/" + info["token"] + ".bin")
        if self.nsweeps == 1:
            return res
        pts, counts, tms = [], [], []
        for sweep in info["sweeps"][:self.nsweeps - 1]:
            if self.drop_frames > 0 and np.random.uniform() < self.drop_frames:
                p, T = np.zeros((0, 5), np.float32), np.full((4, 4), np.nan)
            else:
                p = self.read_file("lidar_point/" + sweep["token"] + ".bin", timestamp=sweep["timestamp"])
                T = np.linalg.inv(info["pose"]) @ sweep["pose"]
            pts.append(p)
            counts.append(len(p))
            tms.append(T)
        res["sweeps"] = {"points": np.concatenate(pts, 0) if pts else np.zeros((0, 5), np.float32),
                         "counts": np.array(counts, np.int64), "transforms": np.stack(tms) if tms else np.zeros((0, 4, 4)),
                         "min_distance": 0.0}
        return res

    def load_box3d(self, res, info):
        annos = info["objects"]
        keep = np.array([ann["num_points"] for ann in annos]).reshape(-1) > 0
        gt_boxes = np.array([ann["box"] for ann in annos]).reshape(-1, 9)[keep]
        gt_names = np.array([ann["label"] for ann in annos])[keep]
        res["annotations"] = {"gt_boxes": gt_boxes.astype(np.float32).copy(), "gt_names": gt_names.copy()}
        return res

    def ground_truth(self):
        """token -> {"boxes" [M, 9] fp32, "names", "num_points" [M]}: every object of the infos."""
        gts = {}
        for info in self.infos:
            objs = info["objects"]
            gts[info["token"]] = {"boxes": np.array([o["box"] for o in objs], np.float32).reshape(-1, 9),
                                  "names": [o["label"] for o in objs],
                                  "num_points": np.array([o["num_points"] for o in objs], np.int64)}
        return gts

    def evaluation(self, detections, output_dir=None):
        from pillarnext_b200.evaluate_waymo import waymo_metrics
        class_names = [n for t in self.tasks for n in t] or CLASS_NAMES
        return waymo_metrics(self.ground_truth(), detections, class_names)
