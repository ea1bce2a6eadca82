"""Synthetic LiDAR scenes with LEARNABLE objects + a dataset in the reference's dataset contract (rows F4 / X2).

The benchmark clouds of synth.py carry random labels (fine for throughput, nothing to learn).  For the accuracy gate of
BASELINE.json (mAP on held-out synthetic scenes, product vs reference algorithm) a detector must be able to learn the
task, so here every ground-truth box is an actual cluster of returns: points sampled on the faces of the box that look
towards the sensor, with a density that falls off with range, standing on a ring-scanned ground plane (ground returns
under a box are removed).  Class-dependent sizes make the classes separable.

SyntheticSceneDataset follows det3d/datasets/base.py (`__len__`, `__getitem__`, `evaluation(detections, output_dir)`,
base.py:48-108) as far as the hot path needs it; label assignment is NOT done on the CPU workers (assign.py) -- the
collated batch carries the raw boxes and the detector builds the targets on the GPU (pnx_assign_labels, row F3).
Global augmentation (`augmentation=`, base.py:97-99) is split the same way: the drop-in transforms of
det3d.datasets.pipelines.augmentation draw their parameters here and the detector applies them on the GPU."""
import numpy as np
import torch

from . import hydra_lite, synth

# nominal (dx, dy, dz) per class, metres (nuScenes / Waymo class vocabulary of the reference configs)
CLASS_SIZES = {
    "car": (4.6, 1.9, 1.7), "truck": (6.9, 2.5, 2.8), "construction_vehicle": (6.4, 2.8, 3.2), "bus": (11.0, 2.9, 3.5),
    "trailer": (12.0, 2.9, 3.9), "barrier": (0.5, 2.5, 1.0), "motorcycle": (2.1, 0.8, 1.5), "bicycle": (1.7, 0.6, 1.3),
    "pedestrian": (0.7, 0.7, 1.8), "traffic_cone": (0.4, 0.4, 1.1), "vehicle": (4.7, 2.1, 1.7), "cyclist": (1.8, 0.8, 1.7),
}
GROUND_Z = -1.84


def _box_surface_points(g, box, n):
    """n points on the faces of `box` (x, y, z, dx, dy, dz, yaw) that face the sensor at the origin."""
    x, y, z, dx, dy, dz, yaw = box
    areas = np.array([dy * dz, dy * dz, dx * dz, dx * dz, dx * dy])           # +x, -x, +y, -y, top
    face = g.choice(5, size=4 * n, p=areas / areas.sum())
    u, v = g.uniform(-0.5, 0.5, 4 * n), g.uniform(-0.5, 0.5, 4 * n)
    loc = np.zeros((4 * n, 3))
    nrm = np.zeros((4 * n, 3))
    for f, (axis, sign) in enumerate(((0, 1), (0, -1), (1, 1), (1, -1), (2, 1))):
        m = face == f
        other = [a for a in range(3) if a != axis]
        loc[m, axis] = sign * 0.5
        loc[m, other[0]] = u[m]
        loc[m, other[1]] = v[m]
        nrm[m, axis] = sign
    loc *= np.array([dx, dy, dz])
    c, s = np.cos(yaw), np.sin(yaw)
    R = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    pts = loc @ R.T + np.array([x, y, z])
    nw = nrm @ R.T
    vis = (nw * (np.array([0.0, 0.0, 0.0]) - pts)).sum(1) > 0                   # outward normal towards the sensor
    pts = pts[vis][:n]
    return pts + g.normal(0, 0.02, pts.shape)


def make_scene(seed, cfg, n_points=6000, n_boxes=12):
    """One frame: points [N, 5] fp32 (x, y, z, intensity, time), gt_boxes [M, 9] fp32, gt_names list[str]."""
    g = np.random.default_rng(90000 + seed)
    names_all = [n for t in cfg["tasks"] for n in t]
    pr = cfg["pc_range"]
    half = min(pr[3], pr[4]) * 0.9
    boxes, names = [], []
    tries = 0
    while len(boxes) < n_boxes and tries < 50 * n_boxes:
        tries += 1
        name = names_all[g.integers(0, len(names_all))]
        size = np.array(CLASS_SIZES.get(name, (2.0, 2.0, 2.0))) * g.uniform(0.9, 1.1, 3)
        xy = g.uniform(-half, half, 2)
        if np.hypot(*xy) < 3.0:
            continue
        if any(np.hypot(xy[0] - b[0], xy[1] - b[1]) < 0.6 * (max(size[:2]) + max(b[3:5])) for b in boxes):
            continue
        yaw = g.uniform(-np.pi, np.pi)
        vel = g.normal(0, 1.0, 2) if name not in ("barrier", "traffic_cone") else np.zeros(2)
        boxes.append(np.array([xy[0], xy[1], GROUND_Z + size[2] / 2, size[0], size[1], size[2], vel[0], vel[1], yaw]))
        names.append(name)
    boxes = np.stack(boxes) if boxes else np.zeros((0, 9))
    # ground: the ring scan of synth.make_frame, minus returns under a box
    n_ground = int(n_points * 0.7)
    ground = synth.make_frame(seed, n_ground, cfg, kind="lidar")[:, :3].astype(np.float64)
    keep = np.ones(len(ground), dtype=bool)
    for b in boxes:
        c, s = np.cos(-b[8]), np.sin(-b[8])
        lx = (ground[:, 0] - b[0]) * c - (ground[:, 1] - b[1]) * s
        ly = (ground[:, 0] - b[0]) * s + (ground[:, 1] - b[1]) * c
        keep &= ~((np.abs(lx) < b[3] / 2) & (np.abs(ly) < b[4] / 2))
    parts = [ground[keep]]
    budget = n_points - int(keep.sum())
    if len(boxes):
        w = np.array([(b[3] * b[5] + b[4] * b[5]) / max(np.hypot(b[0], b[1]), 3.0) ** 1.2 for b in boxes])
        per = np.clip((budget * w / w.sum()).astype(int), 25, 600)
        for b, k in zip(boxes, per):
            parts.append(_box_surface_points(g, b[[0, 1, 2, 3, 4, 5, 8]], int(k)))
    xyz = np.concatenate(parts, 0)
    inten = g.uniform(0, cfg["intensity_max"], (len(xyz), 1))
    t = np.zeros((len(xyz), 1))
    pts = np.concatenate([xyz, inten, t], 1).astype(np.float32)
    return pts[g.permutation(len(pts))], boxes.astype(np.float32), names


class SyntheticSceneDataset(torch.utils.data.Dataset):
    """Frames are generated on the fly from (seed0 + index): an unbounded, reproducible stream; train and held-out
    splits are disjoint seed ranges.

    augmentation: dict of `_target_` nodes (or transform objects) applied to every frame in dict order after the scene
    is made, as the reference's BaseDataset does; each appends its record to the frame's `aug` list."""

    def __init__(self, cfg, n_frames, seed0=0, n_points=6000, n_boxes=12, test_mode=False, class_names=None,
                 augmentation=None, **_):
        self.cfg, self.n_frames, self.seed0, self.n_points, self.n_boxes = cfg, int(n_frames), int(seed0), int(n_points), int(n_boxes)
        self.test_mode = test_mode
        self.class_names = [n for t in cfg["tasks"] for n in t]
        if augmentation and test_mode:
            raise ValueError("augmentation is a training transform: a test_mode dataset must not set it")
        self.augmentations = hydra_lite.instantiate(augmentation) if augmentation else None

    def __len__(self):
        return self.n_frames

    def __getitem__(self, i):
        pts, boxes, names = make_scene(self.seed0 + i, self.cfg, self.n_points, self.n_boxes)
        cls = np.array([self.class_names.index(n) for n in names], dtype=np.int32)
        res = {"points": pts, "gt_boxes_raw": boxes, "gt_classes": cls, "token": "scene_%d" % (self.seed0 + i)}
        if self.augmentations is not None:
            for aug in self.augmentations.values():
                res = aug(res)
        return res

    def ground_truth(self):
        gts = {}
        for i in range(self.n_frames):
            _, boxes, names = make_scene(self.seed0 + i, self.cfg, self.n_points, self.n_boxes)
            gts["scene_%d" % (self.seed0 + i)] = {"boxes": boxes, "names": names}
        return gts

    def evaluation(self, detections, output_dir=None, testset=False):
        """The hook the reference trainer calls at the end of val_epoch (base.py:48-51, trainer.py:165-184)."""
        from .evaluate import detection_map
        return detection_map(self.ground_truth(), detections, self.class_names)


def collate(batch_list):
    """loader/collate.py:6-35 for this dataset: points get the frame index prepended; raw boxes are padded to the
    longest frame (class -1 = padding).  Frames with augmentation records add aug [B, 4, 4] float64: frame i's records
    (code, p0, p1, p2) in slots 0.., the rest zero (empty)."""
    pts = [np.pad(b["points"], ((0, 0), (1, 0)), mode="constant", constant_values=i) for i, b in enumerate(batch_list)]
    m = max(1, max(len(b["gt_classes"]) for b in batch_list))
    boxes = np.zeros((len(batch_list), m, 9), dtype=np.float32)
    boxes[:, :, 3:6] = 1.0
    cls = np.full((len(batch_list), m), -1, dtype=np.int32)
    for i, b in enumerate(batch_list):
        k = len(b["gt_classes"])
        boxes[i, :k] = b["gt_boxes_raw"]
        cls[i, :k] = b["gt_classes"]
    out = {"points": torch.tensor(np.concatenate(pts, 0)), "gt_boxes_raw": torch.tensor(boxes), "gt_classes": torch.tensor(cls),
           "token": [b["token"] for b in batch_list]}
    if any("aug" in b for b in batch_list):
        aug = np.zeros((len(batch_list), 4, 4), dtype=np.float64)
        for i, b in enumerate(batch_list):
            rec = b.get("aug", [])
            if len(rec) > 4:
                raise ValueError("at most 4 augmentation records per frame, got %d" % len(rec))
            if rec:
                aug[i, :len(rec)] = rec
        out["aug"] = torch.tensor(aug)
    return out
