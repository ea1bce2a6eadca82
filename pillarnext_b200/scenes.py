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
det3d.datasets.pipelines.augmentation draw their parameters here and the detector applies them on the GPU.  So is
ground-truth database sampling (`sampler=`, base.py:36-39, 72-96): det3d.datasets.pipelines.sample_ops draws the
candidate objects here, and the detector runs the collision test, the point removal and the paste on the GPU."""
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


def ego_pose(seed, lag, ego_speed):
    """4x4 fp64 transform from the sensor frame `lag` seconds before key frame `seed` to the key frame: the ego drives a
    seeded planar arc (heading, speed up to ego_speed m/s, yaw rate up to 0.3 rad/s) and sits at the origin at lag 0."""
    g = np.random.default_rng([290000, seed])
    heading, speed, rate = g.uniform(-np.pi, np.pi), ego_speed * g.uniform(0.5, 1.0), g.uniform(-0.3, 0.3)
    th = -rate * lag
    c, s = np.cos(th), np.sin(th)
    T = np.eye(4)
    T[:2, :2] = [[c, -s], [s, c]]
    T[:2, 3] = -speed * lag * np.array([np.cos(heading + th / 2), np.sin(heading + th / 2)])
    return T


def make_sweep(seed, k, cfg, boxes, n_points, sweep_interval=0.05, ego_speed=5.0):
    """Past sweep k >= 1 of key frame `seed` (boxes: its gt_boxes [M, 9]), scanned k * sweep_interval seconds earlier:
    each box at centre - v * lag (v = its vx, vy label; barriers and cones do not move), seen from that sweep's sensor
    pose (ego_pose).  Returns (points [N, 5] fp32 in the sweep's sensor frame with time = float32(lag), like a .bin
    file; transform_matrix [4, 4] fp64 sweep -> key frame; box_index [N] int, the box a point was sampled on or -1).
    Its own seeded streams: the key frame stays exactly make_scene(seed)."""
    lag = k * sweep_interval
    T = ego_pose(seed, lag, ego_speed)
    g = np.random.default_rng([390000, seed, k])
    b = boxes.astype(np.float64).copy()
    b[:, :2] -= b[:, 6:8] * lag                                     # key-frame position at the sweep's time
    R, t = T[:2, :2], T[:2, 3]
    b[:, :2] = (b[:, :2] - t) @ R                                   # into the sweep's sensor frame: R^T (c - t)
    b[:, 8] -= np.arctan2(T[1, 0], T[0, 0])
    ground = synth.make_frame(1000003 * (k + 1) + seed, int(n_points * 0.7), cfg, kind="lidar")[:, :3].astype(np.float64)
    keep = np.ones(len(ground), dtype=bool)
    for bb in b:
        c, s = np.cos(-bb[8]), np.sin(-bb[8])
        lx = (ground[:, 0] - bb[0]) * c - (ground[:, 1] - bb[1]) * s
        ly = (ground[:, 0] - bb[0]) * s + (ground[:, 1] - bb[1]) * c
        keep &= ~((np.abs(lx) < bb[3] / 2) & (np.abs(ly) < bb[4] / 2))
    parts, owner = [ground[keep]], [np.full(int(keep.sum()), -1)]
    budget = n_points - int(keep.sum())
    if len(b):
        w = np.array([(bb[3] * bb[5] + bb[4] * bb[5]) / max(np.hypot(bb[0], bb[1]), 3.0) ** 1.2 for bb in b])
        per = np.clip((budget * w / w.sum()).astype(int), 25, 600)
        for j, (bb, m) in enumerate(zip(b, per)):
            parts.append(_box_surface_points(g, bb[[0, 1, 2, 3, 4, 5, 8]], int(m)))
            owner.append(np.full(len(parts[-1]), j))
    xyz, owner = np.concatenate(parts, 0), np.concatenate(owner, 0)
    inten = g.uniform(0, cfg["intensity_max"], (len(xyz), 1))
    pts = np.concatenate([xyz, inten, np.full((len(xyz), 1), np.float32(lag))], 1).astype(np.float32)
    order = g.permutation(len(pts))
    return pts[order], T, owner[order]


def sampling_record(sampler, boxes, names, class_names):
    """The `gts` record of one frame: the candidates sampler.sample_all draws for the scene boxes [M, 9] fp32 named
    `names` (none drawn = zero candidates), their classes as indices into class_names, and numpy's (cos, sin) of the
    scene boxes' yaws."""
    from det3d.datasets.pipelines.sample_ops import numpy_trig
    rec = sampler.sample_all(boxes, np.array(names))
    if rec is None:
        rec = {"gt_names": np.zeros(0, dtype=str), "gt_boxes": np.zeros((0, 9), np.float32),
               "points": np.zeros((0, 5), np.float32), "num_points": np.zeros(0, np.int64),
               "trig": np.zeros((0, 4), np.float32)}
    if rec["points"].shape[1] != 5:
        raise ValueError("the sampler's point_dim must be 5 (x, y, z, intensity, time), got %d" % rec["points"].shape[1])
    unknown = sorted(set(rec["gt_names"]) - set(class_names))
    if unknown:
        raise ValueError("sampled classes %s are not classes of this dataset" % unknown)
    return {"boxes": rec["gt_boxes"], "classes": np.array([class_names.index(n) for n in rec["gt_names"]], np.int32),
            "points": rec["points"], "num_points": rec["num_points"], "trig": rec["trig"],
            "scene_trig": numpy_trig(boxes)}


class SyntheticSceneDataset(torch.utils.data.Dataset):
    """Frames are generated on the fly from (seed0 + index): an unbounded, reproducible stream; train and held-out
    splits are disjoint seed ranges.

    augmentation: dict of `_target_` nodes (or transform objects) applied to every frame in dict order after the scene
    is made, as the reference's BaseDataset does; each appends its record to the frame's `aug` list.

    sampler: the reference's `_partial_` DataBaseSamplerV2 node (or a callable returning a sampler), called once here
    as base.py does.  Each frame then gets a `gts` record before augmentation draws anything: the candidate objects
    (sample_ops.DataBaseSamplerV2.sample_all; none drawn = zero candidates) and numpy's (cos, sin) of the scene boxes'
    yaws.  root_path is where the sampler node's `${data.train_dataset.root_path}` points (the gt database).

    nsweeps, drop_frames: past sweeps accumulated into every frame, as the reference's nuScenes (nsweeps 10) and Waymo
    (nsweeps 3, drop_frames 0.5 in training) datasets do.  With nsweeps > 1 each frame gets a `sweeps` record of its
    nsweeps - 1 past sweeps (make_sweep: the ego and the objects move, sweep_interval seconds apart, the ego at up to
    ego_speed m/s); each is dropped with probability drop_frames by one np.random.uniform() draw per sweep, in sweep
    order and before the sampler and the augmentation draw anything (waymo.py:55-57, base.py:69-99).  The detector
    takes the sweeps into the key frame on the GPU (ops.accumulate_sweeps), dropping the sweep points within
    min_distance of the sensor in x and y (nuScenes' remove_close; 0 = off).  nsweeps = 1 frames are unchanged.

    metric: what evaluation() reports -- "nuscenes" (evaluate.detection_map), "waymo" (evaluate_waymo.waymo_metrics,
    AP / APH at LEVEL_1 and LEVEL_2) or "nds" (evaluate_nuscenes.nuscenes_metrics, the nuScenes detection score with
    its true-positive errors).  For "waymo" and "nds" ground_truth() also hands over each frame's points."""

    def __init__(self, cfg, n_frames, seed0=0, n_points=6000, n_boxes=12, test_mode=False, class_names=None,
                 augmentation=None, sampler=None, root_path=None, metric="nuscenes", nsweeps=1, drop_frames=0.0,
                 sweep_interval=0.05, ego_speed=5.0, min_distance=1.0, **_):
        if int(nsweeps) < 1 or not 0.0 <= drop_frames <= 1.0 or min_distance < 0:
            raise ValueError("nsweeps must be >= 1, drop_frames in [0, 1] and min_distance >= 0, got %r, %r, %r"
                             % (nsweeps, drop_frames, min_distance))
        self.nsweeps, self.drop_frames = int(nsweeps), float(drop_frames)
        self.sweep_interval, self.ego_speed, self.min_distance = float(sweep_interval), float(ego_speed), float(min_distance)
        self.cfg, self.n_frames, self.seed0, self.n_points, self.n_boxes = cfg, int(n_frames), int(seed0), int(n_points), int(n_boxes)
        self.test_mode = test_mode
        if metric not in ("nuscenes", "waymo", "nds"):
            raise ValueError("metric must be 'nuscenes', 'waymo' or 'nds', got %r" % (metric,))
        self.metric = metric
        self.class_names = [n for t in cfg["tasks"] for n in t]
        if augmentation and test_mode:
            raise ValueError("augmentation is a training transform: a test_mode dataset must not set it")
        self.augmentations = hydra_lite.instantiate(augmentation) if augmentation else None
        if sampler and test_mode:
            raise ValueError("sampler is a training transform: a test_mode dataset must not set it")
        self.root_path = root_path
        self.sampler = None
        if sampler:
            self.sampler = (hydra_lite.instantiate(sampler) if isinstance(sampler, dict) else sampler)()

    def __len__(self):
        return self.n_frames

    def __getitem__(self, i):
        pts, boxes, names = make_scene(self.seed0 + i, self.cfg, self.n_points, self.n_boxes)
        cls = np.array([self.class_names.index(n) for n in names], dtype=np.int32)
        res = {"points": pts, "gt_boxes_raw": boxes, "gt_classes": cls, "token": "scene_%d" % (self.seed0 + i)}
        if self.nsweeps > 1:
            res["sweeps"] = self._sweeps(self.seed0 + i, boxes)
        if self.sampler is not None:
            res["gts"] = self._candidates(boxes, names)
        if self.augmentations is not None:
            for aug in self.augmentations.values():
                res = aug(res)
        return res

    def _sweeps(self, seed, boxes):
        kept = [not (self.drop_frames > 0 and np.random.uniform() < self.drop_frames) for _ in range(self.nsweeps - 1)]
        pts, counts, tms = [], [], []
        for k, keep in enumerate(kept, 1):
            if keep:
                p, T, _ = make_sweep(seed, k, self.cfg, boxes, self.n_points, self.sweep_interval, self.ego_speed)
            else:
                p, T = np.zeros((0, 5), np.float32), np.full((4, 4), np.nan)
            pts.append(p)
            counts.append(len(p))
            tms.append(T)
        return {"points": np.concatenate(pts, 0), "counts": np.array(counts, np.int64), "transforms": np.stack(tms),
                "min_distance": self.min_distance}

    def _candidates(self, boxes, names):
        return sampling_record(self.sampler, boxes, names, self.class_names)

    def ground_truth(self):
        gts = {}
        for i in range(self.n_frames):
            pts, boxes, names = make_scene(self.seed0 + i, self.cfg, self.n_points, self.n_boxes)
            gts["scene_%d" % (self.seed0 + i)] = {"boxes": boxes, "names": names}
            if self.metric in ("waymo", "nds"):
                gts["scene_%d" % (self.seed0 + i)]["points"] = pts
        return gts

    def evaluation(self, detections, output_dir=None, testset=False):
        """The hook the reference trainer calls at the end of val_epoch (base.py:48-51, trainer.py:165-184)."""
        if self.metric == "waymo":
            from .evaluate_waymo import waymo_metrics
            return waymo_metrics(self.ground_truth(), detections, self.class_names)
        if self.metric == "nds":
            from .evaluate_nuscenes import nuscenes_metrics
            return nuscenes_metrics(self.ground_truth(), detections, self.class_names)
        from .evaluate import detection_map
        return detection_map(self.ground_truth(), detections, self.class_names)


def collate(batch_list):
    """loader/collate.py:6-35 for this dataset: points get the frame index prepended; raw boxes are padded to the
    longest frame (class -1 = padding).  Frames with augmentation records add aug [B, 4, 4] float64: frame i's records
    (code, p0, p1, p2) in slots 0.., the rest zero (empty).  Frames with sampling records (`gts`) add, with S the most
    candidates of any frame (at least 1):
      gts_boxes [B, S, 9] fp32, gts_classes [B, S] int32 (-1 = padding), gts_trig [B, S, 4] fp32   the candidates
      gts_points [P, 5] fp32, gts_offsets [B S + 1] int32    their stored points; candidate (b, s) owns rows
                                                             gts_offsets[b S + s] .. gts_offsets[b S + s + 1] - 1
      gt_trig [B, M, 2] fp32                                 numpy's (cos, sin) of the scene boxes' yaws
    Frames with past sweeps (`sweeps`) add, with K the most sweeps of any frame (a dropped sweep is an empty slot):
      point_offsets [B + 1] int32              frame f's key-frame points are rows point_offsets[f] .. [f + 1] - 1
      sweep_points [S, 5] fp32, sweep_offsets [B K + 1] int32   sweep (f, k) owns rows sweep_offsets[f K + k] .. - 1
      sweep_transforms [B, K, 4, 4] fp64       sweep -> key frame (NaN = no transform)
      sweep_min_distance float                 the close-point radius of ops.accumulate_sweeps"""
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
    if any("gts" in b for b in batch_list):
        if not all("gts" in b for b in batch_list):
            raise ValueError("either every frame of a batch carries a sampling record (gts) or none does")
        B = len(batch_list)
        s = max(1, max(len(b["gts"]["classes"]) for b in batch_list))
        cb = np.zeros((B, s, 9), dtype=np.float32)
        cb[:, :, 3:6] = 1.0
        cc = np.full((B, s), -1, dtype=np.int32)
        ct = np.zeros((B, s, 4), dtype=np.float32)
        ct[:, :, 0], ct[:, :, 2] = 1.0, 1.0
        st = np.zeros((B, m, 2), dtype=np.float32)
        st[:, :, 0] = 1.0
        counts = np.zeros((B, s), dtype=np.int64)
        for i, b in enumerate(batch_list):
            g = b["gts"]
            k = len(g["classes"])
            cb[i, :k], cc[i, :k], ct[i, :k], counts[i, :k] = g["boxes"], g["classes"], g["trig"], g["num_points"]
            st[i, :len(g["scene_trig"])] = g["scene_trig"]
        off = np.concatenate([[0], np.cumsum(counts.reshape(-1))])
        if off[-1] + len(out["points"]) >= 2 ** 31 - 1:
            raise ValueError("too many points in one batch for int32 offsets")
        pts = [b["gts"]["points"] for b in batch_list]
        out.update(gts_boxes=torch.tensor(cb), gts_classes=torch.tensor(cc), gts_trig=torch.tensor(ct),
                   gts_points=torch.tensor(np.concatenate(pts, 0).astype(np.float32).reshape(-1, 5)),
                   gts_offsets=torch.tensor(off.astype(np.int32)), gt_trig=torch.tensor(st))
    if any("sweeps" in b for b in batch_list):
        if not all("sweeps" in b for b in batch_list):
            raise ValueError("either every frame of a batch carries past sweeps or none does")
        md = {b["sweeps"]["min_distance"] for b in batch_list}
        if len(md) != 1:
            raise ValueError("the frames of a batch must share one min_distance, got %s" % sorted(md))
        B = len(batch_list)
        K = max(1, max(len(b["sweeps"]["counts"]) for b in batch_list))
        counts = np.zeros((B, K), np.int64)
        tms = np.full((B, K, 4, 4), np.nan)
        for i, b in enumerate(batch_list):
            sw = b["sweeps"]
            counts[i, :len(sw["counts"])], tms[i, :len(sw["counts"])] = sw["counts"], sw["transforms"]
        off = np.concatenate([[0], np.cumsum(counts.reshape(-1))])
        if off[-1] + len(out["points"]) >= 2 ** 31 - 1:
            raise ValueError("too many points in one batch for int32 offsets")
        key = np.concatenate([[0], np.cumsum([len(b["points"]) for b in batch_list])])
        out.update(point_offsets=torch.tensor(key.astype(np.int32)),
                   sweep_points=torch.tensor(np.concatenate([b["sweeps"]["points"] for b in batch_list], 0)
                                             .astype(np.float32).reshape(-1, 5)),
                   sweep_offsets=torch.tensor(off.astype(np.int32)), sweep_transforms=torch.tensor(tms),
                   sweep_min_distance=float(md.pop()))
    return out
