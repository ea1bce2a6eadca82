"""Seeded nuScenes and Waymo info trees built from the synthetic scenes of pillarnext_b200.scenes (TEST FIXTURES; pure
numpy plus the scene generator, so they can be written anywhere the package imports).

write_nusc(root, seeds, cfg, ...) writes the nuScenes layout the reference's NuScenesDataset reads:
  samples/LIDAR_TOP/<token>.bin     the key frame of scenes.make_scene, 5 fp32 columns (x, y, z, intensity, ring)
  sweeps/LIDAR_TOP/<token>_<k>.bin  past sweep k of scenes.make_sweep, the same 5 columns, in the sweep's own frame
  <info_name>                       the info pickle: per frame lidar_path, token, sweeps [{lidar_path, transform_matrix
                                    (sweep -> key frame, fp64), time_lag}], ref_from_car, car_from_global (fp64 4x4
                                    from seeded pose quaternions), gt_boxes fp64 [M, 9], gt_names
write_waymo(root, seeds, cfg, ...) writes the Waymo layout of the reference's WaymoDataset:
  lidar_point/<token>.bin           6 fp32 columns (x, y, z, intensity, elongation, no-label-zone flag); the scene's
                                    points carry flag -1, extra rows in no-label zones carry 1
  lidar_point/<token>_<k>.bin       past sweep k, the same layout
  <info_name>                       per frame token, pose (4x4), sweeps [{token, pose, timestamp}], objects [{label,
                                    box [9], num_points}] with num_points the key frame's points in the box

The key frame's points and the sweeps' points and transforms are those of scenes.SyntheticSceneDataset for the same
seed, so a reader over these trees and the synthetic dataset hand the detector the same frames."""
import os
import pickle

import numpy as np

from pillarnext_b200 import scenes

F = np.float32


def quat_matrix(q):
    """3x3 rotation of a unit quaternion (w, x, y, z)."""
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def rigid(q, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = quat_matrix(q), t
    return T


def _pose_quaternions(g):
    """(sensor in car, car in world): (quaternion (w, x, y, z), translation) each, a mostly-yaw rotation."""
    out = []
    for tilt, spread in ((0.01, 2.0), (0.02, 800.0)):
        axis = np.array([g.normal(0, tilt), g.normal(0, tilt), 1.0])
        axis /= np.linalg.norm(axis)
        a = g.uniform(-np.pi, np.pi)
        out.append((np.concatenate([[np.cos(a / 2)], np.sin(a / 2) * axis]), g.uniform(-spread, spread, 3)))
    return out


def _write(root, rel, arr):
    path = os.path.join(root, rel)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.ascontiguousarray(arr, dtype=F).tofile(path)
    return rel


def scene(seed, cfg, n_points, n_boxes, nsweeps):
    """(key points [N, 5], boxes [M, 9] fp32, names, [(sweep points [n, 5], transform, lag)] * (nsweeps - 1)), with
    SyntheticSceneDataset's default sweep_interval (0.05 s) and ego_speed."""
    pts, boxes, names = scenes.make_scene(seed, cfg, n_points, n_boxes)
    sweeps = []
    for k in range(1, nsweeps):
        p, T, _ = scenes.make_sweep(seed, k, cfg, boxes, n_points)
        sweeps.append((p, T, k * 0.05))
    return pts, boxes, names, sweeps


def write_nusc(root, seeds, cfg, n_points=6000, n_boxes=12, nsweeps=10, nan_velocity=0.0, none_transform=False,
               info_name="infos_train_10sweeps_withvelo_filterZero.pkl"):
    """Returns (infos, poses): poses[token] = ((q_cs, t_cs), (q_pose, t_pose)), the quaternions the matrices came from.
    nan_velocity: fraction of boxes whose (vx, vy) is NaN; none_transform: sweep 1 of every frame stored with
    transform_matrix None."""
    g = np.random.default_rng([77, len(seeds)] + [int(s) for s in seeds[:4]])
    infos, poses = [], {}
    for seed in seeds:
        token = "scene_%d" % seed
        pts, boxes, names, sweeps = scene(seed, cfg, n_points, n_boxes, nsweeps)
        ring = g.integers(0, 32, (len(pts), 1)).astype(F)
        lidar_path = _write(root, "samples/LIDAR_TOP/%s.bin" % token, np.concatenate([pts[:, :4], ring], 1))
        sw = []
        for k, (p, T, lag) in enumerate(sweeps, 1):
            rel = _write(root, "sweeps/LIDAR_TOP/%s_%d.bin" % (token, k),
                         np.concatenate([p[:, :4], g.integers(0, 32, (len(p), 1)).astype(F)], 1))
            sw.append({"lidar_path": rel, "transform_matrix": None if (none_transform and k == 1) else T,
                       "time_lag": lag})
        (qc, tc), (qp, tp) = _pose_quaternions(g)
        poses[token] = ((qc, tc), (qp, tp))
        gt = boxes.astype(np.float64)
        gt[g.uniform(0, 1, len(gt)) < nan_velocity, 6:8] = np.nan
        infos.append({"lidar_path": lidar_path, "token": token, "sweeps": sw,
                      "ref_from_car": np.linalg.inv(rigid(qc, tc)), "car_from_global": np.linalg.inv(rigid(qp, tp)),
                      "gt_boxes": gt, "gt_names": np.array(names)})
    with open(os.path.join(root, info_name), "wb") as fh:
        pickle.dump(infos, fh)
    return infos, poses


def write_waymo(root, seeds, cfg, n_points=6000, n_boxes=12, nsweeps=3, identity_pose=False, nlz=0.1, empty_objects=0,
                info_name="waymo_infos_train.pkl"):
    """identity_pose: every key-frame pose is the identity and a sweep's pose is its transform, so inv(pose) @
    sweep_pose is exactly the synthetic transform.  nlz: fraction of extra no-label-zone rows.  empty_objects: labels
    with num_points 0 appended to every frame's objects, boxes beyond the scene (load_box3d drops them)."""
    from det3d.datasets.pipelines.sample_ops import libm_trig
    from oracle.gts_oracle import points_in_boxes
    g = np.random.default_rng([78, len(seeds)] + [int(s) for s in seeds[:4]])

    def layout(p):
        rows = np.concatenate([p[:, :4], g.uniform(0, 1, (len(p), 1)), np.full((len(p), 1), -1.0)], 1)
        extra = np.concatenate([g.uniform(-30, 30, (int(nlz * len(p)), 4)), g.uniform(0, 1, (int(nlz * len(p)), 1)),
                                np.ones((int(nlz * len(p)), 1))], 1)
        at = np.sort(g.integers(0, len(rows) + 1, len(extra)))
        return np.insert(rows, at, extra, axis=0)

    infos = []
    for seed in seeds:
        token = "scene_%d" % seed
        pts, boxes, names, sweeps = scene(seed, cfg, n_points, n_boxes, nsweeps)
        _write(root, "lidar_point/%s.bin" % token, layout(pts))
        q, t = _pose_quaternions(g)[1]
        pose = np.eye(4) if identity_pose else rigid(q, t)
        sw = []
        for k, (p, T, lag) in enumerate(sweeps, 1):
            _write(root, "lidar_point/%s_%d.bin" % (token, k), layout(p))
            sw.append({"token": "%s_%d" % (token, k), "pose": T if identity_pose else pose @ T, "timestamp": lag})
        counts = points_in_boxes(pts, boxes, libm_trig(boxes[:, 8])).sum(0)
        objects = [{"label": n, "box": b.astype(np.float64), "num_points": int(c)} for n, b, c in zip(names, boxes, counts)]
        for k in range(empty_objects):
            objects.append({"label": "pedestrian", "num_points": 0,
                            "box": np.array([cfg["pc_range"][3] + 5.0 + k, 0.0, -1.0, 0.7, 0.7, 1.8, 0.0, 0.0, 0.3])})
        infos.append({"token": token, "pose": pose, "sweeps": sw, "objects": objects})
    with open(os.path.join(root, info_name), "wb") as fh:
        pickle.dump(infos, fh)
    return infos
