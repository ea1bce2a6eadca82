"""Plain-numpy restatement of multi-sweep accumulation (TEST INFRASTRUCTURE, never imported by the product): the
reference's NuScenesDataset.read_sweep / remove_close / load_pointcloud (det3d/datasets/nuscenes/nusc.py) and
WaymoDataset.load_pointcloud (det3d/datasets/waymo/waymo.py), line for line, on the operands scenes.collate packs.
  * nuScenes (min_distance > 0): points_sweep[:3, :] = transform_matrix.dot(vstack((xyz.T, ones)))[:3, :] written back
    into the fp32 array (skipped when the matrix is the NaN "None" marker), then remove_close on the fp32 result;
  * Waymo (min_distance = 0): xyz = (concatenate((xyz, ones), 1) @ rel_pose.T)[:, :3] written back into fp32;
  * per frame: key-frame rows, then sweep 1, 2, ...; the time column is the sweep's stored fp32 value.
numpy's dot / @ go through BLAS, so an element whose exact fp64 value lies next to an fp32 rounding midpoint may come out
one ulp away from the library's fixed-order arithmetic (tests/test_sweeps_cpu.py bounds that).
tests/test_sweeps_cpu.py pins it to the reference's own outputs (tests/golden/ref_sweeps.npz)."""
import numpy as np


def read_sweep(xyzit, transform, min_distance):
    """One sweep, as nusc.py's read_sweep (min_distance > 0) or waymo.py's loop body (min_distance = 0) -> [N', 5] fp32."""
    pts = np.array(xyzit, dtype=np.float32)
    if min_distance > 0:
        ps = pts[:, :4].T.copy()
        if not np.isnan(transform[3, 3]):
            ps[:3, :] = transform.dot(np.vstack((ps[:3, :], np.ones(ps.shape[1]))))[:3, :]
        keep = np.logical_not(np.logical_and(np.abs(ps[0, :]) < min_distance, np.abs(ps[1, :]) < min_distance))
        return np.concatenate([ps.T, pts[:, 4:5]], 1)[keep]
    if not np.isnan(transform[3, 3]):
        pts[:, :3] = (np.concatenate((pts[:, :3], np.ones((pts.shape[0], 1))), axis=1) @ transform.T)[:, :3]
    return pts


def accumulate(points, point_offsets, sweep_points, sweep_offsets, transforms, min_distance):
    """Collated operands (numpy) -> (points_out [n + S, 6] fp32 with the tail rows (B, 0, ...), count)."""
    points, sweep_points = np.asarray(points, np.float32), np.asarray(sweep_points, np.float32)
    B, K = transforms.shape[:2]
    rows = []
    for f in range(B):
        rows.append(points[point_offsets[f]:point_offsets[f + 1]])
        for k in range(K):
            s = f * K + k
            sw = read_sweep(sweep_points[sweep_offsets[s]:sweep_offsets[s + 1]], transforms[f, k], min_distance)
            rows.append(np.concatenate([np.full((len(sw), 1), f, np.float32), sw], 1))
    valid = np.concatenate(rows, 0) if rows else np.zeros((0, 6), np.float32)
    out = np.zeros((len(points) + len(sweep_points), 6), np.float32)
    out[:, 0] = B
    out[:len(valid)] = valid
    return out, len(valid)


def accumulate_example(ex):
    """accumulate() on a collated example (torch CPU tensors) -> a copy of it with the compacted accumulated points and
    without the sweep keys: what a loader that accumulates in numpy would have shipped."""
    import torch
    out, count = accumulate(ex["points"].numpy(), ex["point_offsets"].numpy(), ex["sweep_points"].numpy(),
                            ex["sweep_offsets"].numpy(), ex["sweep_transforms"].numpy(), ex["sweep_min_distance"])
    keys = ("point_offsets", "sweep_points", "sweep_offsets", "sweep_transforms", "sweep_min_distance")
    res = {k: v for k, v in ex.items() if k not in keys}
    res["points"] = torch.from_numpy(out[:count].copy())
    return res


def random_operands(B, sweeps, n, seed):
    """Collated operands of B frames of `sweeps` sweeps (the key frame + sweeps - 1 past ones) of n points each, as numpy:
    points spread over +-50 m (some within the +-1 m square after the transform), each past sweep with a random planar
    rigid transform, sweep 2 of every frame without one (NaN), the last frame's sweep 1 dropped (empty)."""
    g = np.random.default_rng(seed)
    K = sweeps - 1

    def cloud(m):
        xy = np.where(g.uniform(0, 1, (m, 1)) < 0.02, g.uniform(-3, 3, (m, 2)), g.uniform(-50, 50, (m, 2)))
        return np.concatenate([xy, g.uniform(-3, 2, (m, 1)), g.uniform(0, 255, (m, 1))], 1).astype(np.float32)
    key = np.concatenate([np.concatenate([np.full((n, 1), f, np.float32), cloud(n), np.zeros((n, 1), np.float32)], 1)
                          for f in range(B)])
    counts = np.full((B, K), n)
    if K:
        counts[-1, 0] = 0
    tms = np.full((B, K, 4, 4), np.nan)
    sw = []
    for f in range(B):
        for k in range(K):
            th = g.uniform(-0.2, 0.2)
            T = np.eye(4)
            T[:2, :2] = [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]
            T[:3, 3] = g.uniform(-2, 2), g.uniform(-2, 2), g.uniform(-0.1, 0.1)
            if k != 1:
                tms[f, k] = T
            c = cloud(counts[f, k])
            sw.append(np.concatenate([c, np.full((len(c), 1), np.float32(0.05 * (k + 1)))], 1))
    off = np.concatenate([[0], np.cumsum(counts.reshape(-1))]).astype(np.int32)
    return dict(points=key, point_offsets=(np.arange(B + 1) * n).astype(np.int32),
                sweep_points=np.concatenate(sw).astype(np.float32).reshape(-1, 5), sweep_offsets=off, transforms=tms)
