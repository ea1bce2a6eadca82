"""Seeded Waymo-shaped evaluation inputs (TEST INFRASTRUCTURE -- see oracle/__init__.py): ground-truth frames with
points, and detections that are jittered labels plus false positives, in the shapes evaluate_waymo.waymo_metrics takes.
Used by tests/test_waymo_metric_*.py and tools/bench_waymo_eval.py."""
import numpy as np

CLASSES = ["vehicle", "pedestrian", "cyclist"]
SIZES = {"vehicle": (4.7, 2.1, 1.7), "pedestrian": (0.9, 0.9, 1.8), "cyclist": (1.8, 0.8, 1.7)}


def make_frames(seed, n_frames, n_points=180000, n_labels=(60, 30, 5), n_det_max=500, extent=75.0, fp_per_class=(80, 60, 20),
                token0=0):
    """-> (gts, detections, class names).  `extent` sets the half-width of the square the objects lie in: small values
    crowd the boxes together (heavy overlaps).  About a third of the in-box points go to a few boxes only, so box point
    counts span 0 (dropped), 1-5 (LEVEL_2) and more (LEVEL_1)."""
    rng = np.random.default_rng(seed)
    gts, dets = {}, {}
    for fi in range(n_frames):
        boxes, names = [], []
        for c, name in enumerate(CLASSES):
            n = int(n_labels[c])
            size = np.array(SIZES[name]) * rng.uniform(0.8, 1.2, (n, 3))
            xy = rng.uniform(-extent, extent, (n, 2))
            z = rng.uniform(-1.0, 1.0, (n, 1)) + size[:, 2:3] / 2
            yaw = rng.uniform(-np.pi, np.pi, (n, 1))
            b = np.concatenate([xy, z, size, np.zeros((n, 2)), yaw], 1)
            boxes.append(b)
            names += [name] * n
        boxes = np.concatenate(boxes).astype(np.float32)
        m = len(boxes)
        # points: background plus points inside boxes (box weights heavy-tailed so some boxes get few or none)
        n_in = n_points // 3
        w = rng.exponential(1.0, m) ** 3
        owner = rng.choice(m, n_in, p=w / w.sum())
        loc = rng.uniform(-0.45, 0.45, (n_in, 3)) * boxes[owner, 3:6]
        c, s = np.cos(boxes[owner, 8]), np.sin(boxes[owner, 8])
        inside = np.stack([loc[:, 0] * c - loc[:, 1] * s + boxes[owner, 0], loc[:, 0] * s + loc[:, 1] * c + boxes[owner, 1],
                           loc[:, 2] + boxes[owner, 2]], 1)
        bg = np.concatenate([rng.uniform(-extent - 5, extent + 5, (n_points - n_in, 2)),
                             rng.uniform(-2.0, 4.0, (n_points - n_in, 1))], 1)
        pts = np.concatenate([inside, bg]).astype(np.float32)
        pts = np.concatenate([pts, rng.uniform(0, 1, (len(pts), 2)).astype(np.float32)], 1)   # intensity, elongation
        tok = "frame_%d" % (token0 + fi)
        gts[tok] = {"boxes": boxes, "names": names, "points": pts}
        # detections: jittered labels (some flipped by pi), plus false positives near and far from the labels
        db, ds, dl = [], [], []
        for ci, name in enumerate(CLASSES):
            lab = boxes[[i for i, n in enumerate(names) if n == name]]
            keep = lab[rng.uniform(0, 1, len(lab)) < 0.85]
            j = keep.copy()
            j[:, :2] += rng.normal(0, 0.08, (len(j), 2)) * j[:, 3:5]
            j[:, 2] += rng.normal(0, 0.05, len(j)) * j[:, 5]
            j[:, 3:6] *= 1 + rng.normal(0, 0.05, (len(j), 3))
            j[:, 8] += rng.normal(0, 0.15, len(j)) + np.pi * (rng.uniform(0, 1, len(j)) < 0.1)
            n_fp = int(fp_per_class[ci])
            fp = np.zeros((n_fp, 9))
            near = lab[rng.integers(0, max(1, len(lab)), n_fp)] if len(lab) else np.zeros((n_fp, 9))
            fp[:, :2] = np.where(rng.uniform(0, 1, (n_fp, 1)) < 0.5, near[:, :2] + rng.normal(0, 1.0, (n_fp, 2)),
                                 rng.uniform(-extent, extent, (n_fp, 2)))
            fp[:, 2] = rng.uniform(-1, 1, n_fp) + SIZES[name][2] / 2
            fp[:, 3:6] = np.array(SIZES[name]) * rng.uniform(0.8, 1.2, (n_fp, 3))
            fp[:, 8] = rng.uniform(-np.pi, np.pi, n_fp)
            b = np.concatenate([j, fp])[:n_det_max]
            sc = np.concatenate([rng.uniform(0.3, 1.0, len(j)), rng.uniform(0.05, 0.8, n_fp)])[:n_det_max]
            db.append(b)
            ds.append(sc)
            dl.append(np.full(len(b), ci))
        dets[tok] = {"box3d_lidar": np.concatenate(db).astype(np.float32), "scores": np.concatenate(ds).astype(np.float32),
                     "label_preds": np.concatenate(dl).astype(np.int64)}
    return gts, dets, list(CLASSES)
