"""Seeded nuScenes-shaped evaluation inputs (TEST INFRASTRUCTURE -- see oracle/__init__.py): ground-truth frames over the
ten nuScenes classes with points or point counts, and detections that are jittered labels plus false positives, in the
shapes evaluate_nuscenes.nuscenes_metrics takes.  Used by tests/test_nds_metric_*.py and tools/bench_nds_eval.py.

Besides random placement, every frame carries the cases the matching rules decide on: boxes on a 1/8 m grid with
detections exactly 0.5, 1, 2 and 4 m away, a pair of boxes exactly equidistant from one detection, boxes and
detections exactly on the class's range limit, and (tie_scores) scores rounded to two decimals."""
import numpy as np

CLASSES = ["car", "truck", "construction_vehicle", "bus", "trailer", "barrier", "motorcycle", "bicycle", "pedestrian",
           "traffic_cone"]
SIZES = {"car": (4.6, 1.9, 1.7), "truck": (6.9, 2.5, 2.8), "construction_vehicle": (6.4, 2.8, 3.2), "bus": (11.0, 2.9, 3.5),
         "trailer": (12.0, 2.9, 3.9), "barrier": (0.5, 2.5, 1.0), "motorcycle": (2.1, 0.8, 1.5), "bicycle": (1.7, 0.6, 1.3),
         "pedestrian": (0.7, 0.7, 1.8), "traffic_cone": (0.4, 0.4, 1.1)}
WEIGHTS = np.array([0.35, 0.08, 0.02, 0.02, 0.03, 0.12, 0.03, 0.03, 0.2, 0.12])
RANGE = {"car": 50.0, "truck": 50.0, "construction_vehicle": 50.0, "bus": 50.0, "trailer": 50.0, "barrier": 30.0,
         "motorcycle": 40.0, "bicycle": 40.0, "pedestrian": 40.0, "traffic_cone": 30.0}
ATTRS = {"car": ["vehicle.moving", "vehicle.parked", "vehicle.stopped"], "bus": ["vehicle.moving", "vehicle.parked"],
         "bicycle": ["cycle.with_rider", "cycle.without_rider"], "motorcycle": ["cycle.with_rider", "cycle.without_rider"],
         "pedestrian": ["pedestrian.moving", "pedestrian.standing", "pedestrian.sitting_lying_down"]}


def _boxes(rng, names, xy):
    n = len(names)
    size = np.array([SIZES[c] for c in names]).reshape(n, 3) * rng.uniform(0.85, 1.15, (n, 3))
    z = rng.uniform(-1.0, 1.0, (n, 1)) + size[:, 2:3] / 2
    vel = rng.normal(0, 2.0, (n, 2)) * (rng.uniform(0, 1, (n, 1)) < 0.6)
    yaw = rng.uniform(-np.pi, np.pi, (n, 1))
    return np.concatenate([xy, z, size, vel, yaw], 1).astype(np.float32)


def make_frames(seed, n_frames, n_points=30000, n_labels=40, n_det_max=500, extent=55.0, fp_per_frame=120,
                with_attributes=False, tie_scores=True, token0=0):
    """-> (gts, detections, class names).  n_points=None gives each box a "num_points" count (some 0) instead of
    points.  `extent` is the radius of the disc the random objects lie in: small values crowd them together."""
    rng = np.random.default_rng(seed)
    gts, dets = {}, {}
    for fi in range(n_frames):
        n = max(4, int(rng.poisson(n_labels)))
        names = [CLASSES[i] for i in rng.choice(len(CLASSES), n, p=WEIGHTS / WEIGHTS.sum())]
        phi, rad = rng.uniform(-np.pi, np.pi, n), extent * np.sqrt(rng.uniform(0, 1, n))
        xy = np.stack([rad * np.cos(phi), rad * np.sin(phi)], 1)
        grid = rng.uniform(0, 1, n) < 0.3                           # 1/8 m grid: exact fp32 coordinates and offsets
        xy[grid] = np.round(xy[grid] * 8) / 8
        boxes = _boxes(rng, names, xy)
        # exactly on the range limit: (r, 0), (0, -r) or (0.6 r, 0.8 r), all exact in fp32 and in the fp64 radius
        for k in range(2):
            c = CLASSES[rng.integers(0, len(CLASSES))]
            r = RANGE[c]
            p = [(r, 0.0), (0.0, -r), (0.6 * r, 0.8 * r)][rng.integers(0, 3)]
            b = _boxes(rng, [c], np.array([p]))
            boxes, names = np.concatenate([boxes, b]), names + [c]
        # an equidistant pair: boxes at g and g + (2, 0), a detection at g + (1, 0) added below
        g0 = np.round(rng.uniform(-20, 20, 2) * 8) / 8
        c_pair = CLASSES[rng.integers(0, len(CLASSES))]
        pair = _boxes(rng, [c_pair, c_pair], np.array([g0, g0 + [2.0, 0.0]]))
        boxes, names = np.concatenate([boxes, pair]), names + [c_pair, c_pair]
        m = len(boxes)
        nan_vel = rng.uniform(0, 1, m) < 0.03
        boxes[nan_vel, 6:8] = np.nan
        tok = "sample_%d" % (token0 + fi)
        g = {"boxes": boxes, "names": names}
        if n_points is None:
            g["num_points"] = np.where(rng.uniform(0, 1, m) < 0.1, 0, rng.integers(1, 400, m))
        else:
            n_in = n_points // 2
            w = rng.exponential(1.0, m) ** 2
            owner = rng.choice(m, n_in, p=w / w.sum())
            loc = rng.uniform(-0.45, 0.45, (n_in, 3)) * np.nan_to_num(boxes[owner, 3:6])
            c, s = np.cos(boxes[owner, 8]), np.sin(boxes[owner, 8])
            inside = np.stack([loc[:, 0] * c - loc[:, 1] * s + boxes[owner, 0], loc[:, 0] * s + loc[:, 1] * c + boxes[owner, 1],
                               loc[:, 2] + boxes[owner, 2]], 1)
            bg = np.concatenate([rng.uniform(-extent - 5, extent + 5, (n_points - n_in, 2)),
                                 rng.uniform(-2.0, 4.0, (n_points - n_in, 1))], 1)
            pts = np.concatenate([inside, bg]).astype(np.float32)
            g["points"] = np.concatenate([pts, rng.uniform(0, 1, (len(pts), 2)).astype(np.float32)], 1)
        if with_attributes:
            g["attributes"] = [ATTRS[nm][rng.integers(0, len(ATTRS[nm]))] if nm in ATTRS and rng.uniform() < 0.9 else ""
                               for nm in names]
        gts[tok] = g
        # detections: jittered labels, exact threshold offsets from grid boxes, the equidistant one, false positives
        lab = np.array([CLASSES.index(nm) for nm in names])
        keep = rng.uniform(0, 1, m) < 0.85
        j = boxes[keep].copy()
        j[:, :2] += rng.normal(0, 0.4, (len(j), 2))
        j[:, 3:6] *= 1 + rng.normal(0, 0.08, (len(j), 3))
        j[:, 6:8] = np.nan_to_num(j[:, 6:8]) + rng.normal(0, 0.5, (len(j), 2))
        j[:, 8] += rng.normal(0, 0.2, len(j)) + np.pi * (rng.uniform(0, 1, len(j)) < 0.1)
        on_grid = np.nonzero(np.concatenate([grid, np.zeros(m - n, bool)]))[0]
        ex = boxes[on_grid].copy()
        ex[:, 6:8] = np.nan_to_num(ex[:, 6:8])
        off = np.array([0.5, 1.0, 2.0, 4.0])[rng.integers(0, 4, len(ex))]
        ax = rng.integers(0, 2, len(ex))
        ex[np.arange(len(ex)), ax] += off * np.where(rng.uniform(0, 1, len(ex)) < 0.5, -1, 1)
        mid = pair[0].copy()
        mid[0] += 1.0
        mid[6:8] = 0.0
        n_fp = int(fp_per_frame)
        fl = rng.choice(len(CLASSES), n_fp, p=WEIGHTS / WEIGHTS.sum())
        fph, frad = rng.uniform(-np.pi, np.pi, n_fp), (extent + 5) * np.sqrt(rng.uniform(0, 1, n_fp))
        fp = _boxes(rng, [CLASSES[i] for i in fl], np.stack([frad * np.cos(fph), frad * np.sin(fph)], 1))
        near = rng.uniform(0, 1, n_fp) < 0.4
        fp[near, :2] = boxes[rng.integers(0, m, near.sum()), :2] + rng.normal(0, 1.5, (near.sum(), 2))
        db = np.concatenate([j, ex, mid[None], fp])
        dl = np.concatenate([lab[keep], lab[on_grid], [CLASSES.index(c_pair)], fl])
        sc = np.concatenate([rng.uniform(0.3, 1.0, len(j) + len(ex) + 1), rng.uniform(0.05, 0.8, n_fp)])
        if tie_scores:
            sc = np.round(sc, 2)
        perm = rng.permutation(len(db))[:n_det_max]
        dets[tok] = {"box3d_lidar": db[perm].astype(np.float32), "scores": sc[perm].astype(np.float32),
                     "label_preds": dl[perm].astype(np.int64)}
    return gts, dets, list(CLASSES)
