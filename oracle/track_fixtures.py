"""Seeded Waymo-validation-shaped tracking input (TEST FIXTURES; numpy only): n_seq sequences of n_frames frames 0.1 s
apart, three classes.  Each (sequence, class) has its own objects (mostly 10-120, one in ten 450-560), starting within
70 m of an ego that turns and drives slowly, each moving at constant global velocity (the boxes stay within 500 m of
the sensor).  Each object is labelled (with an id and 0, 3 or 50 points) and detected with probability 0.85 (centre
noise 0.15 m, velocity noise 0.3 m/s, in the sensor frame), plus up to 50 false positives per class and frame; at most
max_det detections per class and frame."""
import numpy as np

CLASSES = ["vehicle", "pedestrian", "cyclist"]
DIMS = np.array([(4.5, 2.0, 1.6), (0.8, 0.8, 1.8), (1.8, 0.7, 1.6)], np.float64)
EGO = np.array([1000.0, -300.0])      # the ego's first global position; the objects start within 70 m of it


def waymo_val_shaped(seed, n_seq=200, n_frames=200, max_det=500):
    """-> (detections, frames, gts) keyed by "<context>-<timestamp>" tokens, as track.track and
    evaluate_waymo_tracking.waymo_tracking_metrics take them."""
    g = np.random.default_rng([91, seed])
    dets, frames, gts = {}, {}, {}
    for s in range(n_seq):
        objs = []
        for c in range(3):
            n = int(g.integers(450, 561)) if g.uniform() < 0.1 else int(g.integers(10, 121))
            objs.append((EGO + g.uniform(-70, 70, (n, 2)), g.normal(0, [5.0, 1.0, 3.0][c], (n, 2)), g.uniform(-3, 3, n)))
        yaw0, t0 = g.uniform(-np.pi, np.pi), 1500000000000000 + int(g.integers(0, 10 ** 12))
        ctx = "seg%03d" % s
        for f in range(n_frames):
            ts = t0 + 100000 * f + int(g.integers(-300, 300))
            a = yaw0 + 0.005 * f
            T = np.eye(4)
            T[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
            T[:3, 3] = [EGO[0] + 0.3 * f, EGO[1], 0.3]
            R, t = T[:2, :2], T[:2, 3]
            gb, gn, gi, gp, db, ds, dl = [], [], [], [], [], [], []
            for c, (p0, v, yaw) in enumerate(objs):
                n = len(p0)
                pl = (p0 + v * 0.1 * f - t) @ R                   # R^T (p - t): global -> sensor
                vl = v @ R
                box = np.concatenate([pl, np.zeros((n, 1)), np.broadcast_to(DIMS[c], (n, 3)), vl, yaw[:, None]], 1)
                lab = g.uniform(size=n) < 0.9
                gb.append(box[lab])
                gn += [CLASSES[c]] * int(lab.sum())
                gi += ["%s_%d_%d" % (ctx, c, k) for k in np.nonzero(lab)[0]]
                gp.append(g.choice([0, 3, 50], int(lab.sum())))
                seen = box[g.uniform(size=n) < 0.85].copy()
                seen[:, :2] += g.normal(0, 0.15, (len(seen), 2))
                seen[:, 6:8] += g.normal(0, 0.3, (len(seen), 2))
                nfp = int(g.integers(0, 51))
                fp = np.concatenate([g.uniform(-75, 75, (nfp, 2)), np.zeros((nfp, 1)), np.broadcast_to(DIMS[c], (nfp, 3)),
                                     g.normal(0, 1, (nfp, 2)), g.uniform(-3, 3, (nfp, 1))], 1)
                d = np.concatenate([seen, fp])[:max_det]
                db.append(d)
                ds.append(g.uniform(0.05, 1.0, len(d)))
                dl.append(np.full(len(d), c))
            tok = "%s-%d" % (ctx, ts)
            frames[tok] = dict(sequence=ctx, timestamp=ts, pose=T)
            dets[tok] = dict(box3d_lidar=np.concatenate(db).astype(np.float32), scores=np.concatenate(ds).astype(np.float32),
                             label_preds=np.concatenate(dl).astype(np.int64))
            gts[tok] = dict(boxes=np.concatenate(gb).astype(np.float32), names=gn, ids=gi,
                            num_points=np.concatenate(gp).astype(np.int64), sequence=ctx, timestamp=ts)
    return dets, frames, gts


def write_waymo_sequences(root, seeds, cfg, length=4, n_points=3000, n_boxes=10, info_name="waymo_infos_val.pkl"):
    """A Waymo info tree (the layout of oracle/reader_fixtures.write_waymo: lidar_point/<token>.bin with 6 fp32
    columns, the info pickle) whose frames form real sequences: sequence q is scenes.sequence_frame(seeds[q], k) for
    k < length, token "<context>-<timestamp>", pose = a seeded sensor -> world pose of the first frame times the
    frame's pose, each object with the id of its make_scene box and num_points = the frame's points inside it.
    Returns the infos."""
    import os
    import pickle

    from det3d.datasets.pipelines.sample_ops import libm_trig
    from oracle.gts_oracle import points_in_boxes
    from pillarnext_b200 import scenes
    g = np.random.default_rng([92, len(seeds)])
    infos = []
    for seed in seeds:
        a = g.uniform(-np.pi, np.pi)
        world = np.eye(4)
        world[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
        world[:3, 3] = g.uniform(-500, 500, 3)
        for k in range(length):
            pts, boxes, names, pose = scenes.sequence_frame(seed, k, cfg, n_points, n_boxes)
            ts = scenes.SEQUENCE_T0_US + k * scenes.SEQUENCE_STEP_US
            token = "ctx%d-%d" % (seed, ts)
            rows = np.concatenate([pts[:, :4], np.zeros((len(pts), 1)), np.full((len(pts), 1), -1.0)], 1)
            path = os.path.join(root, "lidar_point", token + ".bin")
            os.makedirs(os.path.dirname(path), exist_ok=True)
            np.ascontiguousarray(rows, dtype=np.float32).tofile(path)
            counts = points_in_boxes(pts, boxes, libm_trig(boxes[:, 8])).sum(0)
            objects = [{"id": "obj%d" % j, "label": n, "box": b.astype(np.float64), "num_points": int(c)}
                       for j, (n, b, c) in enumerate(zip(names, boxes, counts))]
            infos.append({"token": token, "pose": world @ pose, "sweeps": [], "objects": objects})
    with open(os.path.join(root, info_name), "wb") as fh:
        pickle.dump(infos, fh)
    return infos
