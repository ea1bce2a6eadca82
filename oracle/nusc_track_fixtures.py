"""Seeded nuScenes-validation-shaped tracking input (TEST FIXTURES; numpy only): n_scenes scenes of n_frames key frames
0.5 s apart, the ten nuScenes detection classes.  Each scene has about 40 objects within 55 m of an ego that turns and
drives slowly, three in ten starting within 2.5 m of another, each moving at a constant global velocity of its class's
scale; every object is labelled in every frame
(with an id and 0, 3 or 40 points).  Detections: each object seen with probability 0.85 (centre noise 0.2 m, velocity
noise 0.3 m/s, score in [0.3, 1)), low-score duplicates near the objects (centre noise 1 m, score in [0.01, 0.3)), and
false positives anywhere (score in [0.05, 0.6)); at most max_det per frame.  Misses make fragmentations, crowded
duplicates and crossings make identity switches."""
import numpy as np

CLASSES = ["car", "truck", "construction_vehicle", "bus", "trailer", "barrier", "motorcycle", "bicycle", "pedestrian",
           "traffic_cone"]
DIMS = np.array([(4.6, 1.9, 1.7), (6.9, 2.5, 2.8), (6.4, 2.8, 3.2), (11.0, 2.9, 3.5), (12.3, 2.9, 3.9),
                 (0.5, 2.5, 1.0), (2.1, 0.8, 1.5), (1.7, 0.6, 1.3), (0.7, 0.7, 1.8), (0.4, 0.4, 1.1)], np.float64)
SPEED = np.array([5.0, 4.0, 0.5, 5.0, 3.0, 0.0, 5.0, 3.0, 1.0, 0.0])
SHARE = np.array([0.35, 0.1, 0.03, 0.03, 0.04, 0.12, 0.04, 0.04, 0.17, 0.08])
EGO = np.array([400.0, 1200.0])


def nusc_val_shaped(seed, n_scenes=150, n_frames=40, n_objects=40, max_dup=400, max_fp=60, max_det=500):
    """-> (detections, frames, gts) keyed by "<scene>_<frame>" tokens, as track.track and
    evaluate_nuscenes_tracking.nuscenes_tracking_metrics take them (labels index CLASSES)."""
    g = np.random.default_rng([77, seed])
    dets, frames, gts = {}, {}, {}
    for s in range(n_scenes):
        n = int(g.integers(n_objects - 5, n_objects + 6))
        cls = g.choice(len(CLASSES), n, p=SHARE)
        p0 = EGO + g.uniform(-55, 55, (n, 2))
        grouped = g.uniform(size=n) < 0.3                           # parked rows and crowds: next to an earlier object
        grouped[0] = False
        for k in np.nonzero(grouped)[0]:
            p0[k] = p0[int(g.integers(0, k))] + g.uniform(-2.5, 2.5, 2)
        v = g.normal(0, 1, (n, 2)) * SPEED[cls, None]
        yaw = g.uniform(-np.pi, np.pi, n)
        yaw0, t0 = g.uniform(-np.pi, np.pi), 1530000000000000 + int(g.integers(0, 10 ** 12))
        scene = "scene%04d" % s
        for f in range(n_frames):
            ts = t0 + 500000 * f + int(g.integers(-2000, 2000))
            a = yaw0 + 0.01 * f
            T = np.eye(4)
            T[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
            T[:3, 3] = [EGO[0] + 1.0 * f, EGO[1], 1.8]
            R, t = T[:2, :2], T[:2, 3]
            pl = (p0 + v * 0.5 * f - t) @ R                         # R^T (p - t): global -> sensor
            box = np.concatenate([pl, np.zeros((n, 1)), DIMS[cls], v @ R, yaw[:, None]], 1)
            seen = g.uniform(size=n) < 0.85
            det = box[seen].copy()
            det[:, :2] += g.normal(0, 0.2, (len(det), 2))
            det[:, 6:8] += g.normal(0, 0.3, (len(det), 2))
            nd = int(g.integers(0, max_dup + 1))
            src = g.integers(0, n, nd)
            dup = box[src].copy()
            dup[:, :2] += g.normal(0, 1.0, (nd, 2))
            nfp = int(g.integers(0, max_fp + 1))
            fcls = g.integers(0, len(CLASSES), nfp)
            fp = np.concatenate([g.uniform(-60, 60, (nfp, 2)), np.zeros((nfp, 1)), DIMS[fcls], g.normal(0, 1, (nfp, 2)),
                                 g.uniform(-3, 3, (nfp, 1))], 1)
            db = np.concatenate([det, dup, fp])[:max_det]
            ds = np.concatenate([g.uniform(0.3, 1.0, len(det)), g.uniform(0.01, 0.3, nd), g.uniform(0.05, 0.6, nfp)])
            dl = np.concatenate([cls[seen], cls[src], fcls])
            tok = "%s_%02d" % (scene, f)
            frames[tok] = dict(sequence=scene, timestamp=ts, pose=T)
            dets[tok] = dict(box3d_lidar=db.astype(np.float32), scores=ds[:len(db)].astype(np.float32),
                             label_preds=dl[:len(db)].astype(np.int64))
            gts[tok] = dict(boxes=box.astype(np.float32), names=[CLASSES[c] for c in cls],
                            ids=["%s_%d" % (scene, k) for k in range(n)],
                            num_points=g.choice([0, 3, 40], n, p=[0.05, 0.25, 0.7]).astype(np.int64),
                            sequence=scene, timestamp=ts, pose=T)
    return dets, frames, gts
