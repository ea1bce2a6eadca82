"""Sequential numpy restatement of the Waymo-style metric of pillarnext_b200/evaluate_waymo.py (TEST INFRASTRUCTURE --
see oracle/__init__.py): one (frame, class) at a time, one detection at a time, one pair at a time.

The IoU is predict_oracle.aligned_iou3d (the reference's boxes_iou3d_gpu arithmetic, pinned to the reference by
tests/test_predict_cpu.py), detection first; the point counts are gts_oracle.points_in_boxes (the reference's
points_in_boxes_jit arithmetic, pinned by tests/test_gt_sampling_cpu.py) with libm (cosf, sinf).  Heading accuracy and
the curves are float64."""
import math

import numpy as np

from oracle import gts_oracle, predict_oracle as P

IOU_THRESHOLDS = {"vehicle": 0.7, "pedestrian": 0.5, "cyclist": 0.5}


def _np(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def _box7(b):
    b = np.asarray(b, np.float32)
    return b if len(b) == 7 else b[[0, 1, 2, 3, 4, 5, 8]]


def heading_accuracy(a, b):
    d = (float(a) - float(b) + math.pi) % (2 * math.pi) - math.pi
    return 1.0 - min(abs(d), 2 * math.pi - abs(d)) / math.pi


def ap(weights, n_gt):
    """weights in descending score order (TP: 1 or h, FP: None): 100 x area under the monotone precision envelope, with
    precision = sum of TP weights / (sum of TP weights + FP)."""
    if n_gt == 0:
        return float("nan")
    prec, rec, acc, fps = [], [], 0.0, 0
    for w in weights:
        if w is None:
            fps += 1
        else:
            acc += w
        prec.append(acc / (acc + fps) if acc + fps > 0 else 0.0)
        rec.append(acc / n_gt)
    total, prev_rec = 0.0, 0.0
    for i in range(len(weights)):
        env = max(prec[i:])
        total += (rec[i] - prev_rec) * env
        prev_rec = rec[i]
    return 100.0 * total


def waymo_metrics(gts, detections, class_names, iou_thresholds=None):
    """Same inputs and outputs as pillarnext_b200.evaluate_waymo.waymo_metrics."""
    from det3d.datasets.pipelines.sample_ops import libm_trig
    table = dict(IOU_THRESHOLDS, **(iou_thresholds or {}))
    for n in class_names:
        if n not in table:
            raise ValueError("no IoU threshold for class %r" % n)
    per_class = {}
    frames = []
    for t, g in gts.items():
        boxes = [_box7(b) for b in _np(g["boxes"]).reshape(len(g["names"]), -1)]
        b9 = np.zeros((len(boxes), 9), np.float32)
        for j, b in enumerate(boxes):
            b9[j, :6], b9[j, 8] = b[:6], b[6]
        pts = np.asarray(_np(g["points"]), np.float32)[:, :3]
        counts = gts_oracle.points_in_boxes(pts, b9, libm_trig(b9[:, 8])).sum(0) if len(boxes) else np.zeros(0, int)
        d = detections.get(t)
        if d is None:
            dets = []
        else:
            db, ds, dl = _np(d["box3d_lidar"]), _np(d["scores"]), _np(d["label_preds"])
            dets = [(float(np.float32(ds[i])), i, int(dl[i]), _box7(db[i])) for i in range(len(ds))]
        frames.append((list(g["names"]), boxes, counts, dets))
    for c, name in enumerate(class_names):
        thr = np.float32(table[name])
        n_l1 = n_l2 = 0
        results = []                                    # (score, frame, index, matched?, points of the box, h)
        for f, (names, boxes, counts, dets) in enumerate(frames):
            gi = [j for j, n in enumerate(names) if n == name]
            n_l2 += sum(1 for j in gi if counts[j] >= 1)
            n_l1 += sum(1 for j in gi if counts[j] > 5)
            mine = sorted([d for d in dets if d[2] == c], key=lambda d: (-d[0], d[1]))
            used = set()
            for s, i, _, box in mine:
                best, bj = -1.0, -1
                for j in gi:
                    if j in used:
                        continue
                    g = boxes[j]
                    # the oracle's own shortcut: centres farther apart than the half-diagonals plus 1 m share nothing
                    if math.hypot(float(box[0]) - float(g[0]), float(box[1]) - float(g[1])) > \
                            0.5 * (math.hypot(float(box[3]), float(box[4])) + math.hypot(float(g[3]), float(g[4]))) + 1.0:
                        v = 0.0
                    else:
                        v = float(P.aligned_iou3d(box, g))
                    if v > best:
                        best, bj = v, j
                if bj >= 0 and np.float32(best) >= thr:
                    used.add(bj)
                    results.append((s, f, i, True, int(counts[bj]), heading_accuracy(box[6], boxes[bj][6])))
                else:
                    results.append((s, f, i, False, -1, 0.0))
        results.sort(key=lambda r: (-r[0], r[1], r[2]))
        w1, h1, w2, h2 = [], [], [], []
        for s, f, i, hit, npts, h in results:
            if not hit:
                w1.append(None), h1.append(None), w2.append(None), h2.append(None)
                continue
            if npts >= 1:
                w2.append(1.0), h2.append(h)
            if npts > 5:
                w1.append(1.0), h1.append(h)
        per_class[name] = dict(AP_L1=ap(w1, n_l1), APH_L1=ap(h1, n_l1), AP_L2=ap(w2, n_l2), APH_L2=ap(h2, n_l2),
                               n_gt_L1=n_l1, n_gt_L2=n_l2)
    res = {}
    for key in ("AP_L1", "APH_L1", "AP_L2", "APH_L2"):
        vals = [v[key] for v in per_class.values() if v[key] == v[key]]
        res["m" + key] = float(np.mean(vals)) if vals else float("nan")
    res["per_class"] = per_class
    return res


def match_frame(boxes_gt, names, det_boxes, det_scores, det_labels, class_names, thresholds):
    """Per-detection (match index or -1, IoU) of one frame, for comparing the match alone: the IoU is the highest over
    the boxes still unmatched when the detection is visited (0 if none), computed for every pair (no shortcut)."""
    match = np.full(len(det_scores), -1, np.int64)
    iou = np.zeros(len(det_scores), np.float32)
    boxes = [_box7(b) for b in boxes_gt]
    for c, name in enumerate(class_names):
        gi = [j for j, n in enumerate(names) if n == name]
        order = sorted([i for i in range(len(det_scores)) if det_labels[i] == c], key=lambda i: (-float(det_scores[i]), i))
        used = set()
        for i in order:
            best, bj = -1.0, -1
            for j in gi:
                if j in used:
                    continue
                v = float(P.aligned_iou3d(_box7(det_boxes[i]), boxes[j]))
                if v > best:
                    best, bj = v, j
            iou[i] = best if bj >= 0 else 0.0
            if bj >= 0 and np.float32(best) >= np.float32(thresholds[c]):
                used.add(bj)
                match[i] = bj
    return match, iou
