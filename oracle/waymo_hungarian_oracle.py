"""Sequential restatement of evaluate_waymo.waymo_metrics(matching="hungarian") (TEST INFRASTRUCTURE -- see
oracle/__init__.py): one (frame, class, breakdown, cutoff) at a time, the assignment by scipy's linear_sum_assignment on
the fp32 IoU matrix with the infeasible pairs (IoU < threshold, other range, score under the cutoff) excluded, then the
tie rule applied by re-solving with each earlier option fixed.

The IoU is predict_oracle.aligned_iou3d, the point counts gts_oracle.points_in_boxes, as in waymo_metric_oracle.  Totals
are fp64 sums of fp32 IoUs >= 2^-17, which are exact, so equal maxima compare equal."""
import math

import numpy as np
from scipy.optimize import linear_sum_assignment

from oracle import gts_oracle, predict_oracle as P
from oracle.waymo_metric_oracle import IOU_THRESHOLDS, _box7, _np, heading_accuracy

RANGES = ("0-30", "30-50", "50+")


def range_bin(x, y):
    x, y = np.float32(x), np.float32(y)
    r = np.sqrt(np.float32(x * x + y * y))
    return 0 if r < np.float32(30) else (1 if r < np.float32(50) else 2)


def cutoffs(scores, k):
    s = sorted(np.float32(v) for v in scores)
    return [s[(i * len(s)) // k] for i in range(k)] if s else []


def _best(w, fixed):
    """Maximum total of w (a dict (row, col) -> IoU) over one-to-one pairings that contain every pair of `fixed`
    ((row, col or None) in order): the fixed pairs' sum plus linear_sum_assignment on the rest, and that pairing."""
    rows_fixed = {r for r, _ in fixed}
    cols_fixed = {c for _, c in fixed if c is not None}
    rows = sorted({r for r, _ in w} - rows_fixed)
    cols = sorted({c for _, c in w} - cols_fixed)
    total = sum(w[(r, c)] for r, c in fixed if c is not None)
    pairs = {r: c for r, c in fixed}
    if rows and cols:
        a = np.zeros((len(rows), len(cols)))
        for (r, c), v in w.items():
            if r in rows and c in cols:
                a[rows.index(r), cols.index(c)] = v
        ri, ci = linear_sum_assignment(a, maximize=True)
        for i, j in zip(ri, ci):
            if a[i, j] > 0:                                         # a zero is an excluded pair: unmatched
                total += a[i, j]
                pairs[rows[i]] = cols[j]
    return total, pairs


def assign(w, det_order):
    """The maximum-IoU pairing of w with the tie rule: detections in det_order each take the first of (their boxes in
    ascending index, then unmatched) that some maximum agreeing with the earlier choices contains.  -> {det: box}."""
    best, pairs = _best(w, [])
    fixed = []
    for d in det_order:
        for o in sorted(c for r, c in w if r == d) + [None]:
            if any(c == o for _, c in fixed if o is not None):
                continue
            if pairs.get(d) == o:
                fixed.append((d, o))
                break
            total, cand = _best(w, fixed + [(d, o)])
            if total == best:
                fixed.append((d, o))
                pairs = cand
                break
    return {d: c for d, c in fixed if c is not None}


def ap_points(points, n_gt):
    """(TP weight, FP) per cutoff -> 100 x area under the monotone precision envelope, points in ascending recall."""
    if n_gt == 0:
        return float("nan")
    pts = sorted(points, key=lambda p: p[0])
    total, prev = 0.0, 0.0
    for i, (tp, _) in enumerate(pts):
        env = max((t / (t + f) if t + f > 0 else 0.0) for t, f in pts[i:])
        total += (tp / n_gt - prev) * env
        prev = tp / n_gt
    return 100.0 * total


def waymo_metrics(gts, detections, class_names, iou_thresholds=None, num_score_cutoffs=11):
    """Same inputs and outputs as evaluate_waymo.waymo_metrics(..., matching="hungarian")."""
    from det3d.datasets.pipelines.sample_ops import libm_trig
    table = dict(IOU_THRESHOLDS, **(iou_thresholds or {}))
    K = num_score_cutoffs
    frames = []
    for t, g in gts.items():
        boxes = [_box7(b) for b in _np(g["boxes"]).reshape(len(g["names"]), -1)]
        b9 = np.zeros((len(boxes), 9), np.float32)
        for j, b in enumerate(boxes):
            b9[j, :6], b9[j, 8] = b[:6], b[6]
        if "num_points" in g:
            counts = np.asarray(_np(g["num_points"])).reshape(-1)
        else:
            pts = np.asarray(_np(g["points"]), np.float32)[:, :3]
            counts = gts_oracle.points_in_boxes(pts, b9, libm_trig(b9[:, 8])).sum(0) if len(boxes) else np.zeros(0)
        d = detections.get(t)
        dets = []
        if d is not None:
            db, ds, dl = _np(d["box3d_lidar"]), _np(d["scores"]), _np(d["label_preds"])
            dets = [(np.float32(ds[i]) + np.float32(0.0), i, int(dl[i]), _box7(db[i])) for i in range(len(ds))]
        frames.append((list(g["names"]), boxes, counts, dets))
    per_class, per_range = {}, {}
    for c, name in enumerate(class_names):
        thr = np.float32(table[name])
        cuts = cutoffs([s for fr in frames for s, _, lab, _ in fr[3] if lab == c], K)
        # per breakdown b (0: ALL, 1: by range) and region: per cutoff [TP1, TP2, H1, H2, FP], and n_gt
        acc = {(b, r): [[0.0] * 5 for _ in cuts] for b, r in [(0, None), (1, 0), (1, 1), (1, 2)]}
        n_gt = {key: [0, 0] for key in acc}
        for names, boxes, counts, dets in frames:
            gi = [j for j, n in enumerate(names) if n == name]
            grange = {j: range_bin(boxes[j][0], boxes[j][1]) for j in gi}
            for j in gi:
                for key in ((0, None), (1, grange[j])):
                    n_gt[key][0] += counts[j] > 5
                    n_gt[key][1] += counts[j] >= 1
            mine = sorted([d for d in dets if d[2] == c], key=lambda d: (-d[0], d[1]))
            drange = {i: range_bin(box[0], box[1]) for _, i, _, box in mine}
            iou = {}
            for _, i, _, box in mine:
                for j in gi:
                    g = boxes[j]
                    if math.hypot(float(box[0]) - float(g[0]), float(box[1]) - float(g[1])) > \
                            0.5 * (math.hypot(float(box[3]), float(box[4])) + math.hypot(float(g[3]), float(g[4]))) + 1.0:
                        continue
                    v = P.aligned_iou3d(box, g)
                    if np.float32(v) >= thr:
                        iou[(i, j)] = float(np.float32(v))
            for k, cut in enumerate(cuts):
                live = [d for d in mine if d[0] >= cut]
                for b in (0, 1):
                    w = {(i, j): v for (i, j), v in iou.items() if any(d[1] == i for d in live)
                         and (b == 0 or drange[i] == grange[j])}
                    m = assign(w, [d[1] for d in live])
                    for s, i, _, box in live:
                        a = acc[(b, None if b == 0 else drange[i])][k]
                        if i not in m:
                            a[4] += 1
                            continue
                        j = m[i]
                        h = heading_accuracy(box[6], boxes[j][6])
                        if counts[j] > 5:
                            a[0] += 1
                            a[2] += h
                        if counts[j] >= 1:
                            a[1] += 1
                            a[3] += h

        def result(key):
            a, (n1, n2) = acc[key], n_gt[key]
            return dict(AP_L1=ap_points([(x[0], x[4]) for x in a], n1), APH_L1=ap_points([(x[2], x[4]) for x in a], n1),
                        AP_L2=ap_points([(x[1], x[4]) for x in a], n2), APH_L2=ap_points([(x[3], x[4]) for x in a], n2),
                        n_gt_L1=int(n1), n_gt_L2=int(n2))
        per_class[name] = result((0, None))
        per_range[name] = {r: result((1, ri)) for ri, r in enumerate(RANGES)}

    def means(per):
        out = {}
        for key in ("AP_L1", "APH_L1", "AP_L2", "APH_L2"):
            vals = [v[key] for v in per if v[key] == v[key]]
            out["m" + key] = float(np.mean(vals)) if vals else float("nan")
        return out
    res = means(per_class.values())
    res["per_class"] = per_class
    res["per_range"] = per_range
    res["range_means"] = {r: means([per_range[n][r] for n in class_names]) for r in RANGES}
    return res


def frame_assignments(boxes_gt, names, det_boxes, det_scores, det_labels, class_names, thresholds, cut, b, box_index):
    """Per (class) of one frame at one cutoff and breakdown: (the tie-ruled pairing {det: box}, scipy's own maximum
    total, the IoU dict), for comparing the assignment alone.  box_index = the full IoU routine (no shortcut)."""
    out = {}
    for c, name in enumerate(class_names):
        gi = [j for j, n in enumerate(names) if n == name]
        live = sorted([i for i in range(len(det_scores)) if det_labels[i] == c and np.float32(det_scores[i]) >= cut[c]],
                      key=lambda i: (-float(det_scores[i]), i))
        w = {}
        for i in live:
            for j in gi:
                if b == 1 and range_bin(det_boxes[i][0], det_boxes[i][1]) != range_bin(boxes_gt[j][0], boxes_gt[j][1]):
                    continue
                v = np.float32(box_index(i, j))
                if v >= np.float32(thresholds[c]):
                    w[(i, j)] = float(v)
        out[name] = (assign(w, live), _best(w, [])[0], w)
    return out
