"""Sequential restatement of pillarnext_b200.track.track and evaluate_waymo_tracking.waymo_tracking_metrics (TEST
INFRASTRUCTURE -- see oracle/__init__.py), independent of the product.

The tracker walks one (sequence, class) at a time in numpy fp32 scalars, in the order the track.py docstring states
(the pose transform in Python floats, i.e. fp64, rounded once).  The metric walks one (sequence, class, cutoff) at a
time: IoU by predict_oracle.aligned_iou3d, the carry-over in pair order, then waymo_hungarian_oracle.assign (scipy's
linear_sum_assignment plus the tie rule) on the remaining pairs."""
import math

import numpy as np

from oracle import gts_oracle, predict_oracle as P
from oracle.waymo_hungarian_oracle import assign, cutoffs
from oracle.waymo_metric_oracle import IOU_THRESHOLDS, _box7, _np

F32 = np.float32
MAX_DIST = {"vehicle": 2.0, "pedestrian": 1.0, "cyclist": 1.5}


def _order(frames):
    return sorted(frames, key=lambda t: (str(frames[t]["sequence"]), int(frames[t]["timestamp"])))


def _global(T, b):
    x, y, z, vx, vy = (float(F32(b[k])) for k in (0, 1, 2, 6, 7))
    p = (F32(T[0][0] * x + T[0][1] * y + T[0][2] * z + T[0][3]), F32(T[1][0] * x + T[1][1] * y + T[1][2] * z + T[1][3]))
    v = (F32(T[0][0] * vx + T[0][1] * vy), F32(T[1][0] * vx + T[1][1] * vy))
    return p, v


def track(detections, frames, class_names, max_dist=None, max_age=3, min_score=0.0):
    """Same inputs as track.track -> token -> tracking ids [K] int64 (numpy)."""
    table = dict(MAX_DIST, **(max_dist or {}))
    tokens = _order(frames)
    out = {t: np.full(len(_np(detections[t]["scores"])), -1, np.int64) for t in detections}
    seqs = {}
    for t in tokens:
        seqs.setdefault(str(frames[t]["sequence"]), []).append(t)
    for seq_tokens in seqs.values():
        births = []                                        # (frame, class, local id, [(token, det)] of the track)
        members = {}
        for c, name in enumerate(class_names):
            maxd = F32(table[name])
            live, next_id = [], 0                          # [q (x, y), v, local id, misses]
            for f, t in enumerate(seq_tokens):
                dt = F32(0.0) if f == 0 else F32((int(frames[t]["timestamp"]) - int(frames[seq_tokens[f - 1]]["timestamp"])) * 1e-6)
                T = np.asarray(frames[t]["pose"], np.float64).reshape(4, 4).tolist()
                d = detections.get(t)
                dets = []
                if d is not None:
                    b, s, lab = _np(d["box3d_lidar"]), _np(d["scores"]), _np(d["label_preds"])
                    dets = sorted([i for i in range(len(s)) if int(lab[i]) == c],
                                  key=lambda i: (-float(F32(s[i]) + F32(0)), i))
                claimed, born = {}, []
                for i in dets:
                    if not F32(s[i]) >= F32(min_score):
                        continue
                    p, v = _global(T, b[i])
                    bx, by = p[0] - v[0] * dt, p[1] - v[1] * dt
                    best, bj = None, None
                    for j, tr in enumerate(live):
                        if j in claimed:
                            continue
                        dx, dy = bx - tr[0][0], by - tr[0][1]
                        dist = np.sqrt(dx * dx + dy * dy)
                        if dist <= maxd and (best is None or dist < best):
                            best, bj = dist, j
                    if bj is not None:
                        claimed[bj] = (p, v)
                        members[(c, live[bj][2])].append((t, i))
                    else:
                        born.append([p, v, next_id, 0])
                        births.append((f, c, next_id))
                        members[(c, next_id)] = [(t, i)]
                        next_id += 1
                for j, tr in enumerate(live):
                    if j in claimed:
                        tr[0], tr[1], tr[3] = claimed[j][0], claimed[j][1], 0
                    else:
                        tr[0] = (tr[0][0] + tr[1][0] * dt, tr[0][1] + tr[1][1] * dt)
                        tr[3] += 1
                live = [tr for tr in live + born if tr[3] <= max_age]
        for gid, (f, c, local) in enumerate(sorted(births)):
            for t, i in members[(c, local)]:
                out[t][i] = gid
    return out


def tracking_metrics(gts, tracks, class_names, iou_thresholds=None, num_score_cutoffs=11):
    """Same inputs and outputs as evaluate_waymo_tracking.waymo_tracking_metrics."""
    from det3d.datasets.pipelines.sample_ops import libm_trig
    table = dict(IOU_THRESHOLDS, **(iou_thresholds or {}))
    K = num_score_cutoffs
    tokens = _order(gts)
    frames = []
    for t in tokens:
        g = gts[t]
        boxes = [_box7(b) for b in _np(g["boxes"]).reshape(len(g["names"]), -1)]
        b9 = np.zeros((len(boxes), 9), np.float32)
        for j, b in enumerate(boxes):
            b9[j, :6], b9[j, 8] = b[:6], b[6]
        if "num_points" in g:
            counts = np.asarray(_np(g["num_points"])).reshape(-1)
        else:
            pts = np.asarray(_np(g["points"]), np.float32)[:, :3]
            counts = gts_oracle.points_in_boxes(pts, b9, libm_trig(b9[:, 8])).sum(0) if len(boxes) else np.zeros(0)
        d = tracks.get(t)
        dets = []
        if d is not None:
            db, ds, dl, di = _np(d["box3d_lidar"]), _np(d["scores"]), _np(d["label_preds"]), _np(d["tracking_id"])
            dets = [(F32(ds[i]) + F32(0.0), i, int(dl[i]), _box7(db[i]), int(di[i])) for i in range(len(ds)) if di[i] >= 0]
        frames.append((str(g["sequence"]), list(g["names"]), [str(o) for o in g["ids"]], boxes, counts, dets))
    per_class = {}
    for c, name in enumerate(class_names):
        thr = F32(table[name])
        cuts = cutoffs([d[0] for fr in frames for d in fr[5] if d[2] == c], K)
        acc = [[0, 0, 0, 0, 0, 0.0, 0.0, 0] for _ in cuts]   # matches, tp1, mism1, tp2, mism2, dist1, dist2, passing
        n_gt = [0, 0]
        ious = []
        for seq, names, ids, boxes, counts, dets in frames:
            gi = [j for j, n in enumerate(names) if n == name]
            n_gt[0] += sum(counts[j] > 5 for j in gi)
            n_gt[1] += sum(counts[j] >= 1 for j in gi)
            mine = sorted([d for d in dets if d[2] == c], key=lambda d: (-d[0], d[1]))
            iou = {}
            for _, i, _, box, _ in mine:
                for j in gi:
                    g = boxes[j]
                    if math.hypot(float(box[0]) - float(g[0]), float(box[1]) - float(g[1])) > \
                            0.5 * (math.hypot(float(box[3]), float(box[4])) + math.hypot(float(g[3]), float(g[4]))) + 1.0:
                        continue
                    v = F32(P.aligned_iou3d(box, g))
                    if v >= thr:
                        iou[(i, j)] = float(v)
            ious.append(iou)
        for k, cut in enumerate(cuts):
            a = acc[k]
            last = {}
            for (seq, names, ids, boxes, counts, dets), iou in zip(frames, ious):
                live = sorted([d for d in dets if d[2] == c and d[0] >= cut], key=lambda d: (-d[0], d[1]))
                a[7] += len(live)
                tid = {d[1]: d[4] for d in live}
                obj = lambda j: (seq, ids[j])                              # noqa: E731
                kept = {}
                for d in live:
                    for j in sorted(j for (i, j) in iou if i == d[1]):
                        if d[1] in kept or j in kept.values():
                            continue
                        if last.get(obj(j)) == d[4]:
                            kept[d[1]] = j
                w = {(i, j): v for (i, j), v in iou.items() if i in tid and i not in kept and j not in kept.values()}
                m = assign(w, [d[1] for d in live if d[1] not in kept])
                for i, j in list(kept.items()) + sorted(m.items(), key=lambda p: [d[1] for d in live].index(p[0])):
                    o, v = obj(j), iou[(i, j)]
                    mism = o in last and last[o] != tid[i]
                    last[o] = tid[i]
                    a[0] += 1
                    if counts[j] > 5:
                        a[1] += 1
                        a[2] += mism
                        a[5] += 1.0 - v
                    if counts[j] >= 1:
                        a[3] += 1
                        a[4] += mism
                        a[6] += 1.0 - v
        res = {}
        for li, lv in enumerate(("L1", "L2")):
            n = int(n_gt[li])
            res["n_gt_" + lv] = n
            if n == 0:
                vals = dict(MOTA=math.nan, MOTP=math.nan, miss=math.nan, mismatch=math.nan, fp=math.nan,
                            score_cutoff=math.nan)
            elif not cuts:
                vals = dict(MOTA=0.0, MOTP=math.nan, miss=1.0, mismatch=0.0, fp=0.0, score_cutoff=math.nan)
            else:
                best = None
                for k, a in enumerate(acc):
                    tp, mism, fp = a[1 + 2 * li], a[2 + 2 * li], a[7] - a[0]
                    mota = 1.0 - ((n - tp) + mism + fp) / n
                    if best is None or mota > best[0]:
                        best = (mota, tp, mism, fp, a[5 + li], k)
                mota, tp, mism, fp, dist, k = best
                vals = dict(MOTA=mota, MOTP=dist / tp if tp else math.nan, miss=(n - tp) / n, mismatch=mism / n,
                            fp=fp / n, score_cutoff=float(cuts[k]))
            res.update({key + "_" + lv: float(v) for key, v in vals.items()})
        per_class[name] = res
    out = {}
    for lv in ("L1", "L2"):
        for key in ("MOTA", "MOTP"):
            vals = [v[key + "_" + lv] for v in per_class.values() if v["n_gt_" + lv] > 0 and not math.isnan(v[key + "_" + lv])]
            out["m%s_%s" % (key, lv)] = float(np.mean(vals)) if vals else math.nan
    out["per_class"] = per_class
    return out
