"""Sequential restatement of the nuScenes detection score of pillarnext_b200/evaluate_nuscenes.py (TEST INFRASTRUCTURE --
see oracle/__init__.py), written in the devkit's own loop structure: filter the boxes one at a time, then per class and
per distance threshold visit the detections in (score, position) order, each taking an arg-min over its frame's boxes.

The point counts are gts_oracle.points_in_boxes (the reference's points_in_boxes_jit arithmetic, pinned by
tests/test_gt_sampling_cpu.py) with libm (cosf, sinf).  Distances and errors are Python floats (fp64) of the fp32 inputs;
the curves use the same numpy interpolation calls as the devkit."""
import math

import numpy as np

from oracle import gts_oracle

DIST_THS = (0.5, 1.0, 2.0, 4.0)
DIST_TH_TP = 2.0
CLASS_RANGE = {"car": 50.0, "truck": 50.0, "bus": 50.0, "trailer": 50.0, "construction_vehicle": 50.0,
               "pedestrian": 40.0, "motorcycle": 40.0, "bicycle": 40.0, "traffic_cone": 30.0, "barrier": 30.0}
TP_METRICS = [("trans_err", "ATE"), ("scale_err", "ASE"), ("orient_err", "AOE"), ("vel_err", "AVE"), ("attr_err", "AAE")]


def _np(x):
    return x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)


def _box9(b):
    b = [float(v) for v in np.asarray(b, np.float32)]
    return b if len(b) == 9 else b[:6] + [0.0, 0.0, b[6]]


def attribute(name, vx, vy):
    """The detection attribute rule of the reference's nuScenes evaluation, with each class's default attribute."""
    speed = math.sqrt(vx * vx + vy * vy)
    if speed > 0.2:
        if name in ("car", "construction_vehicle", "bus", "truck", "trailer"):
            return "vehicle.moving"
        if name in ("bicycle", "motorcycle"):
            return "cycle.with_rider"
    else:
        if name == "pedestrian":
            return "pedestrian.standing"
        if name == "bus":
            return "vehicle.parked"
    if name in ("car", "truck", "trailer", "construction_vehicle"):
        return "vehicle.parked"
    if name == "bus":
        return "vehicle.moving"
    if name in ("bicycle", "motorcycle"):
        return "cycle.without_rider"
    if name == "pedestrian":
        return "pedestrian.moving"
    if name in ("barrier", "traffic_cone"):
        return "cycle.with_rider"
    return ""


def center_distance(a, b):
    dx, dy = a[0] - b[0], a[1] - b[1]
    return math.sqrt(dx * dx + dy * dy)


def angle_diff(x, y, period):
    diff = (x - y + period / 2) % period - period / 2
    if diff > math.pi:
        diff = diff - 2 * math.pi
    return diff


def scale_iou(g, d):
    inter = min(g[3], d[3]) * min(g[4], d[4]) * min(g[5], d[5])
    vg, vd = g[3] * g[4] * g[5], d[3] * d[4] * d[5]
    return inter / (vg + vd - inter)


def cummean(x):
    if np.isnan(x).all():
        return np.ones(len(x))
    s, n = np.nancumsum(x.astype(float)), np.cumsum(~np.isnan(x))
    return np.divide(s, n, out=np.zeros_like(s), where=n != 0)


def accumulate(gt_boxes, pred_boxes, class_name, dist_th):
    """gt_boxes: token -> list of (name, box9, attr); pred_boxes: list of (token, name, score, box9, attr) in the order
    of the detections.  -> None (no predictions) or (precision, confidence, errors) on the 101 recall points."""
    npos = sum(1 for boxes in gt_boxes.values() for g in boxes if g[0] == class_name)
    if npos == 0:
        return None
    preds = [p for p in pred_boxes if p[1] == class_name]
    confs = [p[2] for p in preds]
    sortind = [i for (v, i) in sorted((v, i) for (i, v) in enumerate(confs))][::-1]
    tp, fp, conf = [], [], []
    data = {k: [] for k, _ in TP_METRICS}
    data["conf"] = []
    taken = set()
    for ind in sortind:
        token, _, score, box, attr = preds[ind]
        min_dist, match = math.inf, None
        for gi, (gname, gbox, _) in enumerate(gt_boxes[token]):
            if gname == class_name and (token, gi) not in taken:
                d = center_distance(gbox, box)
                if d < min_dist:
                    min_dist, match = d, gi
        if min_dist < dist_th:
            taken.add((token, match))
            tp.append(1), fp.append(0), conf.append(score)
            _, gbox, gattr = gt_boxes[token][match]
            data["trans_err"].append(center_distance(gbox, box))
            dvx, dvy = box[6] - gbox[6], box[7] - gbox[7]
            data["vel_err"].append(math.sqrt(dvx * dvx + dvy * dvy))
            data["scale_err"].append(1.0 - scale_iou(gbox, box))
            period = math.pi if class_name == "barrier" else 2 * math.pi
            data["orient_err"].append(abs(angle_diff(gbox[8], box[8], period)))
            data["attr_err"].append(float("nan") if gattr == "" else 1.0 - float(gattr == attr))
            data["conf"].append(score)
        else:
            tp.append(0), fp.append(1), conf.append(score)
    if not data["trans_err"]:
        return None
    tp, fp, conf = np.cumsum(tp).astype(float), np.cumsum(fp).astype(float), np.array(conf)
    prec, rec = tp / (fp + tp), tp / float(npos)
    r = np.linspace(0, 1, 101)
    prec = np.interp(r, rec, prec, right=0)
    conf = np.interp(r, rec, conf, right=0)
    errs = {}
    for k, _ in TP_METRICS:
        tmp = cummean(np.array(data[k]))
        errs[k] = np.interp(conf[::-1], np.array(data["conf"])[::-1], tmp[::-1])[::-1]
    return prec, conf, errs


def calc_ap(md):
    if md is None:
        return 0.0
    p = np.copy(md[0])[11:] - 0.1
    p[p < 0] = 0
    return float(np.mean(p)) / 0.9


def calc_tp(md, key):
    if md is None:
        return 1.0
    nz = np.nonzero(md[1])[0]
    last = nz[-1] if len(nz) else 0
    if last < 11:
        return 1.0
    return float(np.mean(md[2][key][11:last + 1]))


def nuscenes_metrics(gts, detections, class_names, class_range=None):
    """Same inputs and outputs as pillarnext_b200.evaluate_nuscenes.nuscenes_metrics."""
    from det3d.datasets.pipelines.sample_ops import libm_trig
    ranges = dict(CLASS_RANGE, **(class_range or {}))
    for n in class_names:
        if n not in ranges:
            raise ValueError("no detection range for class %r" % n)
    for t, d in detections.items():
        if t not in gts:
            raise ValueError("detections for a token without ground truth: %r" % t)
        if len(d["scores"]) > 500:
            raise ValueError("more than 500 detections in frame %r" % t)
    gt_boxes = {}
    for t, g in gts.items():
        boxes = [_box9(b) for b in _np(g["boxes"]).reshape(len(g["names"]), -1)]
        if "num_points" in g:
            counts = [int(n) for n in _np(g["num_points"])]
        elif "points" in g:
            b9 = np.array(boxes, np.float32).reshape(-1, 9)
            pts = np.asarray(_np(g["points"]), np.float32)[:, :3]
            counts = list(gts_oracle.points_in_boxes(pts, b9, libm_trig(b9[:, 8])).sum(0)) if len(boxes) else []
        else:
            raise ValueError("frame %r has neither num_points nor points" % t)
        kept = []
        for j, (name, box) in enumerate(zip(g["names"], boxes)):
            if name not in class_names:
                continue
            if not math.sqrt(box[0] * box[0] + box[1] * box[1]) < ranges[name]:
                continue
            if counts[j] == 0:
                continue
            attr = g["attributes"][j] if "attributes" in g else attribute(name, box[6], box[7])
            kept.append((name, box, attr))
        gt_boxes[t] = kept
    pred_boxes = []
    for t, d in detections.items():
        db, ds, dl = _np(d["box3d_lidar"]), _np(d["scores"]), _np(d["label_preds"])
        for i in range(len(ds)):
            name, box = class_names[int(dl[i])], _box9(db[i])
            if not math.sqrt(box[0] * box[0] + box[1] * box[1]) < ranges[name]:
                continue
            pred_boxes.append((t, name, float(np.float32(ds[i])), box, attribute(name, box[6], box[7])))
    per_class = {}
    for name in class_names:
        mds = {th: accumulate(gt_boxes, pred_boxes, name, th) for th in DIST_THS}
        aps = [calc_ap(mds[th]) for th in DIST_THS]
        res = {"n_gt": sum(1 for b in gt_boxes.values() for g in b if g[0] == name), "AP": 100.0 * float(np.mean(aps))}
        for th, a in zip(DIST_THS, aps):
            res["AP@%.1f" % th] = 100.0 * a
        for key, short in TP_METRICS:
            if name == "traffic_cone" and key in ("attr_err", "vel_err", "orient_err"):
                res[short] = float("nan")
            elif name == "barrier" and key in ("attr_err", "vel_err"):
                res[short] = float("nan")
            else:
                res[short] = calc_tp(mds[DIST_TH_TP], key)
        per_class[name] = res
    out = {"mAP": float(np.mean([v["AP"] for v in per_class.values()]))}
    total = 5.0 * out["mAP"] / 100.0
    for _, short in TP_METRICS:
        vals = [v[short] for v in per_class.values() if not math.isnan(v[short])]
        out["m" + short] = float(np.mean(vals)) if vals else float("nan")
        total += max(0.0, 1.0 - out["m" + short])
    out["NDS"] = 100.0 * total / 10.0
    out["per_class"] = per_class
    return out
