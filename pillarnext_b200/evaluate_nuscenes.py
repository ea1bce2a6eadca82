"""nuScenes detection score (NDS) with its true-positive errors, restated from the devkit's published definition (the
`detection_cvpr_2019` configuration), because the reference hands nuScenes scoring to the devkit
(det3d/datasets/nuscenes/nusc.py:123-245), which is not installable here.  Float64 throughout unless a step says
otherwise.

  * Inputs.  gts: token -> {"boxes" [M, 9] (x, y, z, dx, dy, dz, vx, vy, yaw), "names" list[str], and either
    "num_points" [M] or "points" [N, >= 3] (x, y, z first)}, optionally "attributes" list[str].  detections: token ->
    the reference's validation_step output {"box3d_lidar" [K, 9], "scores" [K], "label_preds" [K]} (CPU or CUDA tensors,
    or arrays), labels indexing class_names.  Ground-truth boxes whose name is not in class_names are not evaluated.  A
    detection token without ground truth raises ValueError.
  * Cap.  A frame with more than 500 detections raises ValueError before any filtering (the devkit's
    max_boxes_per_sample).
  * Range filter, ground truth and detections alike: a box is kept when sqrt(x^2 + y^2) of its fp32 centre is < r of its
    class (strict).  Defaults: car, truck, bus, trailer, construction_vehicle 50 m; pedestrian, motorcycle, bicycle 40 m;
    traffic_cone, barrier 30 m.  class_range={name: r} overrides or extends them; a class with no range raises ValueError.
  * Point filter: ground-truth boxes with 0 points are dropped.  The counts are "num_points" where a frame gives them,
    otherwise the frame's points inside each box, counted on the GPU with the reference's points_in_boxes_jit test (libm
    cosf / sinf of the yaw), in chunks of frames of at most POINT_BUDGET points.  A frame with neither raises ValueError.
    A dropped box disappears: a detection that would have matched it is a false positive.
  * Visit order, per class: descending score; ties to the HIGHER position, position being the order of the frames in
    `detections`, then the order within the frame (the devkit's sorted((score, i))[::-1]).
  * Matching, per frame, class and threshold d in {0.5, 1, 2, 4} m: each detection in visit order takes the not yet
    matched ground-truth box of its class and frame with the smallest centre distance sqrt(dx^2 + dy^2) (fp64
    differences of the fp32 coordinates), ties to the lower box index; it is a true positive iff that distance is < d.
  * True-positive errors, for each TP of the 2 m match: trans_err = the centre distance; vel_err = |(vx, vy)_det -
    (vx, vy)_gt|_2 (NaN for a NaN ground-truth velocity); scale_err = 1 - V / (V_gt + V_det - V) with V the product of
    the elementwise minima of (dx, dy, dz); orient_err = |((yaw_gt - yaw_det + p/2) mod p) - p/2|, less 2 pi where that
    difference exceeds pi, with the non-negative mod and p = pi for barrier, 2 pi otherwise; attr_err = 1 - [attr_gt ==
    attr_det], NaN when attr_gt is "".
  * Attributes.  A detection's attribute follows the reference's rule (nusc.py:152-185): at speed sqrt(vx^2 + vy^2) >
    0.2 m/s car, truck, bus, trailer and construction_vehicle are vehicle.moving, bicycle and motorcycle
    cycle.with_rider; at or below it pedestrian is pedestrian.standing and bus vehicle.parked; every other case takes
    the class's most frequent attribute in the nuScenes training set (DEFAULT_ATTRIBUTE).  Ground-truth attributes are
    "attributes" where a frame gives them, otherwise derived from the ground-truth velocity by the same rule.
  * Curves, per class and threshold, with npos the class's boxes left by the filters: npos = 0 or no TP gives AP 0 and
    every error 1.  Otherwise cumulative tp and fp, prec = tp / (tp + fp), rec = tp / npos; with r = linspace(0, 1, 101),
    P = interp(r, rec, prec, right=0), conf = interp(r, rec, score, right=0), AP = mean(max(P[11:] - 0.1, 0)) / 0.9.
    Each error: the NaN-aware cumulative mean over the TPs in visit order (all NaN: ones; else nancumsum / count, 0 where
    the count is 0), E = interp(conf[::-1], tp_conf[::-1], cummean[::-1])[::-1], and the class's error is
    mean(E[11 : last + 1]) with last the last index where conf != 0 (0 if none), or 1.0 if last < 11.
  * NaN by rule: traffic_cone's attr, vel and orient errors; barrier's attr and vel errors.
  * Summary: mAP = the mean over ALL class_names of the mean over the four thresholds (a class without ground truth
    counts as 0); mATE .. mAAE = nanmean over the classes; NDS = (5 mAP + sum over the five errors of max(0, 1 - mTP))
    / 10, a NaN mean scoring 0.  mAP, NDS and the per-class APs are reported in percent, the errors in their own units
    (metres, 1 - IoU, radians, m/s, 1 - accuracy).

Known differences from the devkit: the boxes are in the lidar frame, not the global or ego frame, so the range is
measured from the sensor origin; the yaw is used directly instead of through quaternions; there is no bike-rack
filter; the point counts come from the points-in-box test, not from the annotation; ground-truth attributes are derived
from the velocity when absent.

The point counts and the matching run on the GPU (pnx_eval_count_points, pnx_eval_match_center, csrc/det_eval.cu);
filters, attributes and curves are vectorised numpy.  oracle/nds_oracle.py restates the whole definition in the
devkit's own loop structure."""
import math

import numpy as np
import torch

from .evaluate_waymo import _arr, _box9

DIST_THS = (0.5, 1.0, 2.0, 4.0)
DIST_TH_TP = 2.0
MAX_BOXES_PER_SAMPLE = 500
MIN_RECALL = MIN_PRECISION = 0.1
POINT_BUDGET = 1 << 24            # points on the device in one count (16.8 M x 16 bytes)
CLASS_RANGE = {"car": 50.0, "truck": 50.0, "bus": 50.0, "trailer": 50.0, "construction_vehicle": 50.0,
               "pedestrian": 40.0, "motorcycle": 40.0, "bicycle": 40.0, "traffic_cone": 30.0, "barrier": 30.0}
TP_METRICS = (("trans_err", "ATE"), ("scale_err", "ASE"), ("orient_err", "AOE"), ("vel_err", "AVE"), ("attr_err", "AAE"))
NAN_BY_RULE = {"traffic_cone": ("attr_err", "vel_err", "orient_err"), "barrier": ("attr_err", "vel_err")}
ATTRIBUTES = ("vehicle.moving", "vehicle.parked", "vehicle.stopped", "cycle.with_rider", "cycle.without_rider",
              "pedestrian.moving", "pedestrian.standing", "pedestrian.sitting_lying_down")
MOVING_ATTRIBUTE = {"car": "vehicle.moving", "truck": "vehicle.moving", "bus": "vehicle.moving",
                    "trailer": "vehicle.moving", "construction_vehicle": "vehicle.moving",
                    "bicycle": "cycle.with_rider", "motorcycle": "cycle.with_rider"}
STILL_ATTRIBUTE = {"pedestrian": "pedestrian.standing", "bus": "vehicle.parked"}
DEFAULT_ATTRIBUTE = {"car": "vehicle.parked", "truck": "vehicle.parked", "trailer": "vehicle.parked",
                     "construction_vehicle": "vehicle.parked", "bus": "vehicle.moving",
                     "bicycle": "cycle.without_rider", "motorcycle": "cycle.without_rider",
                     "pedestrian": "pedestrian.moving", "barrier": "cycle.with_rider", "traffic_cone": "cycle.with_rider"}
MOVING_SPEED = 0.2


def class_ranges(class_names, class_range=None):
    """Per-class detection range in metres: the defaults above, overridden or extended by `class_range`."""
    table = dict(CLASS_RANGE, **(class_range or {}))
    missing = [n for n in class_names if n not in table]
    if missing:
        raise ValueError("no detection range for classes %s: pass class_range={name: metres}" % missing)
    return np.array([float(table[n]) for n in class_names], np.float64)


class _Vocab:
    """Attribute strings <-> int codes; "" is -1 (no attribute)."""

    def __init__(self):
        self.codes = {"": -1}
        for a in ATTRIBUTES:
            self.code(a)

    def code(self, a):
        return self.codes.setdefault(a, len(self.codes) - 1)

    def encode(self, strings):
        u, inv = np.unique(np.asarray(strings, dtype=str), return_inverse=True)
        return np.array([self.code(str(a)) for a in u], np.int32)[inv.reshape(-1)] if len(u) else np.zeros(0, np.int32)


def derive_attributes(labels, velocity, class_names, vocab):
    """Attribute codes of boxes of class labels [K] (indices into class_names) with velocity [K, 2] fp32: the rule of
    the module docstring, vectorised."""
    tab = [[vocab.code(t.get(n, "")) for n in class_names] for t in (MOVING_ATTRIBUTE, STILL_ATTRIBUTE, DEFAULT_ATTRIBUTE)]
    moving_of, still_of, default_of = (np.array(t + [-1], np.int32) for t in tab)       # label -1 -> the extra slot
    v = np.asarray(velocity, np.float32).astype(np.float64)
    moving = np.sqrt(v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) > MOVING_SPEED
    out = np.where(moving, moving_of[labels], still_of[labels])
    return np.where(out < 0, default_of[labels], out).astype(np.int32)


def _radius(boxes):
    b = boxes.astype(np.float64)
    return np.sqrt(b[..., 0] * b[..., 0] + b[..., 1] * b[..., 1])


def pack(gts, detections, class_names, class_range=None):
    """gts / detections as for nuscenes_metrics -> filtered, keyed and segmented flat arrays (numpy, host); det_pos =
    each kept detection's position in the detections concatenated in the order of `detections`.  The point filter
    waits for the counts (run_device / run_host): gt_classes has the range filter applied only."""
    rng = class_ranges(class_names, class_range)
    tokens = list(gts)
    frame_of = {t: f for f, t in enumerate(tokens)}
    unknown = [t for t in detections if t not in frame_of]
    if unknown:
        raise ValueError("detections for tokens without ground truth: %s" % unknown[:5])
    over = [(t, len(d["scores"])) for t, d in detections.items() if len(d["scores"]) > MAX_BOXES_PER_SAMPLE]
    if over:
        raise ValueError("more than %d detections in frame %s (%d)" % (MAX_BOXES_PER_SAMPLE, over[0][0], over[0][1]))
    B, C = len(tokens), len(class_names)
    vocab = _Vocab()
    # ground truth: flat over all frames, then padded to [B, M]
    sizes = np.array([len(gts[t]["names"]) for t in tokens], np.int64)
    M = int(max(1, sizes.max() if B else 1))
    boxes, names, num_points, points, attrs = [], [], [], [], []
    for t in tokens:
        g = gts[t]
        b = _box9(g["boxes"])
        if len(b) != len(g["names"]):
            raise ValueError("frame %s: %d boxes but %d names" % (t, len(b), len(g["names"])))
        boxes.append(b)
        names.extend(g["names"])
        if "num_points" in g:
            n = _arr(g["num_points"]).reshape(-1).astype(np.int64)
            if len(n) != len(b):
                raise ValueError("frame %s: %d boxes but %d num_points" % (t, len(b), len(n)))
            num_points.append(n)
            points.append(None)
        elif "points" in g:
            num_points.append(np.full(len(b), -1, np.int64))
            points.append(_arr(g["points"], np.float32))
        else:
            raise ValueError("frame %s: ground truth needs num_points or points for the point filter" % t)
        a = g.get("attributes")
        if a is not None and len(a) != len(b):
            raise ValueError("frame %s: %d boxes but %d attributes" % (t, len(b), len(a)))
        attrs.append(a)
    flat = np.concatenate(boxes) if B else np.zeros((0, 9), np.float32)
    nm = np.asarray(names, dtype=str)
    cls = np.full(len(flat), -1, np.int32)
    for c, name in enumerate(class_names):
        cls[nm == name] = c
    cls[(cls >= 0) & ~(_radius(flat) < rng[np.maximum(cls, 0)])] = -1
    derived = derive_attributes(cls, flat[:, 6:8], class_names, vocab)
    start = np.cumsum(sizes) - sizes
    gattr = np.concatenate([derived[s:s + n] if a is None else vocab.encode(a)
                            for s, n, a in zip(start, sizes, attrs)]) if B else np.zeros(0, np.int32)
    fr = np.repeat(np.arange(B), sizes)
    pos = np.arange(len(flat)) - np.repeat(start, sizes)
    gt_boxes = np.zeros((B, M, 9), np.float32)
    gt_boxes[:, :, 3:6] = 1.0
    gt_classes = np.full((B, M), -1, np.int32)
    gt_attr = np.full((B, M), -1, np.int32)
    known = np.full((B, M), -1, np.int64)
    gt_boxes[fr, pos], gt_classes[fr, pos], gt_attr[fr, pos] = flat, cls, gattr
    known[fr, pos] = np.concatenate(num_points) if B else np.zeros(0, np.int64)
    # detections, in the order of `detections` (their position decides score ties)
    db, ds, dl, df = [np.zeros((0, 9), np.float32)], [np.zeros(0, np.float32)], [np.zeros(0, np.int64)], [np.zeros(0, np.int64)]
    for t, d in detections.items():
        b = _box9(d["box3d_lidar"])
        s = _arr(d["scores"], np.float32).reshape(-1)
        lab = _arr(d["label_preds"]).reshape(-1).astype(np.int64)
        if not (len(b) == len(s) == len(lab)):
            raise ValueError("frame %s: box3d_lidar, scores and label_preds differ in length" % t)
        if len(lab) and (lab.min() < 0 or lab.max() >= C):
            raise ValueError("frame %s: label_preds outside [0, %d)" % (t, C))
        if np.isnan(s).any():
            raise ValueError("frame %s: NaN scores" % t)
        db.append(b), ds.append(s), dl.append(lab), df.append(np.full(len(s), frame_of[t], np.int64))
    det_boxes, det_scores, det_labels, det_frames = (np.concatenate(x) for x in (db, ds, dl, df))
    keep = _radius(det_boxes) < rng[det_labels]
    det_pos = np.nonzero(keep)[0]
    det_boxes, det_scores, det_labels, det_frames = det_boxes[keep], det_scores[keep], det_labels[keep], det_frames[keep]
    score64 = det_scores.astype(np.float64)
    seg = det_frames * C + det_labels
    seg_count = np.bincount(seg, minlength=B * C).astype(np.int32)
    return dict(B=B, M=M, C=C, class_names=list(class_names), gt_boxes=gt_boxes, gt_classes=gt_classes, gt_attr=gt_attr,
                num_points=known, points=points, det_boxes=np.ascontiguousarray(det_boxes), det_scores=det_scores,
                det_labels=det_labels, det_frames=det_frames, det_pos=det_pos,
                det_attr=derive_attributes(det_labels, det_boxes[:, 6:8], class_names, vocab),
                order=np.lexsort((-det_pos, -score64, seg)).astype(np.int64),
                visit=np.lexsort((-det_pos, -score64, det_labels)).astype(np.int64),
                seg_start=(np.cumsum(seg_count) - seg_count).astype(np.int32), seg_count=seg_count)


def count_points(pk, count, point_budget=POINT_BUDGET):
    """counts [B, M]: num_points where a frame gives them; the other frames' boxes counted by count(points [n, 4]
    (frame within the chunk, x, y, z), boxes, classes, libm trig) -> [F, M], over chunks of whole frames holding at most
    point_budget points (a larger frame is a chunk of its own)."""
    from det3d.datasets.pipelines.sample_ops import libm_trig
    counts = pk["num_points"].copy()
    chunks, cur, n = [], [], 0
    for f, p in enumerate(pk["points"]):
        if p is None:
            continue
        if cur and n + len(p) > point_budget:
            chunks.append(cur)
            cur, n = [], 0
        cur.append(f)
        n += len(p)
    if cur:
        chunks.append(cur)
    for fr in chunks:
        pts = np.empty((sum(len(pk["points"][f]) for f in fr), 4), np.float32)
        o = 0
        for i, f in enumerate(fr):
            p = pk["points"][f]
            pts[o:o + len(p), 0] = i
            pts[o:o + len(p), 1:] = p[:, :3]
            o += len(p)
        boxes = np.ascontiguousarray(pk["gt_boxes"][fr])
        trig = libm_trig(boxes[:, :, 8]).reshape(len(fr), pk["M"], 2)
        counts[fr] = count(pts, boxes, np.ascontiguousarray(pk["gt_classes"][fr]), trig)
    return counts


def evaluated_classes(pk, counts):
    """gt_classes after both filters: -1 for padding, other classes, boxes out of range and boxes without points."""
    return np.where(counts > 0, pk["gt_classes"], -1).astype(np.int32)


def run_device(pk, point_budget=POINT_BUDGET):
    """Point counts and the match of a pack() on the GPU -> (counts [B, M] int64, match [T, D] int32)."""
    from . import ops
    dev = torch.device("cuda", torch.cuda.current_device())

    def cu(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    counts = count_points(pk, lambda p, b, c, t: ops.eval_count_points(cu(p), cu(b), cu(c), cu(t)).cpu().numpy(),
                          point_budget)
    match = ops.eval_match_center(cu(pk["det_boxes"]), cu(pk["order"]), cu(pk["seg_start"]), cu(pk["seg_count"]),
                                  cu(pk["gt_boxes"]), cu(evaluated_classes(pk, counts)), pk["C"],
                                  cu(np.array(DIST_THS, np.float64)))
    return counts, match.cpu().numpy()


def run_host(pk, point_budget=POINT_BUDGET):
    """The same counts and match through the host twins (pnx_eval_count_points_host, pnx_eval_match_center_host): the
    CPU tests' path to the product logic."""
    from . import ops
    counts = count_points(pk, ops.eval_count_points_host, point_budget)
    match = ops.eval_match_center_host(pk["det_boxes"], pk["order"], pk["seg_start"], pk["seg_count"], pk["gt_boxes"],
                                       evaluated_classes(pk, counts), pk["C"], np.array(DIST_THS, np.float64))
    return counts, match


def cummean(x):
    """NaN-aware cumulative mean; all NaN (or empty) -> ones."""
    if np.isnan(x).all():
        return np.ones(len(x))
    s, n = np.nancumsum(x), np.cumsum(~np.isnan(x))
    return np.divide(s, n, out=np.zeros_like(s), where=n != 0)


def tp_errors(pk, match_tp):
    """The five errors of every detection against its box of the 2 m match (meaningful where match_tp >= 0)."""
    f, j = pk["det_frames"], np.maximum(match_tp, 0)
    g = pk["gt_boxes"][f, j].astype(np.float64)
    d = pk["det_boxes"].astype(np.float64)
    dx, dy = d[:, 0] - g[:, 0], d[:, 1] - g[:, 1]
    dvx, dvy = d[:, 6] - g[:, 6], d[:, 7] - g[:, 7]
    inter = np.minimum(d[:, 3], g[:, 3]) * np.minimum(d[:, 4], g[:, 4]) * np.minimum(d[:, 5], g[:, 5])
    vg, vd = g[:, 3] * g[:, 4] * g[:, 5], d[:, 3] * d[:, 4] * d[:, 5]
    names = np.asarray(pk["class_names"] + [""], dtype=str)
    period = np.where(names[pk["det_labels"]] == "barrier", math.pi, 2 * math.pi)
    yd = np.mod(g[:, 8] - d[:, 8] + period / 2, period) - period / 2
    yd = np.where(yd > math.pi, yd - 2 * math.pi, yd)
    ga = pk["gt_attr"][f, j]
    return {"trans_err": np.sqrt(dx * dx + dy * dy), "vel_err": np.sqrt(dvx * dvx + dvy * dvy),
            "scale_err": 1.0 - inter / (vg + vd - inter), "orient_err": np.abs(yd),
            "attr_err": np.where(ga < 0, np.nan, 1.0 - (ga == pk["det_attr"]))}


def score(pk, counts, match):
    """Match arrays + point counts -> the metric dict of nuscenes_metrics."""
    classes = evaluated_classes(pk, counts)
    visit, lab = pk["visit"], pk["det_labels"]
    bounds = np.searchsorted(lab[visit], np.arange(pk["C"] + 1))
    t_tp = DIST_THS.index(DIST_TH_TP)
    errs = tp_errors(pk, match[t_tp])
    r = np.linspace(0, 1, 101)
    first = round(100 * MIN_RECALL) + 1
    per_class = {}
    for c, name in enumerate(pk["class_names"]):
        npos = int((classes == c).sum())
        sel = visit[bounds[c]:bounds[c + 1]]
        sc = pk["det_scores"][sel].astype(np.float64)
        res = {"n_gt": npos}
        aps, tp_err = [], {k: 1.0 for k, _ in TP_METRICS}
        for t, th in enumerate(DIST_THS):
            tp = match[t, sel] >= 0
            if npos == 0 or not tp.any():                      # the devkit's "no predictions": AP 0, every error 1
                aps.append(0.0)
                continue
            ctp, cfp = np.cumsum(tp).astype(np.float64), np.cumsum(~tp).astype(np.float64)
            prec, rec = ctp / (ctp + cfp), ctp / float(npos)
            p = np.interp(r, rec, prec, right=0)
            conf = np.interp(r, rec, sc, right=0)
            aps.append(float(np.mean(np.maximum(p[first:] - MIN_PRECISION, 0.0))) / (1.0 - MIN_PRECISION))
            if t != t_tp:
                continue
            nz = np.nonzero(conf)[0]
            last = int(nz[-1]) if len(nz) else 0
            for k, _ in TP_METRICS:
                e = np.interp(conf[::-1], sc[tp][::-1], cummean(errs[k][sel[tp]])[::-1])[::-1]
                tp_err[k] = 1.0 if last < first else float(np.mean(e[first:last + 1]))
        for k in NAN_BY_RULE.get(name, ()):
            tp_err[k] = float("nan")
        res["AP"] = 100.0 * float(np.mean(aps))
        for th, a in zip(DIST_THS, aps):
            res["AP@%.1f" % th] = 100.0 * a
        for k, short in TP_METRICS:
            res[short] = tp_err[k]
        per_class[name] = res
    return summarize(per_class)


def summarize(per_class):
    """Per-class AP (percent) and TP errors -> mAP over all classes, the nanmean errors and NDS."""
    out = {"mAP": float(np.mean([v["AP"] for v in per_class.values()])) if per_class else 0.0}
    nds = 5.0 * out["mAP"] / 100.0
    for _, short in TP_METRICS:
        vals = [v[short] for v in per_class.values() if v[short] == v[short]]
        out["m" + short] = float(np.mean(vals)) if vals else float("nan")
        nds += max(0.0, 1.0 - out["m" + short])                 # NaN -> 0, as the devkit's max(0, nan)
    out["NDS"] = 100.0 * nds / 10.0
    out["per_class"] = per_class
    return out


def nuscenes_metrics(gts, detections, class_names, class_range=None):
    """gts / detections as in the module docstring.  Returns {"mAP", "NDS", "mATE", "mASE", "mAOE", "mAVE", "mAAE",
    "per_class": {name: {"AP", "AP@0.5", "AP@1.0", "AP@2.0", "AP@4.0", "ATE", "ASE", "AOE", "AVE", "AAE", "n_gt"}}},
    mAP, NDS and APs in percent."""
    pk = pack(gts, detections, class_names, class_range)
    counts, match = run_device(pk)
    return score(pk, counts, match)
