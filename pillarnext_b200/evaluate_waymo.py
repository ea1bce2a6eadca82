"""Waymo-style 3-D detection metric: AP and APH at LEVEL_1 and LEVEL_2, restated from the published definition (Sun et al.,
CVPR 2020, "Scalability in Perception for Autonomous Driving: Waymo Open Dataset"), because the reference hands Waymo
scoring to the devkit (det3d/datasets/waymo/waymo.py:124 writes a .bin for it), which is not installable here.

  * IoU of a detection and a ground-truth box (x, y, z, dx, dy, dz, yaw): the reference's boxes_iou3d_gpu
    (det3d/core/iou3d_nms/iou3d_nms_utils.py:11-46): the rotated BEV overlap times the height overlap, over
    max(vol_a + vol_b - overlap, 1e-6), in fp32, detection first -- the per-pair arithmetic of the `iou` head target.
  * Thresholds per class: vehicle 0.7, pedestrian 0.5, cyclist 0.5; any other class takes its threshold from the
    `iou_thresholds` mapping (which may also override these).  A class with neither raises ValueError.
  * Difficulty: the frame's points inside each ground-truth box are counted with the reference's points_in_boxes_jit
    test (libm cosf / sinf of the yaw).  A box with 0 points is dropped from evaluation, a box with 1-5 points is
    LEVEL_2, every other box LEVEL_1.
  * Matching, once per (frame, class): the detections are visited in descending score order, ties by lower index; each
    takes the unmatched ground-truth box with the highest IoU >= threshold, ties by lower index, or stays unmatched.
    A detection matched to a dropped (0-point) box is ignored at both levels.
  * Levels: LEVEL_2 uses every remaining box.  LEVEL_1 ignores the LEVEL_2 boxes: they do not count in n_gt, and a
    detection matched to one is removed from the LEVEL_1 curve, as neither TP nor FP.
  * Heading accuracy of a TP: h = 1 - min(|d|, 2 pi - |d|) / pi, d the yaw difference wrapped to [-pi, pi].
  * AP per class: all detections of all frames sorted by descending score (stable over frames in token order, then
    index); cumulative TP and FP; AP = 100 * sum over the curve of (recall step) x (highest precision at any recall >=
    that point), the area under the monotone envelope.  APH: the same with TP replaced by the sum of h, in precision
    (sum h / (sum h + FP), 0 where both are 0) and recall (sum h / n_gt).  mAP / mAPH: the mean over the classes that have ground truth at
    that level; a class without any is NaN and left out of the mean.

Known differences from the devkit: greedy score-ordered matching instead of Hungarian matching, and one curve over all
detections instead of the devkit's score-cutoff quantiles.  No range breakdown.

The point counts and the matching run on the GPU (pnx_eval_count_points, pnx_eval_match, csrc/det_eval.cu); the curves
are float64 numpy.  oracle/waymo_metric_oracle.py restates the whole definition sequentially."""
import numpy as np
import torch

IOU_THRESHOLDS = {"vehicle": 0.7, "pedestrian": 0.5, "cyclist": 0.5}
LEVEL_2_MAX_POINTS = 5


def class_thresholds(class_names, iou_thresholds=None):
    """Per-class IoU thresholds: the defaults above, overridden or extended by `iou_thresholds`."""
    table = dict(IOU_THRESHOLDS, **(iou_thresholds or {}))
    missing = [n for n in class_names if n not in table]
    if missing:
        raise ValueError("no IoU threshold for classes %s: pass iou_thresholds={name: threshold}" % missing)
    return [float(table[n]) for n in class_names]


def _arr(x, dtype=None):
    a = x.detach().cpu().numpy() if hasattr(x, "detach") else np.asarray(x)
    return a if dtype is None else a.astype(dtype, copy=False)


def _box9(boxes):
    """[M, 7] (x, y, z, dx, dy, dz, yaw) or [M, 9] (.., vx, vy, yaw) -> [M, 9] fp32."""
    b = _arr(boxes, np.float32).reshape(len(boxes), -1) if len(boxes) else np.zeros((0, 9), np.float32)
    if b.shape[1] == 9:
        return b
    if b.shape[1] != 7:
        raise ValueError("boxes must have 7 (x, y, z, dx, dy, dz, yaw) or 9 (.., vx, vy, yaw) columns, got %d" % b.shape[1])
    out = np.zeros((len(b), 9), np.float32)
    out[:, :6], out[:, 8] = b[:, :6], b[:, 6]
    return out


def heading_trig(yaw):
    """fp32 (cos, sin) of each fp32 yaw, taken in fp64 and rounded: the trigonometry of the IoU (and of the oracle's)."""
    y = np.asarray(yaw, dtype=np.float32).astype(np.float64).reshape(-1)
    return np.stack([np.cos(y), np.sin(y)], 1).astype(np.float32)


def pack(gts, detections, class_names, iou_thresholds=None):
    """gts / detections as for waymo_metrics -> the flat arrays both kernels take (numpy, host)."""
    from det3d.datasets.pipelines.sample_ops import libm_trig
    thr = np.array(class_thresholds(class_names, iou_thresholds), np.float32)
    tokens = list(gts)
    unknown = sorted(set(detections) - set(tokens))
    if unknown:
        raise ValueError("detections for tokens without ground truth: %s" % unknown[:5])
    B, C = len(tokens), len(class_names)
    cls_of = {n: i for i, n in enumerate(class_names)}
    M = max([1] + [len(gts[t]["names"]) for t in tokens])
    gt_boxes = np.zeros((B, M, 9), np.float32)
    gt_boxes[:, :, 3:6] = 1.0
    gt_classes = np.full((B, M), -1, np.int32)
    points = []
    for f, t in enumerate(tokens):
        g = gts[t]
        b = _box9(g["boxes"])
        if len(b) != len(g["names"]):
            raise ValueError("frame %s: %d boxes but %d names" % (t, len(b), len(g["names"])))
        gt_boxes[f, :len(b)] = b
        gt_classes[f, :len(b)] = [cls_of.get(n, -1) for n in g["names"]]
        p = _arr(g["points"], np.float32)
        q = np.empty((len(p), 4), np.float32)
        q[:, 0] = f
        q[:, 1:] = p[:, :3]
        points.append(q)
    yaw = gt_boxes[:, :, 8].reshape(-1)
    count_trig = libm_trig(yaw).reshape(B, M, 2)
    gt_trig = heading_trig(yaw).reshape(B, M, 2)
    det_boxes, det_scores, det_seg = [np.zeros((0, 9), np.float32)], [np.zeros(0, np.float32)], [np.zeros(0, np.int64)]
    for f, t in enumerate(tokens):
        d = detections.get(t)
        if d is None:
            continue
        b = _box9(d["box3d_lidar"])
        s = _arr(d["scores"], np.float32).reshape(-1)
        lab = _arr(d["label_preds"]).reshape(-1).astype(np.int64)
        if not (len(b) == len(s) == len(lab)):
            raise ValueError("frame %s: box3d_lidar, scores and label_preds differ in length" % t)
        if len(lab) and (lab.min() < 0 or lab.max() >= C):
            raise ValueError("frame %s: label_preds outside [0, %d)" % (t, C))
        if np.isnan(s).any():
            raise ValueError("frame %s: NaN scores" % t)
        det_boxes.append(b)
        det_scores.append(s + np.float32(0.0))                 # -0 -> +0: equal scores order by index
        det_seg.append(f * C + lab)
    det_boxes, det_scores, det_seg = np.concatenate(det_boxes), np.concatenate(det_scores), np.concatenate(det_seg)
    # sort key: segment in the high word, descending score in the low word (fp32 bits made order-preserving)
    u = det_scores.view(np.uint32).astype(np.int64)
    ordered = np.where(det_scores >= 0, u | 0x80000000, (~u) & 0xFFFFFFFF)
    keys = (det_seg << 32) | (0xFFFFFFFF - ordered)
    seg_count = np.bincount(det_seg, minlength=B * C).astype(np.int32)
    seg_start = (np.cumsum(seg_count) - seg_count).astype(np.int32)
    return dict(B=B, M=M, C=C, thresholds=thr, points=np.concatenate(points) if points else np.zeros((0, 4), np.float32),
                gt_boxes=gt_boxes, gt_classes=gt_classes, count_trig=count_trig, gt_trig=gt_trig, det_boxes=det_boxes,
                det_scores=det_scores, det_labels=det_seg % C, det_frames=det_seg // C,
                det_trig=heading_trig(det_boxes[:, 8]), keys=keys, seg_start=seg_start, seg_count=seg_count)


def run_device(pk):
    """Counts and matches of a pack() on the GPU: two kernels, one key sort, one copy back."""
    dev = torch.device("cuda", torch.cuda.current_device())
    from . import ops

    def cu(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=False)
    D, BM = len(pk["det_scores"]), pk["B"] * pk["M"]
    counts = ops.eval_count_points(cu(pk["points"]), cu(pk["gt_boxes"]), cu(pk["gt_classes"]), cu(pk["count_trig"]))
    order = torch.sort(cu(pk["keys"]), stable=True)[1]
    gt_boxes, gt_classes = cu(pk["gt_boxes"]), cu(pk["gt_classes"])
    match, iou, heading = ops.eval_match(cu(pk["det_boxes"]), cu(pk["det_trig"]), order, cu(pk["seg_start"]),
                                         cu(pk["seg_count"]), gt_boxes, gt_classes, cu(pk["gt_trig"]), cu(pk["thresholds"]))
    out = torch.cat([counts.view(-1), match, iou.view(torch.int32), heading.view(torch.int32)]).cpu().numpy()
    return (out[:BM].reshape(pk["B"], pk["M"]), out[BM:BM + D], out[BM + D:BM + 2 * D].view(np.float32),
            out[BM + 2 * D:].view(np.float32))


def run_host(pk):
    """The same counts and matches through the host twins (pnx_eval_*_host): the CPU tests' path to the product logic."""
    from . import ops
    counts = ops.eval_count_points_host(pk["points"], pk["gt_boxes"], pk["gt_classes"], pk["count_trig"])
    order = np.argsort(pk["keys"], kind="stable").astype(np.int64)
    match, iou, heading = ops.eval_match_host(pk["det_boxes"], pk["det_trig"], order, pk["seg_start"], pk["seg_count"],
                                              pk["gt_boxes"], pk["gt_classes"], pk["gt_trig"], pk["thresholds"])
    return counts, match, iou, heading


def _ap(weights, fp, n_gt):
    """weights (TP: 1 or h, FP: 0) and fp (FP: 1) in descending score order -> 100 x the area under the monotone
    precision envelope."""
    if n_gt == 0:
        return float("nan")
    if len(weights) == 0:
        return 0.0
    cw, cf = np.cumsum(np.asarray(weights, np.float64)), np.cumsum(np.asarray(fp, np.float64))
    den = cw + cf
    prec, rec = np.divide(cw, den, out=np.zeros_like(cw), where=den > 0), cw / n_gt
    env = np.maximum.accumulate(prec[::-1])[::-1]
    return 100.0 * float(np.sum(np.diff(rec, prepend=0.0) * env))


def score(pk, counts, match, heading, class_names):
    """Per-detection match results + per-box point counts -> the metric dict of waymo_metrics."""
    per_class = {}
    f, lab, sc = pk["det_frames"], pk["det_labels"], pk["det_scores"]
    npts = np.where(match >= 0, counts[f, np.maximum(match, 0)], -1) if len(match) else np.zeros(0, np.int64)
    for c, name in enumerate(class_names):
        m = pk["gt_classes"] == c
        n_l2 = int((m & (counts >= 1)).sum())
        n_l1 = int((m & (counts > LEVEL_2_MAX_POINTS)).sum())
        sel = np.nonzero(lab == c)[0]
        sel = sel[np.argsort(-sc[sel].astype(np.float64), kind="stable")]
        hit, n, h = match[sel] >= 0, npts[sel], heading[sel].astype(np.float64)
        keep2 = ~hit | (n >= 1)
        keep1 = ~hit | (n > LEVEL_2_MAX_POINTS)
        tp, hw, fp = hit.astype(np.float64), np.where(hit, h, 0.0), (~hit).astype(np.float64)
        per_class[name] = dict(AP_L1=_ap(tp[keep1], fp[keep1], n_l1), APH_L1=_ap(hw[keep1], fp[keep1], n_l1),
                               AP_L2=_ap(tp[keep2], fp[keep2], n_l2), APH_L2=_ap(hw[keep2], fp[keep2], n_l2),
                               n_gt_L1=n_l1, n_gt_L2=n_l2)
    res = {}
    for key in ("AP_L1", "APH_L1", "AP_L2", "APH_L2"):
        vals = [v[key] for v in per_class.values() if v[key] == v[key]]
        res["m" + key] = float(np.mean(vals)) if vals else float("nan")
    res["per_class"] = per_class
    return res


def waymo_metrics(gts, detections, class_names, iou_thresholds=None):
    """gts: token -> {"boxes" [M, 7 or 9] (x, y, z, dx, dy, dz, [vx, vy,] yaw), "names" list[str], "points" [N, >= 3]
    (x, y, z first)}; detections: token -> {"box3d_lidar" [K, 9], "scores" [K], "label_preds" [K]} (the reference's
    validation_step output, single_stage.py:47-59; CPU or CUDA tensors, or arrays), labels indexing class_names.
    Ground-truth boxes whose name is not in class_names are not evaluated.  Returns {"mAP_L1", "mAPH_L1", "mAP_L2",
    "mAPH_L2", "per_class": {name: {AP_L1, APH_L1, AP_L2, APH_L2, n_gt_L1, n_gt_L2}}}, AP values in percent."""
    pk = pack(gts, detections, class_names, iou_thresholds)
    counts, match, _, heading = run_device(pk)
    return score(pk, counts, match, heading, class_names)
