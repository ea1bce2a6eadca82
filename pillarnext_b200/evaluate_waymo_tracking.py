"""Waymo-style tracking metric: CLEAR MOT (Bernardin and Stiefelhagen, 2008) as the Waymo Open Dataset paper applies it
(Sun et al., CVPR 2020), MOTA and MOTP at LEVEL_1 and LEVEL_2, restated from the published definitions.  The devkit
cannot run here, so parity with it is unverified.

The detection metric's conventions (evaluate_waymo.py) are reused unchanged: its IoU routine and class thresholds,
0-point boxes dropped, LEVEL_2 for boxes with 1-5 points with LEVEL_1 ignoring those boxes and their matches, and the
per-class score cutoffs c_k of matching="hungarian" (a detection takes part at cutoff k when its score >= c_k).

  * Frames: each ground-truth frame names its sequence and timestamp; a sequence's frames are taken in ascending
    timestamp.  Each box carries its object id; an object is (sequence, class, id).  Detections carry the tracker's
    "tracking_id"; those with id < 0 are left out.
  * Per (sequence, class, cutoff), frames in order, with the pairs (detection, box) of IoU >= the class threshold whose
    detection passes the cutoff:
      - Carry-over: a pair whose detection carries the id of the object's last match is kept, pairs taken in order
        (detections in descending score, ties by lower index; each one's boxes by ascending index), each unless its
        detection or box is already kept.
      - Assignment: the remaining pairs (neither side kept) take the exact maximum-sum-IoU assignment with the tie
        rule of matching="hungarian".
      - Counts: a match whose id differs from the id of the object's previous match (if it had one) is a mismatch;
        every match then records its id as the object's last.  Unmatched detections are false positives, unmatched
        boxes misses, and the sum of (1 - IoU) runs over the matches.  At a level, matches to boxes outside the level
        are neither TP nor FP, and the level's boxes alone count in n_gt.
  * Results, per class and level: MOTA = 1 - (miss + mismatch + FP) / n_gt and MOTP = sum(1 - IoU) / matches at each
    cutoff; the class reports the cutoff with the highest MOTA (ties: lower cutoff) with its MOTA, MOTP and its miss,
    mismatch and FP rates (each over n_gt).  A class without detections has MOTA 0, miss rate 1 and MOTP NaN; without
    ground truth every value is NaN.  mMOTA / mMOTP: the means over the classes that have ground truth at that level
    (NaN values left out).

The pairs and components run on the GPU (pnx_eval_pairs, pnx_eval_components), the frame-by-frame carry-over,
assignment and counts in pnx_eval_mot (csrc/det_eval.cu: one warp per (sequence, class, cutoff)); the final sums are
float64 numpy.  oracle/track_oracle.py restates the definition sequentially (scipy's linear_sum_assignment plus the
tie rule)."""
import numpy as np
import torch

from . import evaluate_waymo as EW
from .track import frame_order

LEVELS = ("L1", "L2")


def pack(gts, tracks, class_names, iou_thresholds=None, num_score_cutoffs=11):
    """evaluate_waymo.pack_hungarian over the frames in (sequence, timestamp) order and the tracked detections, plus
    the tracking ids, each box's object index and the sequences' first frames."""
    for t, g in gts.items():
        for key in ("ids", "sequence", "timestamp"):
            if key not in g:
                raise ValueError("frame %s: ground truth needs %r for tracking" % (t, key))
        if len(g["ids"]) != len(g["names"]):
            raise ValueError("frame %s: %d ids but %d names" % (t, len(g["ids"]), len(g["names"])))
    tokens, seqs, seq_start = frame_order(gts)
    dets, det_ids = {}, []
    for t in tokens:
        d = tracks.get(t)
        if d is None:
            continue
        tid = EW._arr(d["tracking_id"], np.int64).reshape(-1)
        keep = tid >= 0
        if len(tid) and tid.max() >= 2 ** 31:
            raise ValueError("frame %s: tracking ids must be < 2^31" % t)
        dets[t] = {k: EW._arr(d[k])[keep] for k in ("box3d_lidar", "scores", "label_preds")}
        det_ids.append(tid[keep])
    unknown = sorted(set(tracks) - set(gts))
    if unknown:
        raise ValueError("tracks for tokens without ground truth: %s" % unknown[:5])
    pk = EW.pack_hungarian({t: gts[t] for t in tokens}, dets, class_names, iou_thresholds, num_score_cutoffs)
    gt_obj = np.full((pk["B"], pk["M"]), -1, np.int32)
    objects = {}
    s = 0
    for f, t in enumerate(tokens):
        while f >= seq_start[s + 1]:
            s += 1
        names, ids = gts[t]["names"], gts[t]["ids"]
        gt_obj[f, :len(names)] = [objects.setdefault((s, n, str(i)), len(objects)) if c >= 0 else -1
                                  for n, i, c in zip(names, ids, pk["gt_classes"][f, :len(names)].tolist())]
    pk.update(tokens=tokens, sequences=seqs, seq_start=seq_start, gt_obj=gt_obj, n_obj=len(objects),
              det_id=(np.concatenate(det_ids) if det_ids else np.zeros(0, np.int64)).astype(np.int32))
    return pk


def run_device(pk):
    """Point counts and the per-(sequence, class, cutoff) counts of a pack() on the GPU."""
    from . import ops
    dev = torch.device("cuda", torch.cuda.current_device())

    def cu(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    counts = ops.eval_count_points(cu(pk["points"]), cu(pk["gt_boxes"]), cu(pk["gt_classes"]), cu(pk["count_trig"]))
    npts = torch.where(cu(pk["num_points"]) >= 0, cu(pk["num_points"]), counts.long()).to(torch.int32)
    order = torch.sort(cu(pk["keys"]), stable=True)[1]
    start, e_det, e_box, e_iou, _ = ops.eval_pairs(cu(pk["det_boxes"]), cu(pk["det_trig"]), order, cu(pk["seg_start"]),
                                                   cu(pk["seg_count"]), cu(pk["gt_boxes"]), cu(pk["gt_classes"]),
                                                   cu(pk["gt_trig"]), cu(pk["thresholds"]))
    comp_start, comp_nedge, grouped = ops.eval_components(start, e_det, e_box, pk["M"], pk["C"])
    mot, dist = ops.eval_mot(start, e_det, e_box, e_iou, grouped, comp_start, comp_nedge, cu(pk["det_pass"]),
                             cu(pk["det_id"]), cu(pk["gt_obj"].reshape(-1)), npts.view(-1), cu(pk["seq_start"]),
                             pk["M"], pk["C"], pk["K"], pk["n_obj"])
    return npts.cpu().numpy(), mot.cpu().numpy(), dist.cpu().numpy()


def run_host(pk):
    """The same through the host twins (the CPU tests' path to the product logic)."""
    from . import ops
    counts = ops.eval_count_points_host(pk["points"], pk["gt_boxes"], pk["gt_classes"], pk["count_trig"])
    npts = EW.known_counts(pk, counts).astype(np.int32)
    order = np.argsort(pk["keys"], kind="stable").astype(np.int64)
    start, e_det, e_box, e_iou, _ = ops.eval_pairs_host(pk["det_boxes"], pk["det_trig"], order, pk["seg_start"],
                                                        pk["seg_count"], pk["gt_boxes"], pk["gt_classes"],
                                                        pk["gt_trig"], pk["thresholds"])
    comp_start, comp_nedge, grouped = ops.eval_components_host(start, e_det, e_box, pk["M"], pk["C"])
    mot, dist = ops.eval_mot_host(start, e_det, e_box, e_iou, grouped, comp_start, comp_nedge, pk["det_pass"],
                                  pk["det_id"], pk["gt_obj"].reshape(-1), npts.reshape(-1), pk["seq_start"], pk["M"],
                                  pk["C"], pk["K"], pk["n_obj"])
    return npts, mot, dist


def score(pk, npts, mot, dist, class_names):
    """Point counts [B, M] + pnx_eval_mot's counts [S, C, K, 5] and dist [S, C, K, 2] -> the metric dict."""
    tot, dsum = mot.sum(0), dist.sum(0)                          # [C, K, 5], [C, K, 2]
    per_class = {}
    for c, name in enumerate(class_names):
        m = pk["gt_classes"] == c
        n_gt = {"L1": int((m & (npts > EW.LEVEL_2_MAX_POINTS)).sum()), "L2": int((m & (npts >= 1)).sum())}
        cuts = pk["cutoffs"][c]
        passes = pk["det_pass"][pk["det_labels"] == c]
        res = {}
        for li, lv in enumerate(LEVELS):
            n = n_gt[lv]
            res["n_gt_" + lv] = n
            if n == 0:
                vals = dict(MOTA=np.nan, MOTP=np.nan, miss=np.nan, mismatch=np.nan, fp=np.nan, score_cutoff=np.nan)
            elif len(cuts) == 0:
                vals = dict(MOTA=0.0, MOTP=np.nan, miss=1.0, mismatch=0.0, fp=0.0, score_cutoff=np.nan)
            else:
                k_all = np.arange(len(cuts))
                tp = tot[c, k_all, 1 + 2 * li].astype(np.float64)
                mism = tot[c, k_all, 2 + 2 * li].astype(np.float64)
                fp = np.array([(passes > k).sum() for k in k_all], np.float64) - tot[c, k_all, 0]
                mota = 1.0 - ((n - tp) + mism + fp) / n
                k = int(np.argmax(mota))
                vals = dict(MOTA=float(mota[k]), MOTP=float(dsum[c, k, li] / tp[k]) if tp[k] else np.nan,
                            miss=float((n - tp[k]) / n), mismatch=float(mism[k] / n), fp=float(fp[k] / n),
                            score_cutoff=float(cuts[k]))
            res.update({key + "_" + lv: float(v) for key, v in vals.items()})
        per_class[name] = res
    out = {}
    for lv in LEVELS:
        for key in ("MOTA", "MOTP"):
            vals = [v[key + "_" + lv] for v in per_class.values() if v["n_gt_" + lv] > 0 and v[key + "_" + lv] == v[key + "_" + lv]]
            out["m%s_%s" % (key, lv)] = float(np.mean(vals)) if vals else float("nan")
    out["per_class"] = per_class
    return out


def waymo_tracking_metrics(gts, tracks, class_names, iou_thresholds=None, num_score_cutoffs=11, host=False):
    """gts: token -> evaluate_waymo.waymo_metrics' ground truth plus "ids" [M] (object ids), "sequence" and "timestamp";
    tracks: token -> track.track's output (predict's dict plus "tracking_id").  Returns {"mMOTA_L1", "mMOTP_L1",
    "mMOTA_L2", "mMOTP_L2", "per_class": {name: {MOTA_L1, MOTP_L1, miss_L1, mismatch_L1, fp_L1, score_cutoff_L1,
    n_gt_L1, and the same for L2}}}; MOTA and MOTP as fractions, the rates over n_gt.  host=True runs the host twins."""
    pk = pack(gts, tracks, class_names, iou_thresholds, num_score_cutoffs)
    npts, mot, dist = (run_host if host else run_device)(pk)
    return score(pk, npts, mot, dist, class_names)


def track_and_score(gts, detections, class_names, iou_thresholds=None, num_score_cutoffs=11, **track_kw):
    """track.track over the frames of gts (each with "sequence", "timestamp" and "pose"), then waymo_tracking_metrics:
    -> (tracks, metrics)."""
    from .track import track
    tracks = track(detections, gts, class_names, **track_kw)
    return tracks, waymo_tracking_metrics(gts, tracks, class_names, iou_thresholds, num_score_cutoffs)
