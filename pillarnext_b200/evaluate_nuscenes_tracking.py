"""nuScenes tracking metric: AMOTA / AMOTP and the CLEAR MOT counts of the nuScenes tracking task (Caesar et al., CVPR
2020), with MOTAR and its average over recalls as AB3DMOT defines them (Weng et al., IROS 2020), restated from the
published definitions.  The devkit cannot run here, so parity with it is unverified; the rules below are this
project's.

  * Inputs.  gts: token -> evaluate_nuscenes.nuscenes_metrics' ground truth ("boxes", "names", "points" or
    "num_points") plus "ids" [M] (object ids), "sequence" (the scene) and "timestamp"; "pose" is read by the tracker
    only.  tracks: token -> track.track's output (labels indexing class_names, plus "tracking_id").  A scene's frames
    are taken in ascending timestamp.
  * Classes.  The tracking classes are bicycle, bus, car, motorcycle, pedestrian, trailer and truck; those present in
    class_names are scored, in class_names' order.  Detections and boxes of every other class (barrier, traffic_cone,
    construction_vehicle) are ignored on both sides, as are detections with tracking id < 0.
  * Filters: evaluate_nuscenes unchanged, applied to what is left: a frame with more than 500 detections raises
    ValueError, the per-class range filter on boxes and detections, and ground-truth boxes with 0 points dropped (the
    points counted on the GPU where a frame gives no "num_points").  P = a class's boxes after the filters.
  * Pairs.  Within a (scene, class) and frame, a detection and a box form a pair when their BEV centre distance d
    (fp64 differences of the fp32 coordinates, evaluate_nuscenes' arithmetic) is < 2.0 m, strictly; d is kept as fp32.
  * Frame step, per (scene, class, score cutoff c), frames in order; only detections with score >= c take part.  An
    object is (scene, class, id).
      1. Carry-over: a pair whose detection carries the object's last matched id is kept, pairs taken in order
         (detections in descending score, ties by lower index; each one's boxes by ascending index), each unless its
         detection or box is already kept.
      2. Assignment: the remaining pairs (neither side kept) take an exact assignment with, first, the most pairs and
         then, among those, the smallest sum of d; ties by the Hungarian mode's rule (detections in visit order, each
         taking the first possible of its boxes by ascending index, then "unmatched").  The assignment maximises the
         integer weight 2^40 - round(d 2^26) per pair (d 2^26 is exact in fp64; round half up).  A component's matches
         are at most its boxes, <= 4096 = 2^12, each rounded distance is <= 2^27 (d <= 2), so the distances of any
         assignment sum to < 2^40: one more pair always outweighs any difference in distance, and the most pairs
         come first exactly.  Distances closer than 2^-27 m may tie.
      3. Counts: TP = matches; FP = detections taking part and left unmatched; FN = boxes left unmatched; IDS = matches
         whose id differs from the object's last matched id (if it has one); FRAG = matches of an object that was
         matched before and has a box in a frame after that match (so was unmatched in between); sum d over the
         matches.  Every match then records its id and frame as the object's last.
  * Thresholds, per class.  One pass with every detection taking part records which detections are matched; their
    scores sorted in descending order give, for each recall r_k in numpy's linspace(0.1, 1.0, 40), the cutoff c_k =
    the score of the n_k-th match with n_k = ceil(r_k P) (fp64).  With fewer than n_k matches (or P = 0) r_k is
    unreached.  Then one pass per reached c_k.
  * Results, per class: MOTAR_k = max(0, 1 - (IDS + FP + FN - (1 - r_k) P) / (r_k P)); AMOTA = the sum over the
    reached k / 40 (an unreached k counts 0); as r_k is the target recall and a cutoff's pass may make more than r_k P
    matches, MOTAR_k and AMOTA can exceed 1.  MOTP_k = sum d / TP (2.0 when TP = 0); AMOTP = the mean over all 40 k,
    an unreached k counting 2.0 m.  At the reached k with the highest MOTA = max(0, 1 - (FN + FP + IDS) / P) (ties to
    the lower k) the class reports MOTA, MOTP, recall = TP / P, IDS, FRAG, FP, FN and the cutoff.  No ground truth:
    every value NaN.  No reached k (no detections, or too few matches): AMOTA 0, AMOTP 2.0, MOTA 0, MOTP NaN, recall
    0, IDS, FRAG and FP 0, FN = P, cutoff NaN.
  * Overall: AMOTA, AMOTP, MOTA, MOTP and recall are means over the classes with ground truth (NaN values left out);
    IDS, FRAG, FP and FN are their sums.

Not covered: the devkit's ground-truth track interpolation, its bike-rack filter, and the TID / LGD metrics.

The point counts, the pairs (pnx_eval_pairs_center), their components (pnx_eval_components) and both passes
(pnx_eval_mot_center: one warp per (scene, class, cutoff), csrc/det_eval.cu) run on the GPU; thresholds and the final
sums are float64 numpy.  oracle/nusc_track_oracle.py restates the definition sequentially (scipy's
linear_sum_assignment plus the tie rule)."""
import math

import numpy as np
import torch

from . import evaluate_nuscenes as EN
from .evaluate_waymo import _arr
from .track import frame_order

TRACKING_NAMES = ("bicycle", "bus", "car", "motorcycle", "pedestrian", "trailer", "truck")
PAIR_DIST = 2.0
RECALLS = np.linspace(0.1, 1.0, 40)
MOTP_UNREACHED = 2.0


def tracking_classes(class_names):
    """The tracking classes among class_names, in class_names' order."""
    return [n for n in class_names if n in TRACKING_NAMES]


def pack(gts, tracks, class_names, class_range=None):
    """evaluate_nuscenes.pack over the frames in (scene, timestamp) order and the tracked detections of the tracking
    classes, plus their tracking ids, the visit order and the scenes' first frames."""
    for t, g in gts.items():
        for key in ("ids", "sequence", "timestamp"):
            if key not in g:
                raise ValueError("frame %s: ground truth needs %r for tracking" % (t, key))
        if len(g["ids"]) != len(g["names"]):
            raise ValueError("frame %s: %d ids but %d names" % (t, len(g["ids"]), len(g["names"])))
    unknown = sorted(set(tracks) - set(gts))
    if unknown:
        raise ValueError("tracks for tokens without ground truth: %s" % unknown[:5])
    tcls = tracking_classes(class_names)
    to_t = np.array([tcls.index(n) if n in tcls else -1 for n in class_names] + [-1], np.int64)
    tokens, seqs, seq_start = frame_order(gts)
    dets, det_ids = {}, []
    for t in tokens:
        d = tracks.get(t)
        if d is None:
            continue
        lab = _arr(d["label_preds"]).reshape(-1).astype(np.int64)
        tid = _arr(d["tracking_id"]).reshape(-1).astype(np.int64)
        if len(lab) != len(tid):
            raise ValueError("frame %s: %d labels but %d tracking ids" % (t, len(lab), len(tid)))
        if len(lab) and (lab.min() < 0 or lab.max() >= len(class_names)):
            raise ValueError("frame %s: label_preds outside [0, %d)" % (t, len(class_names)))
        if len(tid) and tid.max() >= 2 ** 31:
            raise ValueError("frame %s: tracking ids must be < 2^31" % t)
        keep = (to_t[lab] >= 0) & (tid >= 0)
        dd = {"box3d_lidar": EN._box9(d["box3d_lidar"])[keep], "scores": _arr(d["scores"], np.float32).reshape(-1)[keep],
              "label_preds": to_t[lab[keep]]}
        dets[t] = dd
        det_ids.append(tid[keep])
    if not tcls:
        raise ValueError("no tracking class among %s" % list(class_names))
    pk = EN.pack({t: gts[t] for t in tokens}, dets, tcls, class_range)
    seg = pk["det_frames"] * pk["C"] + pk["det_labels"]
    D = len(seg)
    pk.update(tokens=tokens, sequences=seqs, seq_start=seq_start, tracking_names=tcls,
              det_id=(np.concatenate(det_ids) if det_ids else np.zeros(0, np.int64))[pk["det_pos"]].astype(np.int32),
              order=np.lexsort((np.arange(D), -pk["det_scores"].astype(np.float64), seg)).astype(np.int64))
    return pk


def objects(pk, gts, classes):
    """gt_obj [B M] (object index, -1 for a box left out) and gt_prev [B M] (the frame of the object's previous box
    that the filters left, -1 for none) over the evaluated boxes, and the number of objects."""
    B, M = classes.shape
    gt_obj, gt_prev = np.full((B, M), -1, np.int32), np.full((B, M), -1, np.int32)
    index, last = {}, {}
    s = 0
    for f, t in enumerate(pk["tokens"]):
        while f >= pk["seq_start"][s + 1]:
            s += 1
        ids = gts[t]["ids"]
        for j in np.nonzero(classes[f] >= 0)[0]:
            key = (s, int(classes[f, j]), str(ids[j]))
            gt_obj[f, j] = index.setdefault(key, len(index))
            gt_prev[f, j] = last.get(key, -1)
            last[key] = f
    return gt_obj.reshape(-1), gt_prev.reshape(-1), len(index)


def cutoffs(pk, classes, matched):
    """Per class, the cutoffs of the reached recalls in recall order (descending scores) -> list of fp32 arrays."""
    out = []
    for c in range(pk["C"]):
        P = int((classes == c).sum())
        ms = np.sort(pk["det_scores"][(pk["det_labels"] == c) & (matched != 0)])[::-1]
        n = np.ceil(RECALLS * P).astype(np.int64)
        out.append(ms[n[(n >= 1) & (n <= len(ms))] - 1] if P else np.zeros(0, np.float32))
    return out


def cutoff_passes(pk, cuts):
    """det_pass [D]: the cutoffs each detection passes, counted from the lowest (kernel cutoff j = R_c - 1 - k)."""
    det_pass = np.zeros(len(pk["det_labels"]), np.int32)
    for c, cut in enumerate(cuts):
        sel = pk["det_labels"] == c
        det_pass[sel] = np.searchsorted(cut[::-1], pk["det_scores"][sel], side="right")
    return det_pass


def _passes(ops_, pk, gts, counts, device):
    """The shared body of run_device / run_host: ops_ = (pairs, components, mot, to) of one side."""
    pairs, components, mot, to = ops_
    classes = EN.evaluated_classes(pk, counts)
    gt_obj, gt_prev, n_obj = objects(pk, gts, classes)
    B, M, C, D = pk["B"], pk["M"], pk["C"], len(pk["det_labels"])
    start, e_det, e_box, e_dist = pairs(to(pk["det_boxes"]), to(pk["order"]), to(pk["seg_start"]), to(pk["seg_count"]),
                                        to(pk["gt_boxes"]), to(classes), C, PAIR_DIST)
    comp_start, comp_nedge, grouped = components(start, e_det, e_box, M, C)
    common = (to(pk["det_id"]), to(gt_obj), to(gt_prev), to(pk["seq_start"]), M, C)
    _, _, matched = mot(start, e_det, e_box, e_dist, grouped, comp_start, comp_nedge, to(np.ones(D, np.int32)),
                        *common, 1, n_obj, want_matched=True)
    matched = matched.cpu().numpy() if device else matched
    cuts = cutoffs(pk, classes, matched)
    n, dist, _ = mot(start, e_det, e_box, e_dist, grouped, comp_start, comp_nedge, to(cutoff_passes(pk, cuts)),
                     *common, len(RECALLS), n_obj)
    if device:
        n, dist = n.cpu().numpy(), dist.cpu().numpy()
    return dict(classes=classes, matched=matched, cutoffs=cuts, counts=n, dist=dist)


def run_device(pk, gts):
    """Point counts, pairs, the threshold pass and the cutoff pass of a pack() on the GPU."""
    from . import ops
    dev = torch.device("cuda", torch.cuda.current_device())

    def cu(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    counts = EN.count_points(pk, lambda p, b, c, t: ops.eval_count_points(cu(p), cu(b), cu(c), cu(t)).cpu().numpy())
    return _passes((ops.eval_pairs_center, ops.eval_components, ops.eval_mot_center, cu), pk, gts, counts, True)


def run_host(pk, gts):
    """The same through the host twins (the CPU tests' path to the product logic)."""
    from . import ops
    counts = EN.count_points(pk, ops.eval_count_points_host)
    return _passes((ops.eval_pairs_center_host, ops.eval_components_host, ops.eval_mot_center_host, np.ascontiguousarray),
                   pk, gts, counts, False)


def score(pk, res):
    """run_device / run_host's result -> the metric dict."""
    classes, cuts = res["classes"], res["cutoffs"]
    tot, dsum = res["counts"].sum(0), res["dist"].sum(0)               # [C, K, 3], [C, K]
    det_pass = cutoff_passes(pk, cuts)
    nan = float("nan")
    per_class = {}
    for c, name in enumerate(pk["tracking_names"]):
        P = int((classes == c).sum())
        R = len(cuts[c])
        out = {"n_gt": P}
        if P == 0:
            out.update(AMOTA=nan, AMOTP=nan, MOTA=nan, MOTP=nan, recall=nan, IDS=nan, FRAG=nan, FP=nan, FN=nan,
                       score_cutoff=nan)
        elif R == 0:
            out.update(AMOTA=0.0, AMOTP=MOTP_UNREACHED, MOTA=0.0, MOTP=nan, recall=0.0, IDS=0, FRAG=0, FP=0, FN=P,
                       score_cutoff=nan)
        else:
            j = R - 1 - np.arange(R)                                    # kernel cutoff of recall k
            tp, ids, frag = (tot[c, j, q].astype(np.float64) for q in range(3))
            passes = det_pass[pk["det_labels"] == c]
            fp = np.array([(passes > jj).sum() for jj in j], np.float64) - tp
            fn = P - tp
            r = RECALLS[:R]
            motar = np.maximum(0.0, 1.0 - (ids + fp + fn - (1.0 - r) * P) / (r * P))
            motp = np.where(tp > 0, dsum[c, j] / np.maximum(tp, 1), MOTP_UNREACHED)
            mota = np.maximum(0.0, 1.0 - (fn + fp + ids) / P)
            k = int(np.argmax(mota))
            out.update(AMOTA=float(motar.sum() / len(RECALLS)),
                       AMOTP=float((motp.sum() + MOTP_UNREACHED * (len(RECALLS) - R)) / len(RECALLS)),
                       MOTA=float(mota[k]), MOTP=float(motp[k]), recall=float(tp[k] / P), IDS=int(ids[k]),
                       FRAG=int(frag[k]), FP=int(fp[k]), FN=int(fn[k]), score_cutoff=float(cuts[c][k]))
        per_class[name] = out
    summary = {}
    scored = [v for v in per_class.values() if v["n_gt"] > 0]
    for key in ("AMOTA", "AMOTP", "MOTA", "MOTP", "recall"):
        vals = [v[key] for v in scored if not math.isnan(v[key])]
        summary[key] = float(np.mean(vals)) if vals else nan
    for key in ("IDS", "FRAG", "FP", "FN"):
        summary[key] = int(sum(v[key] for v in scored)) if scored else nan
    summary["per_class"] = per_class
    return summary


def nuscenes_tracking_metrics(gts, tracks, class_names, class_range=None, host=False):
    """gts / tracks as in the module docstring -> {"AMOTA", "AMOTP", "MOTA", "MOTP", "recall", "IDS", "FRAG", "FP",
    "FN", "per_class": {tracking class: the same keys plus "score_cutoff" and "n_gt"}}, fractions and metres.
    host=True runs the host twins."""
    pk = pack(gts, tracks, class_names, class_range)
    res = (run_host if host else run_device)(pk, gts)
    return score(pk, res)


def track_detections(frames, detections, class_names, host=False, **track_kw):
    """track.track over the tracking classes' detections, with track.NUSCENES_MAX_DIST overridden by any max_dist
    given; frames: token -> {"sequence", "timestamp", "pose"}.  -> token -> the tracking classes' detections (labels
    indexing class_names, numpy) plus "tracking_id"."""
    from .track import NUSCENES_MAX_DIST, track
    track_kw["max_dist"] = dict(NUSCENES_MAX_DIST, **(track_kw.get("max_dist") or {}))
    tcls = tracking_classes(class_names)
    to_t = np.array([tcls.index(n) if n in tcls else -1 for n in class_names], np.int64)
    sub = {}
    for t, d in detections.items():
        lab = _arr(d["label_preds"]).reshape(-1).astype(np.int64)
        keep = to_t[lab] >= 0
        sub[t] = {"box3d_lidar": EN._box9(d["box3d_lidar"])[keep],
                  "scores": _arr(d["scores"], np.float32).reshape(-1)[keep], "label_preds": to_t[lab[keep]]}
    back = np.array([class_names.index(n) for n in tcls], np.int64)
    tracks = {}
    for t, d in track(sub, frames, tcls, host=host, **track_kw).items():
        d = dict(d)
        d["label_preds"] = back[np.asarray(d["label_preds"])]
        tracks[t] = d
    return tracks


def track_and_score(gts, detections, class_names, class_range=None, host=False, **track_kw):
    """track_detections over the frames of gts (each with "sequence", "timestamp" and "pose"), then
    nuscenes_tracking_metrics -> (tracks, metrics)."""
    tracks = track_detections(gts, detections, class_names, host=host, **track_kw)
    return tracks, nuscenes_tracking_metrics(gts, tracks, class_names, class_range, host=host)
