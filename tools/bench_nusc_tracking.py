"""nuScenes tracking and its AMOTA / AMOTP metric on a nuScenes-validation-shaped input, timed with CUDA events.

  python tools/bench_nusc_tracking.py [--scenes 150] [--frames 40] [--repeats 3] [--oracle-scenes 3] [--json OUT]

Input: oracle/nusc_track_fixtures.nusc_val_shaped (scenes x key frames 0.5 s apart, ten classes, about 40 boxes and up
to 500 detections per frame).  Timed, each after one warm-up call, the median of --repeats:
  track_greedy     ops.track_greedy on device operands already packed and sorted (the tracking classes only);
  pairs            ops.eval_pairs_center on the packed device operands (count pass, prefix sum, write pass);
  threshold pass   ops.eval_mot_center with every detection taking part and the matched flags (one row per (scene,
                   class));
  cutoff pass      ops.eval_mot_center over the 40 recall cutoffs (scenes x tracking classes x 40 rows);
  whole call       evaluate_nuscenes_tracking.track_and_score from the host dicts, packing included (one call, after
                   the kernels above are warm).
The oracle (oracle/nusc_track_oracle.py) is timed per scene on the first --oracle-scenes scenes.  The card name and
power limit are printed with the numbers, because every number depends on them.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_tracking import timed  # noqa: E402
from gemm_shape_table import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=150)
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--oracle-scenes", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_nusc_tracking.py needs a CUDA device")
    from oracle import nusc_track_oracle as O
    from oracle.nusc_track_fixtures import CLASSES, nusc_val_shaped
    from pillarnext_b200 import evaluate_nuscenes as EN, evaluate_nuscenes_tracking as ENT, ops, track as TR
    dets, frames, gts = nusc_val_shaped(0, args.scenes, args.frames)

    def cu(a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()
    tcls = ENT.tracking_classes(CLASSES)
    res = {}

    def whole():
        res["tracks"], res["m"] = ENT.track_and_score(gts, dets, CLASSES)
    whole()                                                    # warm every kernel once
    tracks = res["tracks"]
    sub = {t: dict(box3d_lidar=d["box3d_lidar"], scores=d["scores"], label_preds=np.array(
        [tcls.index(CLASSES[c]) for c in d["label_preds"]], np.int64)) for t, d in tracks.items()}
    pk = TR.pack(sub, gts, tcls, TR.NUSCENES_MAX_DIST)
    tr = [cu(pk[k]) for k in ("boxes", "scores")] + [torch.sort(cu(pk["keys"]), stable=True)[1]] + \
        [cu(pk[k]) for k in ("seg_start", "seg_count", "poses", "times", "seq_start", "max_dist")]
    t_track = timed(lambda: ops.track_greedy(*tr, 3, 0.0), args.repeats)

    mp = ENT.pack(gts, tracks, CLASSES)
    counts = EN.count_points(mp, lambda p, b, c, t: ops.eval_count_points(cu(p), cu(b), cu(c), cu(t)).cpu().numpy())
    classes = EN.evaluated_classes(mp, counts)
    gt_obj, gt_prev, n_obj = ENT.objects(mp, gts, classes)
    pair_args = [cu(mp[k]) for k in ("det_boxes", "order", "seg_start", "seg_count", "gt_boxes")] + [cu(classes)]
    t_pairs = timed(lambda: ops.eval_pairs_center(*pair_args, mp["C"], ENT.PAIR_DIST), args.repeats)
    start, e_det, e_box, e_dist = ops.eval_pairs_center(*pair_args, mp["C"], ENT.PAIR_DIST)
    comp_start, comp_nedge, grouped = ops.eval_components(start, e_det, e_box, mp["M"], mp["C"])
    D = len(mp["det_labels"])
    head = (start, e_det, e_box, e_dist, grouped, comp_start, comp_nedge)
    tail = (cu(mp["det_id"]), cu(gt_obj), cu(gt_prev), cu(mp["seq_start"]), mp["M"], mp["C"])
    ones = cu(np.ones(D, np.int32))
    t_thr = timed(lambda: ops.eval_mot_center(*head, ones, *tail, 1, n_obj, want_matched=True), args.repeats)
    matched = ops.eval_mot_center(*head, ones, *tail, 1, n_obj, want_matched=True)[2].cpu().numpy()
    passes = cu(ENT.cutoff_passes(mp, ENT.cutoffs(mp, classes, matched)))
    K = len(ENT.RECALLS)
    t_cut = timed(lambda: ops.eval_mot_center(*head, passes, *tail, K, n_obj), args.repeats)
    t_whole = timed(whole, 1, warm=False)

    seqs = sorted({str(g["sequence"]) for g in gts.values()})[:args.oracle_scenes]
    keep = [t for t in gts if str(gts[t]["sequence"]) in seqs]
    t0 = time.perf_counter()
    O.tracking_metrics({t: gts[t] for t in keep}, {t: tracks[t] for t in keep}, CLASSES)
    t_oracle = (time.perf_counter() - t0) * 1000.0 / max(1, len(seqs))

    out = dict(card=card(), scenes=args.scenes, frames=args.frames, detections=int(D), pairs=int(len(e_det)),
               cutoff_rows=int((len(mp["seq_start"]) - 1) * mp["C"] * K), track_greedy_ms=t_track, pairs_ms=t_pairs,
               threshold_pass_ms=t_thr, cutoff_pass_ms=t_cut, whole_call_ms=t_whole, oracle_ms_per_scene=t_oracle,
               metrics={k: v for k, v in res["m"].items() if k != "per_class"})
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
