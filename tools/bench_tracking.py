"""Tracking and its CLEAR-MOT metric on a Waymo-validation-shaped input, timed with CUDA events.

  python tools/bench_tracking.py [--sequences 200] [--frames 200] [--repeats 3] [--json OUT]

Input: oracle/track_fixtures.waymo_val_shaped (sequences x frames, three classes, up to 500 detections per class and
frame).  Timed, each after one warm-up call, the median of --repeats:
  track_greedy  ops.track_greedy on device operands already packed and sorted (the tracker kernels and the status read);
  eval_mot      ops.eval_mot on the device pairs and components (the per-(sequence, class, cutoff) walk);
  whole call    track.track + evaluate_waymo_tracking.waymo_tracking_metrics from the host dicts, packing included
                (one call, after the kernels above are warm: most of it is host-side packing).
The card name and power limit are printed with the numbers, because every number depends on them.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gemm_shape_table import card  # noqa: E402


def timed(fn, repeats, warm=True):
    if warm:
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sequences", type=int, default=200)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_tracking.py needs a CUDA device")
    from oracle.track_fixtures import CLASSES, waymo_val_shaped
    from pillarnext_b200 import evaluate_waymo_tracking as EWT, ops, track as TR
    dets, frames, gts = waymo_val_shaped(0, args.sequences, args.frames)

    def cu(a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()
    pk = TR.pack(dets, frames, CLASSES)
    tr = [cu(pk[k]) for k in ("boxes", "scores")] + [torch.sort(cu(pk["keys"]), stable=True)[1]] + \
        [cu(pk[k]) for k in ("seg_start", "seg_count", "poses", "times", "seq_start", "max_dist")]
    t_track = timed(lambda: ops.track_greedy(*tr, 3, 0.1), args.repeats)
    tracks = TR.track(dets, frames, CLASSES, min_score=0.1)
    mp = EWT.pack(gts, tracks, CLASSES)
    npts, _, _ = EWT.run_device(mp)
    order = torch.sort(cu(mp["keys"]), stable=True)[1]
    start, e_det, e_box, e_iou, _ = ops.eval_pairs(cu(mp["det_boxes"]), cu(mp["det_trig"]), order, cu(mp["seg_start"]),
                                                   cu(mp["seg_count"]), cu(mp["gt_boxes"]), cu(mp["gt_classes"]),
                                                   cu(mp["gt_trig"]), cu(mp["thresholds"]))
    comp_start, comp_nedge, grouped = ops.eval_components(start, e_det, e_box, mp["M"], mp["C"])
    mot_args = (start, e_det, e_box, e_iou, grouped, comp_start, comp_nedge, cu(mp["det_pass"]), cu(mp["det_id"]),
                cu(mp["gt_obj"].reshape(-1)), cu(npts.reshape(-1)), cu(mp["seq_start"]), mp["M"], mp["C"], mp["K"],
                mp["n_obj"])
    t_mot = timed(lambda: ops.eval_mot(*mot_args), args.repeats)
    res = {}

    def whole():
        res["m"] = EWT.waymo_tracking_metrics(gts, TR.track(dets, frames, CLASSES, min_score=0.1), CLASSES)
    t_whole = timed(whole, 1, warm=False)
    out = dict(card=card(), sequences=args.sequences, frames=args.frames, detections=int(len(pk["scores"])),
               pairs=int(len(e_det)), track_greedy_ms=t_track, eval_mot_ms=t_mot, whole_call_ms=t_whole,
               metrics={k: v for k, v in res["m"].items() if k != "per_class"})
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
