#!/usr/bin/env python
"""Time the nuScenes detection score (pillarnext_b200/evaluate_nuscenes.py) on a nuScenes-val-shaped seeded input: 6019
frames with about 40 labels over the ten classes and up to 500 detections each (jittered labels plus false positives).
One nuscenes_metrics call scores the whole set, twice: once with per-box num_points given, once with --points points
per frame counted on the GPU.  Reports CUDA-event times of the match and the point count, the wall time of each whole
call, the sequential oracle's time on an --oracle-frames subset with the largest difference from the product over every
reported number, and the card's name and power limit, as one JSON line.

  python tools/bench_nds_eval.py --frames 6019 --points 30000
"""
import argparse
import json
import math
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_waymo_eval import Timer, card  # noqa: E402
from oracle import nds_fixtures, nds_oracle  # noqa: E402
from pillarnext_b200 import evaluate_nuscenes as EN  # noqa: E402


def max_diff(a, b):
    out = 0.0
    for k, v in a.items():
        if k == "per_class":
            for name in v:
                out = max(out, max_diff(v[name], b[k][name]))
        elif not (math.isnan(v) and math.isnan(b[k])):
            out = max(out, abs(v - b[k]))
    return out


def timed(gts, dets, classes):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = EN.nuscenes_metrics(gts, dets, classes)
    torch.cuda.synchronize()
    return res, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=6019)
    ap.add_argument("--points", type=int, default=30000)
    ap.add_argument("--oracle-frames", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    warm_g, warm_d, classes = nds_fixtures.make_frames(args.seed + 999, 2, n_points=1000)
    EN.nuscenes_metrics(warm_g, warm_d, classes)
    out = {"card": card(), "frames": args.frames}
    t0 = time.perf_counter()
    gts, dets, classes = nds_fixtures.make_frames(args.seed, args.frames, n_points=None, fp_per_frame=460)
    gen_s = time.perf_counter() - t0
    out["detections"] = int(sum(len(d["scores"]) for d in dets.values()))
    out["labels"] = int(sum(len(g["names"]) for g in gts.values()))
    with Timer("eval_match_center") as tm:
        res, wall = timed(gts, dets, classes)
    out.update(num_points_match_ms=round(tm.ms, 2), num_points_nuscenes_metrics_s=round(wall, 2),
               num_points_NDS=res["NDS"], num_points_mAP=res["mAP"])
    del gts, dets
    t0 = time.perf_counter()
    gts, dets, classes = nds_fixtures.make_frames(args.seed + 1, args.frames, n_points=args.points, fp_per_frame=460)
    gen_s += time.perf_counter() - t0
    with Timer("eval_count_points") as tc, Timer("eval_match_center") as tm:
        res, wall = timed(gts, dets, classes)
    out.update(points_per_frame=args.points, points_count_ms=round(tc.ms, 2), points_match_ms=round(tm.ms, 2),
               points_nuscenes_metrics_s=round(wall, 2), points_NDS=res["NDS"])
    del gts, dets
    gts, dets, classes = nds_fixtures.make_frames(args.seed + 5000, args.oracle_frames, n_points=args.points,
                                                  fp_per_frame=460)
    t0 = time.perf_counter()
    want = nds_oracle.nuscenes_metrics(gts, dets, classes)
    oracle_s = time.perf_counter() - t0
    got, wall = timed(gts, dets, classes)
    out.update(oracle_frames=args.oracle_frames, oracle_s_per_frame=round(oracle_s / args.oracle_frames, 4),
               product_s_per_frame_on_subset=round(wall / args.oracle_frames, 4),
               product_s_per_frame_full_set=round(out["points_nuscenes_metrics_s"] / args.frames, 5),
               oracle_vs_product_max_abs_diff=max_diff(got, want), input_generation_s=round(gen_s, 1))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
