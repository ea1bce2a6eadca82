#!/usr/bin/env python
"""Time the Waymo-style evaluation (pillarnext_b200/evaluate_waymo.py) on Waymo-val-shaped seeded input: 180k points and
about 60 vehicle, 30 pedestrian and 5 cyclist labels per frame, detections = jittered labels plus false positives (at
most 500 per class).  waymo_metrics runs on chunks of --chunk frames (the points of 2000 frames alone take 8.6 GB).
Reports CUDA-event times of the point count, the match and the whole waymo_metrics call per 1000 frames, the sequential
oracle's time on a 20-frame subset, and the card's name and power limit, as one JSON line.  --matching hungarian (or
both) also times matching="hungarian" on the same frames: its pair, component and assignment passes and the whole call,
against oracle/waymo_hungarian_oracle.py.

  python tools/bench_waymo_eval.py --frames 2000 --chunk 200 --matching both
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import waymo_fixtures, waymo_hungarian_oracle, waymo_metric_oracle  # noqa: E402
from pillarnext_b200 import evaluate_waymo as EW, ops  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name()


class Timer:
    """CUDA-event time of every call of ops.<name> (wrapped for the run)."""

    def __init__(self, name):
        self.name, self.fn, self.ms, self.ev = name, getattr(ops, name), 0.0, []

    def __enter__(self):
        def wrapped(*a, **k):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = self.fn(*a, **k)
            e.record()
            self.ev.append((s, e))
            return out
        setattr(ops, self.name, wrapped)
        return self

    def __exit__(self, *a):
        setattr(ops, self.name, self.fn)
        torch.cuda.synchronize()
        self.ms = sum(s.elapsed_time(e) for s, e in self.ev)


def run_chunks(args, matching, names):
    """Whole-call and per-entry-point CUDA-event ms over all chunks, and the first chunk's result."""
    timers = [Timer(n) for n in names]
    total_ms = gen_s = 0.0
    first = None
    for t in timers:
        t.__enter__()
    try:
        for c0 in range(0, args.frames, args.chunk):
            t0 = time.perf_counter()
            gts, dets, classes = waymo_fixtures.make_frames(args.seed + c0, min(args.chunk, args.frames - c0), token0=c0)
            gen_s += time.perf_counter() - t0
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s.record()
            r = EW.waymo_metrics(gts, dets, classes, matching=matching)
            e.record()
            torch.cuda.synchronize()
            total_ms += s.elapsed_time(e)
            first = first or r
    finally:
        for t in timers:
            t.__exit__()
    return total_ms, {t.name: t.ms for t in timers}, first, gen_s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--chunk", type=int, default=200)
    ap.add_argument("--oracle-frames", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--matching", choices=("greedy", "hungarian", "both"), default="greedy")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    warm_g, warm_d, classes = waymo_fixtures.make_frames(args.seed + 999, 2)
    EW.waymo_metrics(warm_g, warm_d, classes)
    EW.waymo_metrics(warm_g, warm_d, classes, matching="hungarian")
    per_k = 1000.0 / args.frames
    out = {"card": card(), "frames": args.frames, "chunk": args.chunk}
    gts, dets, classes = waymo_fixtures.make_frames(args.seed + 5000, args.oracle_frames)
    if args.matching in ("greedy", "both"):
        total_ms, ms, first, gen_s = run_chunks(args, "greedy", ("eval_count_points", "eval_match"))
        t0 = time.perf_counter()
        want = waymo_metric_oracle.waymo_metrics(gts, dets, classes)
        oracle_s = time.perf_counter() - t0
        got = EW.waymo_metrics(gts, dets, classes)
        out.update({
            "count_ms_per_1000_frames": round(ms["eval_count_points"] * per_k, 3),
            "match_ms_per_1000_frames": round(ms["eval_match"] * per_k, 3),
            "waymo_metrics_ms_per_1000_frames": round(total_ms * per_k, 1),
            "oracle_s_per_frame": round(oracle_s / args.oracle_frames, 3), "oracle_frames": args.oracle_frames,
            "oracle_vs_product_mAPH_L2": [want["mAPH_L2"], got["mAPH_L2"]],
            "first_chunk_mAPH_L2": first["mAPH_L2"], "input_generation_s": round(gen_s, 1)})
    if args.matching in ("hungarian", "both"):
        names = ("eval_count_points", "eval_pairs", "eval_components", "eval_assign")
        total_ms, ms, first, gen_s = run_chunks(args, "hungarian", names)
        t0 = time.perf_counter()
        want = waymo_hungarian_oracle.waymo_metrics(gts, dets, classes)
        oracle_s = time.perf_counter() - t0
        got = EW.waymo_metrics(gts, dets, classes, matching="hungarian")
        h = {n + "_ms_per_1000_frames": round(ms[n] * per_k, 3) for n in names}
        h.update({"waymo_metrics_ms_per_1000_frames": round(total_ms * per_k, 1),
                  "oracle_s_per_frame": round(oracle_s / args.oracle_frames, 3),
                  "oracle_vs_product_mAPH_L2": [want["mAPH_L2"], got["mAPH_L2"]],
                  "first_chunk_mAPH_L2": first["mAPH_L2"],
                  "first_chunk_range_mAPH_L2": {r: v["mAPH_L2"] for r, v in first["range_means"].items()},
                  "input_generation_s": round(gen_s, 1)})
        out["hungarian"] = h
    print(json.dumps(out))


if __name__ == "__main__":
    main()
