"""Eval-mode throughput and peak memory of the detector, single pass and with double-flip test-time augmentation.

  python tools/bench_eval.py [--config nusc] [--frames 6] [--steps 20] [--warmup 5] [--json OUT]

Builds the bench.py model (seeded, untrained) in eval mode and times `model(example)` -- forward, decode, NMS and the copy
of the detections to the host -- on synthetic lidar batches with CUDA events, for post_processing.double_flip False and
True.  Peak memory is torch.cuda.max_memory_allocated over the timed window.  When the 4 x frames double-flip batch
does not fit, the out-of-memory error is reported and the largest batch that fits (halving the frames) is measured
instead.  The card name, power limit and SM clocks are printed with the numbers, because every number depends on them.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from gemm_shape_table import card  # noqa: E402


def measure(model, batches, double_flip, steps, warmup):
    model.post_processing["double_flip"] = double_flip
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    with torch.no_grad():
        for i in range(warmup):
            model(batches[i % len(batches)])
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n_det = 0
        t0.record()
        for i in range(steps):
            dets = model(batches[i % len(batches)])
            n_det += sum(d["scores"].numel() for d in dets.values())
        t1.record()
        torch.cuda.synchronize()
    frames = len(batches[0]["token"])
    ms = t0.elapsed_time(t1) / steps
    return dict(double_flip=double_flip, frames=frames, ms_per_batch=ms, frames_per_s=1000.0 * frames / ms,
                peak_mem_gib=torch.cuda.max_memory_allocated() / 2 ** 30, detections_per_frame=n_det / steps / frames)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="nusc")
    ap.add_argument("--frames", type=int, default=None, help="frames per batch (default: the config's frames_per_gpu)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_eval.py needs a CUDA device")
    from pillarnext_b200 import modules, synth
    dev = torch.device("cuda", 0)
    sel = synth.BENCH_CONFIGS[args.config]
    cfg = sel["cfg"]
    frames = args.frames or cfg["frames_per_gpu"]
    torch.manual_seed(0)
    model = modules.build_pillarnext_b(cfg).to(dev).eval()
    model.post_processing = dict(cfg["post_processing"])

    def make_batches(n):
        out = []
        for b in range(2):
            ex = synth.make_batch([b * n + f for f in range(n)], sel["points"], cfg, kind="lidar", n_boxes=40,
                                  sweeps=sel["sweeps"], rings=sel["rings"])
            out.append(dict(points=ex["points"].to(dev), token=["f%d" % (b * n + f) for f in range(n)]))
        return out

    gpu = card()
    print("card: %s" % gpu)
    print(sel["label"] % sel["points"])
    results = []
    for double_flip in (False, True):
        n = frames
        while n >= 1:
            try:
                r = measure(model, make_batches(n), double_flip, args.steps, args.warmup)
                break
            except torch.cuda.OutOfMemoryError as e:
                print("double_flip=%s, %d frames (%d forward frames): out of memory: %s" % (
                    double_flip, n, 4 * n if double_flip else n, str(e).splitlines()[0]))
                r = dict(double_flip=double_flip, frames=n, oom=True)
                results.append(r)
                torch.cuda.empty_cache()
                n //= 2
        else:
            continue
        results.append(r)
        print("double_flip=%-5s %d frames (%3d forward frames): %8.2f ms/batch  %7.2f frames/s  peak %6.2f GiB  %.0f det/frame"
              % (double_flip, r["frames"], 4 * r["frames"] if double_flip else r["frames"], r["ms_per_batch"],
                 r["frames_per_s"], r["peak_mem_gib"], r["detections_per_frame"]))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(card=gpu, config=args.config, steps=args.steps, results=results), fh, indent=1)


if __name__ == "__main__":
    main()
