"""Cost of the GPU global augmentation: the kernel alone, and its share of a training step.

  python tools/bench_aug.py [--iters 200] [--rounds 5] [--steps 10] [--json OUT]

1. ops.global_aug (one pnx_global_aug launch) on 6 frames x 30k points (the nuScenes bench shape) and 6 frames x 265k
   points, 40 boxes per frame, the reference's four transforms on every frame.  CUDA events around `--iters` back-to-back
   calls after a warm-up; GB/s counts the bytes the algorithm has to move, 48 per point (24 read, 24 written) and 72 per
   box, over the kernel time.
2. The bench.py `nusc` training step (forward, backward, AdamW) on raw-ground-truth examples with and without `aug`
   records, the two arms alternated `--rounds` times, `--steps` steps each, CUDA events; the median per arm is reported.
The card name, power limit and SM clocks are printed with the numbers, because every number depends on them.
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

N_BOXES = 40


def aug_records(frames, seed):
    from det3d.datasets.pipelines import augmentation as A
    chain = [A.Rotation([-0.785, 0.785]), A.Scaling([0.9, 1.1]), A.Translation(0.5), A.Flip([0.5, 0.5])]
    np.random.seed(seed)
    aug = np.zeros((frames, 4, 4))
    for f in range(frames):
        res = {}
        for op in chain:
            res = op(res)
        aug[f] = res["aug"]
    return torch.from_numpy(aug)


def time_kernel(frames, points, iters, dev):
    from pillarnext_b200 import ops, synth
    seeds = list(range(frames))
    pts = synth.make_batch(seeds, points, kind="uniform", with_labels=False)["points"].to(dev)
    boxes = synth.make_gt_batch(seeds, N_BOXES)[0].to(dev)
    aug = aug_records(frames, 0).to(dev)
    for _ in range(20):
        ops.global_aug(pts, boxes, aug)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        ops.global_aug(pts, boxes, aug)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / iters
    nbytes = 48 * pts.shape[0] + 72 * boxes.shape[0] * boxes.shape[1]
    return dict(frames=frames, points_per_frame=points, n_points=int(pts.shape[0]), boxes=frames * N_BOXES, ms=ms,
                us=1000 * ms, bytes=nbytes, gb_per_s=nbytes / (ms * 1e-3) / 1e9)


def time_steps(rounds, steps, warmup, dev):
    from pillarnext_b200 import modules, synth
    sel = synth.BENCH_CONFIGS["nusc"]
    cfg = sel["cfg"]
    frames = cfg["frames_per_gpu"]
    torch.manual_seed(0)
    model = modules.build_pillarnext_b(cfg).to(dev).train()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, betas=(0.9, 0.99), weight_decay=0.01, fused=True)
    plain, augmented = [], []
    for b in range(2):
        seeds = [b * frames + f for f in range(frames)]
        ex = synth.make_batch(seeds, sel["points"], cfg, kind="lidar", sweeps=sel["sweeps"], rings=sel["rings"],
                              with_labels=False)
        gt_b, gt_c = synth.make_gt_batch(seeds, N_BOXES, cfg)
        raw = dict(points=ex["points"].to(dev), token=ex["token"], gt_boxes_raw=gt_b.to(dev), gt_classes=gt_c.to(dev))
        plain.append(raw)
        augmented.append(dict(raw, aug=aug_records(frames, 100 + b).to(dev)))

    def step(ex):
        loss, _ = model(ex)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)

    def window(batches):
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for i in range(steps):
            step(batches[i % 2])
        t1.record()
        torch.cuda.synchronize()
        return t0.elapsed_time(t1) / steps

    for i in range(warmup):
        step(plain[i % 2])
        step(augmented[i % 2])
    ms = {"plain": [], "aug": []}
    for _ in range(rounds):
        ms["plain"].append(window(plain))
        ms["aug"].append(window(augmented))
    med = {k: float(np.median(v)) for k, v in ms.items()}
    return dict(frames=frames, points_per_frame=sel["points"], rounds=rounds, steps=steps, ms=ms, median_ms=med,
                overhead_pct=100.0 * (med["aug"] - med["plain"]) / med["plain"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_aug.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = card()
    print("card: %s" % gpu)
    kernel = [time_kernel(6, n, args.iters, dev) for n in (30000, 265000)]
    for r in kernel:
        print("ops.global_aug %d frames x %dk points + %d boxes: %7.2f us  %7.1f GB/s (%.1f MB)"
              % (r["frames"], r["points_per_frame"] // 1000, r["boxes"], r["us"], r["gb_per_s"], r["bytes"] / 1e6))
    st = time_steps(args.rounds, args.steps, args.warmup, dev)
    print("nusc training step, %d frames x %dk points, median of %d rounds x %d steps: without aug %.2f ms, with aug %.2f ms "
          "(%+.2f %%)" % (st["frames"], st["points_per_frame"] // 1000, st["rounds"], st["steps"], st["median_ms"]["plain"],
                          st["median_ms"]["aug"], st["overhead_pct"]))
    print("  per-round ms without aug: %s" % " ".join("%.2f" % v for v in st["ms"]["plain"]))
    print("  per-round ms with aug:    %s" % " ".join("%.2f" % v for v in st["ms"]["aug"]))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(card=gpu, kernel=kernel, step=st), fh, indent=1)


if __name__ == "__main__":
    main()
