"""Cost of the GPU ground-truth database sampling: the kernels alone, and their share of a training step.

  python tools/bench_gts.py [--iters 200] [--rounds 5] [--steps 10] [--json OUT]

1. ops.gt_sample (select, mark, scan, write) on 6 frames x 30k points (the nuScenes bench shape) and 6 frames x 265k
   points, 40 scene boxes and 40 candidates per frame in the ten class calls of the reference's nuScenes groups, 200
   stored points per candidate.  CUDA events around `--iters` back-to-back calls after a warm-up.  GB/s counts the bytes
   the algorithm has to move over the kernel time: 24 B read + 24 B written per scene point, 20 B read + 24 B written
   per candidate point, 48 B per scene box and 56 B per candidate read, 40 B per output box written.
2. The bench.py `nusc` training step (forward, backward, AdamW) on raw-ground-truth examples with and without sampling
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

NUSC_GROUPS = [2, 3, 7, 4, 6, 2, 6, 6, 2, 2]       # the reference nuScenes sampler's group maxima, 40 in all
PTS_PER_CAND = 200


def candidates(gt_boxes, n_classes, seed, dev):
    """Sampling records for a collated batch: scene trig, 40 candidates per frame (class ids cycled into the task's
    classes), PTS_PER_CAND stored points each."""
    from det3d.datasets.pipelines.sample_ops import libm_trig, numpy_trig
    rng = np.random.default_rng(seed)
    B, M = gt_boxes.shape[:2]
    S = sum(NUSC_GROUPS)
    gb = gt_boxes.cpu().numpy()
    st = numpy_trig(gb.reshape(-1, 9)).reshape(B, M, 2)
    cb = np.concatenate([rng.uniform(-50, 50, (B, S, 2)), rng.uniform(-2, 0, (B, S, 1)), rng.uniform(0.5, 8, (B, S, 2)),
                         rng.uniform(1, 3, (B, S, 1)), rng.normal(0, 1, (B, S, 2)), rng.uniform(-np.pi, np.pi, (B, S, 1))],
                        2).astype(np.float32)
    cc = np.tile(np.repeat(np.arange(10) % n_classes, NUSC_GROUPS), (B, 1)).astype(np.int32)
    ct = np.concatenate([numpy_trig(cb.reshape(-1, 9)), libm_trig(cb.reshape(-1, 9)[:, -1])], 1).reshape(B, S, 4)
    off = (np.arange(B * S + 1) * PTS_PER_CAND).astype(np.int32)
    cp = np.concatenate([rng.uniform(-1.5, 1.5, (off[-1], 3)), rng.uniform(0, 255, (off[-1], 1)),
                         np.zeros((off[-1], 1))], 1).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return dict(gt_trig=t(st), gts_boxes=t(cb), gts_classes=t(cc), gts_trig=t(ct), gts_points=t(cp), gts_offsets=t(off))


def time_kernel(frames, points, iters, dev):
    from pillarnext_b200 import ops, synth
    seeds = list(range(frames))
    pts = synth.make_batch(seeds, points, kind="uniform", with_labels=False)["points"].to(dev)
    boxes, classes = (t.to(dev) for t in synth.make_gt_batch(seeds, 40))
    c = candidates(boxes, 3, 0, dev)
    args = (pts, boxes, classes.to(torch.int32), c["gt_trig"], c["gts_boxes"], c["gts_classes"], c["gts_trig"],
            c["gts_points"], c["gts_offsets"])
    for _ in range(20):
        out = ops.gt_sample(*args)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        ops.gt_sample(*args)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / iters
    n, P = pts.shape[0], c["gts_points"].shape[0]
    B, M, S = boxes.shape[0], boxes.shape[1], c["gts_boxes"].shape[1]
    nbytes = 48 * n + 44 * P + 48 * B * M + 56 * B * S + 40 * B * (M + S)
    return dict(frames=frames, points_per_frame=points, n_points=int(n), candidate_points=int(P), candidates=B * S,
                accepted=int(out[3].sum().item()), valid_rows=int(out[4].item()), ms=ms, us=1000 * ms, bytes=nbytes,
                gb_per_s=nbytes / (ms * 1e-3) / 1e9)


def time_steps(rounds, steps, warmup, dev):
    from pillarnext_b200 import modules, synth
    sel = synth.BENCH_CONFIGS["nusc"]
    cfg = sel["cfg"]
    frames = cfg["frames_per_gpu"]
    torch.manual_seed(0)
    model = modules.build_pillarnext_b(cfg).to(dev).train()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, betas=(0.9, 0.99), weight_decay=0.01, fused=True)
    n_classes = sum(len(t) for t in cfg["tasks"])
    plain, sampled = [], []
    for b in range(2):
        seeds = [b * frames + f for f in range(frames)]
        ex = synth.make_batch(seeds, sel["points"], cfg, kind="lidar", sweeps=sel["sweeps"], rings=sel["rings"],
                              with_labels=False)
        gt_b, gt_c = synth.make_gt_batch(seeds, 40, cfg)
        raw = dict(points=ex["points"].to(dev), token=ex["token"], gt_boxes_raw=gt_b.to(dev),
                   gt_classes=gt_c.to(dev).to(torch.int32))
        plain.append(raw)
        sampled.append(dict(raw, **candidates(gt_b, n_classes, 100 + b, dev)))

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
        step(sampled[i % 2])
    ms = {"plain": [], "gts": []}
    for _ in range(rounds):
        ms["plain"].append(window(plain))
        ms["gts"].append(window(sampled))
    med = {k: float(np.median(v)) for k, v in ms.items()}
    return dict(frames=frames, points_per_frame=sel["points"], rounds=rounds, steps=steps, ms=ms, median_ms=med,
                overhead_pct=100.0 * (med["gts"] - med["plain"]) / med["plain"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_gts.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = card()
    print("card: %s" % gpu)
    kernel = [time_kernel(6, n, args.iters, dev) for n in (30000, 265000)]
    for r in kernel:
        print("ops.gt_sample %d frames x %dk points, %d candidates (%d accepted, %d points): %7.2f us  %7.1f GB/s (%.1f MB)"
              % (r["frames"], r["points_per_frame"] // 1000, r["candidates"], r["accepted"], r["candidate_points"], r["us"],
                 r["gb_per_s"], r["bytes"] / 1e6))
    st = time_steps(args.rounds, args.steps, args.warmup, dev)
    print("nusc training step, %d frames x %dk points, median of %d rounds x %d steps: without sampling %.2f ms, with "
          "sampling %.2f ms (%+.2f %%)" % (st["frames"], st["points_per_frame"] // 1000, st["rounds"], st["steps"],
                                           st["median_ms"]["plain"], st["median_ms"]["gts"], st["overhead_pct"]))
    print("  per-round ms without sampling: %s" % " ".join("%.2f" % v for v in st["ms"]["plain"]))
    print("  per-round ms with sampling:    %s" % " ".join("%.2f" % v for v in st["ms"]["gts"]))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(card=gpu, kernel=kernel, step=st), fh, indent=1)


if __name__ == "__main__":
    main()
