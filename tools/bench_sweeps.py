"""Cost of the GPU multi-sweep accumulation: the kernels alone, their share of a training step, and the numpy loader work
they replace.

  python tools/bench_sweeps.py [--iters 200] [--rounds 5] [--steps 10] [--json OUT]

1. ops.accumulate_sweeps (mark, scan, write) at 6 frames x 10 sweeps x 26.5k points (the nuScenes ten-sweep size of
   SURVEY.md section 8d) and 3 frames x 3 sweeps x 180k points (Waymo's three-frame size), min_distance 1.0, random
   planar transforms (oracle/sweeps_oracle.random_operands).  CUDA events around `--iters` back-to-back calls after a
   warm-up.  GB/s counts the bytes the algorithm has to move over the kernel time: 24 B read per key-frame point, 20 B
   per sweep point, 24 B written per output row (24 n + 20 S + 24 (n + S)); the second read of the sweep rows that the
   mark / write split makes is not counted.
2. The bench.py `nusc` training step (forward, backward, AdamW) on the same 30k-point frames, once as merged clouds
   and once as a 3k-point key frame plus nine 3k-point sweeps that the step accumulates, the two arms alternated
   `--rounds` times, `--steps` steps each, CUDA events; the median per arm is reported.
3. HOST time: the reference's numpy accumulation (read_sweep + remove_close + concatenate, oracle/sweeps_oracle.py) of
   one 10 x 26.5k-point frame, the data-loader work the GPU stage removes.
The card name, power limit and SM clocks are printed with the numbers, because every number depends on them.
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

from gemm_shape_table import card  # noqa: E402
from oracle import sweeps_oracle as O  # noqa: E402

OPS = ("points", "point_offsets", "sweep_points", "sweep_offsets", "transforms")


def time_kernel(frames, sweeps, points, iters, dev):
    from pillarnext_b200 import ops
    a = O.random_operands(frames, sweeps, points, seed=0)
    args = [torch.from_numpy(a[k]).to(dev) for k in OPS]
    for _ in range(20):
        _, count = ops.accumulate_sweeps(*args, 1.0)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        ops.accumulate_sweeps(*args, 1.0)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / iters
    n, S = len(a["points"]), len(a["sweep_points"])
    nbytes = 24 * n + 20 * S + 24 * (n + S)
    return dict(frames=frames, sweeps=sweeps, points_per_sweep=points, n_points=n, sweep_points=S,
                valid_rows=int(count.item()), ms=ms, us=1000 * ms, bytes=nbytes, gb_per_s=nbytes / (ms * 1e-3) / 1e9)


def split_sweeps(points, frames, n_sweeps, seed):
    """A merged [N, 6] cloud of `frames` equal frames -> the sweep keys of scenes.collate: each frame's first 1/n_sweeps
    is its key frame, the rest n_sweeps - 1 sweeps taken back by a small random planar motion (the step moves them
    forward again)."""
    g = np.random.default_rng(seed)
    p = points.numpy().reshape(frames, -1, 6)
    m = p.shape[1] // n_sweeps
    K = n_sweeps - 1
    tms = np.zeros((frames, K, 4, 4))
    sw = []
    for f in range(frames):
        for k in range(K):
            th = g.uniform(-0.05, 0.05)
            T = np.eye(4)
            T[:2, :2] = [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]
            T[:2, 3] = g.uniform(-1, 1, 2)
            tms[f, k] = T
            q = p[f, m * (k + 1):m * (k + 2), 1:].astype(np.float64)
            q[:, :3] = (np.c_[q[:, :3], np.ones(len(q))] @ np.linalg.inv(T).T)[:, :3]
            sw.append(q.astype(np.float32))
    key = p[:, :m].reshape(-1, 6)
    return dict(points=torch.from_numpy(np.ascontiguousarray(key)),
                point_offsets=torch.from_numpy((np.arange(frames + 1) * m).astype(np.int32)),
                sweep_points=torch.from_numpy(np.concatenate(sw)),
                sweep_offsets=torch.from_numpy((np.arange(frames * K + 1) * m).astype(np.int32)),
                sweep_transforms=torch.from_numpy(tms), sweep_min_distance=1.0)


def time_steps(rounds, steps, warmup, dev):
    from pillarnext_b200 import modules, synth
    sel = synth.BENCH_CONFIGS["nusc"]
    cfg = sel["cfg"]
    frames = cfg["frames_per_gpu"]
    torch.manual_seed(0)
    model = modules.build_pillarnext_b(cfg).to(dev).train()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, betas=(0.9, 0.99), weight_decay=0.01, fused=True)
    plain, swept = [], []
    for b in range(2):
        seeds = [b * frames + f for f in range(frames)]
        ex = synth.make_batch(seeds, sel["points"], cfg, kind="lidar", sweeps=sel["sweeps"], rings=sel["rings"],
                              with_labels=False)
        gt_b, gt_c = synth.make_gt_batch(seeds, 40, cfg)
        raw = dict(token=ex["token"], gt_boxes_raw=gt_b.to(dev), gt_classes=gt_c.to(dev).to(torch.int32))
        plain.append(dict(raw, points=ex["points"].to(dev)))
        sw = split_sweeps(ex["points"], frames, 10, 100 + b)
        swept.append(dict(raw, **{k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in sw.items()}))

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
        step(swept[i % 2])
    ms = {"merged": [], "sweeps": []}
    for _ in range(rounds):
        ms["merged"].append(window(plain))
        ms["sweeps"].append(window(swept))
    med = {k: float(np.median(v)) for k, v in ms.items()}
    return dict(frames=frames, points_per_frame=sel["points"], rounds=rounds, steps=steps, ms=ms, median_ms=med,
                overhead_pct=100.0 * (med["sweeps"] - med["merged"]) / med["merged"])


def time_numpy(repeats=5):
    a = O.random_operands(1, 10, 26500, seed=1)
    args = [a[k] for k in OPS]
    O.accumulate(*args, 1.0)
    t = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        O.accumulate(*args, 1.0)
        t.append(time.perf_counter() - t0)
    return dict(frame_points=len(a["points"]) + len(a["sweep_points"]), host_ms=1000 * float(np.median(t)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_sweeps.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    gpu = card()
    print("card: %s" % gpu)
    kernel = [time_kernel(6, 10, 26500, args.iters, dev), time_kernel(3, 3, 180000, args.iters, dev)]
    for r in kernel:
        print("ops.accumulate_sweeps %d frames x %d sweeps x %.1fk points (%d valid of %d rows): %7.2f us  %7.1f GB/s "
              "(%.1f MB)" % (r["frames"], r["sweeps"], r["points_per_sweep"] / 1000, r["valid_rows"],
                             r["n_points"] + r["sweep_points"], r["us"], r["gb_per_s"], r["bytes"] / 1e6))
    st = time_steps(args.rounds, args.steps, args.warmup, dev)
    print("nusc training step, %d frames x %dk points, median of %d rounds x %d steps: merged clouds %.2f ms, key frame + "
          "9 sweeps accumulated in the step %.2f ms (%+.2f %%)" % (st["frames"], st["points_per_frame"] // 1000,
                                                                   st["rounds"], st["steps"], st["median_ms"]["merged"],
                                                                   st["median_ms"]["sweeps"], st["overhead_pct"]))
    print("  per-round ms merged: %s" % " ".join("%.2f" % v for v in st["ms"]["merged"]))
    print("  per-round ms sweeps: %s" % " ".join("%.2f" % v for v in st["ms"]["sweeps"]))
    host = time_numpy()
    print("HOST time: numpy accumulation of one %d-point frame (10 sweeps x 26.5k), the loader work this removes: %.2f ms"
          % (host["frame_points"], host["host_ms"]))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(card=gpu, kernel=kernel, step=st, host=host), fh, indent=1)


if __name__ == "__main__":
    main()
