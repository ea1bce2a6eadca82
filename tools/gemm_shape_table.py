"""Per-shape table of the tensor-core GEMMs of one training step: calls, ms, TFLOP/s and share of the step.

  python tools/gemm_shape_table.py [--config nusc] [--steps 10] [--warmup 5] [--json OUT]

Builds the bench.py model and synthetic batches, times --steps plain steps with CUDA events (the step time), then runs one
probe step with ops.PROFILE on: CUDA events around every igemm / igemm_win / wgrad launch, tagged by shape.  Rows are
grouped by (kind, tag), sorted by time.  The card name, power limit and SM clocks are printed with the table, because
every number in it depends on them.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=" + q, "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:  # the table is still worth printing without it
        return "%s (nvidia-smi unavailable: %s)" % (torch.cuda.get_device_name(), e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="nusc")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the rows as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("gemm_shape_table.py needs a CUDA device")
    from pillarnext_b200 import modules, ops, synth
    dev = torch.device("cuda", 0)
    sel = synth.BENCH_CONFIGS[args.config]
    cfg = sel["cfg"]
    frames = cfg["frames_per_gpu"]
    torch.manual_seed(0)
    model = modules.build_pillarnext_b(cfg).to(dev).train()
    opt = torch.optim.AdamW(list(model.parameters()), lr=1e-4, betas=(0.9, 0.99), weight_decay=0.01, fused=True)
    batches = []
    for b in range(4):
        ex = synth.make_batch([b * frames + f for f in range(frames)], sel["points"], cfg, kind="lidar", n_boxes=40,
                              sweeps=sel["sweeps"], rings=sel["rings"])
        batches.append({k: ([e.to(dev) for e in v] if isinstance(v, list) and torch.is_tensor(v[0]) else
                            (v.to(dev) if torch.is_tensor(v) else v)) for k, v in ex.items()})

    def step(ex):
        loss, _ = model(ex)
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)

    for i in range(max(args.warmup, 4)):
        step(batches[i % 4])
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(args.steps):
        step(batches[i % 4])
    t1.record()
    torch.cuda.synchronize()
    step_ms = t0.elapsed_time(t1) / args.steps

    ops.PROFILE = []
    step(batches[0])
    torch.cuda.synchronize()
    prof, ops.PROFILE = ops.PROFILE, None
    rows = {}
    for kind, flops, _nbytes, a, b, tag in prof:
        r = rows.setdefault((kind, tag), [0, 0.0, 0.0])
        r[0] += 1
        r[1] += a.elapsed_time(b)
        r[2] += flops
    out = []
    gpu = card()
    print("card: %s" % gpu)
    print("step: %.2f ms (%d steps, CUDA events, profiler off)" % (step_ms, args.steps))
    print("%-10s %-34s %5s %9s %8s %7s" % ("kind", "tag", "calls", "ms", "TFLOP/s", "share"))
    for (kind, tag), (n, ms, fl) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
        out.append(dict(kind=kind, tag=tag, calls=n, ms=ms, tflops=fl / ms / 1e9, share=ms / step_ms))
        print("%-10s %-34s %5d %9.3f %8.1f %6.1f%%" % (kind, tag, n, ms, fl / ms / 1e9, 100 * ms / step_ms))
    for kinds in (("igemm",), ("igemm_win",), ("igemm", "igemm_win"), ("wgrad",)):
        sel_rows = [r for r in out if r["kind"] in kinds]
        ms = sum(r["ms"] for r in sel_rows)
        fl = sum(r["tflops"] * r["ms"] * 1e9 for r in sel_rows)
        if ms > 0:
            print("total %-28s %5d %9.3f %8.1f %6.1f%%  (%.2f TFLOP)" % (
                "+".join(kinds), sum(r["calls"] for r in sel_rows), ms, fl / ms / 1e9, 100 * ms / step_ms, fl / 1e12))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(card=gpu, step_ms=step_ms, rows=out), fh, indent=1)


if __name__ == "__main__":
    main()
