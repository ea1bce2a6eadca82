#!/usr/bin/env python
"""bench.py -- frames/sec of the PillarNeXt-B hot path (BASELINE.json metric) on N GPUs of one node.

  python bench.py --gpus 1 --steps K --warmup W                       (N=1)
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
         bench.py --gpus N --steps K --warmup W                       (N>1, one rank per GPU, NCCL)
  python bench.py --impl reference ...                                 (the reference's algorithm on host CPU cores)
  python bench.py ... --dump-outputs DIR                               (also write the last timed step's results as .npy)

A "step" = one training pass of the hot path over one batch of synthetic nuScenes-shaped frames:
reader (voxelize + PillarFeatureNet) -> sparse ResNet-18 -> ASPP -> CenterHead -> CenterPoint loss -> backward
(-> NCCL gradient all-reduce when N>1) -> AdamW step.  Weights are random-init PillarNeXt-B
(10,379,782 parameters), data is synthetic (no dataset / checkpoint is reachable), compute is bf16
tensor-core GEMMs with fp32 accumulation (reader fp32).  Prints ONE JSON line on rank 0.
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "frames/sec PillarNeXt-B fwd+bwd"


def workload(sel, points, frames):
    return (sel["label"] % points) + ", bf16, fwd+loss+bwd+AdamW, %d frames/GPU/step" % frames


def peaks():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as fh:
            p = json.load(fh)
        return dict(hbm=p["hbm_gbs"], tf_burst=p["bf16_tflops"], tf_sust=p.get("bf16_tflops_sustained", p["bf16_tflops"]), src="measured")
    except Exception:
        return dict(hbm=3350.0, tf_burst=989.0, tf_sust=989.0, src="H100 SXM data sheet")


class ClockSampler(threading.Thread):
    """nvidia-smi clocks / throttle reasons sampled during the timed region."""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.rows, self.stop_flag, self.proc = index, [], False, None

    def run(self):
        q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
            "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q, "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            for line in self.proc.stdout:
                self.rows.append(line.strip())
                if self.stop_flag:
                    break
        except Exception:
            pass

    def finish(self):
        self.stop_flag = True
        if self.proc is not None:
            try:
                self.proc.terminate()
            except Exception:
                pass
        sm, mx, reasons = [], 0, set()
        for r in self.rows:
            f = [x.strip() for x in r.split(",")]
            try:
                sm.append(float(f[0]))
                mx = max(mx, float(f[1]))
                for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[2:6]):
                    if val.lower().startswith("active"):
                        reasons.add(name)
            except Exception:
                continue
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx or None, "reasons": sorted(reasons), "samples": len(sm)}


def to_device(ex, dev, non_blocking=False):
    out = {}
    for k, v in ex.items():
        if torch.is_tensor(v):
            out[k] = v.to(dev, non_blocking=non_blocking)
        elif isinstance(v, list) and v and torch.is_tensor(v[0]):
            out[k] = [e.to(dev, non_blocking=non_blocking) for e in v]
        else:
            out[k] = v
    return out


class DeviceSlots:
    """Double-buffered device staging for the end-to-end arm: two sets of device buffers sized for the largest batch,
    filled by non-blocking copies from pinned host memory (what a prefetching loader keeps) -- the timed steps then
    never touch the caching allocator for their inputs (a side-stream allocation pattern that changes from batch to
    batch cost a one-off ~20 ms somewhere in the first dozen steps and made a 5-step e2e number irreproducible)."""

    def __init__(self, host_batches, dev, n_slots=2):
        self.slots = []
        for _ in range(n_slots):
            bufs = {}
            for ex in host_batches:
                for k, v in ex.items():
                    if torch.is_tensor(v):
                        cur = bufs.get(k)
                        if cur is None or cur.numel() < v.numel():
                            bufs[k] = torch.empty(v.numel(), dtype=v.dtype, device=dev)
            self.slots.append(bufs)

    def load(self, slot, ex):
        out = {}
        for k, v in ex.items():
            if torch.is_tensor(v):
                d = self.slots[slot][k][:v.numel()].view(v.shape)
                d.copy_(v, non_blocking=True)
                out[k] = d
            else:
                out[k] = v
        return out


def pin(ex):
    out = {}
    for k, v in ex.items():
        if torch.is_tensor(v):
            out[k] = v.pin_memory()
        elif isinstance(v, list) and v and torch.is_tensor(v[0]):
            out[k] = [e.pin_memory() for e in v]
        else:
            out[k] = v
    return out


def nbytes(ex):
    n = 0
    for v in ex.values():
        if torch.is_tensor(v):
            n += v.numel() * v.element_size()
        elif isinstance(v, list) and v and torch.is_tensor(v[0]):
            n += sum(e.numel() * e.element_size() for e in v)
    return n


# ------------------------------------------------------------------------------------------------- reference arm
def cpu_reference_step(cfg, sd, ex, frames):
    """The reference's algorithm (oracle port: fp32 torch CPU restatement of reader / sparse backbone
    (gather-GEMM form) / ASPP / CenterHead / loss, oracle/pillarnext_oracle.py) fwd+bwd on `frames` frames."""
    from oracle import pillarnext_oracle as O
    p = {k: v.clone().requires_grad_(v.dtype.is_floating_point and "running" not in k) for k, v in sd.items()}
    preds = O.detector_forward(ex["points"], p, cfg, frames, train=True, backbone="gather")
    loss, _ = O.center_loss(ex, preds, cfg["weight"], cfg["code_weights"], cfg["with_reg_iou"], cfg["voxel_size"],
                            cfg["pc_range"], cfg["out_size_factor"], with_iou="iou" in cfg["common_heads"])
    loss.backward()
    return float(loss)


def run_cpu_baseline(cfg, n_points, steps, warmup, sel=None):
    from pillarnext_b200 import modules, synth
    torch.manual_seed(0)
    sd = {k: v.detach().clone() for k, v in modules.build_pillarnext_b(cfg).state_dict().items()}
    sw, rg = (sel["sweeps"], sel["rings"]) if sel else (10, 32)
    exs = [synth.make_batch([100 + i], n_points, cfg, kind="lidar", n_boxes=40, sweeps=sw, rings=rg) for i in range(2)]
    for i in range(warmup):
        cpu_reference_step(cfg, sd, exs[i % 2], 1)
    t0 = time.perf_counter()
    for i in range(steps):
        cpu_reference_step(cfg, sd, exs[i % 2], 1)
    dt = time.perf_counter() - t0
    return steps / dt, dt / steps


def main_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    from pillarnext_b200 import synth
    sel = synth.BENCH_CONFIGS[args.config]
    cfg = sel["cfg"]
    args.points = args.points or sel["points"]
    if int(os.environ.get("WORLD_SIZE", "1")) > 1 and "OMP_NUM_THREADS" in os.environ:
        torch.set_num_threads(os.cpu_count() or 1)      # torchrun pins OMP_NUM_THREADS=1: rank 0 alone runs this arm, on all cores
    steps, warmup = min(args.steps, 3), min(args.warmup, 1)
    fps, spf = run_cpu_baseline(cfg, args.points, steps, warmup, sel)
    cores = torch.get_num_threads()
    sample = "%d timed single-frame fwd+loss+bwd steps (%d pts) of the fp32 oracle port, %d torch CPU threads" % (steps, args.points, cores)
    line = {"impl": "reference", "metric": METRIC, "value": fps, "unit": "frames/s", "n_gpus": args.gpus, "steps": steps,
            "warmup": warmup, "ms_per_step": spf * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic", "config": {"workload": workload(sel, args.points, 1), "note": "CPU port of the reference algorithm (spconv/torch_scatter absent: oracle restatement)"},
            "cpu_baseline": {"value": fps, "unit": "frames/s", "cores": cores, "kind": "port", "sample": sample},
            "e2e": {"value": fps, "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


def dump_outputs(out_dir, model, loss, logs):
    """The loss, logged terms and updated model state (after AdamW) of a training step: one .npy per array, float32
    (integer counters float64)."""
    os.makedirs(out_dir, exist_ok=True)
    arrays = {"loss": loss}

    def flatten(name, v):
        if torch.is_tensor(v) or isinstance(v, (int, float)):
            arrays[name] = v
        elif isinstance(v, dict):
            for k, e in v.items():
                flatten("%s.%s" % (name, k), e)
        elif isinstance(v, (list, tuple)):
            for i, e in enumerate(v):
                flatten("%s.%d" % (name, i), e)

    flatten("logs", logs)
    for k, v in model.state_dict().items():
        arrays["state." + k] = v
    total = 0
    for name, v in arrays.items():
        v = v.detach().cpu() if torch.is_tensor(v) else torch.tensor(v)
        a = v.numpy().astype(np.float32 if v.is_floating_point() else np.float64)
        total += a.nbytes
        np.save(os.path.join(out_dir, name + ".npy"), a)
    assert total <= 64 << 20, "dumped outputs exceed 64 MB (%d bytes)" % total


# ------------------------------------------------------------------------------------------------- GPU arm
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--config", default="nusc", choices=["nusc", "waymo180k", "waymo540k"],
                    help="BASELINE.json configs[1] (default, the config the metric is quoted on) / [3] / [4]")
    ap.add_argument("--frames", type=int, default=0, help="frames per GPU per step (default: the reference's 6 nuScenes / 3 Waymo, docs/RUN.md:9,34)")
    ap.add_argument("--points", type=int, default=0, help="points per frame (default: the config's)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--sync-bn", action="store_true", help="SyncBatchNorm semantics (reference default sync_batchnorm: True) instead of local BN")
    ap.add_argument("--voxelize-sweep", action="store_true", help="also report voxelizer GB/s over batch sizes")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last timed step's loss, logged terms and updated model state as DIR/<name>.npy")
    args = ap.parse_args()
    if args.impl == "reference":
        return main_reference(args)

    import torch.distributed as dist
    from pillarnext_b200 import modules, ops, synth
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    nccl_log = None
    if not torch.cuda.is_available():
        raise RuntimeError("bench.py needs a CUDA device: the product has no CPU path")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        # NCCL's own log (communicator init: nranks, rings/trees, NVLS) goes to a per-process file so stdout stays the one
        # JSON line; rank 0 echoes the communicator lines to stderr at the end
        if os.environ.get("NCCL_DEBUG", "").upper() not in ("INFO", "TRACE"):
            os.environ["NCCL_DEBUG"] = "INFO"
            os.environ.setdefault("NCCL_DEBUG_SUBSYS", "INIT")
        if "NCCL_DEBUG_FILE" not in os.environ:
            logdir = os.path.join(ROOT, "gpurun_out") if os.path.isdir(os.path.join(ROOT, "gpurun_out")) else "/tmp"
            os.environ["NCCL_DEBUG_FILE"] = os.path.join(logdir, "nccl.%h.%p.log")
            nccl_log = os.environ["NCCL_DEBUG_FILE"].replace("%h", os.uname().nodename).replace("%p", str(os.getpid()))
        else:
            nccl_log = None
        dist.init_process_group("nccl", device_id=dev)
    warmup = max(args.warmup, 5)     # >= one untimed step per distinct synthetic batch (4): the caching allocator has seen every size
    sel = synth.BENCH_CONFIGS[args.config]
    cfg = sel["cfg"]
    args.frames = args.frames or cfg["frames_per_gpu"]
    args.points = args.points or sel["points"]
    torch.manual_seed(0)
    model = modules.build_pillarnext_b(cfg, sync_batchnorm=args.sync_bn and world > 1).to(dev).train()
    params = [p for p in model.parameters()]
    opt = torch.optim.AdamW(params, lr=1e-4, betas=(0.9, 0.99), weight_decay=0.01, fused=True)
    nb = 4                                                     # distinct synthetic batches, rotated
    host = [pin(synth.make_batch([rank * 1000 + b * args.frames + f for f in range(args.frames)], args.points, cfg,
                                 kind="lidar", n_boxes=40, sweeps=sel["sweeps"], rings=sel["rings"])) for b in range(nb)]
    resident = [to_device(h, dev) for h in host]
    # end-to-end arm: the host ships the raw ground truth (36 B/object) and the targets are built on the GPU (row F3:
    # pnx_assign_labels), instead of the dense heat-map labels the reference's loader workers produce (5.5 MB/frame)
    host_raw = []
    for b in range(nb):
        gt_b, gt_c = synth.make_gt_batch([rank * 1000 + b * args.frames + f for f in range(args.frames)], 40, cfg)
        host_raw.append(pin({"points": host[b]["points"], "token": host[b]["token"], "gt_boxes_raw": gt_b, "gt_classes": gt_c}))
    from pillarnext_b200.parallel import BucketedGradAllReduce, default_buckets
    reducer = BucketedGradAllReduce(default_buckets(model))     # head | neck | backbone+reader, overlapped with the backward

    last = {}

    def step(ex):
        loss, logs = model(ex)
        loss.backward()
        reducer.finish()
        opt.step()
        opt.zero_grad(set_to_none=True)
        last["loss"], last["logs"] = loss, logs
        return loss

    copy_stream = torch.cuda.Stream(device=dev)
    slots = DeviceSlots(host_raw, dev)
    loss_host = [torch.zeros(1, dtype=torch.float32).pin_memory() for _ in range(2)]
    loss_ev = [torch.cuda.Event() for _ in range(2)]

    def timed(n, e2e):
        # Python's cyclic GC is collected here and held off during the timed steps (a generation-2 pass over the autograd
        # graph objects of a step costs tens of ms at an arbitrary point; trainers at this scale schedule it explicitly too)
        gc.collect()
        gc.disable()
        try:
            return _timed(n, e2e)
        finally:
            gc.enable()

    def _timed(n, e2e):
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        if e2e:
            # end to end: every step copies ITS inputs from pinned host memory and one step's loss is read back to the
            # host, all inside the timed region.  Like a training loop with a prefetching loader and lazy logging,
            # the copy of step i+1 runs on a side stream during step i and the loss of step i is read after step
            # i+1 has been enqueued (the last one before the closing event).
            nxt = None
            prev_loss = None
            for i in range(n):
                if nxt is None:
                    with torch.cuda.stream(copy_stream):
                        nxt = (slots.load(i & 1, host_raw[i % nb]), torch.cuda.Event())
                        nxt[1].record(copy_stream)
                ex, ev = nxt
                torch.cuda.current_stream().wait_event(ev)
                if i + 1 < n:
                    copy_stream.wait_stream(torch.cuda.current_stream())   # slot (i+1)&1 was read by step i-1: free again
                    with torch.cuda.stream(copy_stream):
                        nxt = (slots.load((i + 1) & 1, host_raw[(i + 1) % nb]), torch.cuda.Event())
                        nxt[1].record(copy_stream)
                loss = step(ex)
                # device -> host read of the step's result: async copy into pinned memory + event, consumed one step
                # later (a plain .item() would synchronise the whole stream, i.e. also the step just enqueued)
                slot = i & 1
                loss_host[slot].copy_(loss.detach().reshape(1), non_blocking=True)
                loss_ev[slot].record()
                if prev_loss is not None:
                    loss_ev[prev_loss].synchronize()
                    _ = float(loss_host[prev_loss][0])
                prev_loss = slot
            if prev_loss is not None:
                loss_ev[prev_loss].synchronize()
                _ = float(loss_host[prev_loss][0])
        else:
            for i in range(n):
                step(resident[i % nb])
        t1.record()
        torch.cuda.synchronize()
        ms = torch.tensor([t0.elapsed_time(t1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            dist.barrier()
        return ms.item()

    for i in range(warmup):
        step(resident[i % nb])
    sampler = ClockSampler(local) if rank == 0 else None
    if sampler:
        sampler.start()
    l0 = ops.LAUNCHES
    ms = timed(args.steps, False)
    launches = ops.LAUNCHES - l0
    clocks = sampler.finish() if sampler else None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, model, last["loss"], last["logs"])
    timed(2 * nb + 2, True)             # untimed: every distinct batch once through the copy stream's allocator pool and the read-back path
    ms_e2e = timed(args.steps, True)
    # host-side enqueue time of one step (python + autograd + ctypes launches), no synchronisation inside
    torch.cuda.synchronize()
    th = time.perf_counter()
    for i in range(2):
        step(resident[i % nb])
    host_ms = (time.perf_counter() - th) / 2 * 1e3
    torch.cuda.synchronize()
    frames_total = args.frames * world * args.steps
    value = frames_total / (ms / 1e3)
    e2e = frames_total / (ms_e2e / 1e3)

    # ---- roofline of the dominant kernel family (wgmma implicit GEMM + weight-gradient GEMM), one probe step with
    #      CUDA events around every launch on the launching stream
    ops.PROFILE = []
    step(resident[0])
    torch.cuda.synchronize()
    prof, ops.PROFILE = ops.PROFILE, None
    agg = {}
    for kind, flops, nb_, a, b, _tag in prof:
        d = agg.setdefault(kind, [0.0, 0.0, 0])
        d[0] += flops
        d[1] += a.elapsed_time(b)
        d[2] += 1
    pk = peaks()
    gemm_ms = sum(v[1] for v in agg.values())
    gemm_fl = sum(v[0] for v in agg.values())
    ig = [sum(agg.get(k, [0.0, 0.0, 0])[i] for k in ("igemm", "igemm_win")) for i in range(3)]
    ig[1] = max(ig[1], 1e-9)
    roof = {"bound": "tensor", "kernel": "igemm_kernel + igemm_win_kernel (wgmma implicit GEMM: cp.async row gather / TMA window producers; fwd+dgrad)",
            "achieved": ig[0] / (ig[1] * 1e-3) / 1e12, "peak": pk["tf_sust"], "unit": "TFLOP/s",
            "frac": ig[0] / (ig[1] * 1e-3) / 1e12 / pk["tf_sust"], "traffic": None, "traffic_detail": None, "peak_source": pk["src"] + " (bf16)",
            "launches": ig[2], "flops_per_step": ig[0], "share_of_step": ig[1] / (ms / args.steps),
            "wgrad": {"achieved": agg["wgrad"][0] / (agg["wgrad"][1] * 1e-3) / 1e12, "launches": agg["wgrad"][2],
                      "share_of_step": agg["wgrad"][1] / (ms / args.steps)} if "wgrad" in agg else None,
            "note": "executed MMA flops (zero-filled absent neighbours included); per-launch CUDA events in a probe step"}

    if args.config == "nusc" and args.frames == 6:
        tr = traffic_from_profile(("igemm_kernel", "igemm_win_kernel"))
        if tr:
            roof["traffic"] = tr["bytes_per_launch"]
            roof["traffic_detail"] = dict(tr, unit="bytes of DRAM traffic per launch, averaged over the %d igemm launches of one step "
                                                   "(ncu launch list, same workload)" % tr["launches"],
                                          algorithmic_note="bound is tensor: DRAM traffic is reported for completeness, "
                                                           "flops per launch = flops_per_step / launches")
    # ---- voxelizer HBM roofline (second half of the BASELINE metric): many frames per launch so bytes >= 64 MB
    vox = None
    if rank == 0:
        vox = voxelize_roofline(dev, sel, pk)

    line = None
    if rank == 0:
        cpu = None
        if not args.no_cpu_baseline:
            torch.cuda.synchronize()
            fps, spf = run_cpu_baseline(cfg, args.points, 1, 0, sel)
            cpu = {"value": fps, "unit": "frames/s", "cores": torch.get_num_threads(), "kind": "port",
                   "sample": "1 single-frame fwd+loss+bwd step (%d pts) of the fp32 oracle port on the host CPU (%.1f s)" % (args.points, spf)}
        line = {"metric": METRIC, "value": value, "unit": "frames/s", "n_gpus": world, "steps": args.steps, "warmup": warmup,
                "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
                "dtype": "bf16", "data": "synthetic",
                "config": {"workload": workload(sel, args.points, args.frames), "name": args.config, "global_batch": args.frames * world,
                           "parallelism": "dp%d (frames sharded, bucketed NCCL gradient all-reduce overlapped with the backward, %s BatchNorm)" % (world, "synchronised" if (args.sync_bn and world > 1) else "local"),
                           "l2": "per-step activation working set (GBs) >> 50 MB L2; 4 distinct input batches rotated",
                           "timed_step": "reader+backbone+neck+head fwd, loss, bwd, grad all-reduce (N>1), AdamW",
                           "gc": "Python cyclic GC collected before and disabled inside each timed region"},
                "e2e": {"value": e2e, "unit": "frames/s", "h2d_bytes_per_step": nbytes(host_raw[0]), "d2h_bytes_per_step": 4,
                        "ms_per_step": ms_e2e / args.steps,
                        "pipeline": "inside the timed region every step: pinned-host -> device copy of its inputs = points + raw ground-truth "
                                    "boxes (side stream, overlapping the previous step), label assignment on the GPU (pnx_assign_labels), "
                                    "and a 4-byte loss read-back (async copy to pinned memory + event, consumed one step late)"},
                "gpu": torch.cuda.get_device_name(dev), "peak_memory_gb": torch.cuda.max_memory_allocated(dev) / 1e9,
                "gpu_launches": launches, "host_enqueue_ms_per_step": host_ms, "clocks": clocks, "roofline": roof, "voxelize": vox, "cpu_baseline": cpu}
        print(json.dumps(line))
        if world > 1 and nccl_log and os.path.exists(nccl_log):
            with open(nccl_log) as fh:
                comm = [ln.strip() for ln in fh if "nranks" in ln or "NVLS" in ln][:6]
            for ln in comm:
                print(ln, file=sys.stderr)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def traffic_from_profile(kernel_prefixes, path=None):
    """DRAM bytes per launch (dram__bytes_read.sum + dram__bytes_write.sum) of a kernel family, from the committed ncu
    launch list of one training step of the nuScenes bench config (profiles/launches_r2_summary.txt, produced by
    tools/ncu_round2.sh + tools/launch_summary.py).  None when the file is absent."""
    path = path or os.path.join(ROOT, "profiles", "launches_r2_summary.txt")
    if not os.path.exists(path):
        return None
    tot, n = 0.0, 0
    with open(path) as fh:
        for ln in fh:
            f = ln.split()
            if ln.startswith("#") or len(f) < 7:
                continue
            name = " ".join(f[6:])
            if any(k in name for k in kernel_prefixes):
                tot += (float(f[3]) + float(f[4])) * 1e6
                n += int(f[2])
    return {"bytes_per_launch": tot / n, "launches": n, "source": os.path.relpath(path, ROOT)} if n else None


def voxelize_roofline(dev, sel, pk):
    """Index-generation voxelizer (pnx_voxelize: V1-V2) swept over frames per launch on the selected config's point
    clouds.  Algorithmic bytes (SURVEY 8d): 24*N + 4*Nv + 12*P; the headline entry is the largest launch (>= 64 MB of
    algorithmic bytes, input larger than the 50 MB L2 so every timed iteration streams from HBM)."""
    from pillarnext_b200 import ops, synth
    cfg, n = sel["cfg"], sel["points"]
    nbase = 16 if n <= 60000 else 4
    base = [synth.make_frame(5000 + i, n, cfg, "lidar", sweeps=sel["sweeps"], rings=sel["rings"]) for i in range(nbase)]
    sweep = []
    tiled = None
    for total in (480000, 1920000, 7680000):
        frames = max(1, total // n)
        pts = synth.collate_points([base[i % nbase] for i in range(frames)]).to(dev)
        v = ops.voxelize(pts, frames, cfg["voxel_size"], cfg["pc_range"], buckets=False)
        tiled = v.status is not None
        P = int(v.counts[0].item())
        Nv = int((v.pillar_of_point[:pts.shape[0]] >= 0).sum().item())
        for _ in range(3):
            ops.voxelize(pts, frames, cfg["voxel_size"], cfg["pc_range"], buckets=False)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = 10
        t0.record()
        for _ in range(reps):
            ops.voxelize(pts, frames, cfg["voxel_size"], cfg["pc_range"], buckets=False)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / reps
        alg = 24.0 * pts.shape[0] + 4.0 * Nv + 12.0 * P
        sweep.append({"frames_per_launch": frames, "points": int(pts.shape[0]), "pillars": P, "algorithmic_bytes": alg, "ms": ms, "kernels": "frame-tiled" if tiled else "global-bitmap",
                      "achieved": alg / (ms * 1e-3) / 1e9, "frac": alg / (ms * 1e-3) / 1e9 / pk["hbm"]})
        if total == 7680000 and ops.lib().pnx_voxelize_frames_supported(frames, *[int(x) for x in ops.grid_size_xy(cfg["voxel_size"], cfg["pc_range"])]):
            # the alternative design (bitmap slices in shared memory), for the record: bit-exact, measured slower
            f = lambda: ops.voxelize(pts, frames, cfg["voxel_size"], cfg["pc_range"], buckets=False, frame_sorted="force")
            f().check_order()
            for _ in range(2):
                f()
            torch.cuda.synchronize()
            t0.record()
            for _ in range(reps):
                f()
            t1.record()
            torch.cuda.synchronize()
            sweep[-1]["frame_tiled_ms"] = t0.elapsed_time(t1) / reps
        del pts, v
    best = sweep[-1]
    return {"bound": "hbm", "kernel": "pnx_voxelize", "achieved": best["achieved"], "peak": pk["hbm"],
            "unit": "GB/s", "frac": best["frac"], "peak_source": pk["src"], "sweep": sweep,
            "note": "index generation (pillar id per point + sorted-unique coords); bytes = 24*N + 4*Nv + 12*P; the largest launch reads "
                    "%.0f MB of points (> L2), back-to-back launches, CUDA events" % (24.0 * best["points"] / 1e6)}


if __name__ == "__main__":
    main()
