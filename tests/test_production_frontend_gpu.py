"""The front end of a production training step -- voxelizer, PillarFeatureNet (PFN), sparse rulebook, densify, weight
repack, label assignment and the IoU target -- checked at the configuration the bench runs, against exact or float64
references.

One bf16 training step (the bench's end-to-end arm: raw ground truth, labels assigned on the GPU) of each bench config
(`nusc` 6 x 30k points, `waymo180k` 3 x 180k, `waymo540k` 3 x 540k multi-sweep) runs with ops.voxelize, pfn_forward,
pfn_backward, level_dilate, nbr_table, scatter_dense, pack_weights, assign_labels and aligned_iou3d
wrapped through pytest's MonkeyPatch: each call passes through unchanged and its device inputs and outputs are kept (the
Voxels, the Levels, the neighbour tables, the dfeat the backbone sends back, clones of the PFN parameters before the
step).  Frame 0 of every config carries an injected hot pillar (HOT_POINTS points plus HOT_DUPS exact duplicates), so one
bucket spans several 256-point CTA tiles of the PFN backward.  After the step a fused AdamW step runs and every cached
bf16 weight operand is rewritten by pnx_pack_weights.  The configs are recorded one after another and each model is
freed before the next, so the peak memory is that of one bench step plus what is kept.  The library handle is also
replaced by a proxy that notes every pnx_* entry point called (test_every_front_end_entry_point_is_covered).

What is compared:
- voxelizer: coords, pillar_of_point, P, Nv, the CSR buckets, the occupancy bitmap, inblk and blockpref bit for bit
  against oracle.pillarnext_oracle.voxelize, a plain occupancy grid and numpy prefix sums; the bench's roofline launches
  (480k / 1.92M / 7.68M points) through both kernel families, bit for bit with each other, the largest one against a numpy
  unique reference.
- PFN forward / backward: against a float64 evaluation on the GPU, within bounds k u sum|terms| (u = 2^-24) computed from
  the data, with k from the kernels' accumulation lengths (see _pfn_forward_ref and _pfn_backward_ref).
- rulebook and densify: bitmaps, counts, coords, inblk / blockpref, the forward, transposed and submanifold neighbour
  tables and scatter_dense / its gather, exactly, against max_pool2d / nonzero / a vectorised brute force / index_put.
- weight repack: bit for bit against WLayout.pack_fwd / pack_dgrad.
- label assignment and the aligned IoU: against synth.assign_labels and ops.aligned_iou3d_host with the tolerances of
  tests/test_assign_gpu.py and tests/test_iou_loss_gpu.py."""
import time
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import pillarnext_oracle as O
from pillarnext_b200 import _lib, modules, ops, synth
from pillarnext_b200 import functional as Fn

pytestmark = pytest.mark.gpu

CONFIGS = ("nusc", "waymo180k", "waymo540k")
U = 2.0 ** -24
HOT_POINTS, HOT_DUPS = 4000, 1000
ROOFLINE_TOTALS = (480000, 1920000, 7680000)       # bench.py voxelize_roofline
BIG = 2 ** 62

# Entry points the front end of the step calls, and the test here that checks each one.
COVERED = {
    "pnx_voxelize": "test_voxelizer_bit_exact_at_bench_shapes, test_voxelizer_roofline_launches",
    "pnx_voxelize_frames": "test_voxelizer_roofline_launches (frame_sorted='force')",
    "pnx_bucketize": "test_voxelizer_bit_exact_at_bench_shapes (CSR buckets)",
    "pnx_pfn_mean": "test_pfn_forward_matches_float64 (decoration through the mean)",
    "pnx_pfn_lin0": "test_pfn_forward_matches_float64",
    "pnx_pfn_max0": "test_pfn_forward_matches_float64",
    "pnx_pfn_lin1": "test_pfn_forward_matches_float64",
    "pnx_pfn_max1": "test_pfn_forward_matches_float64",
    "pnx_pfn_backward": "test_pfn_backward_matches_float64",
    "pnx_sites_dilate": "test_rulebook_and_densify_exact",
    "pnx_scan_blocks": "test_rulebook_and_densify_exact (blockpref)",
    "pnx_sites_coords": "test_rulebook_and_densify_exact",
    "pnx_nbr_table": "test_rulebook_and_densify_exact",
    "pnx_scatter_dense": "test_rulebook_and_densify_exact",
    "pnx_pack_weights": "test_weight_repack_bit_exact",
    "pnx_assign_labels": "test_assign_labels_at_e2e_shapes",
    "pnx_aligned_iou3d": "test_aligned_iou3d_at_loss_shapes",
}
# Host-side queries the front end makes: they launch nothing.
NO_LAUNCH = {"pnx_voxelize_bitmap_words", "pnx_voxelize_frames_supported", "pnx_voxelize_frames_scratch",
             "pnx_blockcnt_size", "pnx_sites_out_dim"}


# ------------------------------------------------------------------------------------------------- recording
def _hot_pillar(cfg, frame):
    """HOT_POINTS points inside one pillar of `frame` plus HOT_DUPS exact copies of some of them ([n, 6] fp32)."""
    g = np.random.default_rng(11)
    vs, pr = cfg["voxel_size"], cfg["pc_range"]
    gx, gy = (int(x) for x in ops.grid_size_xy(vs, pr)[:2])
    ix, iy = gx // 2 + 37, gy // 2 - 29
    u = g.uniform(0.1, 0.9, size=(HOT_POINTS, 2))
    p = np.stack([pr[0] + (ix + u[:, 0]) * vs[0], pr[1] + (iy + u[:, 1]) * vs[1], g.uniform(-1.5, 0.5, HOT_POINTS),
                  g.uniform(0, cfg["intensity_max"], HOT_POINTS), np.zeros(HOT_POINTS)], 1)
    p = np.concatenate([p, p[g.choice(HOT_POINTS, HOT_DUPS, replace=False)]]).astype(np.float32)
    return F.pad(torch.from_numpy(p), (1, 0), value=float(frame))


def _bench_example(name):
    """The bench's first end-to-end batch of config `name` (rank 0: frame seeds 0 .. B-1), with the hot pillar appended
    to frame 0 (the points stay grouped by frame)."""
    sel = synth.BENCH_CONFIGS[name]
    cfg = sel["cfg"]
    seeds = list(range(cfg["frames_per_gpu"]))
    ex = synth.make_batch(seeds, sel["points"], cfg, kind="lidar", n_boxes=40, sweeps=sel["sweeps"], rings=sel["rings"],
                          with_labels=False)
    pts = ex["points"]
    n0 = int((pts[:, 0] == 0).sum())
    pts = torch.cat([pts[:n0], _hot_pillar(cfg, 0), pts[n0:]])
    gt_b, gt_c = synth.make_gt_batch(seeds, 40, cfg)
    return {"points": pts, "token": ex["token"], "gt_boxes_raw": gt_b, "gt_classes": gt_c}


class Recorder:
    def __init__(self, real):
        self.real, self.called, self.cur = real, set(), None

    def proxy(self):
        rec = self

        class Proxy:
            def __getattr__(self, name):
                if name.startswith("pnx_"):
                    rec.called.add(name)
                return getattr(rec.real, name)
        return Proxy()


def _clone(t):
    return t.detach().clone() if torch.is_tensor(t) else t


def _wrappers(rec):
    """name -> wrapper of ops.<name> that keeps what the checks need in rec.cur (the config being recorded)."""
    real = {n: getattr(ops, n) for n in ("voxelize", "pfn_forward", "pfn_backward", "level_dilate", "nbr_table",
                                         "scatter_dense", "pack_weights", "assign_labels", "aligned_iou3d")}

    def voxelize(*a, **kw):
        v = real["voxelize"](*a, **kw)
        rec.cur.vox.append((a, kw, v))
        return v

    def pfn_forward(v, w0, bn0, w1, bn1, training, eps=1e-3, momentum=0.01, **kw):
        prm = dict(w0=w0, g0=bn0[0], b0=bn0[1], rm0=bn0[2], rv0=bn0[3], w1=w1, g1=bn1[0], b1=bn1[1], rm1=bn1[2], rv1=bn1[3])
        prm = {k: _clone(t) for k, t in prm.items()}
        fwd = real["pfn_forward"](v, w0, bn0, w1, bn1, training, eps=eps, momentum=momentum, **kw)
        rec.cur.pfn = types.SimpleNamespace(v=v, prm=prm, fwd=fwd, eps=eps, momentum=momentum, training=training,
                                            rm0=_clone(bn0[2]), rv0=_clone(bn0[3]), rm1=_clone(bn1[2]), rv1=_clone(bn1[3]))
        return fwd

    def pfn_backward(v, fwd, dfeat, w1, gamma0, gamma1):
        out = real["pfn_backward"](v, fwd, dfeat, w1, gamma0, gamma1)
        rec.cur.pfn.dfeat = dfeat.clone()
        rec.cur.pfn.grads = [t.clone() for t in out]
        return out

    def level_dilate(src, stride):
        lv = real["level_dilate"](src, stride)
        rec.cur.dilate.append((src, stride, lv))
        return lv

    def nbr_table(dst, src, stride, transposed):
        nbr = real["nbr_table"](dst, src, stride, transposed)
        rec.cur.nbr.append((dst, src, stride, transposed, nbr))
        return nbr

    def scatter_dense(feat, lv, channels, canvas=None, gather=False):
        out = real["scatter_dense"](feat, lv, channels, canvas=canvas, gather=gather)
        rec.cur.dense.append((lv, channels, gather, feat.clone(), out.clone()))     # gather: feat is the output
        return out

    def pack_weights(table, n, total):
        rec.cur.packs.append(int(n))
        return real["pack_weights"](table, n, total)

    def assign_labels(gt_boxes, gt_cls, tasks, voxel_size, pc_range, out_size_factor, **kw):
        out = real["assign_labels"](gt_boxes, gt_cls, tasks, voxel_size, pc_range, out_size_factor, **kw)
        rec.cur.assign.append((gt_boxes.clone(), gt_cls.clone(), tasks, voxel_size, pc_range, out_size_factor, kw, out))
        return out

    def aligned_iou3d(a, b):
        out = real["aligned_iou3d"](a, b)
        rec.cur.iou.append((a.detach().clone(), b.detach().clone(), out.clone()))
        return out
    return dict(voxelize=voxelize, pfn_forward=pfn_forward, pfn_backward=pfn_backward, level_dilate=level_dilate,
                nbr_table=nbr_table, scatter_dense=scatter_dense, pack_weights=pack_weights, assign_labels=assign_labels,
                aligned_iou3d=aligned_iou3d)


def _record(rec, name, dev):
    sel = synth.BENCH_CONFIGS[name]
    cfg = sel["cfg"]
    r = types.SimpleNamespace(name=name, cfg=cfg, vox=[], pfn=None, dilate=[], nbr=[], dense=[], packs=[], assign=[],
                              iou=[], pack_entries=None, pack_step_entries=None)
    rec.cur = r
    ex = _bench_example(name)
    ex = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in ex.items()}
    torch.manual_seed(0)
    model = modules.build_pillarnext_b(cfg).to(dev).train()
    opt = torch.optim.AdamW(list(model.parameters()), lr=1e-4, betas=(0.9, 0.99), weight_decay=0.01, fused=True)
    loss, _ = model(ex)
    loss.backward()
    torch.cuda.synchronize()
    r.pack_step_entries = _pack_entries()
    opt.step()
    opt.zero_grad(set_to_none=True)
    r.packs = []
    Fn._repack_all(torch.device(dev))                   # what the next step's first packed() call does
    torch.cuda.synchronize()
    r.pack_entries = _pack_entries()
    r.step_peak = torch.cuda.max_memory_allocated()
    del model, opt, loss, ex
    torch.cuda.empty_cache()
    return r


def _pack_entries():
    """(kind, which, flip, fp32 weight, cached bf16 operand) of every non-split cached operand of a live parameter."""
    out = []
    for k, e in list(Fn._pack_cache.items()):
        w = e[1]()
        if w is None or w.data_ptr() != e[3] or k[4] != 0:
            continue
        out.append((k[3], k[1], k[2], w.detach().clone(), e[2].clone()))
    return out


T0 = {}


@pytest.fixture(scope="module")
def steps():
    T0["t"] = time.perf_counter()
    dev = "cuda:%d" % torch.cuda.current_device()
    torch.cuda.reset_peak_memory_stats()
    rec = Recorder(_lib.lib())
    prev = Fn.set_precision("bf16"), ops.set_deterministic(False)      # the production step
    out = {}
    with pytest.MonkeyPatch.context() as mp:
        proxy = rec.proxy()
        mp.setattr(_lib, "lib", lambda: proxy)
        mp.setattr(ops, "lib", lambda: proxy)
        for n, f in _wrappers(rec).items():
            mp.setattr(ops, n, f)
        try:
            for name in CONFIGS:
                out[name] = _record(rec, name, dev)
                print("\n%s: recorded, peak %.2f GB" % (name, out[name].step_peak / 2 ** 30))
        finally:
            Fn.set_precision(prev[0])
            ops.set_deterministic(prev[1])
    out["_called"] = rec.called
    return out


# ------------------------------------------------------------------------------------------------- helpers
def _worst(t):
    """Largest entry with NaN counted as +inf."""
    return t.double().nan_to_num(nan=float("inf")).max().item() if t.numel() else 0.0


def _ratio(err, bound):
    return _worst(err / (bound + 1e-300))


def _popcount(words):
    """Popcount of int32 words (numpy)."""
    return np.unpackbits(np.ascontiguousarray(words).view(np.uint8)).reshape(-1, 32).sum(1).astype(np.int64)


def _prefix_fails(bm, inblk, blockpref, what):
    """inblk (exclusive prefix of the word popcounts inside each 32-word block) and blockpref (exclusive prefix of the
    block totals, then the total) against numpy."""
    pc = _popcount(bm.cpu().numpy()).reshape(-1, 32)
    incl = np.cumsum(pc, 1)
    want_in = (incl - pc).reshape(-1)
    want_bp = np.concatenate([[0], np.cumsum(incl[:, -1])])
    bad = []
    if not np.array_equal(inblk.cpu().numpy().astype(np.int64) & 0xFFFF, want_in):
        bad.append("%s: inblk differs from the numpy in-block prefix" % what)
    if not np.array_equal(blockpref[:len(want_bp)].cpu().numpy().astype(np.int64), want_bp):
        bad.append("%s: blockpref differs from the numpy block prefix" % what)
    return bad


def _mask_words(mask, nw):
    """The nw bitmap words (int32) of a [B, U, V] bool mask: bit v % 32 of word (b U + u) ceil(V / 32) + v / 32, every
    other bit and word zero."""
    B, Uu, V = mask.shape
    vw = (V + 31) // 32
    assert nw >= (B * Uu * vw + 31) // 32 * 32 and nw % 32 == 0, nw
    b, u, v = torch.nonzero(mask, as_tuple=True)
    w = torch.zeros(nw, dtype=torch.int64, device=mask.device)
    w.index_add_(0, (b * Uu + u) * vw + v // 32, torch.ones_like(v) << (v % 32))   # distinct bits: the sum is the OR
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


# ------------------------------------------------------------------------------------------------- voxelizer
def _oracle(r):
    """oracle.pillarnext_oracle.voxelize of the step's points (cached on the record)."""
    if getattr(r, "oracle", None) is None:
        r.oracle = O.voxelize(r.vox[0][2].points.cpu(), r.cfg["voxel_size"], r.cfg["pc_range"])
    return r.oracle


def _vox_fails(v, ref):
    """Failures of one voxelizer result against the oracle, the occupancy grid and the numpy prefixes; the bucket sizes."""
    P, Nv = v.sync_counts()
    bad = []
    if P != ref["coords"].shape[0] or Nv != int(ref["keep"].sum()):
        return ["P / Nv %d / %d, oracle %d / %d" % (P, Nv, ref["coords"].shape[0], int(ref["keep"].sum()))], None
    dev = v.coords.device
    rc = ref["coords"].to(dev)
    if not torch.equal(v.coords[:P], rc):
        bad.append("pillar coords differ from the oracle")
    pop_ref = ref["pillar_of_point"].to(dev)
    if not torch.equal(v.pillar_of_point[:v.n].long(), pop_ref):
        bad.append("pillar_of_point differs from the oracle")
    off = v.bucket_off[:P + 1].long()
    bp = v.bucket_pts[:Nv].long()
    sizes = off[1:] - off[:-1]
    if off[0] != 0 or off[-1] != Nv or bool((sizes <= 0).any()):
        bad.append("bucket offsets are not a partition of the Nv kept points")
    else:
        seg = torch.repeat_interleave(torch.arange(P, device=dev), sizes)
        if not torch.equal(pop_ref[bp], seg):
            bad.append("a bucket holds a point of another pillar")
        same = seg[1:] == seg[:-1]
        if not bool((bp[1:][same] > bp[:-1][same]).all()):
            bad.append("point ids inside a bucket are not ascending")
        if not torch.equal(torch.sort(bp)[0], torch.nonzero(ref["keep"]).flatten().to(dev)):
            bad.append("the buckets do not hold every kept point exactly once")
    occ = torch.zeros(v.batch, v.gx, v.gy, dtype=torch.bool, device=dev)
    occ[rc[:, 0].long(), rc[:, 2].long(), rc[:, 1].long()] = True
    if not torch.equal(v.bitmap, _mask_words(occ, v.bitmap.numel())):
        bad.append("occupancy bitmap differs from the plain grid")
    bad += _prefix_fails(v.bitmap, v.inblk, v.blockpref, "voxelizer")
    return bad, sizes


def test_voxelizer_bit_exact_at_bench_shapes(steps):
    """The step's own voxelizer call of each config (bench points plus the hot pillar), bit for bit."""
    failures = []
    for name in CONFIGS:
        r = steps[name]
        assert len(r.vox) == 1, "the step voxelized %d times" % len(r.vox)
        (a, kw, v) = r.vox[0]
        bad, sizes = _vox_fails(v, _oracle(r))
        biggest = int(sizes.max()) if sizes is not None else -1
        print("%-9s N %d  P %d  Nv %d  largest bucket %d points  %s" % (name, v.n, v.P, v.Nv, biggest, bad or "bit-exact"))
        failures += ["%s: %s" % (name, b) for b in bad]
        assert biggest > 3 * 256, "%s: largest bucket %d does not span several 256-point PFN backward tiles" % (name, biggest)
    assert not failures, "\n".join(failures)


def _numpy_voxelize(pts, cfg):
    """(coords (b, y, x) int32 in (b, x, y) order, pillar_of_point) by np.unique of the cell key: the reference's fp32
    arithmetic (pillar_encoder.py:95-110)."""
    vs = np.asarray(cfg["voxel_size"], dtype=np.float32)
    lo = np.asarray(cfg["pc_range"][:3], dtype=np.float32)
    gx, gy = (int(x) for x in ops.grid_size_xy(cfg["voxel_size"], cfg["pc_range"])[:2])
    pc = (pts[:, 1:4] - lo) / vs
    keep = (pc[:, 0] >= 0) & (pc[:, 0] < gx) & (pc[:, 1] >= 0) & (pc[:, 1] < gy)
    xi, yi = pc[keep, 0].astype(np.int64), pc[keep, 1].astype(np.int64)
    b = pts[keep, 0].astype(np.int64)
    key = (b * gx + xi) * gy + yi
    uniq, inv = np.unique(key, return_inverse=True)
    coords = np.stack([uniq // (gx * gy), uniq % gy, (uniq // gy) % gx], 1).astype(np.int32)
    pop = np.full(pts.shape[0], -1, dtype=np.int64)
    pop[keep] = inv.reshape(-1)
    return coords, pop


def test_voxelizer_roofline_launches(steps):
    """bench.py's voxelize_roofline launches (the config's base clouds concatenated to 480k / 1.92M / 7.68M points) through
    the global-bitmap and the frame-tiled kernels: bit for bit with each other, the largest against numpy."""
    failures = []
    dev = "cuda"
    for name in CONFIGS:
        sel = synth.BENCH_CONFIGS[name]
        cfg, n = sel["cfg"], sel["points"]
        nbase = 16 if n <= 60000 else 4
        base = [synth.make_frame(5000 + i, n, cfg, "lidar", sweeps=sel["sweeps"], rings=sel["rings"]) for i in range(nbase)]
        gx, gy = (int(x) for x in ops.grid_size_xy(cfg["voxel_size"], cfg["pc_range"])[:2])
        for total in ROOFLINE_TOTALS:
            frames = max(1, total // n)
            pts = synth.collate_points([base[i % nbase] for i in range(frames)])
            pd = pts.to(dev)
            a = ops.voxelize(pd, frames, cfg["voxel_size"], cfg["pc_range"])
            b = ops.voxelize(pd, frames, cfg["voxel_size"], cfg["pc_range"], frame_sorted="force")
            tiled = b.status is not None
            if ops.voxelize_frames_supported(frames, gx, gy) and not tiled:
                failures.append("%s %d frames: the frame-tiled kernels did not run" % (name, frames))
            b.check_order()
            pa, pb = a.sync_counts(), b.sync_counts()
            P = pa[0]
            same = (pa == pb and torch.equal(a.coords[:P], b.coords[:P]) and torch.equal(a.pillar_of_point, b.pillar_of_point)
                    and torch.equal(a.bitmap, b.bitmap) and torch.equal(a.inblk, b.inblk)
                    and torch.equal(a.blockpref, b.blockpref) and torch.equal(a.bucket_off[:P + 1], b.bucket_off[:P + 1])
                    and torch.equal(a.bucket_pts[:pa[1]], b.bucket_pts[:pb[1]]))
            note = "kernel families bit-identical" if same else "FAIL: kernel families differ"
            if not same:
                failures.append("%s %d frames: the frame-tiled result differs from the global-bitmap one" % (name, frames))
            bad = _prefix_fails(a.bitmap, a.inblk, a.blockpref, "%s %d frames" % (name, frames))
            if total == ROOFLINE_TOTALS[-1]:
                coords, pop = _numpy_voxelize(pts.numpy(), cfg)
                if P != coords.shape[0] or not np.array_equal(a.coords[:P].cpu().numpy(), coords):
                    bad.append("%s %d frames: coords differ from numpy unique" % (name, frames))
                if not np.array_equal(a.pillar_of_point[:a.n].cpu().numpy().astype(np.int64), pop):
                    bad.append("%s %d frames: pillar_of_point differs from numpy unique" % (name, frames))
                note += ", numpy unique reference matched" if not bad else ""
            failures += bad
            print("%-9s %3d frames %8d points P %8d (%s): %s" % (name, frames, pts.shape[0], P,
                                                                "frame-tiled" if tiled else "global only", note))
            del a, b, pd
        torch.cuda.empty_cache()
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------- PFN
def _pfn_inputs(p):
    """Per-point quantities in bucket order (q = position in bucket_pts): the decorated features in fp64, the pillar of each
    point, and the first-order bound e_dec of the kernel's fp32 decoration error."""
    v = p.v
    P, Nv = v.sync_counts()
    dev = v.points.device
    off = v.bucket_off[:P + 1].long()
    n_p = (off[1:] - off[:-1]).double()
    pid = torch.repeat_interleave(torch.arange(P, device=dev), off[1:] - off[:-1])
    X = v.points[v.bucket_pts[:Nv].long()].double()
    xyz = X[:, 1:4]
    mean = torch.zeros(P, 3, dtype=torch.float64, device=dev).index_add_(0, pid, xyz) / n_p[:, None]
    amean = torch.zeros(P, 3, dtype=torch.float64, device=dev).index_add_(0, pid, xyz.abs()) / n_p[:, None]
    vs = torch.tensor([v.vs_x, v.vs_y], dtype=torch.float64, device=dev)
    lo = torch.tensor([v.min_x, v.min_y], dtype=torch.float64, device=dev)
    cell = v.coords[:P][:, [2, 1]].double() * vs
    center = cell + vs / 2 + lo
    fcl = xyz - mean[pid]
    fce = X[:, 1:3] - center[pid]
    dec = torch.cat([X[:, 1:6], fcl, fce], 1)
    # pfn_mean: an in-order fp32 sum of n points, then a division: |err| <= (n - 1) u mean|x| + u |mean|; the subtraction
    # adds u |f|.  The cell centre: three fp32 roundings of magnitude <= |cell| + vs + |lo|, then u |f|.
    em = U * ((n_p[:, None] - 1) * amean + mean.abs())
    e_dec = torch.cat([torch.zeros_like(X[:, 1:6]), em[pid] + U * fcl.abs(),
                       3 * U * (cell.abs() + vs + lo.abs())[pid] + U * fce.abs()], 1)
    return types.SimpleNamespace(P=P, Nv=Nv, pid=pid, n_p=n_p, dec=dec, e_dec=e_dec, dev=dev)


def _amax(x, pid, P):
    return torch.zeros(P, x.shape[1], dtype=x.dtype, device=x.device).scatter_reduce(
        0, pid[:, None].expand_as(x), x, "amax", include_self=False)


def _pfn_forward_ref(p, d):
    """float64 PFN forward with the BatchNorm affine the kernels applied (sc, sh), and the first-order bound of each kernel
    output.  lin0: 10 fp32 fma per output, |err| <= 11 u sum_k |w0_ok dec_k| (gamma_10 < 11 u) plus the decoration
    error through |W0|; lin1: 64 fp32 fma per output, <= 65 u sum_k |w1_ok in_k| plus the layer-0 error through |W1|.
    The BatchNorm affine is one fmaf (u |result|) and max / ReLU are 1-Lipschitz, so a pillar's bound is the largest
    bound of its points."""
    f = p.fwd
    W0, W1 = p.prm["w0"].double(), p.prm["w1"].double()
    sc0, sh0, sc1, sh1 = (f[k].double() for k in ("sc0", "sh0", "sc1", "sh1"))
    y0 = d.dec @ W0.t()
    e_y0 = 11 * U * (d.dec.abs() @ W0.abs().t()) + d.e_dec @ W0.abs().t()
    pre0 = y0 * sc0 + sh0
    h0 = pre0.clamp(min=0)
    e_h0 = sc0.abs() * e_y0 + U * pre0.abs()
    x0m, e_x0m = _amax(h0, d.pid, d.P), _amax(e_h0, d.pid, d.P)
    inp = torch.cat([h0, x0m[d.pid]], 1)
    e_in = torch.cat([e_h0, e_x0m[d.pid]], 1)
    del pre0, e_h0
    y1 = inp @ W1.t()
    e_y1 = 65 * U * (inp.abs() @ W1.abs().t()) + e_in @ W1.abs().t()
    pre1 = y1 * sc1 + sh1
    feat = _amax(pre1.clamp(min=0), d.pid, d.P)
    e_feat = _amax(sc1.abs() * e_y1 + U * pre1.abs(), d.pid, d.P)
    return types.SimpleNamespace(y0=y0, e_y0=e_y0, x0m=x0m, e_x0m=e_x0m, inp=inp, e_in=e_in, y1=y1, e_y1=e_y1, feat=feat,
                                 e_feat=e_feat)


def _stat_check(y, e_y, mean_k, invstd_k, gamma, beta, sc_k, sh_k, rm0, rv0, rm_k, rv_k, eps, mom):
    """Batch statistics, running statistics and the BatchNorm affine of one PFN layer against fp64 on y (the fp64 layer
    output), within the bound of the kernel's sums: each thread's y (error e_y) squared in fp32 (u), summed over a warp in
    fp32 (5 levels), the warps' partials in fp64: |err(sum y)| <= 6 u sum|y| + sum e_y, |err(sum y^2)| <= 7 u sum y^2 +
    2 sum |y| e_y; the finalize and the fp32 stores add a few u of each quantity.  Returns (failures, notes, relative bound
    of invstd, absolute bounds of mean, scale and shift)."""
    N = y.shape[0]
    mu = y.mean(0)
    var = ((y - mu) ** 2).mean(0)
    d_mean = (6 * U * y.abs().sum(0) + e_y.sum(0)) / N + 2 * U * mu.abs()
    d_var = (7 * U * (y * y).sum(0) + 2 * (y.abs() * e_y).sum(0)) / N + 2 * mu.abs() * d_mean + 4 * U * (var + mu * mu)
    istd = 1 / torch.sqrt(var + eps)
    d_istd = istd * (0.5 * d_var / (var + eps) + 4 * U)
    g, b = gamma.double(), beta.double()
    sc, sh = g * istd, b - mu * g * istd
    d_sc = g.abs() * d_istd + 2 * U * sc.abs()
    d_sh = mu.abs() * d_sc + sc.abs() * d_mean + 4 * U * (b.abs() + (mu * sc).abs())
    rm = (1 - mom) * rm0.double() + mom * mu
    rv = (1 - mom) * rv0.double() + mom * var * N / (N - 1)
    d_rm = mom * d_mean + 4 * U * ((1 - mom) * rm0.double().abs() + mom * mu.abs())
    d_rv = mom * d_var * N / (N - 1) + 4 * U * ((1 - mom) * rv0.double().abs() + mom * var * N / (N - 1))
    checks = [("mean", mean_k, mu, d_mean), ("invstd", invstd_k, istd, d_istd), ("scale", sc_k, sc, d_sc),
              ("shift", sh_k, sh, d_sh), ("running_mean", rm_k, rm, d_rm), ("running_var", rv_k, rv, d_rv)]
    bad, notes = [], []
    for nm, got, want, bound in checks:
        r = _ratio((got.double() - want).abs(), bound)
        notes.append("%s %.2f" % (nm, r))
        if not r <= 1.0:
            bad.append("%s off by %.3g x its bound" % (nm, r))
    return bad, " ".join(notes), _worst(d_istd / istd), d_mean, d_sc, d_sh


def _routing(val_k, out_k, pid, P):
    """First point in bucket order whose kernel-side value relu(fmaf(y, sc, sh)) equals the pillar's kernel max (> 0):
    the arg-max the backward kernels route the gradient to (pfn_bwd_max1 / pfn_bwd_max0).  BIG where there is none."""
    q = torch.arange(val_k.shape[0], device=val_k.device)[:, None].expand_as(val_k)
    hit = (val_k == out_k[pid]) & (out_k[pid] > 0)
    pos = torch.where(hit, q, torch.full_like(q, BIG))
    return torch.full((P, val_k.shape[1]), BIG, dtype=torch.long, device=val_k.device).scatter_reduce(
        0, pid[:, None].expand_as(val_k), pos, "amin", include_self=True)


def _kernel_relu(y, sc, sh):
    return (y.double() * sc.double() + sh.double()).float().clamp(min=0)


def _pfn_backward_ref(p, d, fr, dfeat, stat):
    """float64 gradients of sum(feat * dfeat) with the kernels' discrete decisions (ReLU gates and first arg-max of each
    max, taken from the kernel's own fp32 forward values) and fp64 batch statistics, plus bounds.

    The weight gradients are sums over points of dy (x) input, accumulated per 256-point CTA tile in fp32 (fmaf: gamma_256
    <= 257 u of sum |dy input|) and across tiles in fp64: k = 257.  dy = A (g - sum g / N - xhat sum g xhat / N) is a
    handful of fp32 operations on terms of magnitude |A| (|g| + |sum g| / N + |xhat sum g xhat| / N) (8 u of that, plus the
    relative bound of the batch statistics from _stat_check, plus xhat's share of the forward error).  The layer-0
    gradient g0 comes from d_in = dy1 W1 (64 fma: 65 u sum |dy1 w1|) and, at the arg-max point, the in-order fp32 sum of
    the pillar's n x0max gradients (n u of their absolute sum)."""
    f = p.fwd
    P, Nv, pid = d.P, d.Nv, d.pid
    eps = p.eps
    val1 = _kernel_relu(f["y1"][:Nv], f["sc1"], f["sh1"])
    arg1 = _routing(val1, f["feat"][:P], pid, P)
    del val1
    val0 = _kernel_relu(f["y0"][:Nv], f["sc0"], f["sh0"])
    arg0 = _routing(val0, f["x0max"][:P], pid, P)
    gate0 = (val0 > 0).double()
    del val0
    lf = {k: p.prm[k].double().requires_grad_() for k in ("w0", "g0", "b0", "w1", "g1", "b1")}
    v1, c1 = arg1 < BIG, arg1.clamp(max=Nv - 1)
    v0, c0 = arg0 < BIG, arg0.clamp(max=Nv - 1)
    y0 = d.dec @ lf["w0"].t()
    mu0, var0 = y0.mean(0).detach(), y0.var(0, unbiased=False).detach()
    z0 = (y0 - y0.mean(0)) / torch.sqrt(y0.var(0, unbiased=False) + eps) * lf["g0"] + lf["b0"]
    z0.retain_grad()
    h0 = z0 * gate0
    x0m = h0.gather(0, c0) * v0
    inp = torch.cat([h0, x0m[pid]], 1)
    y1 = inp @ lf["w1"].t()
    mu1, var1 = y1.mean(0).detach(), y1.var(0, unbiased=False).detach()
    z1 = (y1 - y1.mean(0)) / torch.sqrt(y1.var(0, unbiased=False) + eps) * lf["g1"] + lf["b1"]
    z1.retain_grad()
    feat = z1.gather(0, c1) * v1
    (feat * dfeat[:P].double()).sum().backward()
    ref = {k: t.grad.detach() for k, t in lf.items()}
    g1, g0 = z1.grad.detach(), z0.grad.detach()
    inp = inp.detach()
    del z0, z1, h0, x0m, y0, y1, feat
    N = float(Nv)
    absW1 = p.prm["w1"].double().abs()

    def bn_terms(g, y, mu, var, gamma, e_y, rel_stat):
        istd = 1 / torch.sqrt(var + eps)
        xh = (y - mu) * istd
        A = gamma.double() * istd
        sg, sgx = g.sum(0), (g * xh).sum(0)
        mag = A.abs() * (g.abs() + sg.abs() / N + xh.abs() * sgx.abs() / N)
        e_dy = (8 * U + rel_stat) * mag + (A * sgx / N).abs() * istd * e_y
        return mag, e_dy, xh, istd

    rel1, rel0 = stat
    # fr (the forward reference) applied the kernel's BatchNorm-0 affine, this one the fp64 statistics: their difference
    # is within the affine's bound (d_sc0 |y0| + d_sh0) and joins the input and y1 errors
    ext = rel0[2] * fr.y0.abs() + rel0[3]
    ext = torch.cat([ext, _amax(ext, pid, P)[pid]], 1)
    e_in = fr.e_in + ext
    e_y1 = fr.e_y1 + ext @ absW1.t()
    del ext
    mag1, e_dy1, xh1, istd1 = bn_terms(g1, fr.y1, mu1, var1, p.prm["g1"], e_y1, rel1[0])
    b_w1 = 257 * U * (mag1.t() @ inp.abs()) + e_dy1.t() @ inp.abs() + mag1.t() @ e_in
    b_g1 = (g1.abs() * (istd1 * (e_y1 + rel1[1]) + xh1.abs() * (rel1[0] + 3 * U))).sum(0)
    b_b1 = U * g1.abs().sum(0)
    Dm = mag1 @ absW1                                            # |d_in| terms
    ED = 65 * U * Dm + e_dy1 @ absW1                             # error of d_in
    del mag1, e_dy1, xh1
    Dsum = torch.zeros(P, 32, dtype=torch.float64, device=d.dev).index_add_(0, pid, Dm[:, 32:])
    EDsum = torch.zeros(P, 32, dtype=torch.float64, device=d.dev).index_add_(0, pid, ED[:, 32:]) + d.n_p[:, None] * U * Dsum
    at_arg = (torch.arange(Nv, device=d.dev)[:, None] == c0[pid]) & v0[pid]
    e_g0 = gate0 * (ED[:, :32] + torch.where(at_arg, EDsum[pid], torch.zeros((), dtype=torch.float64, device=d.dev)))
    del Dm, ED, Dsum, EDsum, at_arg
    mag0, e_dy0, xh0, istd0 = bn_terms(g0, fr.y0, mu0, var0, p.prm["g0"], fr.e_y0, rel0[0])
    A0 = (p.prm["g0"].double() * istd0).abs()
    e_dy0 = e_dy0 + A0 * (e_g0 + e_g0.sum(0) / N + xh0.abs() * (e_g0 * xh0.abs()).sum(0) / N)
    b_w0 = 257 * U * (mag0.t() @ d.dec.abs()) + e_dy0.t() @ d.dec.abs() + mag0.t() @ d.e_dec
    b_g0 = (e_g0 * xh0.abs() + g0.abs() * (istd0 * (fr.e_y0 + rel0[1]) + xh0.abs() * (rel0[0] + 3 * U))).sum(0)
    b_b0 = e_g0.sum(0) + U * g0.abs().sum(0)
    bounds = dict(w0=b_w0, w1=b_w1, g0=b_g0, b0=b_b0, g1=b_g1, b1=b_b1)
    for k in bounds:                                             # the fp32 result
        bounds[k] = bounds[k] + U * ref[k].abs() + 1e-30
    return ref, bounds, types.SimpleNamespace(arg1=arg1, inp=inp, g1=g1, mu1=mu1, var1=var1)


_PFN = {}


def _pfn(steps, name):
    """Forward reference, statistics and backward references of config `name` (cached: one config at a time)."""
    if name in _PFN:
        return _PFN[name]
    _PFN.clear()
    torch.cuda.empty_cache()
    p = steps[name].pfn
    d = _pfn_inputs(p)
    fr = _pfn_forward_ref(p, d)
    f = p.fwd
    s0 = _stat_check(fr.y0, fr.e_y0, f["mean0"], f["invstd0"], p.prm["g0"], p.prm["b0"], f["sc0"], f["sh0"], p.prm["rm0"],
                     p.prm["rv0"], p.rm0, p.rv0, p.eps, p.momentum)
    s1 = _stat_check(fr.y1, fr.e_y1, f["mean1"], f["invstd1"], p.prm["g1"], p.prm["b1"], f["sc1"], f["sh1"], p.prm["rm1"],
                     p.prm["rv1"], p.rm1, p.rv1, p.eps, p.momentum)
    stat = (s1[2:], s0[2:])
    _PFN[name] = types.SimpleNamespace(p=p, d=d, fr=fr, s0=s0, s1=s1, stat=stat, bwd={})
    return _PFN[name]


def _bwd(c, which):
    """(kernel gradients, fp64 reference, bounds, extras) for dfeat = the recorded one or a seeded Gaussian."""
    if which in c.bwd:
        return c.bwd[which]
    c.bwd.clear()
    p = c.p
    if which == "recorded":
        dfeat, got = p.dfeat, p.grads
    else:
        gen = torch.Generator(device=p.dfeat.device).manual_seed(17)
        dfeat = torch.randn(p.dfeat.shape, generator=gen, device=p.dfeat.device)
        got = ops.pfn_backward(p.v, p.fwd, dfeat, p.prm["w1"], p.prm["g0"], p.prm["g1"])
    ref, bounds, ex = _pfn_backward_ref(p, c.d, c.fr, dfeat, c.stat)
    got = dict(zip(("w0", "w1", "g0", "b0", "g1", "b1"), got))
    c.bwd[which] = (got, ref, bounds, ex, dfeat)
    return c.bwd[which]


def test_pfn_forward_matches_float64(steps):
    """feat within its bound, feat_bf16 = round-to-nearest of feat, batch / running statistics and the BatchNorm affine."""
    failures = []
    for name in CONFIGS:
        c = _pfn(steps, name)
        f, P = c.p.fwd, c.d.P
        err = (f["feat"][:P].double() - c.fr.feat).abs()
        r = _ratio(err, c.fr.e_feat + 1e-30)
        bad = [] if r <= 1.0 else ["feat off by %.3g x its bound" % r]
        if not torch.equal(f["feat_bf16"][:P], f["feat"][:P].bfloat16()):
            bad.append("feat_bf16 is not the round-to-nearest of feat")
        bad += ["BN0 " + b for b in c.s0[0]] + ["BN1 " + b for b in c.s1[0]]
        print("%-9s P %d Nv %d largest bucket %d: feat max err %.2e, err/bound %.3f (bound max %.2e); BN0 err/bound %s; "
              "BN1 %s  %s" % (name, P, c.d.Nv, int(c.d.n_p.max()), _worst(err), r, _worst(c.fr.e_feat), c.s0[1], c.s1[1],
                             "ok" if not bad else "FAIL: " + "; ".join(bad)))
        failures += ["%s: %s" % (name, b) for b in bad]
    assert not failures, "\n".join(failures)


def _grad_fails(got, ref, bounds):
    bad, notes = [], []
    for k in ("w0", "w1", "g0", "b0", "g1", "b1"):
        r = _ratio((got[k].double() - ref[k]).abs(), bounds[k])
        notes.append("d%s %.1e" % (k, r))
        if not r <= 1.0:
            bad.append("d%s off by %.3g x its bound" % (k, r))
    return bad, " ".join(notes)


def test_pfn_backward_matches_float64(steps):
    """dW0, dW1, dgamma0/1, dbeta0/1 with the dfeat the backbone sent back and with a seeded Gaussian dfeat."""
    failures = []
    for name in CONFIGS:
        c = _pfn(steps, name)
        for which in ("recorded", "gaussian"):
            got, ref, bounds, _, _ = _bwd(c, which)
            bad, note = _grad_fails(got, ref, bounds)
            print("%-9s dfeat %-8s err/bound: %s  %s" % (name, which, note, "ok" if not bad else "FAIL: " + "; ".join(bad)))
            failures += ["%s %s dfeat: %s" % (name, which, b) for b in bad]
    assert not failures, "\n".join(failures)


def test_self_check_pfn_dw1_comparison_catches_a_dropped_cta_block(steps):
    """The dW1 comparison fails when the reference leaves out one 256-point CTA block of the backward (the block with the
    largest sum |dy1| |input|, one of about 700)."""
    name = CONFIGS[0]
    c = _pfn(steps, name)
    got, ref, bounds, ex, dfeat = _bwd(c, "recorded")
    assert not _grad_fails(got, ref, bounds)[0]
    # dy1 (fp64 BatchNorm backward of the routed dfeat); the share of dW1 of one CTA block of points taken out
    mu1, istd1 = ex.mu1, 1 / torch.sqrt(ex.var1 + c.p.eps)
    xh = (c.fr.y1 - mu1) * istd1
    N = float(c.d.Nv)
    g1 = ex.g1
    dy1 = c.p.prm["g1"].double() * istd1 * (g1 - g1.sum(0) / N - xh * (g1 * xh).sum(0) / N)
    share = torch.zeros(-(-c.d.Nv // 256), dtype=torch.float64, device=dy1.device).index_add_(
        0, torch.arange(c.d.Nv, device=dy1.device) // 256, dy1.abs().sum(1) * ex.inp.abs().sum(1))
    q0 = int(share.argmax()) * 256
    blk = slice(q0, min(q0 + 256, c.d.Nv))
    dropped = dict(ref, w1=ref["w1"] - dy1[blk].t() @ ex.inp[blk])
    bad, note = _grad_fails(got, dropped, bounds)
    print("%s: reference dW1 without points %d..%d: %s" % (name, blk.start, blk.stop, note))
    assert any(b.startswith("dw1") for b in bad), "a dW1 reference without one CTA block goes unnoticed"


# ------------------------------------------------------------------------------------------------- rulebook
def _unpack_mask(lv):
    vw = (lv.V + 31) // 32
    w = lv.bm[:lv.batch * lv.U * vw].long() & 0xFFFFFFFF
    bits = (w.view(lv.batch, lv.U, vw, 1) >> torch.arange(32, device=w.device)) & 1
    return bits.reshape(lv.batch, lv.U, vw * 32)[:, :, :lv.V].bool()


def _index_grid(mask):
    idx = torch.full(mask.shape, -1, dtype=torch.long, device=mask.device)
    idx[mask] = torch.arange(int(mask.sum()), device=mask.device)
    return idx


def _fwd_table(dc, idx_src, stride):
    """[n_dst, 9] brute-force table: row of the source site at (u s + ku - 1, v s + kv - 1), tap ku * 3 + kv, -1 absent."""
    B, Us, Vs = idx_src.shape
    exp = torch.full((dc.shape[0], 9), -1, dtype=torch.long, device=dc.device)
    for ku in range(3):
        for kv in range(3):
            u = dc[:, 1] * stride + ku - 1
            v = dc[:, 2] * stride + kv - 1
            ok = (u >= 0) & (u < Us) & (v >= 0) & (v < Vs)
            exp[ok, ku * 3 + kv] = idx_src[dc[ok, 0], u[ok], v[ok]]
    return exp


def _level_fails(lv, mask, what):
    """Bitmap (every word, padding included), count, coords and prefixes of one level against its mask."""
    bad = []
    if not torch.equal(lv.bm, _mask_words(mask, lv.bm.numel())):
        bad.append("%s: bitmap differs from the reference mask" % what)
    n = int(mask.sum())
    if int(lv.count.item()) != n or lv.n != n:
        bad.append("%s: count %d / n %s, reference %d" % (what, int(lv.count.item()), lv.n, n))
    elif not torch.equal(lv.coords[:n].long(), torch.nonzero(mask)):
        bad.append("%s: coords differ from nonzero(mask)" % what)
    bad += _prefix_fails(lv.bm, lv.inblk, lv.blockpref, what)
    return bad


def _pyramid(r):
    """Levels 0..4 of the recorded pyramid and their reference masks (level 0: the oracle's occupancy grid; level s + 1:
    max_pool2d(3, stride, 1) of level s)."""
    v = r.vox[0][2]
    lv0 = r.dilate[0][0]
    levels, strides = [lv0], []
    for src, stride, out in r.dilate:
        assert src is levels[-1], "dilations out of order"
        levels.append(out)
        strides.append(stride)
    ref = _oracle(r)["coords"].to(v.coords.device).long()
    m = torch.zeros(v.batch, v.gx, v.gy, dtype=torch.bool, device=v.coords.device)
    m[ref[:, 0], ref[:, 2], ref[:, 1]] = True
    masks = [m]
    for s in strides:
        masks.append(F.max_pool2d(masks[-1].float().unsqueeze(1), 3, s, 1)[:, 0] > 0)
    return levels, masks, strides


def _table_fails(r, levels, masks):
    """Every recorded neighbour table (forward, transposed, submanifold) against the brute force."""
    pos = {id(lv): i for i, lv in enumerate(levels)}
    bad, kinds = [], set()
    for dst, src, stride, transposed, nbr in r.nbr:
        i, j = pos[id(dst)], pos[id(src)]
        if transposed:                                   # rows: sites of the finer level i; entries: coarse level j
            kinds.add("transposed")
            fc = torch.nonzero(masks[j])
            fwd = _fwd_table(fc, _index_grid(masks[i]), stride)
            exp = torch.full((int(masks[i].sum()), 9), -1, dtype=torch.long, device=fwd.device)
            ii, tt = torch.nonzero(fwd >= 0, as_tuple=True)
            exp[fwd[ii, tt], tt] = ii
        else:
            kinds.add("submanifold" if i == j else "forward")
            exp = _fwd_table(torch.nonzero(masks[i]), _index_grid(masks[j]), stride)
        if not torch.equal(nbr[:exp.shape[0]].long(), exp):
            n = int((nbr[:exp.shape[0]].long() != exp).sum())
            bad.append("%s table level %d <- %d (stride %d): %d entries differ" % (
                "transposed" if transposed else "forward", i, j, stride, n))
    return bad, kinds


def _dense_fails(r, levels):
    bad = []
    for lv, C, gather, feat, canvas in r.dense:
        n = lv.n
        c = lv.coords[:n].long()
        if not gather:
            exp = torch.zeros(lv.batch, lv.V, lv.U, C, dtype=torch.bfloat16, device=feat.device)
            exp[c[:, 0], c[:, 2], c[:, 1]] = feat[:n]
            if not torch.equal(canvas, exp):
                bad.append("scatter_dense canvas differs from index_put (level %d x %d)" % (lv.U, lv.V))
            back = torch.empty_like(feat[:n])
            ops.scatter_dense(back, lv, C, canvas=canvas.clone(), gather=True)
            if not torch.equal(back, feat[:n]):
                bad.append("scatter / gather round trip differs (level %d x %d)" % (lv.U, lv.V))
        elif not torch.equal(feat[:n], canvas[c[:, 0], c[:, 2], c[:, 1]]):
            bad.append("scatter_dense gather differs from indexing the canvas (level %d x %d)" % (lv.U, lv.V))
    return bad


def test_rulebook_and_densify_exact(steps):
    failures, partial = [], []
    for name in CONFIGS:
        r = steps[name]
        levels, masks, strides = _pyramid(r)
        assert len(levels) == 5, "levels 0..4"
        bad = []
        for i, (lv, m) in enumerate(zip(levels, masks)):
            bad += _level_fails(lv, m, "level %d (%d x %d x %d)" % (i, lv.batch, lv.U, lv.V))
            if lv.V % 32:
                partial.append("%s level %d: V = %d, %d words per row" % (name, i, lv.V, (lv.V + 31) // 32))
        tb, kinds = _table_fails(r, levels, masks)
        bad += tb
        assert kinds == {"forward", "transposed", "submanifold"}, kinds
        bad += _dense_fails(r, levels)
        assert r.dense and any(g for _, _, g, _, _ in r.dense), "no densify forward and gather recorded"
        print("%-9s levels %s, sites %s, %d tables, %d densify calls: %s" % (
            name, " ".join("%dx%dx%d" % (lv.batch, lv.U, lv.V) for lv in levels), [lv.n for lv in levels], len(r.nbr),
            len(r.dense), "exact" if not bad else "FAIL: " + "; ".join(bad)))
        failures += ["%s: %s" % (name, b) for b in bad]
    print("levels ending their rows in a partially valid word: %d\n  %s" % (len(partial), "\n  ".join(partial)))
    assert len(partial) >= 8, partial
    assert not failures, "\n".join(failures)


def test_self_check_rulebook_comparisons_fail(steps):
    """One neighbour-table entry changed in the last frame of the last level, and two site coords swapped inside a 32-word
    block that straddles a row, each fail their comparison."""
    r = steps[CONFIGS[0]]
    levels, masks, _ = _pyramid(r)
    last = levels[-1]
    ent = [e for e in r.nbr if e[0] is last and not e[3]]
    dst, src, stride, transposed, nbr = ent[0]
    row = int((last.coords[:last.n, 0] == last.batch - 1).nonzero().max())
    t = int((nbr[row] >= 0).nonzero()[0])
    bad_nbr = nbr.clone()
    bad_nbr[row, t] += 1
    mod = types.SimpleNamespace(**vars(r))
    mod.nbr = [(dst, src, stride, transposed, bad_nbr)]
    tb, _ = _table_fails(mod, levels, masks)
    print("neighbour table with entry (%d, %d) changed: %s" % (row, t, tb))
    assert tb, "a changed neighbour-table entry goes unnoticed"
    # two consecutive sites of one 32-word block in different rows (u) of a level whose rows end in a partial word
    i = next(k for k, lv in enumerate(levels) if lv.V % 32)
    lv = levels[i]
    c = lv.coords[:lv.n].long()
    vw = (lv.V + 31) // 32
    blk = ((c[:, 0] * lv.U + c[:, 1]) * vw + c[:, 2] // 32) // 32
    k = int(((blk[1:] == blk[:-1]) & (c[1:, 1] != c[:-1, 1])).nonzero()[0])
    swapped = types.SimpleNamespace(**vars(lv))
    swapped.coords = lv.coords.clone()
    swapped.coords[[k, k + 1]] = lv.coords[[k + 1, k]]
    lb = _level_fails(swapped, masks[i], "level %d" % i)
    print("level %d coords %d and %d swapped (block %d, rows %d / %d): %s" % (i, k, k + 1, int(blk[k]), int(c[k, 1]),
                                                                            int(c[k + 1, 1]), lb))
    assert any("coords differ" in b for b in lb), "two swapped site coords go unnoticed"


# ------------------------------------------------------------------------------------------------- weight repack
def test_weight_repack_bit_exact(steps):
    """Every cached (weight, layout, which, flip) operand after the step (packed by torch) and after a fused AdamW step
    (rewritten by pnx_pack_weights, 256 entries per launch) equals WLayout.pack_fwd / pack_dgrad bit for bit."""
    failures = []
    for name in CONFIGS:
        r = steps[name]
        assert r.pack_entries and r.packs, "%s: no repack ran" % name
        assert sum(r.packs) == len(r.pack_entries) and len(r.packs) == -(-len(r.pack_entries) // 256), \
            (name, r.packs, len(r.pack_entries))
        for stage, entries in (("after the step", r.pack_step_entries), ("after AdamW", r.pack_entries)):
            n_bad = 0
            for kind, which, flip, w, pk in entries:
                lay = Fn.WLayout(kind)
                want = lay.pack_fwd(w) if which == "fwd" else lay.pack_dgrad(w, flip)
                if not torch.equal(pk, want):
                    n_bad += 1
                    failures.append("%s %s: %s %s flip=%s %s differs" % (name, stage, kind, which, flip, tuple(w.shape)))
            print("%-9s %-14s %d packed operands (%d pnx_pack_weights launches): %d differ" % (
                name, stage, len(entries), len(r.packs), n_bad))
        changed = sum(not torch.equal(a[3], b[3]) for a, b in zip(r.pack_step_entries, r.pack_entries))
        assert changed > 0, "AdamW changed no packed weight"
    assert not failures, "\n".join(failures[:20])


# ------------------------------------------------------------------------------------------------- labels and IoU
def _assign_fails(got, boxes, cls, cfg, max_objs, what):
    """pnx_assign_labels against synth.assign_labels: ind / mask / cat exact, hm 1e-6, anno_box 2e-6, gt_boxes exact."""
    names_all = [n for t in cfg["tasks"] for n in t]
    want = []
    for b in range(boxes.shape[0]):
        names = [names_all[c] if c >= 0 else "ignored_class" for c in cls[b].tolist()]
        want.append(synth.assign_labels(boxes[b].numpy(), names, cfg=cfg, max_objs=max_objs))
    bad = []
    for t in range(len(cfg["tasks"])):
        for key in ("ind", "mask", "cat"):
            w = torch.stack([torch.tensor(want[b][key][t]) for b in range(len(want))])
            if not torch.equal(got[key][t].cpu(), w):
                bad.append("%s task %d: %s differs" % (what, t, key))
        for key, tol in (("hm", 1e-6), ("anno_box", 2e-6), ("gt_boxes", 0.0)):
            w = torch.stack([torch.tensor(want[b][key][t]) for b in range(len(want))])
            g = got[key][t].cpu()
            d = torch.where(torch.isnan(g) & torch.isnan(w), torch.zeros_like(g), (g - w).abs())
            if g.shape != w.shape or not _worst(d) <= tol:
                bad.append("%s task %d: %s off by %.3g (tolerance %g)" % (what, t, key, _worst(d), tol))
    return bad, want


def test_assign_labels_at_e2e_shapes(steps):
    """The e2e arm's raw ground truth of each config, and one frame of 600 boxes of one class (past max_objs = 500)."""
    failures = []
    for name in CONFIGS:
        r = steps[name]
        assert len(r.assign) == 1
        boxes, cls, tasks, vs, pr, osf, kw, got = r.assign[0]
        bad, _ = _assign_fails(got, boxes.cpu(), cls.cpu(), r.cfg, kw["max_objs"], name + " e2e")
        n_pos = [int(m.sum()) for m in got["mask"]]
        cfg = r.cfg
        b600, _ = synth.make_gt(77, 600, cfg)
        b600 = torch.from_numpy(b600)[None]
        c600 = torch.zeros(1, 600, dtype=torch.int32)
        g600 = ops.assign_labels(b600.cuda(), c600.cuda(), cfg["tasks"], cfg["voxel_size"], cfg["pc_range"],
                                 cfg["out_size_factor"], **kw)
        b2, want = _assign_fails(g600, b600, c600, cfg, kw["max_objs"], name + " 600 boxes")
        bad += b2
        kept = int(g600["mask"][0].sum())
        if kept != kw["max_objs"] or int(want[0]["mask"][0].sum()) != kw["max_objs"]:
            bad.append("%s 600 boxes: %d objects kept, the reference truncates at %d" % (name, kept, kw["max_objs"]))
        print("%-9s e2e %d frames x %d boxes, positives per task %s; 600 boxes of one class -> %d kept: %s" % (
            name, boxes.shape[0], boxes.shape[1], n_pos, kept, "ok" if not bad else "FAIL: " + "; ".join(bad)))
        failures += bad
    assert not failures, "\n".join(failures)


def test_aligned_iou3d_at_loss_shapes(steps):
    """Every recorded aligned-IoU call (the `iou` head's target) against the host twin, 3e-6 absolute; the Waymo loss
    launches 3 frames x 500 slots."""
    failures, shapes = [], set()
    for name in CONFIGS:
        for a, b, out in steps[name].iou:
            shapes.add((name, a.shape[0]))
            want = torch.from_numpy(ops.aligned_iou3d_host(a.cpu().numpy(), b.cpu().numpy()))
            err = _worst((out.cpu() - want).abs())
            if not err < 3e-6:
                failures.append("%s n = %d: IoU off by %.3g" % (name, a.shape[0], err))
            print("%-9s aligned IoU n = %d: max err %.2e vs host twin" % (name, a.shape[0], err))
    assert any(n == "waymo540k" and k == 3 * 500 for n, k in shapes) and any(
        n == "waymo180k" and k == 3 * 500 for n, k in shapes), shapes
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------- completeness
def test_every_front_end_entry_point_is_covered(steps):
    """Every pnx_* entry point the three steps called is covered here, replayed by a sibling production test, or a host
    query that launches nothing."""
    from test_production_rowwise_gpu import ARG_MAPS, EXCLUDED, GEMM_REPLAYED
    called = steps["_called"]
    print("\nentry points called: %s" % ", ".join(sorted(called)))
    missing = sorted(n for n in called if n not in COVERED and n not in NO_LAUNCH and n not in ARG_MAPS
                     and n not in GEMM_REPLAYED and not ("launches nothing" in EXCLUDED.get(n, "")))
    assert not missing, "entry points the step calls that no production test covers: %s" % missing
    assert {n for n in COVERED if n != "pnx_voxelize_frames"} <= called, sorted(set(COVERED) - called)
    stale = sorted(n for n in COVERED if "test_production_frontend_gpu" not in EXCLUDED.get(n, ""))
    assert not stale, "EXCLUDED of tests/test_production_rowwise_gpu.py does not point these here: %s" % stale
    print("wall time of the file so far %.1f s, peak GPU memory %.2f GB" % (
        time.perf_counter() - T0["t"], torch.cuda.max_memory_allocated() / 2 ** 30))
