"""Thin host wrappers: torch device buffers + current stream -> libpnx C-ABI calls.

This module is the only caller of libpnx: every entry point, including the host twins (`*_host`: the CPU builds of
kernels, which take numpy arrays), is reached through a wrapper here.
torch is used here for device memory, streams and dtype plumbing only; all compute is in libpnx.
"""
import ctypes

import numpy as np
import torch

from ._lib import check, lib, ptr, sm_count, stream

# ---- instrumentation used by bench.py: kernel-launch counter and optional per-call CUDA-event timing
LAUNCHES = 0            # number of libpnx kernels launched so far (each wrapper adds its own kernel count)
PROFILE = None          # when a list: (kind, flops, bytes, start_event, end_event) per tensor-core GEMM call


def _count(n):
    global LAUNCHES
    LAUNCHES += n


# --------------------------------------------------------------------------------- operand checks
_NUMPY = {torch.float32: np.dtype(np.float32), torch.float64: np.dtype(np.float64), torch.int32: np.dtype(np.int32),
          torch.int64: np.dtype(np.int64)}


def _want(t, dtype, shape, what, host=False):
    """Check one operand of a libpnx call and return it C-contiguous.  A device entry point takes a CUDA tensor of
    `dtype`; a host twin (host=True) takes a numpy array of the same element type.  A wrong dtype or shape raises here
    instead of being read as garbage by the library."""
    if host:
        ok, kind = isinstance(t, np.ndarray) and t.dtype == _NUMPY[dtype], "a numpy %s array" % _NUMPY[dtype]
    else:
        ok, kind = isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype, "a CUDA %s tensor" % dtype
    if not ok or tuple(t.shape) != tuple(shape):
        raise ValueError("%s must be %s of shape %s, got %s %s %s" % (what, kind, tuple(shape), type(t).__name__,
                                                                    getattr(t, "dtype", None), tuple(getattr(t, "shape", ()))))
    return np.ascontiguousarray(t) if host else t.contiguous()


def _hp(a):
    """Address of a host twin's operand (a C-contiguous numpy array)."""
    return a.ctypes.data


class _Timed:
    def __init__(self, kind, flops, nbytes, tag=""):
        self.rec = None
        if PROFILE is not None:
            self.rec = [kind, flops, nbytes, torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True), tag]

    def __enter__(self):
        if self.rec is not None:
            self.rec[3].record()

    def __exit__(self, *a):
        if self.rec is not None:
            self.rec[4].record()
            PROFILE.append(tuple(self.rec))


# --------------------------------------------------------------------------------- per-step zero arena
class ZeroArena:
    """The small zero-initialised accumulators of one training step (BatchNorm statistics, reduction buffers, the fp32
    weight-gradient accumulators: ~130 tensors, ~45 MB) carved out of ONE buffer that is cleared by a single memset at
    the start of the step, instead of one fill kernel each.  Inactive (plain torch.zeros) until begin_step() is called;
    the views are only valid until the next begin_step()."""

    def __init__(self):
        self.buf, self.off, self.need, self.active = None, 0, 0, False

    def begin_step(self, device):
        cap = self.buf.numel() if self.buf is not None else 0
        want = max(self.need, self.off)
        if self.buf is None or self.buf.device != device or want > cap:
            self.buf = torch.empty(max(int(want * 1.25), 64 << 20), dtype=torch.uint8, device=device)
        self.buf.zero_()
        self.off, self.need, self.active = 0, 0, True

    def zeros(self, shape, dtype, device):
        n = 1
        for s in (shape if isinstance(shape, (tuple, list)) else (shape,)):
            n *= int(s)
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        if not self.active or self.buf is None or self.buf.device != device:
            return torch.zeros(shape, dtype=dtype, device=device)
        start = (self.off + 255) // 256 * 256
        self.need = max(self.need, start + nbytes)
        if start + nbytes > self.buf.numel():       # first step(s): grow at the next begin_step, plain allocation now
            self.off = start + nbytes
            return torch.zeros(shape, dtype=dtype, device=device)
        self.off = start + nbytes
        return self.buf[start:start + nbytes].view(dtype).view(shape)


ARENA = ZeroArena()


def zeros(shape, dtype, device):
    return ARENA.zeros(shape, dtype, device)


# --------------------------------------------------------------------------------- geometry
def grid_size_xy(voxel_size, pc_range):
    """Same float64 arithmetic as the reference (pillar_encoder.py:87-89)."""
    vs = np.array(voxel_size, dtype=np.float64)
    pr = np.array(pc_range, dtype=np.float64)
    g = (pr[3:] - pr[:3]) / vs
    return np.round(g).astype(np.int64)


def _f32(x):
    return float(np.float32(x))


class Voxels:
    """Result of the voxelizer: fixed-capacity device buffers + device counts {P, Nv}."""

    def __init__(self):
        self.P = None
        self.Nv = None

    def sync_counts(self):
        if self.P is None:
            if getattr(self, "status", None) is not None:
                c = torch.cat([self.counts, self.status]).cpu()
                self.check_order(c[2])
            else:
                c = self.counts.cpu()
            self.P, self.Nv = int(c[0]), int(c[1])
        return self.P, self.Nv

    def check_order(self, status_value=None):
        """Raise if the frame-tiled voxelizer found the points not grouped by frame (status_value: the already fetched
        host copy of self.status; fetched here, with a synchronisation, when omitted)."""
        if getattr(self, "status", None) is None:
            return
        bad = int(self.status.item()) if status_value is None else int(status_value)
        if bad:
            raise RuntimeError("pnx_voxelize_frames: %d point(s) lie outside their frame's range -- the points are not grouped "
                               "by ascending batch index; use voxelize(..., frame_sorted=False)" % bad)


# The frame-tiled kernels (pnx_voxelize_frames) are bit-exact with the global-bitmap ones, but every slice re-processes all
# points of its frame and its bitmap sweep costs as much as the points, so they only run on request
# (frame_sorted="force"; bench.py reports their time next to the production kernels); None = never chosen automatically.
FRAME_TILED_MIN_CTAS = None


def bitmap_words(batch, gx, gy):
    """Words of the occupancy bitmap of a batch x gx x gy grid, padded to whole 32-word blocks (pnx_voxelize_bitmap_words)."""
    return lib().pnx_voxelize_bitmap_words(batch, gx, gy)


def voxelize_frames_supported(batch, gx, gy):
    """CTAs the frame-tiled voxelizer (pnx_voxelize_frames) would launch for this geometry; 0 = not supported."""
    return lib().pnx_voxelize_frames_supported(batch, gx, gy)


def voxelize(points, batch, voxel_size, pc_range, buckets=True, frame_sorted=False):
    """V1-V2 index generation (pnx_voxelize) and, with buckets=True, the CSR grouping the PFN needs
    (pnx_bucketize). points [N,6] fp32 cuda (b,x,y,z,i,t).
    frame_sorted=True: the points are grouped by frame in ascending batch index (what collate produces) -> the
    frame-tiled kernels (pnx_voxelize_frames: bitmap slices in shared memory) MAY be used: "force" = whenever the geometry
    allows, True = when FRAME_TILED_MIN_CTAS says so (never, today: see there).  The order is verified on the device:
    `v.status` (int32 [1]) is non-zero when it did not hold and the outputs must be discarded -- check it at the next
    host synchronisation (Voxels.check_order(), modules.build_pyramid does) and re-run with frame_sorted=False."""
    assert points.is_cuda and points.dtype == torch.float32 and points.dim() == 2 and points.shape[1] == 6, \
        "points must be a CUDA float32 [N, 6] tensor (batch_idx, x, y, z, intensity, time)"
    points = points.contiguous()
    if points.data_ptr() % 16:
        points = points.clone()
    n = points.shape[0]
    g = grid_size_xy(voxel_size, pc_range)
    gx, gy = int(g[0]), int(g[1])
    dev = points.device
    L = lib()
    words = bitmap_words(batch, gx, gy)
    cap_p = min(n, batch * gx * gy)
    v = Voxels()
    v.points, v.n, v.batch, v.gx, v.gy, v.cap_p = points, n, batch, gx, gy, cap_p
    v.min_x, v.min_y = _f32(pc_range[0]), _f32(pc_range[1])
    v.vs_x, v.vs_y = _f32(voxel_size[0]), _f32(voxel_size[1])
    i32 = dict(dtype=torch.int32, device=dev)
    v.bitmap = torch.empty(words, **i32)
    v.blockcnt = torch.empty(L.pnx_blockcnt_size(words // 32), **i32)
    v.inblk = torch.empty(words, dtype=torch.int16, device=dev)
    v.blockpref = torch.empty(words // 32 + 1, **i32)
    cell = torch.empty(max(n, 1), **i32)
    v.pillar_of_point = torch.empty(max(n, 1), **i32)
    v.coords = torch.empty(max(cap_p, 1), 3, **i32)
    bucket_cnt = torch.empty(2 * (cap_p + 1), **i32) if buckets else None
    v.counts = torch.zeros(2, **i32)
    v.status = None
    n_cta = voxelize_frames_supported(batch, gx, gy) if (frame_sorted and n > 0) else 0
    if n_cta > 0 and (frame_sorted == "force" or (FRAME_TILED_MIN_CTAS is not None and n_cta >= FRAME_TILED_MIN_CTAS)):
        scratch = torch.empty(L.pnx_voxelize_frames_scratch(batch), **i32)
        v.status = scratch[0:1]
        _count(4)
        check(L.pnx_voxelize_frames(ptr(points), n, batch, v.min_x, v.min_y, v.vs_x, v.vs_y, gx, gy, ptr(v.bitmap), ptr(v.inblk),
                                    ptr(v.blockcnt), ptr(v.blockpref), ptr(cell), ptr(v.pillar_of_point), ptr(v.coords), cap_p,
                                    ptr(bucket_cnt) if buckets else None, ptr(v.counts), ptr(scratch), stream()))
    else:
        _count(5 if n > 0 else 3)
        check(L.pnx_voxelize(ptr(points), n, batch, v.min_x, v.min_y, v.vs_x, v.vs_y, gx, gy, ptr(v.bitmap), ptr(v.inblk),
                             ptr(v.blockcnt), ptr(v.blockpref), ptr(cell), ptr(v.pillar_of_point), ptr(v.coords), cap_p,
                             ptr(bucket_cnt) if buckets else None, ptr(v.counts), stream()))
    if buckets:
        scratch = torch.empty(cap_p // 2048 + 4, **i32)
        v.bucket_off = torch.empty(cap_p + 1, **i32)
        bucket_tmp = torch.empty(max(n, 1), **i32)
        v.bucket_pts = torch.empty(max(n, 1), **i32)
        _count(5 if n > 0 else 3)
        check(L.pnx_bucketize(ptr(v.pillar_of_point), n, cap_p, ptr(bucket_cnt), ptr(scratch), ptr(v.bucket_off),
                              ptr(bucket_tmp), ptr(v.bucket_pts), ptr(v.counts), stream()))
    return v


def pillar_mean(v):
    """Per-pillar mean of (x, y, z) (pnx_pfn_mean; pillar_encoder.py:113-114 scatter_mean): [cap_p, 3] fp32, rows >= P
    undefined.  Needs the CSR buckets (voxelize(..., buckets=True))."""
    mean = torch.empty(max(v.cap_p, 1), 3, dtype=torch.float32, device=v.points.device)
    _count(1)
    check(lib().pnx_pfn_mean(ptr(v.points), ptr(v.bucket_off), ptr(v.bucket_pts), ptr(v.counts), v.cap_p, ptr(mean), stream()))
    return mean


# --------------------------------------------------------------------------------- BatchNorm stats
def bn_finalize(stats, channels, count_ptr, count_mult, gamma, beta, eps, momentum, running_mean, running_var,
                want_saved=True):
    dev = stats.device
    scale = torch.empty(channels, dtype=torch.float32, device=dev)
    shift = torch.empty_like(scale)
    mean = torch.empty_like(scale) if want_saved else None
    invstd = torch.empty_like(scale) if want_saved else None
    _count(1)
    check(lib().pnx_bn_finalize(ptr(stats), channels, ptr(count_ptr) if count_ptr is not None else None,
                                int(count_mult), ptr(gamma), ptr(beta), float(eps), float(momentum),
                                ptr(running_mean) if running_mean is not None else None,
                                ptr(running_var) if running_var is not None else None,
                                ptr(scale), ptr(shift), ptr(mean) if want_saved else None,
                                ptr(invstd) if want_saved else None, stream()))
    return scale, shift, mean, invstd


def bn_eval_affine(gamma, beta, rm, rv, eps):
    c = gamma.shape[0]
    scale = torch.empty(c, dtype=torch.float32, device=gamma.device)
    shift = torch.empty_like(scale)
    _count(1)
    check(lib().pnx_bn_eval_affine(c, ptr(gamma), ptr(beta), ptr(rm), ptr(rv), float(eps), ptr(scale), ptr(shift),
                                   stream()))
    return scale, shift


# --------------------------------------------------------------------------------- PFN forward
def _sync_stats(stats, count):
    """SyncBatchNorm (reference tools/train.py:55-56): batch statistics over the points of ALL ranks.
    stats fp64 [2C] local sums, count = device int tensor [1] -> (global stats, global count as device int32 [1])."""
    import torch.distributed as dist
    pack = torch.cat([stats, count.to(torch.float64)])
    dist.all_reduce(pack)
    return pack[:-1], pack[-1:].round().to(torch.int32)


def pfn_forward(v, w0, bn0, w1, bn1, training, eps=1e-3, momentum=0.01, want_f32=True, sync=False):
    """P1-P3. bn0/bn1 = (gamma, beta, running_mean, running_var). Returns dict with feat (fp32 [capP,64]),
    feat_bf16, and everything the backward needs.  sync: SyncBatchNorm statistics (all-reduced over the ranks)."""
    L = lib()
    dev = v.points.device
    f32 = dict(dtype=torch.float32, device=dev)
    n, cap_p = max(v.n, 1), max(v.cap_p, 1)
    out = {}
    mean = torch.empty(cap_p, 3, **f32)
    y0 = torch.empty(n, 32, **f32)
    y1 = torch.empty(n, 64, **f32)
    x0max = torch.empty(cap_p, 32, **f32)
    stats = torch.zeros(2 * 32 + 2 * 64, dtype=torch.float64, device=dev)
    s0, s1 = stats[:64], stats[64:]
    nv_ptr = v.counts[1:2]
    tr = 1 if training else 0
    _count(5)
    check(L.pnx_pfn_mean(ptr(v.points), ptr(v.bucket_off), ptr(v.bucket_pts), ptr(v.counts), v.cap_p, ptr(mean),
                         stream()))
    check(L.pnx_pfn_lin0(ptr(v.points), ptr(v.bucket_pts), ptr(v.pillar_of_point), ptr(v.coords), ptr(mean),
                         ptr(v.counts), v.n, v.min_x, v.min_y, v.vs_x, v.vs_y, ptr(w0), ptr(y0), ptr(s0), tr,
                         stream()))
    sync = bool(sync and training)
    s0f, s1f, nv_bn = s0, s1, nv_ptr
    if sync:
        s0f, nv_bn = _sync_stats(s0, nv_ptr)
    if training:
        sc0, sh0, m0, i0 = bn_finalize(s0f, 32, nv_bn, 1, bn0[0], bn0[1], eps, momentum, bn0[2], bn0[3])
    else:
        sc0, sh0 = bn_eval_affine(bn0[0], bn0[1], bn0[2], bn0[3], eps)
        m0 = i0 = None
    check(L.pnx_pfn_max0(ptr(y0), ptr(v.bucket_off), ptr(v.counts), v.cap_p, ptr(sc0), ptr(sh0), ptr(x0max),
                         stream()))
    check(L.pnx_pfn_lin1(ptr(y0), ptr(x0max), ptr(v.bucket_pts), ptr(v.pillar_of_point), ptr(v.counts), v.n,
                         ptr(sc0), ptr(sh0), ptr(w1), ptr(y1), ptr(s1), tr, stream()))
    if sync:
        s1f, _ = _sync_stats(s1, nv_ptr)
    if training:
        sc1, sh1, m1, i1 = bn_finalize(s1f, 64, nv_bn, 1, bn1[0], bn1[1], eps, momentum, bn1[2], bn1[3])
    else:
        sc1, sh1 = bn_eval_affine(bn1[0], bn1[1], bn1[2], bn1[3], eps)
        m1 = i1 = None
    feat = torch.empty(cap_p, 64, **f32) if want_f32 else None
    feat_bf16 = torch.empty(cap_p, 64, dtype=torch.bfloat16, device=dev)
    check(L.pnx_pfn_max1(ptr(y1), ptr(v.bucket_off), ptr(v.counts), v.cap_p, ptr(sc1), ptr(sh1),
                         ptr(feat) if want_f32 else None, ptr(feat_bf16), stream()))
    out.update(feat=feat, feat_bf16=feat_bf16, mean=mean, y0=y0, y1=y1, x0max=x0max, sc0=sc0, sh0=sh0, sc1=sc1,
               sh1=sh1, mean0=m0, invstd0=i0, mean1=m1, invstd1=i1, bn_count=nv_bn if sync else None)
    return out


def pfn_backward(v, fwd, dfeat, w1, gamma0, gamma1):
    """Backward of pfn_forward (training mode). dfeat fp32 [>=P, 64] contiguous.
    Returns dW0 [32,10], dW1 [64,64], dgamma0, dbeta0, dgamma1, dbeta1 (fp32)."""
    dev = dfeat.device
    n, cap_p = max(v.n, 1), max(v.cap_p, 1)
    assert dfeat.dtype == torch.float32 and dfeat.is_contiguous() and dfeat.shape[0] >= min(v.P or 0, cap_p)
    if dfeat.shape[0] < cap_p:
        full = torch.zeros(cap_p, 64, dtype=torch.float32, device=dev)
        full[:dfeat.shape[0]] = dfeat
        dfeat = full
    argq1 = torch.empty(cap_p, 64, dtype=torch.int32, device=dev)
    d_x0 = torch.empty(n, 32, dtype=torch.float32, device=dev)
    dxm = torch.empty(n, 32, dtype=torch.float32, device=dev)
    red = torch.zeros(64 + 128, dtype=torch.float64, device=dev)
    dW0 = torch.zeros(32, 10, dtype=torch.float64, device=dev)      # fp64 accumulators (cross-CTA atomics, order-insensitive)
    dW1 = torch.zeros(64, 64, dtype=torch.float64, device=dev)
    _count(4)
    bn_count = fwd.get("bn_count")

    def run(phases, red_buf):
        check(lib().pnx_pfn_backward(ptr(v.points), ptr(v.bucket_off), ptr(v.bucket_pts), ptr(v.pillar_of_point),
                                     ptr(v.coords), ptr(v.counts), v.n, v.cap_p, v.min_x, v.min_y, v.vs_x, v.vs_y,
                                     ptr(fwd["mean"]), ptr(fwd["y0"]), ptr(fwd["y1"]), ptr(fwd["x0max"]), ptr(fwd["feat"]),
                                     ptr(dfeat), ptr(w1), ptr(fwd["sc0"]), ptr(fwd["sh0"]), ptr(fwd["mean0"]),
                                     ptr(fwd["invstd0"]), ptr(gamma0), ptr(fwd["sc1"]), ptr(fwd["sh1"]), ptr(fwd["mean1"]),
                                     ptr(fwd["invstd1"]), ptr(gamma1), ptr(argq1), ptr(d_x0), ptr(dxm), ptr(red_buf), ptr(dW0),
                                     ptr(dW1), phases, ptr(bn_count) if bn_count is not None else None, stream()))

    if bn_count is None:
        run(0, red)
    else:
        # SyncBatchNorm backward: the two per-channel sums of each BN are all-reduced between the phase that produces
        # them and the phase that applies them; dgamma / dbeta stay local (DDP averages parameter gradients)
        import torch.distributed as dist
        glob = torch.zeros_like(red)
        run(1, red)
        glob[64:] = red[64:]
        dist.all_reduce(glob[64:])
        run(2, glob)
        run(4, red)
        glob[:64] = red[:64]
        dist.all_reduce(glob[:64])
        run(8, glob)
    r = red.float()
    return dW0.float(), dW1.float(), r[32:64], r[0:32], r[128:192], r[64:128]


# --------------------------------------------------------------------------------- sites / rulebook
class Level:
    """Active-site set of one backbone level: bitmap (b,u,v), inblk (u16 per word), blockpref, coords [n,3], count."""
    pass


def level_from_bitmap(bm, blockpref, count, batch, U, V, inblk=None):
    """Wrap an existing bitmap (e.g. the voxelizer's level 0); inblk is computed here when not given."""
    lv = Level()
    lv.bm, lv.blockpref, lv.count, lv.batch, lv.U, lv.V = bm, blockpref, count, batch, U, V
    if inblk is None:
        inblk = torch.empty(bm.numel(), dtype=torch.int16, device=bm.device)
        _count(1)
        check(lib().pnx_sites_inblock(ptr(bm), bm.numel(), ptr(inblk), stream()))
    lv.inblk = inblk
    lv.n = None
    lv.coords = None
    return lv


def level_from_mask_words(bm, batch, U, V):
    """Level from a raw bitmap (words padded to whole blocks): block counts, scan and in-block prefix."""
    assert bm.numel() % 32 == 0
    blocks = bm.numel() // 32
    inblk = torch.empty(bm.numel(), dtype=torch.int16, device=bm.device)
    _count(1)
    check(lib().pnx_sites_inblock(ptr(bm), bm.numel(), ptr(inblk), stream()))
    cnt = torch.zeros(lib().pnx_blockcnt_size(blocks), dtype=torch.int32, device=bm.device)
    # block counts = in-block prefix of the last word + its popcount (host-side torch plumbing, used by tests and by
    # modules.SparseResNet for coordinates that do not come from the voxelizer)
    w = bm.view(-1, 32)
    pc = torch.zeros_like(w)
    x = w.clone().to(torch.int64) & 0xFFFFFFFF
    for _ in range(32):
        pc += (x & 1).to(torch.int32)
        x >>= 1
    cnt[:blocks] = pc.sum(1)
    so = (blocks + 3) // 4 * 4
    nsb = (blocks + 1023) // 1024
    padded = torch.zeros(nsb * 1024, dtype=torch.int32, device=bm.device)
    padded[:blocks] = cnt[:blocks]
    cnt[so:so + nsb] = padded.view(nsb, 1024).sum(1)
    blockpref = torch.empty(blocks + 1, dtype=torch.int32, device=bm.device)
    count = torch.empty(1, dtype=torch.int32, device=bm.device)
    _count(1)
    check(lib().pnx_scan_blocks(ptr(cnt), blocks, ptr(blockpref), ptr(count), stream()))
    return level_from_bitmap(bm, blockpref, count, batch, U, V, inblk=inblk)


def level_dilate(src, stride):
    L = lib()
    uo, vo = L.pnx_sites_out_dim(src.U, stride), L.pnx_sites_out_dim(src.V, stride)
    words = (src.batch * uo * ((vo + 31) // 32) + 31) // 32 * 32
    dev = src.bm.device
    bm = torch.empty(words, dtype=torch.int32, device=dev)
    inblk = torch.empty(words, dtype=torch.int16, device=dev)
    cnt = torch.empty(L.pnx_blockcnt_size(words // 32), dtype=torch.int32, device=dev)
    blockpref = torch.empty(words // 32 + 1, dtype=torch.int32, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    _count(2)
    check(L.pnx_sites_dilate(ptr(src.bm), src.batch, src.U, src.V, stride, ptr(bm), ptr(inblk), ptr(cnt), stream()))
    check(L.pnx_scan_blocks(ptr(cnt), words // 32, ptr(blockpref), ptr(count), stream()))
    return level_from_bitmap(bm, blockpref, count, src.batch, uo, vo, inblk=inblk)


def level_coords(lv, n):
    lv.n = n
    lv.coords = torch.empty(max(n, 1), 3, dtype=torch.int32, device=lv.bm.device)
    _count(1)
    check(lib().pnx_sites_coords(ptr(lv.bm), ptr(lv.blockpref), ptr(lv.inblk), lv.batch, lv.U, lv.V, ptr(lv.coords), n,
                                 stream()))
    return lv.coords


def nbr_table(dst, src, stride, transposed):
    nbr = torch.empty(max(dst.n, 1), 9, dtype=torch.int32, device=dst.bm.device)
    _count(1)
    check(lib().pnx_nbr_table(ptr(dst.coords), ptr(dst.count), dst.n, ptr(src.bm), ptr(src.blockpref), ptr(src.inblk),
                              src.batch, src.U, src.V, stride, 1 if transposed else 0, ptr(nbr), stream()))
    return nbr


def scatter_dense(feat, lv, channels, canvas=None, gather=False):
    """feat [n,C] bf16 <-> canvas [B, V(y), U(x), C] bf16."""
    if canvas is None:
        canvas = torch.zeros(lv.batch, lv.V, lv.U, channels, dtype=torch.bfloat16, device=feat.device)
    _count(1)
    check(lib().pnx_scatter_dense(ptr(feat), ptr(lv.coords), ptr(lv.count), lv.n, channels, lv.batch, lv.U, lv.V,
                                  ptr(canvas), 1 if gather else 0, stream()))
    return canvas


# --------------------------------------------------------------------------------- implicit GEMM
def _bnr_args(bnr, cout):
    """Trailing C-ABI arguments of the fused BatchNorm-backward reduce (None: off).  bnr: functional.BNInfo."""
    if bnr is None:
        return (None, 0, None, None, None, None, None, 0)
    assert bnr.raw.dtype == torch.bfloat16 and bnr.C == cout and bnr.red.numel() == 2 * cout
    return (ptr(bnr.raw), bnr.raw.stride(0), ptr(bnr.scale), ptr(bnr.shift), ptr(bnr.mean), ptr(bnr.invstd), ptr(bnr.red), cout)


def bnr_eligible(cout, out_fp32=False, shuffle=False):
    """The fused reduce lives in the bf16 staged (coalesced) store of the GEMM epilogues: 64-column granularity."""
    return (not out_fp32) and (not shuffle) and cout % 64 == 0


def pick_block_n(cout):
    for bn in (256, 192, 128, 64, 32, 16):
        if cout % bn == 0:
            return bn
    raise ValueError("Cout %d is not a multiple of 16" % cout)


def igemm(A, M, w_packed, taps, cin, cout, out, *, lda=None, ldc=None, nbr=None, dense=None, bias=None, stats=None,
          stats_mod=None, shuffle=False, relu=False, block_n=None, addend=None, segs=None, a_lo_off=0, bnr=None):
    """out[m, :cout] = sum_t A[nbr(m,t)] @ W[t]^T.  w_packed [taps, cout, cin] bf16.
    dense = (Hout, Wout, Hin, Win, kw, mul, dil, pad) or None.
    segs: fp32-grade split mode -- list of (A piece, W piece) K segments in execution order; A rows hold piece p at
    column p*a_lo_off + c, w_packed is [taps, cout, pieces*cin] (see include/pnx.h "split rows")."""
    assert A.dtype == torch.bfloat16 and w_packed.dtype == torch.bfloat16 and w_packed.is_contiguous()
    nseg, seg_code = 1, 0
    if segs:
        nseg = len(segs)
        for i, (ap, wp) in enumerate(segs):
            seg_code |= ((ap << 2) | wp) << (4 * i)
    w_pieces = (max(wp for _, wp in segs) + 1) if segs else 1
    assert tuple(w_packed.shape) == (taps, cout, cin * w_pieces), (tuple(w_packed.shape), (taps, cout, cin), segs)
    lda = A.stride(0) if lda is None else lda
    ldc = out.stride(-2) if ldc is None else ldc
    bn = block_n or pick_block_n(cout)
    d = dense or (0, 0, 0, 0, 1, 1, 1, 0)
    out_fp32 = 1 if out.dtype == torch.float32 else 0
    assert out.dtype in (torch.float32, torch.bfloat16)
    sC = stats.numel() // 2 if stats is not None else 0
    _count(1)
    add_f32 = 1 if (addend is not None and addend.dtype == torch.float32) else 0
    with _Timed("igemm", 2.0 * M * taps * cin * cout * nseg, 2.0 * M * (cin * min(taps, 2) + cout) + 2.0 * taps * cin * cout,
                "M%d_T%d_K%d_N%d_bn%d%s" % (M, taps, cin, cout, bn, "_tbl" if nbr is not None else ("_dense" if dense else ""))):
      check(lib().pnx_igemm(ptr(A), lda, A.shape[0], M, taps, cin, ptr(w_packed), cout, bn, ptr(nbr) if nbr is not None else None,
                          1 if dense else 0, d[0], d[1], d[2], d[3], d[4], d[5], d[6], d[7], ptr(out), ldc, out_fp32,
                          ptr(bias) if bias is not None else None, ptr(stats) if stats is not None else None, sC,
                          stats_mod or (sC if sC else 1), 1 if shuffle else 0, 1 if relu else 0,
                          ptr(addend) if addend is not None else None, addend.stride(0) if addend is not None else 0,
                          int(nseg), int(a_lo_off), int(seg_code), add_f32, *_bnr_args(bnr, cout), sm_count(), stream()))
    return out


WIN_BASE_OFF = 0   # measured on H100: the 128B swizzle is applied on absolute smem address bits, so row-shifted wgmma
                   # descriptors need NO matrix base offset (tests/test_igemm_win_gpu.py checks both conventions)


def win_eligible(dense, n_cols, k_cols, out_fp32=False, shuffle=False):
    """Dense 3x3 stride-1 dilation-1 'same' conv whose image rows tile into 128-pixel chunks with <= 15 % waste."""
    if dense is None or out_fp32 or shuffle:
        return False
    Ho, Wo, Hi, Wi, kw, mul, dil, pad = dense
    if not (kw == 3 and mul == 1 and dil == 1 and pad == 1 and Ho == Hi and Wo == Wi):
        return False
    if n_cols % 64 or k_cols % 64:
        return False
    xc = (Wo + 127) // 128
    return xc * 128 <= 1.15 * Wo


def conv3x3_win(A, B, H, W, w_packed, cin, cout, out, *, bias=None, stats=None, relu=False, block_n=None, base_off=None, bnr=None):
    """Dense 3x3 'same' conv with TMA-folded im2col (pnx_conv3x3_win). A bf16 rows [B*H*W, >=cin]; out bf16."""
    assert A.dtype == torch.bfloat16 and out.dtype == torch.bfloat16 and tuple(w_packed.shape) == (9, cout, cin)
    if block_n:
        bn = block_n
    elif cin == 64 and cout % 128 == 0:
        bn = 128            # weights-stationary variant: the nine [128 x 64] tiles stay in shared memory
    else:
        bn = 192 if cout % 192 == 0 else (128 if cout % 128 == 0 else 64)
    M = B * H * W
    _count(1)
    with _Timed("igemm_win", 2.0 * M * 9 * cin * cout, 2.0 * M * (cin * 3 + cout), "M%d_K%d_N%d_bn%d" % (M, cin, cout, bn)):
      check(lib().pnx_conv3x3_win(ptr(A), A.stride(0), B, H, W, cin, ptr(w_packed), cout, bn, ptr(out), out.stride(0),
                                ptr(bias) if bias is not None else None, ptr(stats) if stats is not None else None,
                                stats.numel() // 2 if stats is not None else 0, 1 if relu else 0,
                                WIN_BASE_OFF if base_off is None else base_off, *_bnr_args(bnr, cout), sm_count(), stream()))
    return out


DETERMINISTIC = False     # set through functional.set_deterministic


def set_deterministic(on):
    """Library side of functional.set_deterministic: fp64 accumulation of the BatchNorm statistics in the GEMM epilogues
    (pnx_set_deterministic).  pnx_wgrad reduces its K splits in split order in either mode."""
    global DETERMINISTIC
    prev, DETERMINISTIC = DETERMINISTIC, bool(on)
    lib().pnx_set_deterministic(1 if on else 0)
    return prev


def wgrad_splits(x_channels, y_channels, taps, M, sms=None):
    """Number of K splits pnx_wgrad uses for the shape (a pure function of it; sms defaults to this device's SM count)."""
    return lib().pnx_wgrad_splits(x_channels, y_channels, taps, M, sm_count() if sms is None else sms)


def wgrad(X, x_channels, Y, y_channels, M, taps, dW, *, nbr=None, dense=None, shuffle=False, gathered=None):
    """dW[t, x, y] += sum_m X[m, x] * Y[g(m,t), y]; X direct, Y gathered; dW fp32 [taps, x_channels, y_channels]."""
    assert X.dtype == torch.bfloat16 and Y.dtype == torch.bfloat16 and dW.dtype == torch.float32
    assert tuple(dW.shape) == (taps, x_channels, y_channels) and dW.is_contiguous()
    if x_channels != 64 and x_channels % 128 != 0:
        # the kernel tiles X in 128-channel blocks (or one 64-channel block): split e.g. 448 = 384 + 64 column slices of X
        # (seven sibling heads of a Waymo task); each part accumulates into its own zeroed buffer, added to its dW rows
        assert x_channels % 64 == 0 and x_channels > 64, "x_channels must be a multiple of 64"
        main = x_channels // 128 * 128
        for x0, x1 in ((0, main), (main, x_channels)):
            part = torch.zeros(taps, x1 - x0, y_channels, dtype=torch.float32, device=dW.device)
            wgrad(X[:, x0:x1], x1 - x0, Y, y_channels, M, taps, part, nbr=nbr, dense=dense, shuffle=shuffle, gathered=gathered)
            dW[:, x0:x1] += part
        return dW
    d = dense or (0, 0, 0, 0, 1, 1, 1, 0)
    if gathered is None:
        gathered = nbr is not None or dense is not None or shuffle
    # one slab per K split, added in split order (not fp32 atomics): the weight gradient is the same from run to run
    splits = wgrad_splits(x_channels, y_channels, taps, M)
    partials = torch.empty(max(splits, 1) * taps * x_channels * y_channels, dtype=torch.float32, device=dW.device)
    _count(2)
    with _Timed("wgrad", 2.0 * M * taps * x_channels * y_channels, 2.0 * M * (x_channels + taps * y_channels),
                "M%d_T%d_X%d_Y%d" % (M, taps, x_channels, y_channels)):
      check(lib().pnx_wgrad(ptr(X), X.stride(0), x_channels, ptr(Y), Y.stride(0), Y.shape[0], y_channels, 1 if gathered else 0, M,
                          taps, ptr(nbr) if nbr is not None else None, d[0], d[1], d[2], d[3], d[4], d[5], d[6], d[7],
                          1 if shuffle else 0, ptr(dW), ptr(partials) if partials is not None else None, sm_count(), stream()))
    return dW


# --------------------------------------------------------------------------------- row-wise kernels
def bn_apply(x, M, C, scale, shift, y, res=None, relu=True):
    _count(1)
    check(lib().pnx_bn_apply(ptr(x), x.stride(0), M, C, ptr(scale), ptr(shift), ptr(res) if res is not None else None,
                             res.stride(0) if res is not None else 8, 1 if relu else 0, ptr(y), y.stride(0), stream()))
    return y


def bn_bwd_reduce(dy, y, x, M, C, mean, invstd, relu, affine=None, red=None):
    """Reduce pass of the BatchNorm backward (pnx_bn_bwd_reduce) -> red fp64 [2C] (sum g = dbeta, sum g*xhat = dgamma)
    of the gated gradient g, added into `red` (default: a zeroed buffer of the step's arena).  y=None (no residual): the
    ReLU mask is recomputed from x with affine=(scale, shift) of the forward."""
    fs, fh = affine if affine is not None else (None, None)
    if red is None:
        red = zeros(2 * C, torch.float64, dy.device)
    _count(1)
    check(lib().pnx_bn_bwd_reduce(ptr(dy), dy.stride(0), ptr(y), y.stride(0) if y is not None else 8, ptr(x), x.stride(0),
                                  M, C, ptr(mean), ptr(invstd), 1 if relu else 0, ptr(fs), ptr(fh), ptr(red), stream()))
    return red


def bn_bwd_apply(dy, y, x, M, C, mean, invstd, gamma, red, count, relu, affine, dx, dres=None, dres_accumulate=False,
                 count_dev=None):
    """Apply pass of the BatchNorm backward (pnx_bn_bwd_apply): writes dx (and dres) from the sums red of the reduce
    pass.  relu=False when dy already is the gated g (the reduce pass ran in the epilogue of the GEMM that produced it).
    count_dev: the population as a device int32 [1] (SyncBatchNorm), used instead of the host count."""
    fs, fh = affine if affine is not None else (None, None)
    _count(1)
    check(lib().pnx_bn_bwd_apply(ptr(dy), dy.stride(0), ptr(y), y.stride(0) if y is not None else 8, ptr(x), x.stride(0),
                                 M, C, ptr(mean), ptr(invstd), ptr(gamma), ptr(red), float(max(count, 1)), ptr(count_dev),
                                 1 if relu else 0, ptr(fs), ptr(fh), ptr(dx), dx.stride(0), ptr(dres),
                                 dres.stride(0) if dres is not None else 8, 1 if dres_accumulate else 0, stream()))
    return dx


def bn_bwd(dy, y, x, M, C, mean, invstd, gamma, count, relu, dx, dres=None, dres_accumulate=False, affine=None, red=None):
    """Both passes of the BatchNorm backward: bn_bwd_reduce, then bn_bwd_apply with the host count.  Returns red.
    red given: the reduce pass already happened in the epilogue of the GEMM that produced dy (which is then the gated
    g, so the apply pass runs without a ReLU mask)."""
    if red is None:
        red = bn_bwd_reduce(dy, y, x, M, C, mean, invstd, relu, affine)
    else:
        relu = False
    bn_bwd_apply(dy, y, x, M, C, mean, invstd, gamma, red, count, relu, affine, dx, dres=dres, dres_accumulate=dres_accumulate)
    return red


def add_rows(a, b, M, C):
    _count(1)
    check(lib().pnx_add_rows(ptr(a), a.stride(0), ptr(b), b.stride(0), M, C, stream()))
    return a


def add_relu(a, b, M, C, y):
    _count(1)
    check(lib().pnx_add_relu(ptr(a), a.stride(0), ptr(b), b.stride(0), M, C, ptr(y), y.stride(0), stream()))
    return y


def relu_bwd(dy, y, M, C, g, accumulate=False):
    _count(1)
    check(lib().pnx_relu_bwd(ptr(dy), dy.stride(0), ptr(y), y.stride(0), M, C, ptr(g), g.stride(0),
                             1 if accumulate else 0, stream()))
    return g


# --------------------------------------------------------------------------------- fp32-grade split rows
# A "split" activation is a bf16 tensor [M, P*C]: piece 0 = bf16(v) in columns [0, C), piece 1 = bf16(v - piece 0) in
# [C, 2C), ... (include/pnx.h, "split rows"; P = split_pieces(), 2 or 3).  The wrappers take (tensor-or-view, piece
# offset in elements) per operand.
SEGMENTS = {2: [(1, 1), (1, 0), (0, 1), (0, 0)],                       # (A piece, W piece), smallest products first
            3: [(2, 0), (0, 2), (1, 1), (1, 0), (0, 1), (0, 0)]}       # 2^-16-sized terms, 2^-8-sized terms, hi*hi


def split_pieces(set_to=None):
    if set_to is not None:
        lib().pnx_split_set_pieces(int(set_to))
    return lib().pnx_split_get_pieces()


def split_segments():
    return SEGMENTS[split_pieces()]


def to_pieces(p):
    """fp32 [..., K] -> bf16 [..., P*K] = [piece 0 | piece 1 | ...] (packed weights of the split mode)."""
    out, rem = [], p.float()
    for _ in range(split_pieces()):
        q = rem.to(torch.bfloat16)
        out.append(q)
        rem = rem - q.float()
    return torch.cat(out, -1).contiguous()


def rows_split(x, C=None, out=None, lo=None):
    """fp32 rows [M, >=C] -> split rows.  out/lo: write into an existing buffer (view) with the lo half at +lo."""
    assert x.dtype == torch.float32 and x.stride(-1) == 1
    M = x.shape[0]
    C = x.shape[1] if C is None else C
    if out is None:
        out = torch.empty(M, split_pieces() * C, dtype=torch.bfloat16, device=x.device)
        lo = C
    _count(1)
    check(lib().pnx_rows_split(ptr(x), x.stride(0), M, C, ptr(out), out.stride(0), int(lo), stream()))
    return out


def rows_merge(x, C, lo, out=None, accumulate=False):
    """split rows -> fp32 [M, C] (hi + lo)."""
    M = x.shape[0]
    if out is None:
        out = torch.empty(M, C, dtype=torch.float32, device=x.device)
    _count(1)
    check(lib().pnx_rows_merge(ptr(x), x.stride(0), int(lo), M, C, ptr(out), out.stride(0), 1 if accumulate else 0, stream()))
    return out


def bn_apply_split(x, M, C, scale, shift, y, y_lo, res=None, res_lo=0, relu=True):
    _count(1)
    check(lib().pnx_bn_apply_split(ptr(x), x.stride(0), M, C, ptr(scale), ptr(shift), ptr(res) if res is not None else None,
                                   res.stride(0) if res is not None else 16, int(res_lo) if res is not None else 16, 1 if relu else 0,
                                   ptr(y), y.stride(0), int(y_lo), stream()))
    return y


def bn_bwd_reduce_split(dy, dy_lo, y, y_lo, x, M, C, mean, invstd, relu, affine):
    L = lib()
    part = torch.empty(L.pnx_bn_bwd_reduce_split_scratch(C), dtype=torch.float64, device=dy.device)
    red = torch.empty(2 * C, dtype=torch.float64, device=dy.device)
    fs, fh = affine if affine is not None else (None, None)
    _count(2)
    check(L.pnx_bn_bwd_reduce_split(ptr(dy), dy.stride(0), int(dy_lo), ptr(y) if y is not None else None,
                                    y.stride(0) if y is not None else 16, int(y_lo) if y is not None else 16, ptr(x), x.stride(0), M, C,
                                    ptr(mean), ptr(invstd), 1 if relu else 0, ptr(fs) if fs is not None else None,
                                    ptr(fh) if fh is not None else None, ptr(part), ptr(red), stream()))
    return red


def bn_bwd_apply_split(dy, dy_lo, y, y_lo, x, M, C, mean, invstd, gamma, red, count, relu, affine, dx, dx_lo, dres=None, dres_lo=0):
    fs, fh = affine if affine is not None else (None, None)
    _count(1)
    check(lib().pnx_bn_bwd_apply_split(ptr(dy), dy.stride(0), int(dy_lo), ptr(y) if y is not None else None,
                                       y.stride(0) if y is not None else 16, int(y_lo) if y is not None else 16, ptr(x), x.stride(0), M, C,
                                       ptr(mean), ptr(invstd), ptr(gamma), ptr(red), float(max(count, 1)), 1 if relu else 0,
                                       ptr(fs) if fs is not None else None, ptr(fh) if fh is not None else None, ptr(dx), dx.stride(0),
                                       int(dx_lo), ptr(dres) if dres is not None else None,
                                       dres.stride(0) if dres is not None else 16, int(dres_lo) if dres is not None else 16, stream()))
    return dx


def add_relu_split(a, a_lo, b, b_lo, M, C, y, y_lo):
    _count(1)
    check(lib().pnx_add_relu_split(ptr(a), a.stride(0), int(a_lo), ptr(b), b.stride(0), int(b_lo), M, C, ptr(y), y.stride(0),
                                   int(y_lo), stream()))
    return y


def relu_bwd_split(dy_f32, y, y_lo, M, C, g, g_lo):
    _count(1)
    check(lib().pnx_relu_bwd_split(ptr(dy_f32), dy_f32.stride(0), ptr(y), y.stride(0), int(y_lo), M, C, ptr(g), g.stride(0),
                                   int(g_lo), stream()))
    return g


def wgrad_split(X, x_lo, x_channels, Y, y_lo, y_channels, M, taps, dW, **kw):
    """Weight gradient of split operands: one launch per (X piece, Y piece) segment, smallest products first, all
    accumulating into the same dW."""
    for xp, yp in split_segments():
        wgrad(X[:, xp * x_lo:xp * x_lo + x_channels], x_channels, Y[:, yp * y_lo:yp * y_lo + y_channels], y_channels, M, taps, dW, **kw)
    return dW


# --------------------------------------------------------------------------------- head final convs: 9-tap stencil
def tap_gather_sum(Z, cpt, bias, B, H, W, out):
    """out [B*H*W, 16] fp32 = bias + the sum over the 9 taps of the stencil of Z [B*H*W, >= 9*cpt] fp32, column
    tap*cpt + j (pnx_tap_gather_sum)."""
    _count(1)
    check(lib().pnx_tap_gather_sum(ptr(Z), Z.stride(0), cpt, ptr(bias), B, H, W, ptr(out), stream()))
    return out


def tap_scatter(dout, B, H, W, dZ, nz, cpt, lo_off=0):
    """Backward of tap_gather_sum (pnx_tap_scatter): dZ [B*H*W, nz] bf16 (columns >= 9*cpt zeroed) from dout fp32;
    lo_off > 0: all pieces of a split-rows dZ, piece q at column q*lo_off + c."""
    _count(1)
    check(lib().pnx_tap_scatter(ptr(dout), B, H, W, ptr(dZ), dZ.stride(0), nz, cpt, lo_off, stream()))
    return dZ


# --------------------------------------------------------------------------------- L1: fused CenterPoint loss
def center_loss_task(out, dout, labels, task, weight, code_weights, with_iou, acc):
    """Loss partial sums of one task into acc fp64 [16] (zeroed) and the gradient dout (pnx_center_loss_task).
    out/dout [B*H*W, npad] fp32; labels: the task's hm / anno_box / ind / mask / cat / gt_boxes (assign_labels);
    task: its geometry B, H, W, npad, C, M, column offsets `off` and the sx, sy, ox, oy of the box encoding."""
    cw, cwp = _host_floats(code_weights, 10)
    o = task["off"]
    _count(2)
    check(lib().pnx_center_loss_task(ptr(out), ptr(dout), ptr(labels["hm"]), ptr(labels["anno_box"]), ptr(labels["ind"]),
                                     ptr(labels["mask"]), ptr(labels["cat"]), ptr(labels["gt_boxes"]), task["B"], task["H"],
                                     task["W"], task["npad"], task["C"], task["M"], o["reg"], o["height"], o["dim"], o["rot"],
                                     o["vel"], o["hm"], task["sx"], task["sy"], task["ox"], task["oy"], weight, cwp,
                                     1 if with_iou else 0, ptr(acc), stream()))
    return dout


def center_loss_finalize(acc, weights_dev, code_w_dev, with_iou_dev, res, total):
    """acc [T, 16] fp64 of center_loss_task -> res [T, 16] per-task losses and total [1] (pnx_center_loss_finalize)."""
    _count(1)
    check(lib().pnx_center_loss_finalize(ptr(acc), acc.shape[0], ptr(weights_dev), ptr(code_w_dev), ptr(with_iou_dev),
                                         ptr(res), ptr(total), stream()))
    return res, total


# --------------------------------------------------------------------------------- F3: label assignment
_cls_tables = {}


def pack_weights(table, n, total):
    """pnx_pack_weights: rewrite all bf16 packed operands described by the device table (functional._repack_all)."""
    _count(1)
    check(lib().pnx_pack_weights(ptr(table), int(n), int(total), stream()))


def assign_labels(gt_boxes, gt_cls, tasks, voxel_size, pc_range, out_size_factor, max_objs=500, gaussian_overlap=0.1,
                  min_radius=2):
    """AssignLabel + collate on the GPU (pnx_assign_labels): gt_boxes [B, N, 9] fp32 cuda, gt_cls [B, N] int32 cuda
    (index into the flattened class list of `tasks`, < 0 = ignored) -> dict of per-task lists hm / anno_box / ind /
    mask / cat / gt_boxes in the reference's collate format (det3d/datasets/pipelines/assign.py, loader/collate.py)."""
    assert gt_boxes.is_cuda and gt_boxes.dtype == torch.float32 and gt_boxes.dim() == 3 and gt_boxes.shape[2] == 9
    assert gt_cls.is_cuda and gt_cls.dtype == torch.int32 and tuple(gt_cls.shape) == tuple(gt_boxes.shape[:2])
    gt_boxes, gt_cls = gt_boxes.contiguous(), gt_cls.contiguous()
    dev = gt_boxes.device
    B, N = gt_cls.shape
    key = (tuple(tuple(t) for t in tasks), dev)
    if key not in _cls_tables:
        ct = [ti for ti, t in enumerate(tasks) for _ in t]
        ci = [ni for t in tasks for ni, _ in enumerate(t)]
        _cls_tables[key] = (torch.tensor(ct, dtype=torch.int32, device=dev), torch.tensor(ci, dtype=torch.int32, device=dev))
    cls_task, cls_id = _cls_tables[key]
    g = grid_size_xy(voxel_size, pc_range)
    out = {k: [] for k in ("hm", "anno_box", "ind", "mask", "cat", "gt_boxes")}
    L = lib()
    obj = torch.empty(B, max(N, 1), 4, dtype=torch.int32, device=dev)
    for t, task in enumerate(tasks):
        osf = int(out_size_factor[t])
        W, H = int(g[0]) // osf, int(g[1]) // osf
        hm = torch.zeros(B, len(task), H, W, dtype=torch.float32, device=dev)
        anno = torch.zeros(B, max_objs, 10, dtype=torch.float32, device=dev)
        ind = torch.zeros(B, max_objs, dtype=torch.int64, device=dev)
        mask = torch.zeros(B, max_objs, dtype=torch.uint8, device=dev)
        cat = torch.zeros(B, max_objs, dtype=torch.int64, device=dev)
        gtb = torch.zeros(B, max_objs, 7, dtype=torch.float32, device=dev)
        _count(2)
        check(L.pnx_assign_labels(ptr(gt_boxes), ptr(gt_cls), B, N, ptr(cls_task), ptr(cls_id), cls_task.numel(), t,
                                  float(voxel_size[0]), float(voxel_size[1]), float(pc_range[0]), float(pc_range[1]), osf,
                                  float(gaussian_overlap), int(min_radius), int(max_objs), len(task), H, W, ptr(hm), ptr(anno),
                                  ptr(ind), ptr(mask), ptr(cat), ptr(gtb), ptr(obj), stream()))
        for k, v in (("hm", hm), ("anno_box", anno), ("ind", ind), ("mask", mask), ("cat", cat), ("gt_boxes", gtb)):
            out[k].append(v)
    return out


# --------------------------------------------------------------------------------- F1: decode + rotated NMS
def _host_floats(vals, n):
    a = (ctypes.c_float * n)(*([float(v) for v in vals] + [0.0] * (n - len(vals))))
    return a, ctypes.addressof(a)


def _decode_params(offs, osf, voxel_size, pc_range, score_thr, post_center_range, rectifier):
    """The decode parameters of the F1 entry points and their host twins, after (out, ld, B, H, W, C): -> (the host
    arrays they point to, to be kept alive across the calls; the arguments)."""
    offs_a = (ctypes.c_int * 7)(*[int(o) for o in offs])
    r6, r6p = _host_floats(post_center_range, 6)
    rc, rcp = _host_floats(rectifier, 8)
    return (offs_a, r6, rc), (ctypes.addressof(offs_a), float(osf), float(voxel_size[0]), float(voxel_size[1]),
                              float(pc_range[0]), float(pc_range[1]), float(score_thr), r6p, rcp)


def det_postprocess(out, B, H, W, C, offs, osf, voxel_size, pc_range, score_thr, post_center_range, rectifier, nms_thr,
                    pre_max, post_max, label_offset=0, double_flip=False):
    """One task of CenterHead.predict (centerhead.py:231-384): `out` = channels-last head output [B*H*W, ld] fp32,
    offs = column offsets (reg, height, dim, rot, vel, hm, iou or -1).  Returns det_box [B*C, post_max, 9], det_score
    [B*C, post_max], det_label [B*C, post_max] (int64, + label_offset) and keep_count [B*C] -- all on the device, no
    host synchronisation.  Segment s = frame * C + class.  The candidate ordering is one device sort (torch.sort of
    the 64-bit keys the decode kernel builds); decode, IoU mask, greedy sweep and gather are libpnx kernels.
    double_flip=True: `out` is the head output of a flip4_points batch, [4B*H*W, ld] (frame 4b + k = copy k of frame b);
    the decode merges the four copies of each pixel (pnx_det_*_flip4, include/pnx.h) and the results are those of the
    B original frames."""
    assert out.dtype == torch.float32 and out.is_cuda and out.dim() == 2 and out.shape[0] == (4 if double_flip else 1) * B * H * W
    dev = out.device
    M, nseg = B * H * W, B * C
    alive, params = _decode_params(offs, osf, voxel_size, pc_range, score_thr, post_center_range, rectifier)
    nt, ntp = _host_floats(nms_thr, 8)
    common = (ptr(out), out.stride(0), B, H, W, C) + params
    keys = torch.empty(M, dtype=torch.int64, device=dev)
    seg_count = torch.empty(nseg, dtype=torch.int32, device=dev)
    L = lib()
    keys_fn, nms_fn, gather_fn = ((L.pnx_det_keys_flip4, L.pnx_det_nms_flip4, L.pnx_det_gather_flip4) if double_flip else
                                  (L.pnx_det_keys, L.pnx_det_nms, L.pnx_det_gather))
    _count(1)
    check(keys_fn(*common, ptr(keys), ptr(seg_count), stream()))
    order = torch.sort(keys, stable=True)[1]        # tied scores: ascending pixel index, whatever sort torch picks
    seg_start = (torch.cumsum(seg_count, 0, dtype=torch.int32) - seg_count).contiguous()
    col_blocks = (pre_max + 63) // 64
    mask = torch.empty(nseg * pre_max * col_blocks, dtype=torch.int64, device=dev)
    keep = torch.empty(nseg * post_max, dtype=torch.int32, device=dev)
    keep_count = torch.empty(nseg, dtype=torch.int32, device=dev)
    _count(2)
    check(nms_fn(*common, ntp, ptr(order), ptr(seg_start), ptr(seg_count), int(pre_max), int(post_max), ptr(mask),
                        ptr(keep), ptr(keep_count), stream()))
    det_box = torch.empty(nseg, post_max, 9, dtype=torch.float32, device=dev)
    det_score = torch.empty(nseg, post_max, dtype=torch.float32, device=dev)
    det_label = torch.empty(nseg, post_max, dtype=torch.int64, device=dev)
    _count(1)
    check(gather_fn(*common, ptr(order), ptr(seg_start), ptr(keep), ptr(keep_count), int(post_max), int(label_offset),
                    ptr(det_box), ptr(det_score), ptr(det_label), stream()))
    return det_box, det_score, det_label, keep_count


def det_decode_host(out, B, H, W, C, offs, osf, voxel_size, pc_range, score_thr, post_center_range, rectifier,
                    double_flip=False):
    """Host twin of the decode of det_postprocess (pnx_det_decode_host, pnx_det_decode_flip4_host with double_flip):
    `out` numpy fp32 [B*H*W (4B*H*W with double_flip), ld] -> keep [B*H*W] bool (score above the threshold and centre in
    post_center_range), box [B*H*W, 9] fp32, score fp32, label int32 (meaningful where keep) of every output pixel."""
    need = max(offs[0] + 2, offs[1] + 1, offs[2] + 3, offs[3] + 2, offs[4] + 2, offs[5] + C, offs[6] + 1)
    ld = out.shape[1] if out.ndim == 2 else 0
    if ld < need:
        raise ValueError("out must have at least %d columns for these offsets, got shape %s" % (need, out.shape))
    M = B * H * W
    out = _want(out, torch.float32, ((4 if double_flip else 1) * M, ld), "out", host=True)
    alive, params = _decode_params(offs, osf, voxel_size, pc_range, score_thr, post_center_range, rectifier)
    keep = np.zeros(M, bool)
    box, score, label = np.zeros((M, 9), np.float32), np.zeros(M, np.float32), np.zeros(M, np.int32)
    fn = lib().pnx_det_decode_flip4_host if double_flip else lib().pnx_det_decode_host
    for m in range(M):
        rc = fn(_hp(out), ld, B, H, W, C, *params, m, _hp(box[m]), _hp(score[m:]), _hp(label[m:]))
        if rc < 0:
            check(rc)
        keep[m] = rc == 1
    return keep, box, score, label


def det_iou_bev_host(a, b):
    """Rotated bird's-eye-view IoU of the NMS (pnx_det_iou_bev_host) of each pair a[i], b[i]: numpy fp32 [n, 7]
    (x, y, z, dx, dy, dz, heading) -> [n] fp32."""
    return _box_pairs_host(lib().pnx_det_iou_bev_host, a, b)


def _box_pairs_host(fn, a, b):
    """fn(box7_a, box7_b) -> float of a host twin on each pair of rows of a, b (numpy fp32 [n, 7]) -> [n] fp32."""
    n = len(a)
    a, b = _want(a, torch.float32, (n, 7), "a", host=True), _want(b, torch.float32, (n, 7), "b", host=True)
    return np.array([fn(_hp(a[i]), _hp(b[i])) for i in range(n)], np.float32)


def flip4_points(points):
    """Double-flip test-time augmentation: points [N, 6] (b, x, y, z, i, t) fp32 cuda -> [4N, 6], copy k of point i at row
    k*N + i in frame 4b + k (k = 1: y -> -y, k = 2: x -> -x, k = 3: both; pnx_flip4_points).  The rows are NOT grouped by
    frame: voxelize them with frame_sorted=False."""
    assert points.is_cuda and points.dtype == torch.float32 and points.dim() == 2 and points.shape[1] == 6, \
        "points must be a CUDA float32 [N, 6] tensor (batch_idx, x, y, z, intensity, time)"
    points = points.contiguous()
    out = torch.empty(4 * points.shape[0], 6, dtype=torch.float32, device=points.device)
    _count(1)
    check(lib().pnx_flip4_points(ptr(points), points.shape[0], ptr(out), stream()))
    return out


def _global_aug_operands(points, gt_boxes, aug, host=False):
    B, M = gt_boxes.shape[:2] if gt_boxes.ndim == 3 else (0, 0)
    return (_want(points, torch.float32, (len(points), 6), "points (batch_idx, x, y, z, intensity, time)", host),
            _want(gt_boxes, torch.float32, (B, M, 9), "gt_boxes", host),
            _want(aug, torch.float64, (B, 4, 4), "aug", host))


def global_aug(points, gt_boxes, aug):
    """Global training augmentation on the GPU (pnx_global_aug, include/pnx.h): points [N, 6] (b, x, y, z, i, t) fp32
    cuda, raw boxes [B, M, 9] fp32 cuda and the collated records aug [B, 4, 4] fp64 cuda (det3d.datasets.pipelines.
    augmentation) -> (points, boxes), new tensors with the reference's numpy results to the bit.  The inputs are left
    untouched and the point order is kept, so frame-sorted points stay frame-sorted."""
    points, gt_boxes, aug = _global_aug_operands(points, gt_boxes, aug)
    pts_out, box_out = torch.empty_like(points), torch.empty_like(gt_boxes)
    B, M = gt_boxes.shape[:2]
    _count(1)
    check(lib().pnx_global_aug(ptr(points), points.shape[0], ptr(gt_boxes), B, M, ptr(aug), ptr(pts_out), ptr(box_out),
                               stream()))
    return pts_out, box_out


def global_aug_host(points, gt_boxes, aug):
    """Host twin of global_aug (pnx_global_aug_host): the same operands as numpy arrays -> (points, boxes), new arrays."""
    points, gt_boxes, aug = _global_aug_operands(points, gt_boxes, aug, host=True)
    pts_out, box_out = np.empty_like(points), np.empty_like(gt_boxes)
    B, M = gt_boxes.shape[:2]
    check(lib().pnx_global_aug_host(_hp(points), len(points), _hp(gt_boxes), B, M, _hp(aug), _hp(pts_out), _hp(box_out)))
    return pts_out, box_out


def _gt_sample_operands(points, gt_boxes, gt_classes, gt_trig, cand_boxes, cand_classes, cand_trig, cand_points,
                        cand_offsets, host=False):
    B, M = gt_boxes.shape[:2] if gt_boxes.ndim == 3 else (0, 0)
    S = cand_boxes.shape[1] if cand_boxes.ndim == 3 else 0
    f32, i32 = torch.float32, torch.int32
    return [_want(t, dtype, shape, what, host) for t, dtype, shape, what in (
        (points, f32, (len(points), 6), "points"), (gt_boxes, f32, (B, M, 9), "gt_boxes"),
        (gt_classes, i32, (B, M), "gt_classes"), (gt_trig, f32, (B, M, 2), "gt_trig"),
        (cand_boxes, f32, (B, S, 9), "cand_boxes"), (cand_classes, i32, (B, S), "cand_classes"),
        (cand_trig, f32, (B, S, 4), "cand_trig"), (cand_points, f32, (len(cand_points), 5), "cand_points"),
        (cand_offsets, i32, (B * S + 1,), "cand_offsets"))]


def gt_sample(points, gt_boxes, gt_classes, gt_trig, cand_boxes, cand_classes, cand_trig, cand_points, cand_offsets):
    """Ground-truth database sampling on the GPU (pnx_gt_sample, include/pnx.h): the reference's collision test,
    scene-point removal and paste for the candidates scenes.collate packed (gts_* keys; all CUDA tensors):
    points [N, 6] fp32, scene boxes [B, M, 9] fp32, classes [B, M] int32, gt_trig [B, M, 2] fp32, candidates
    [B, S, 9] / [B, S] / [B, S, 4], cand_points [P, 5] fp32, cand_offsets [B S + 1] int32 ->
    (points [N + P, 6], boxes [B, M + S, 9], classes [B, M + S] int32, accepted [B, S] int32, count [1] int32 cuda).
    The rows past `count` have batch index B, which the voxelizers drop; the host does not wait for the count.  Frames
    stay in order, each with its pasted objects' points first, so frame-sorted input stays frame-sorted."""
    p, b, c, t, cb, cc, ct, cp, co = _gt_sample_operands(points, gt_boxes, gt_classes, gt_trig, cand_boxes, cand_classes,
                                                         cand_trig, cand_points, cand_offsets)
    n, (B, M), S, P = len(p), b.shape[:2], cb.shape[1], len(cp)
    dev = p.device
    pts_out = torch.empty((n + P, 6), dtype=torch.float32, device=dev)
    box_out = torch.empty((B, M + S, 9), dtype=torch.float32, device=dev)
    cls_out = torch.empty((B, M + S), dtype=torch.int32, device=dev)
    accepted = torch.empty((B, S), dtype=torch.int32, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    ws = torch.empty(max(4, lib().pnx_gt_sample_workspace(n, B, S)), dtype=torch.uint8, device=dev)
    _count(1)
    check(lib().pnx_gt_sample(ptr(p), n, ptr(b), ptr(c), ptr(t), B, M, ptr(cb), ptr(cc), ptr(ct), S, ptr(cp), ptr(co), P,
                              ptr(pts_out), ptr(box_out), ptr(cls_out), ptr(accepted), ptr(count), ptr(ws), stream()))
    return pts_out, box_out, cls_out, accepted, count


def gt_sample_host(points, gt_boxes, gt_classes, gt_trig, cand_boxes, cand_classes, cand_trig, cand_points, cand_offsets):
    """Host twin of gt_sample (pnx_gt_sample_host): the same operands as numpy arrays -> (points, boxes, classes,
    accepted, count), the first four new arrays and count an int."""
    p, b, c, t, cb, cc, ct, cp, co = _gt_sample_operands(points, gt_boxes, gt_classes, gt_trig, cand_boxes, cand_classes,
                                                         cand_trig, cand_points, cand_offsets, host=True)
    n, (B, M), S, P = len(p), b.shape[:2], cb.shape[1], len(cp)
    pts_out = np.full((n + P, 6), np.nan, np.float32)          # every row is written: a NaN left over is a twin's bug
    box_out, cls_out = np.zeros((B, M + S, 9), np.float32), np.zeros((B, M + S), np.int32)
    accepted, count = np.zeros((B, S), np.int32), np.zeros(1, np.int32)
    check(lib().pnx_gt_sample_host(_hp(p), n, _hp(b), _hp(c), _hp(t), B, M, _hp(cb), _hp(cc), _hp(ct), S, _hp(cp), _hp(co),
                                   P, _hp(pts_out), _hp(box_out), _hp(cls_out), _hp(accepted), _hp(count)))
    return pts_out, box_out, cls_out, accepted, int(count[0])


def _sweeps_operands(points, point_offsets, sweep_points, sweep_offsets, transforms, host=False):
    B, K = transforms.shape[:2] if transforms.ndim == 4 else (len(point_offsets) - 1, 0)
    f32, i32 = torch.float32, torch.int32
    return [_want(t, dtype, shape, what, host) for t, dtype, shape, what in (
        (points, f32, (len(points), 6), "points (batch_idx, x, y, z, intensity, time)"),
        (point_offsets, i32, (B + 1,), "point_offsets"), (sweep_points, f32, (len(sweep_points), 5), "sweep_points"),
        (sweep_offsets, i32, (B * K + 1,), "sweep_offsets"), (transforms, torch.float64, (B, K, 4, 4), "transforms"))]


def accumulate_sweeps(points, point_offsets, sweep_points, sweep_offsets, transforms, min_distance):
    """Multi-sweep accumulation on the GPU (pnx_accumulate_sweeps, include/pnx.h): the reference's nuScenes / Waymo
    load_pointcloud for the sweeps scenes.collate packed (all CUDA tensors): key-frame points [n, 6] fp32 with frame f
    owning rows point_offsets[f] .. point_offsets[f + 1] - 1 ([B + 1] int32), sweep_points [S, 5] fp32 in each sweep's
    frame, sweep_offsets [B K + 1] int32 (sweep (f, k) = segment f K + k), transforms [B, K, 4, 4] fp64 (NaN [3][3] = no
    transform), min_distance (1.0 nuScenes, 0 = off) -> (points [n + S, 6], count [1] int32 cuda).  Per frame, its key
    points then its sweeps in order; the rows past `count` have batch index B, which the voxelizers drop; the host does
    not wait for the count.  The inputs are left untouched."""
    p, po, sp, so, tr = _sweeps_operands(points, point_offsets, sweep_points, sweep_offsets, transforms)
    n, S, (B, K) = len(p), len(sp), tr.shape[:2]
    dev = p.device
    pts_out = torch.empty((n + S, 6), dtype=torch.float32, device=dev)
    count = torch.empty(1, dtype=torch.int32, device=dev)
    ws = torch.empty(max(4, lib().pnx_accumulate_sweeps_workspace(S, B)), dtype=torch.uint8, device=dev)
    _count(3 if min_distance > 0 else 2)
    check(lib().pnx_accumulate_sweeps(ptr(p), n, ptr(po), B, ptr(sp), S, ptr(so), K, ptr(tr), float(min_distance),
                                      ptr(pts_out), ptr(count), ptr(ws), stream()))
    return pts_out, count


def accumulate_sweeps_host(points, point_offsets, sweep_points, sweep_offsets, transforms, min_distance):
    """Host twin of accumulate_sweeps (pnx_accumulate_sweeps_host): the same operands as numpy arrays -> (points, count),
    points a new array and count an int."""
    p, po, sp, so, tr = _sweeps_operands(points, point_offsets, sweep_points, sweep_offsets, transforms, host=True)
    n, S, (B, K) = len(p), len(sp), tr.shape[:2]
    pts_out = np.full((n + S, 6), np.nan, np.float32)           # every row is written: a NaN left over is a twin's bug
    count = np.zeros(1, np.int32)
    check(lib().pnx_accumulate_sweeps_host(_hp(p), n, _hp(po), B, _hp(sp), S, _hp(so), K, _hp(tr), float(min_distance),
                                           _hp(pts_out), _hp(count)))
    return pts_out, int(count[0])


def _row_shape(t, min_cols, what):
    """Shape (n, c) of a [n, >= min_cols] operand; raises otherwise."""
    shape = tuple(getattr(t, "shape", ()))
    if len(shape) != 2 or shape[1] < min_cols:
        raise ValueError("%s must be [n, >= %d], got shape %s" % (what, min_cols, shape))
    return shape


def _points_in_boxes_operands(points, boxes, trig, host=False):
    m = len(boxes)
    return (_want(points, torch.float32, _row_shape(points, 3, "points"), "points", host),
            _want(boxes, torch.float32, (m, 9), "boxes", host), _want(trig, torch.float32, (m, 2), "trig", host))


def points_in_boxes(points, boxes, trig):
    """The point test of gt_sample on the GPU (pnx_points_in_boxes, the reference's points_in_rbbox): points fp32
    [n, >= 3] (x, y, z first), boxes [m, 9] fp32, trig [m, 2] fp32 = libm (cosf, sinf) of each yaw, all CUDA -> inside
    [n, m] bool cuda, equal to points_in_boxes_host to the bit."""
    points, boxes, trig = _points_in_boxes_operands(points, boxes, trig)
    n, m = len(points), len(boxes)
    inside = torch.empty((n, m), dtype=torch.uint8, device=points.device)
    if n * m:
        _count(1)
    check(lib().pnx_points_in_boxes(ptr(points), n, points.shape[1], ptr(boxes), ptr(trig), m, ptr(inside), stream()))
    return inside.view(torch.bool)


def points_in_boxes_host(points, boxes, trig):
    """The point test of gt_sample on the host (pnx_points_in_boxes_host, the reference's points_in_rbbox): points numpy
    fp32 [n, >= 3] (x, y, z first), boxes [m, 9] fp32, trig [m, 2] fp32 = libm (cosf, sinf) of each yaw -> inside
    [n, m] bool."""
    points, boxes, trig = _points_in_boxes_operands(points, boxes, trig, host=True)
    m = len(boxes)
    inside = np.zeros((len(points), m), np.uint8)
    check(lib().pnx_points_in_boxes_host(_hp(points), len(points), points.shape[1], _hp(boxes), _hp(trig), m, _hp(inside)))
    return inside.astype(bool)


def aligned_iou3d(boxes_a, boxes_b):
    """[n, 7] x [n, 7] fp32 (x, y, z, dx, dy, dz, heading) -> [n] aligned 3-D IoU (iou3d_nms_utils.py:45-87)."""
    assert boxes_a.shape == boxes_b.shape and boxes_a.shape[-1] == 7 and boxes_a.is_cuda
    a, b = boxes_a.contiguous().float(), boxes_b.contiguous().float()
    out = torch.empty(a.shape[0], dtype=torch.float32, device=a.device)
    _count(1)
    check(lib().pnx_aligned_iou3d(ptr(a), ptr(b), a.shape[0], ptr(out), stream()))
    return out


def aligned_iou3d_host(a, b):
    """Host twin of aligned_iou3d (pnx_aligned_iou3d_host): numpy fp32 [n, 7] x [n, 7] -> [n] fp32."""
    return _box_pairs_host(lib().pnx_aligned_iou3d_host, a, b)


# --------------------------------------------------------------------------------- Waymo-style evaluation
def _count_points_operands(boxes, classes, trig, host=False):
    B, M = boxes.shape[:2] if boxes.ndim == 3 else (0, 0)
    return (_want(boxes, torch.float32, (B, M, 9), "boxes", host), _want(classes, torch.int32, (B, M), "classes", host),
            _want(trig, torch.float32, (B, M, 2), "trig", host))


def eval_count_points(points, boxes, classes, trig):
    """Points inside each ground-truth box (pnx_eval_count_points, include/pnx.h), with the reference's
    points_in_boxes_jit test: points [N, >= 4] fp32 (batch_idx, x, y, z, ...), boxes [B, M, 9] fp32, classes [B, M]
    int32 (-1 = padding), trig [B, M, 2] fp32 libm (cosf, sinf) of each yaw, all CUDA -> counts [B, M] int32 cuda."""
    _want(points, torch.float32, _row_shape(points, 4, "points"), "points")
    points = points if points.stride(1) == 1 else points.contiguous()
    row = points.stride(0) if points.shape[0] > 1 else points.shape[1]    # an empty or one-row tensor's stride is arbitrary
    boxes, classes, trig = _count_points_operands(boxes, classes, trig)
    B, M = classes.shape
    counts = torch.empty((B, M), dtype=torch.int32, device=boxes.device)
    _count(1)
    check(lib().pnx_eval_count_points(ptr(points), points.shape[0], row, ptr(boxes), ptr(classes), ptr(trig), B, M,
                                      ptr(counts), stream()))
    return counts


def eval_count_points_host(points, boxes, classes, trig):
    """Host twin of eval_count_points (pnx_eval_count_points_host): the same operands as numpy arrays -> counts [B, M]
    int32."""
    points = _want(points, torch.float32, _row_shape(points, 4, "points"), "points", host=True)
    boxes, classes, trig = _count_points_operands(boxes, classes, trig, host=True)
    B, M = classes.shape
    counts = np.zeros((B, M), np.int32)
    check(lib().pnx_eval_count_points_host(_hp(points), len(points), points.shape[1], _hp(boxes), _hp(classes), _hp(trig),
                                           B, M, _hp(counts)))
    return counts


def _eval_match_operands(det_boxes, det_trig, order, seg_start, seg_count, gt_boxes, gt_classes, gt_trig, thresholds,
                         host=False):
    D, C = len(det_boxes), len(thresholds)
    B, M = gt_boxes.shape[:2] if gt_boxes.ndim == 3 else (0, 0)
    f32, i32 = torch.float32, torch.int32
    return [_want(t, dtype, shape, what, host) for t, dtype, shape, what in (
        (det_boxes, f32, (D, 9), "det_boxes"), (det_trig, f32, (D, 2), "det_trig"), (order, torch.int64, (D,), "order"),
        (seg_start, i32, (B * C,), "seg_start"), (seg_count, i32, (B * C,), "seg_count"),
        (gt_boxes, f32, (B, M, 9), "gt_boxes"), (gt_classes, i32, (B, M), "gt_classes"),
        (gt_trig, f32, (B, M, 2), "gt_trig"), (thresholds, f32, (C,), "thresholds"))]


def eval_match(det_boxes, det_trig, order, seg_start, seg_count, gt_boxes, gt_classes, gt_trig, thresholds):
    """Greedy score-ordered matching per (frame, class) segment (pnx_eval_match, include/pnx.h), all CUDA:
    det_boxes [D, 9] fp32, det_trig [D, 2] fp32 (cos, sin) of each yaw, order [D] int64 (detections sorted by segment
    f C + c, then descending score, ties by lower index), seg_start / seg_count [B C] int32, gt_boxes [B, M, 9] fp32,
    gt_classes [B, M] int32 (-1 = padding), gt_trig [B, M, 2] fp32, thresholds [C] fp32 ->
    (match [D] int32 box index within the frame or -1, iou [D] fp32, heading accuracy [D] fp32)."""
    db, dt, od, ss, sc, gb, gc, gt, th = _eval_match_operands(det_boxes, det_trig, order, seg_start, seg_count, gt_boxes,
                                                              gt_classes, gt_trig, thresholds)
    D, (B, M), C = len(db), gb.shape[:2], len(th)
    dev = db.device
    match = torch.empty(D, dtype=torch.int32, device=dev)
    iou = torch.empty(D, dtype=torch.float32, device=dev)
    heading = torch.empty(D, dtype=torch.float32, device=dev)
    _count(1)
    check(lib().pnx_eval_match(ptr(db), ptr(dt), D, ptr(od), ptr(ss), ptr(sc), ptr(gb), ptr(gc), ptr(gt), B, M, C, ptr(th),
                               ptr(match), ptr(iou), ptr(heading), stream()))
    return match, iou, heading


def eval_match_host(det_boxes, det_trig, order, seg_start, seg_count, gt_boxes, gt_classes, gt_trig, thresholds):
    """Host twin of eval_match (pnx_eval_match_host): the same operands as numpy arrays -> (match, iou, heading)."""
    db, dt, od, ss, sc, gb, gc, gt, th = _eval_match_operands(det_boxes, det_trig, order, seg_start, seg_count, gt_boxes,
                                                              gt_classes, gt_trig, thresholds, host=True)
    D, (B, M), C = len(db), gb.shape[:2], len(th)
    match, iou, heading = np.zeros(D, np.int32), np.zeros(D, np.float32), np.zeros(D, np.float32)
    check(lib().pnx_eval_match_host(_hp(db), _hp(dt), D, _hp(od), _hp(ss), _hp(sc), _hp(gb), _hp(gc), _hp(gt), B, M, C,
                                    _hp(th), _hp(match), _hp(iou), _hp(heading)))
    return match, iou, heading


def eval_pairs(det_boxes, det_trig, order, seg_start, seg_count, gt_boxes, gt_classes, gt_trig, thresholds):
    """The feasible pairs (IoU >= the class threshold) of every (frame, class) segment (pnx_eval_pairs, include/pnx.h),
    operands as for eval_match, all CUDA -> (edge_start [B C] int32, e_det [E] int32 detection index, e_box [E] int32
    f M + j, e_iou [E] fp32, e_head [E] fp32 heading accuracy as eval_match's), each segment's pairs from edge_start
    on.  One count pass, one prefix sum, one host read of E, one write pass."""
    db, dt, od, ss, sc, gb, gc, gt, th = _eval_match_operands(det_boxes, det_trig, order, seg_start, seg_count, gt_boxes,
                                                              gt_classes, gt_trig, thresholds)
    D, (B, M), C = len(db), gb.shape[:2], len(th)
    dev = db.device
    count = torch.zeros(B * C, dtype=torch.int32, device=dev)
    args = (ptr(db), ptr(dt), D, ptr(od), ptr(ss), ptr(sc), ptr(gb), ptr(gc), ptr(gt), B, M, C, ptr(th))
    _count(2)
    check(lib().pnx_eval_pairs(*args, None, ptr(count), None, None, None, None, stream()))
    end = torch.cumsum(count, 0, dtype=torch.int64)
    E = int(end[-1]) if B * C else 0
    start = (end - count).to(torch.int32)
    e_det, e_box = (torch.empty(E, dtype=torch.int32, device=dev) for _ in range(2))
    e_iou, e_head = (torch.empty(E, dtype=torch.float32, device=dev) for _ in range(2))
    if E:
        check(lib().pnx_eval_pairs(*args, ptr(start), ptr(count), ptr(e_det), ptr(e_box), ptr(e_iou), ptr(e_head),
                                   stream()))
    return start, e_det, e_box, e_iou, e_head


def eval_pairs_host(det_boxes, det_trig, order, seg_start, seg_count, gt_boxes, gt_classes, gt_trig, thresholds):
    """Host twin of eval_pairs (pnx_eval_pairs_host): the same operands as numpy arrays -> the same five arrays."""
    db, dt, od, ss, sc, gb, gc, gt, th = _eval_match_operands(det_boxes, det_trig, order, seg_start, seg_count, gt_boxes,
                                                              gt_classes, gt_trig, thresholds, host=True)
    D, (B, M), C = len(db), gb.shape[:2], len(th)
    count = np.zeros(B * C, np.int32)
    args = (_hp(db), _hp(dt), D, _hp(od), _hp(ss), _hp(sc), _hp(gb), _hp(gc), _hp(gt), B, M, C, _hp(th))
    check(lib().pnx_eval_pairs_host(*args, None, _hp(count), None, None, None, None))
    start = (np.cumsum(count, dtype=np.int64) - count).astype(np.int32)
    E = int(count.sum(dtype=np.int64))
    e_det, e_box = np.zeros(E, np.int32), np.zeros(E, np.int32)
    e_iou, e_head = np.zeros(E, np.float32), np.zeros(E, np.float32)
    if E:
        check(lib().pnx_eval_pairs_host(*args, _hp(start), _hp(count), _hp(e_det), _hp(e_box), _hp(e_iou), _hp(e_head)))
    return start, e_det, e_box, e_iou, e_head


def _eval_components_operands(edge_start, e_det, e_box, host=False):
    E = len(e_det)
    i32 = torch.int32
    return [_want(t, i32, shape, what, host) for t, shape, what in (
        (edge_start, (len(edge_start),), "edge_start"), (e_det, (E,), "e_det"), (e_box, (E,), "e_box"))]


def _edge_count(start, E):
    """Pairs per segment from the segments' first pair and the total E."""
    if isinstance(start, np.ndarray):
        return (np.append(start[1:], E) - start).astype(np.int32)
    return (torch.cat([start[1:], start.new_full((1,), E)]) - start).to(torch.int32)


def eval_components(edge_start, e_det, e_box, M, n_classes):
    """Connected components of each segment's feasible pairs (pnx_eval_components, include/pnx.h), all CUDA:
    edge_start [B C] int32 and e_det / e_box [E] int32 of eval_pairs, M boxes per frame, C = n_classes ->
    (comp_start [E] int32, comp_nedge [E] int32, grouped [E] int32): for each component's first pair, where its pairs
    begin in grouped and how many there are; -1 and 0 for every other pair."""
    st, ed, eb = _eval_components_operands(edge_start, e_det, e_box)
    E, C = len(ed), int(n_classes)
    B = len(st) // C
    count = _edge_count(st, E)
    root, comp_start, comp_nedge, grouped = (torch.empty(E, dtype=torch.int32, device=ed.device) for _ in range(4))
    _count(1)
    check(lib().pnx_eval_components(ptr(st), ptr(count), B, int(M), C, E, ptr(ed), ptr(eb), ptr(root), ptr(comp_start),
                                    ptr(comp_nedge), ptr(grouped), stream()))
    return comp_start, comp_nedge, grouped


def eval_components_host(edge_start, e_det, e_box, M, n_classes):
    """Host twin of eval_components (pnx_eval_components_host): numpy in, numpy out."""
    st, ed, eb = _eval_components_operands(edge_start, e_det, e_box, host=True)
    E, C = len(ed), int(n_classes)
    B = len(st) // C
    count = _edge_count(st, E)
    root, comp_start, comp_nedge, grouped = (np.zeros(E, np.int32) for _ in range(4))
    check(lib().pnx_eval_components_host(_hp(st), _hp(count), B, int(M), C, E, _hp(ed), _hp(eb), _hp(root),
                                         _hp(comp_start), _hp(comp_nedge), _hp(grouped)))
    return comp_start, comp_nedge, grouped


def _eval_assign_operands(grouped, comp_start, comp_nedge, e_det, e_box, e_iou, e_head, det_pass, det_range, gt_range,
                          host=False):
    E, D = len(e_det), len(det_pass)
    f32, i32 = torch.float32, torch.int32
    return [_want(t, dtype, shape, what, host) for t, dtype, shape, what in (
        (grouped, i32, (E,), "grouped"), (comp_start, i32, (E,), "comp_start"), (comp_nedge, i32, (E,), "comp_nedge"),
        (e_det, i32, (E,), "e_det"), (e_box, i32, (E,), "e_box"), (e_iou, f32, (E,), "e_iou"),
        (e_head, f32, (E,), "e_head"), (det_pass, i32, (D,), "det_pass"), (det_range, i32, (D,), "det_range"),
        (gt_range, i32, (len(gt_range),), "gt_range"))]


def _component_lists(comp_nedge, xp):
    """Roots of the components the one-warp solver takes, roots of the larger ones, the larger ones' exclusive prefix
    sum of pairs (their workspace offsets) and their total.  xp = torch or numpy."""
    warp = lib().pnx_eval_assign_warp_pairs()
    if xp is torch:
        small = torch.nonzero((comp_nedge > 0) & (comp_nedge <= warp)).view(-1).to(torch.int32)
        large = torch.nonzero(comp_nedge > warp).view(-1)
        n = comp_nedge[large].to(torch.int64)
        end = torch.cumsum(n, 0)
        return small, large.to(torch.int32), end - n, int(end[-1]) if len(n) else 0
    small = np.nonzero((comp_nedge > 0) & (comp_nedge <= warp))[0].astype(np.int32)
    large = np.nonzero(comp_nedge > warp)[0]
    n = comp_nedge[large].astype(np.int64)
    return small, large.astype(np.int32), np.cumsum(n) - n, int(n.sum())


def eval_assign(grouped, comp_start, comp_nedge, e_det, e_box, e_iou, e_head, det_pass, det_range, gt_range, M, K):
    """Maximum-IoU assignment of every component, per breakdown and score cutoff (pnx_eval_assign, include/pnx.h), all
    CUDA: the pairs and components of eval_pairs / eval_components, det_pass [D] int32 (cutoffs each detection passes),
    det_range [D] and gt_range [B M] int32 range bins, M, K cutoffs -> (match [2, K, D] int32, the box index within the
    frame or -1; heading [2, K, D] fp32, the matched pair's e_head or 0), breakdown 0: all pairs; 1: pairs within one
    range bin.  The components are listed by size on the device (one host read of the counts), and only the larger
    ones get workspace."""
    ops_ = _eval_assign_operands(grouped, comp_start, comp_nedge, e_det, e_box, e_iou, e_head, det_pass, det_range,
                                 gt_range)
    E, D = len(ops_[3]), len(ops_[7])
    dev = ops_[7].device
    small, large, large_off, large_pairs = _component_lists(ops_[2], torch)
    match = torch.empty((2, int(K), D), dtype=torch.int32, device=dev)
    heading = torch.empty((2, int(K), D), dtype=torch.float32, device=dev)
    ws = torch.empty(max(1, lib().pnx_eval_assign_workspace(large_pairs)), dtype=torch.uint8, device=dev)
    _count(2)
    check(lib().pnx_eval_assign(E, *[ptr(t) for t in ops_[:7]], ptr(small), len(small), ptr(large), ptr(large_off),
                                len(large), large_pairs, D, *[ptr(t) for t in ops_[7:]], int(M), int(K), ptr(match),
                                ptr(heading), ptr(ws), stream()))
    return match, heading


def eval_assign_host(grouped, comp_start, comp_nedge, e_det, e_box, e_iou, e_head, det_pass, det_range, gt_range, M, K):
    """Host twin of eval_assign (pnx_eval_assign_host): numpy in -> (match [2, K, D] int32, heading [2, K, D] fp32)."""
    ops_ = _eval_assign_operands(grouped, comp_start, comp_nedge, e_det, e_box, e_iou, e_head, det_pass, det_range,
                                 gt_range, host=True)
    E, D = len(ops_[3]), len(ops_[7])
    small, large, large_off, large_pairs = _component_lists(ops_[2], np)
    match, heading = np.zeros((2, int(K), D), np.int32), np.zeros((2, int(K), D), np.float32)
    check(lib().pnx_eval_assign_host(E, *[_hp(t) for t in ops_[:7]], _hp(small), len(small), _hp(large),
                                     _hp(large_off), len(large), large_pairs, D, *[_hp(t) for t in ops_[7:]], int(M),
                                     int(K), _hp(match), _hp(heading)))
    return match, heading


# --------------------------------------------------------------------------------- nuScenes detection score
def _eval_match_center_operands(det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes, n_classes, dist_ths,
                                host=False):
    D, T, C = len(det_boxes), len(dist_ths), int(n_classes)
    B, M = gt_boxes.shape[:2] if gt_boxes.ndim == 3 else (0, 0)
    f32, i32 = torch.float32, torch.int32
    return [_want(t, dtype, shape, what, host) for t, dtype, shape, what in (
        (det_boxes, f32, (D, 9), "det_boxes"), (order, torch.int64, (D,), "order"),
        (seg_start, i32, (B * C,), "seg_start"), (seg_count, i32, (B * C,), "seg_count"),
        (gt_boxes, f32, (B, M, 9), "gt_boxes"), (gt_classes, i32, (B, M), "gt_classes"),
        (dist_ths, torch.float64, (T,), "dist_ths"))]


def eval_match_center(det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes, n_classes, dist_ths):
    """Centre-distance matching per (frame, class) segment and distance threshold (pnx_eval_match_center,
    include/pnx.h), all CUDA: det_boxes [D, 9] fp32, order [D] int64 (detections sorted by segment f C + c, then in
    visit order), seg_start / seg_count [B C] int32, gt_boxes [B, M, 9] fp32, gt_classes [B, M] int32 in [0, C) (-1 =
    padding or filtered out), C = n_classes, dist_ths [T] fp64 -> match [T, D] int32, the box index within the frame
    or -1."""
    db, od, ss, sc, gb, gc, th = _eval_match_center_operands(det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes,
                                                             n_classes, dist_ths)
    D, (B, M), T, C = len(db), gb.shape[:2], len(th), int(n_classes)
    match = torch.empty((T, D), dtype=torch.int32, device=db.device)
    _count(1)
    check(lib().pnx_eval_match_center(ptr(db), D, ptr(od), ptr(ss), ptr(sc), ptr(gb), ptr(gc), B, M, C, ptr(th), T,
                                      ptr(match), stream()))
    return match


def eval_match_center_host(det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes, n_classes, dist_ths):
    """Host twin of eval_match_center (pnx_eval_match_center_host): the same operands as numpy arrays -> match [T, D]
    int32."""
    db, od, ss, sc, gb, gc, th = _eval_match_center_operands(det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes,
                                                             n_classes, dist_ths, host=True)
    D, (B, M), T, C = len(db), gb.shape[:2], len(th), int(n_classes)
    match = np.zeros((T, D), np.int32)
    check(lib().pnx_eval_match_center_host(_hp(db), D, _hp(od), _hp(ss), _hp(sc), _hp(gb), _hp(gc), B, M, C, _hp(th), T,
                                           _hp(match)))
    return match


# --------------------------------------------------------------------------------- tracking
def _track_operands(boxes, scores, order, seg_start, seg_count, poses, times, seq_start, max_dist, host=False):
    D, F, C = len(boxes), len(poses), len(max_dist)
    f32, i32, i64 = torch.float32, torch.int32, torch.int64
    return [_want(t, dtype, shape, what, host) for t, dtype, shape, what in (
        (boxes, f32, (D, 9), "boxes"), (scores, f32, (D,), "scores"), (order, i64, (D,), "order"),
        (seg_start, i32, (F * C,), "seg_start"), (seg_count, i32, (F * C,), "seg_count"),
        (poses, torch.float64, (F, 4, 4), "poses"), (times, i64, (F,), "times"),
        (seq_start, i32, (len(seq_start),), "seq_start"), (max_dist, f32, (C,), "max_dist"))]


def _track_status(status, C):
    if status:
        raise ValueError("sequence %d, class %d: more than %d live tracks at once" %
                         ((status - 1) // C, (status - 1) % C, lib().pnx_track_max_tracks()))


def track_greedy(boxes, scores, order, seg_start, seg_count, poses, times, seq_start, max_dist, max_age, min_score):
    """The greedy velocity tracker (pnx_track_greedy, include/pnx.h), all CUDA: boxes [D, 9] fp32, scores [D] fp32,
    order [D] int64 (by segment f C + c, then descending score), seg_start / seg_count [F C] int32, poses [F, 4, 4]
    fp64, times [F] int64 microseconds, seq_start [S + 1] int32, max_dist [C] fp32 -> track_id [D] int64 (-1 below
    min_score).  Reads the largest segment and one status word back: raises ValueError when a (sequence, class)
    exceeds the track capacity."""
    ops_ = _track_operands(boxes, scores, order, seg_start, seg_count, poses, times, seq_start, max_dist)
    D, F, C, S = len(ops_[0]), len(ops_[5]), len(ops_[8]), len(ops_[7]) - 1
    dev = ops_[0].device
    per_row = torch.zeros(S * C + 1, dtype=torch.int64, device=dev)
    if D:
        seq_of_frame = torch.repeat_interleave(torch.arange(S, device=dev), (ops_[7][1:] - ops_[7][:-1]).long(),
                                               output_size=F)
        row_of_seg = (seq_of_frame[:, None] * C + torch.arange(C, device=dev)).view(-1)
        per_row.index_add_(0, row_of_seg + 1, ops_[4].long())
    row_det_start = torch.cumsum(per_row, 0)[:-1].contiguous()
    local_id, scratch = (torch.empty(max(D, 1), dtype=torch.int32, device=dev) for _ in range(2))
    births = torch.empty(max(S * C, 1), dtype=torch.int32, device=dev)
    track_id = torch.empty(D, dtype=torch.int64, device=dev)
    status = torch.empty(1, dtype=torch.int32, device=dev)
    # slots enough for every track that can be live (matched or born in the last max_age + 1 frames, plus this
    # frame's births), at most the library's capacity: a smaller table keeps more warps per SM
    cap = min(lib().pnx_track_max_tracks(), (int(max_age) + 2) * max(1, int(ops_[4].max()) if F * C else 1))
    _count(2)
    check(lib().pnx_track_greedy(ptr(ops_[0]), ptr(ops_[1]), D, *[ptr(t) for t in ops_[2:8]], S, F, C, ptr(ops_[8]),
                                 int(max_age), float(min_score), cap, ptr(row_det_start), ptr(local_id), ptr(births),
                                 ptr(scratch), ptr(track_id), ptr(status), stream()))
    _track_status(int(status.item()), C)
    return track_id


def track_greedy_host(boxes, scores, order, seg_start, seg_count, poses, times, seq_start, max_dist, max_age, min_score):
    """Host twin of track_greedy (pnx_track_greedy_host): the same operands as numpy arrays -> track_id [D] int64."""
    ops_ = _track_operands(boxes, scores, order, seg_start, seg_count, poses, times, seq_start, max_dist, host=True)
    D, F, C, S = len(ops_[0]), len(ops_[5]), len(ops_[8]), len(ops_[7]) - 1
    track_id, status = np.zeros(D, np.int64), np.zeros(1, np.int32)
    check(lib().pnx_track_greedy_host(_hp(ops_[0]), _hp(ops_[1]), D, *[_hp(t) for t in ops_[2:8]], S, F, C,
                                      _hp(ops_[8]), int(max_age), float(min_score), _hp(track_id), _hp(status)))
    _track_status(int(status[0]), C)
    return track_id


def _eval_mot_operands(edge_start, e_det, e_box, e_iou, grouped, comp_start, comp_nedge, det_pass, det_id, gt_obj,
                       gt_points, seq_start, host=False):
    E, D, BM = len(e_det), len(det_pass), len(gt_obj)
    i32 = torch.int32
    return [_want(t, dtype, shape, what, host) for t, dtype, shape, what in (
        (edge_start, i32, (len(edge_start),), "edge_start"), (grouped, i32, (E,), "grouped"),
        (comp_start, i32, (E,), "comp_start"), (comp_nedge, i32, (E,), "comp_nedge"), (e_det, i32, (E,), "e_det"),
        (e_box, i32, (E,), "e_box"), (e_iou, torch.float32, (E,), "e_iou"), (det_pass, i32, (D,), "det_pass"),
        (det_id, i32, (D,), "det_id"), (gt_obj, i32, (BM,), "gt_obj"), (gt_points, i32, (BM,), "gt_points"),
        (seq_start, i32, (len(seq_start),), "seq_start"))]


def _mot_cap(comp_nedge):
    """Pairs one row's assignment state must hold: the largest component, at least the one-warp size + 2."""
    big = int(comp_nedge.max()) if len(comp_nedge) else 0
    return max(big, lib().pnx_eval_assign_warp_pairs() + 2)


def eval_mot(edge_start, e_det, e_box, e_iou, grouped, comp_start, comp_nedge, det_pass, det_id, gt_obj, gt_points,
             seq_start, M, n_classes, K, n_obj):
    """CLEAR-MOT frame matching per (sequence, class, cutoff) (pnx_eval_mot, include/pnx.h), all CUDA: the pairs of
    eval_pairs, the components of eval_components, det_pass / det_id [D] int32, gt_obj / gt_points [B M] int32,
    seq_start [S + 1] int32 -> (counts [S, C, K, 5] int64, dist [S, C, K, 2] fp64).  One host read (the largest
    component) sizes the workspace: every (sequence, class, cutoff) row gets 164 B per pair of the largest component
    anywhere plus 4 B per box slot, so S C K (164 cap + 4 M) bytes in all (Waymo val: 6600 rows, 37 MB at the
    one-warp minimum of 34 pairs; a crowd component of 2000 pairs would take 2.2 GB)."""
    ops_ = _eval_mot_operands(edge_start, e_det, e_box, e_iou, grouped, comp_start, comp_nedge, det_pass, det_id,
                              gt_obj, gt_points, seq_start)
    st = ops_[0]
    E, D, S, C, B = len(ops_[4]), len(ops_[7]), len(ops_[11]) - 1, int(n_classes), len(st) // int(n_classes)
    dev = st.device
    cap = _mot_cap(ops_[3])
    count = _edge_count(st, E)
    counts = torch.empty((S, C, int(K), 5), dtype=torch.int64, device=dev)
    dist = torch.empty((S, C, int(K), 2), dtype=torch.float64, device=dev)
    last_id = torch.empty(max(1, int(K) * int(n_obj)), dtype=torch.int32, device=dev)
    ws = torch.empty(max(1, lib().pnx_eval_mot_workspace(S * C * int(K), int(M), cap)), dtype=torch.uint8, device=dev)
    _count(1)
    check(lib().pnx_eval_mot(ptr(st), ptr(count), E, *[ptr(t) for t in ops_[1:7]], D,
                             *[ptr(t) for t in ops_[7:]], S, B, int(M), C, int(K), int(n_obj), cap, ptr(last_id),
                             ptr(counts), ptr(dist), ptr(ws), stream()))
    return counts, dist


def eval_mot_host(edge_start, e_det, e_box, e_iou, grouped, comp_start, comp_nedge, det_pass, det_id, gt_obj,
                  gt_points, seq_start, M, n_classes, K, n_obj):
    """Host twin of eval_mot (pnx_eval_mot_host): numpy in -> (counts [S, C, K, 5] int64, dist [S, C, K, 2] fp64)."""
    ops_ = _eval_mot_operands(edge_start, e_det, e_box, e_iou, grouped, comp_start, comp_nedge, det_pass, det_id,
                              gt_obj, gt_points, seq_start, host=True)
    st = ops_[0]
    E, D, S, C, B = len(ops_[4]), len(ops_[7]), len(ops_[11]) - 1, int(n_classes), len(st) // int(n_classes)
    cap = _mot_cap(ops_[3])
    count = _edge_count(st, E)
    counts, dist = np.zeros((S, C, int(K), 5), np.int64), np.zeros((S, C, int(K), 2), np.float64)
    last_id = np.zeros(max(1, int(K) * int(n_obj)), np.int32)
    check(lib().pnx_eval_mot_host(_hp(st), _hp(count), E, *[_hp(t) for t in ops_[1:7]], D,
                                  *[_hp(t) for t in ops_[7:]], S, B, int(M), C, int(K), int(n_obj), cap,
                                  _hp(last_id), _hp(counts), _hp(dist)))
    return counts, dist


# --------------------------------------------------------------------------------- nuScenes tracking
def _eval_pairs_center_operands(det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes, n_classes, host=False):
    D, C = len(det_boxes), int(n_classes)
    B, M = gt_boxes.shape[:2] if gt_boxes.ndim == 3 else (0, 0)
    f32, i32 = torch.float32, torch.int32
    return [_want(t, dtype, shape, what, host) for t, dtype, shape, what in (
        (det_boxes, f32, (D, 9), "det_boxes"), (order, torch.int64, (D,), "order"),
        (seg_start, i32, (B * C,), "seg_start"), (seg_count, i32, (B * C,), "seg_count"),
        (gt_boxes, f32, (B, M, 9), "gt_boxes"), (gt_classes, i32, (B, M), "gt_classes"))]


def eval_pairs_center(det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes, n_classes, max_dist):
    """The pairs of every (frame, class) segment with centre distance < max_dist (pnx_eval_pairs_center,
    include/pnx.h), operands as for eval_match_center, all CUDA -> (edge_start [B C] int32, e_det [E] int32, e_box [E]
    int32 f M + j, e_dist [E] fp32).  One count pass, one prefix sum, one host read of E, one write pass."""
    db, od, ss, sc, gb, gc = _eval_pairs_center_operands(det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes,
                                                         n_classes)
    D, (B, M), C = len(db), gb.shape[:2], int(n_classes)
    dev = db.device
    count = torch.zeros(B * C, dtype=torch.int32, device=dev)
    args = (ptr(db), D, ptr(od), ptr(ss), ptr(sc), ptr(gb), ptr(gc), B, M, C, float(max_dist))
    _count(2)
    check(lib().pnx_eval_pairs_center(*args, None, ptr(count), None, None, None, stream()))
    end = torch.cumsum(count, 0, dtype=torch.int64)
    E = int(end[-1]) if B * C else 0
    start = (end - count).to(torch.int32)
    e_det, e_box = (torch.empty(E, dtype=torch.int32, device=dev) for _ in range(2))
    e_dist = torch.empty(E, dtype=torch.float32, device=dev)
    if E:
        check(lib().pnx_eval_pairs_center(*args, ptr(start), ptr(count), ptr(e_det), ptr(e_box), ptr(e_dist), stream()))
    return start, e_det, e_box, e_dist


def eval_pairs_center_host(det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes, n_classes, max_dist):
    """Host twin of eval_pairs_center (pnx_eval_pairs_center_host): numpy in -> the same four arrays."""
    db, od, ss, sc, gb, gc = _eval_pairs_center_operands(det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes,
                                                         n_classes, host=True)
    D, (B, M), C = len(db), gb.shape[:2], int(n_classes)
    count = np.zeros(B * C, np.int32)
    args = (_hp(db), D, _hp(od), _hp(ss), _hp(sc), _hp(gb), _hp(gc), B, M, C, float(max_dist))
    check(lib().pnx_eval_pairs_center_host(*args, None, _hp(count), None, None, None))
    start = (np.cumsum(count, dtype=np.int64) - count).astype(np.int32)
    E = int(count.sum(dtype=np.int64))
    e_det, e_box, e_dist = np.zeros(E, np.int32), np.zeros(E, np.int32), np.zeros(E, np.float32)
    if E:
        check(lib().pnx_eval_pairs_center_host(*args, _hp(start), _hp(count), _hp(e_det), _hp(e_box), _hp(e_dist)))
    return start, e_det, e_box, e_dist


def eval_mot_center(edge_start, e_det, e_box, e_dist, grouped, comp_start, comp_nedge, det_pass, det_id, gt_obj,
                    gt_prev, seq_start, M, n_classes, K, n_obj, want_matched=False):
    """nuScenes tracking's frame matching per (scene, class, cutoff) (pnx_eval_mot_center, include/pnx.h), all CUDA:
    the pairs of eval_pairs_center, the components of eval_components, det_pass / det_id [D] int32, gt_obj / gt_prev
    [B M] int32, seq_start [S + 1] int32 -> (counts [S, C, K, 3] int64 matches / identity switches / fragmentations,
    dist [S, C, K] fp64, matched [D] uint8 or None).  want_matched needs K = 1.  The workspace is eval_mot's: every
    (scene, class, cutoff) row gets 164 B per pair of the largest component anywhere plus 4 B per box slot, S C K (164
    cap + 4 M) bytes (nuScenes val shape, 150 x 7 x 40 = 42,000 rows: a largest component of 159 pairs takes 1.1 GB; it
    grows linearly with the densest crowd of detections, 14 GB at 2000 pairs)."""
    ops_ = _eval_mot_operands(edge_start, e_det, e_box, e_dist, grouped, comp_start, comp_nedge, det_pass, det_id,
                              gt_obj, gt_prev, seq_start)
    st = ops_[0]
    E, D, S, C, B = len(ops_[4]), len(ops_[7]), len(ops_[11]) - 1, int(n_classes), len(st) // int(n_classes)
    dev = st.device
    cap = _mot_cap(ops_[3])
    count = _edge_count(st, E)
    counts = torch.empty((S, C, int(K), 3), dtype=torch.int64, device=dev)
    dist = torch.empty((S, C, int(K)), dtype=torch.float64, device=dev)
    last_id, last_frame = (torch.empty(max(1, int(K) * int(n_obj)), dtype=torch.int32, device=dev) for _ in range(2))
    matched = torch.empty(D, dtype=torch.uint8, device=dev) if want_matched else None
    ws = torch.empty(max(1, lib().pnx_eval_mot_workspace(S * C * int(K), int(M), cap)), dtype=torch.uint8, device=dev)
    _count(1)
    check(lib().pnx_eval_mot_center(ptr(st), ptr(count), E, *[ptr(t) for t in ops_[1:7]], D,
                                    *[ptr(t) for t in ops_[7:]], S, B, int(M), C, int(K), int(n_obj), cap,
                                    ptr(last_id), ptr(last_frame), ptr(counts), ptr(dist), ptr(matched), ptr(ws),
                                    stream()))
    return counts, dist, matched


def eval_mot_center_host(edge_start, e_det, e_box, e_dist, grouped, comp_start, comp_nedge, det_pass, det_id, gt_obj,
                         gt_prev, seq_start, M, n_classes, K, n_obj, want_matched=False):
    """Host twin of eval_mot_center (pnx_eval_mot_center_host): numpy in -> (counts, dist, matched or None)."""
    ops_ = _eval_mot_operands(edge_start, e_det, e_box, e_dist, grouped, comp_start, comp_nedge, det_pass, det_id,
                              gt_obj, gt_prev, seq_start, host=True)
    st = ops_[0]
    E, D, S, C, B = len(ops_[4]), len(ops_[7]), len(ops_[11]) - 1, int(n_classes), len(st) // int(n_classes)
    cap = _mot_cap(ops_[3])
    count = _edge_count(st, E)
    counts, dist = np.zeros((S, C, int(K), 3), np.int64), np.zeros((S, C, int(K)), np.float64)
    last_id, last_frame = (np.zeros(max(1, int(K) * int(n_obj)), np.int32) for _ in range(2))
    matched = np.zeros(D, np.uint8) if want_matched else None
    check(lib().pnx_eval_mot_center_host(_hp(st), _hp(count), E, *[_hp(t) for t in ops_[1:7]], D,
                                         *[_hp(t) for t in ops_[7:]], S, B, int(M), C, int(K), int(n_obj), cap,
                                         _hp(last_id), _hp(last_frame), _hp(counts), _hp(dist),
                                         None if matched is None else _hp(matched)))
    return counts, dist, matched
