"""Every BatchNorm, row-wise, stencil and loss kernel launch of a production training step, replayed at its production
launch configuration against a float64 reference.

One bf16 training step of the bench model (nusc: 6 frames, waymo180k: 3 frames) and one eval-mode forward (nusc) run
with the library handle (`_lib.lib`, `ops.lib`) replaced by a proxy.  For the entry points in ARG_MAPS the proxy keeps
the scalars of each call (M, C, every leading dimension, flags, counts, eps / momentum, offsets, geometry) and whether
each pointer argument is null, never an operand, and passes the call through; it also notes every other `pnx_*` entry
point the step calls.  Each unique configuration is then replayed on fresh operands with the recorded leading
dimensions, and once more with each operand's leading dimension widened by a different multiple of 8 elements (a
stride mix-up between operands then reads the wrong rows).  Every operand buffer carries GUARD_ROWS rows past M, and
columns past C when its leading dimension leaves room, filled with a NaN sentinel: a read there shows as a NaN in the
result, a write there as a changed sentinel.  Every comparison fails on a NaN (test_self_check_a_nan_in_a_kernel_output
checks each one).

What is compared:
- add_relu / relu_bwd / add_rows and tap_scatter: bit for bit against torch (fp32 sum or gate, then bf16 rounding).
- tap_gather_sum: bit for bit on small-integer Z and bias (every fp32 sum exact).
- bn_apply and bn_bwd_apply's dx: within one bf16 ulp of the fp64 result, plus the fp32 evaluation floor of the kernel's
  folded coefficients; the fraction of elements that are not the fp64 result rounded to bf16 is bounded.  dres exact.
- bn_bwd_reduce: bit for bit on small-integer dy / x / y, where every fp32 and fp64 sum is exact (one missing row
  fails); and on bf16 Gaussian inputs against fp64, within the worst-case bound of an fp32 sum of L terms
  (L = rows one thread accumulates): |err(sum g)| <= (L + 1) u sum|g| and
  |err(sum g xhat)| <= (L + 1) u invstd (sum|g x| + |mean| sum|g|), u = 2^-24.
- bn_finalize / bn_eval_affine: the torch BatchNorm formulas in fp64 (running statistics with both BatchNorm families'
  eps / momentum, and n = 1).
- the fused CenterPoint loss at the production map and label shapes, with edge cases injected, against
  oracle.pillarnext_oracle.center_loss in float64; the loss finalize against its formula.

Every BatchNorm replay gives a few channels |mean| / std up to 30 ("large-mean channels"), where the raw-moment reduce
and the E[x^2] - mean^2 variance cancel; their error relative to the centred quantity is reported next to what bf16
storage of x already costs there, and must stay below it."""
import ctypes
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from pillarnext_b200 import _lib, modules, ops, synth
from pillarnext_b200 import functional as Fn

pytestmark = pytest.mark.gpu

GUARD_ROWS = 64
CHUNK_BYTES = 1 << 28                    # fp64 reference temporaries per row chunk
SENT = {torch.bfloat16: (torch.int16, 0x7FC1), torch.float32: (torch.int32, 0x7FC00001)}   # NaNs no kernel produces
U = 2.0 ** -24
LARGE_MEAN = (30.0, -30.0, 10.0, -3.0)   # |mean| / std of the large-mean channels

# Argument names and ctypes kinds (P pointer, I int, L long long, F float, D double) of the recorded entry points, in the
# order of include/pnx.h.  tests/test_rowwise_recorder_cpu.py checks them against _lib._SIGS.
ARG_MAPS = {
    "pnx_bn_finalize": "stats:P channels:I count_ptr:P count_mult:L gamma:P beta:P eps:F momentum:F running_mean:P running_var:P "
                       "scale:P shift:P mean_out:P invstd_out:P stream:P",
    "pnx_bn_eval_affine": "channels:I gamma:P beta:P running_mean:P running_var:P eps:F scale:P shift:P stream:P",
    "pnx_bn_apply": "x:P ldx:L M:L C:I scale:P shift:P res:P ldr:L relu:I y:P ldy:L stream:P",
    "pnx_bn_bwd_reduce": "dy:P lddy:L y:P ldy:L x:P ldx:L M:L C:I mean:P invstd:P relu:I fscale:P fshift:P red:P stream:P",
    "pnx_bn_bwd_apply": "dy:P lddy:L y:P ldy:L x:P ldx:L M:L C:I mean:P invstd:P gamma:P red:P count:D count_dev:P relu:I "
                        "fscale:P fshift:P dx:P lddx:L dres:P lddres:L dres_accumulate:I stream:P",
    "pnx_add_rows": "a:P lda:L b:P ldb:L M:L C:I stream:P",
    "pnx_add_relu": "a:P lda:L b:P ldb:L M:L C:I y:P ldy:L stream:P",
    "pnx_relu_bwd": "dy:P lddy:L y:P ldy:L M:L C:I g:P ldg:L accumulate:I stream:P",
    "pnx_tap_gather_sum": "Z:P ldz:L cpt:I bias16:P B:I H:I W:I out:P stream:P",
    "pnx_tap_scatter": "dout:P B:I H:I W:I dZ:P ldz:L nz:I cpt:I lo_off:L stream:P",
    "pnx_center_loss_task": "out:P dout:P hm_gt:P anno:P ind:P mask:P cat:P gt_boxes:P B:I H:I W:I npad:I C:I M:I "
                            "off_reg:I off_height:I off_dim:I off_rot:I off_vel:I off_hm:I sx:F sy:F ox:F oy:F weight:F "
                            "code_w_host:P with_iou:I acc:P stream:P",
    "pnx_center_loss_finalize": "acc:P n_tasks:I weights_dev:P code_w_dev:P with_iou_dev:P res:P total:P stream:P",
}


def arg_map(name):
    return [tuple(a.split(":")) for a in ARG_MAPS[name].split()]


GEMM_REPLAYED = {"pnx_igemm", "pnx_conv3x3_win", "pnx_wgrad"}       # tests/test_production_gemms_gpu.py
EXCLUDED = {
    **dict.fromkeys(("pnx_voxelize", "pnx_voxelize_frames", "pnx_bucketize"),
                    "voxelizer at the bench's shapes: tests/test_production_frontend_gpu.py"),
    **dict.fromkeys(("pnx_sites_dilate", "pnx_scan_blocks", "pnx_sites_coords", "pnx_nbr_table", "pnx_scatter_dense"),
                    "sparse rulebook and densify of the recorded pyramids: tests/test_production_frontend_gpu.py"),
    **dict.fromkeys(("pnx_pfn_mean", "pnx_pfn_lin0", "pnx_pfn_max0", "pnx_pfn_lin1", "pnx_pfn_max1", "pnx_pfn_backward"),
                    "PillarFeatureNet against float64 at the bench's shapes: tests/test_production_frontend_gpu.py"),
    "pnx_pack_weights": "weight repack after AdamW: tests/test_production_frontend_gpu.py",
    "pnx_assign_labels": "label assignment at the e2e shapes: tests/test_production_frontend_gpu.py",
    "pnx_aligned_iou3d": "IoU target of the Waymo `iou` head loss: tests/test_production_frontend_gpu.py",
    "pnx_scan_u32": "called inside pnx_bucketize (tests/test_production_frontend_gpu.py); launches nothing of its own here",
    **dict.fromkeys(("pnx_voxelize_frames_scratch", "pnx_voxelize_frames_supported", "pnx_voxelize_bitmap_words",
                     "pnx_blockcnt_size", "pnx_sites_out_dim"), "host-side size / geometry query; launches nothing"),
    "pnx_sites_inblock": "not called by the step (the voxelizer writes level 0's inblk): tests/test_rulebook_gpu.py",
    "pnx_wgrad_splits": "host-side query of the weight-gradient split count; launches nothing",
    "pnx_set_deterministic": "mode switch; launches nothing",
    "pnx_split_get_pieces": "mode query of the split precision path; launches nothing",
    "pnx_last_error": "error string of a failed call",
    "pnx_abi_version": "version query; launches nothing",
    "pnx_sm_count": "device query; launches nothing",
}


# ------------------------------------------------------------------------------------------------- recording
class Recorder:
    """The library handle's proxy: keeps one record per unique configuration of the entry points in `maps` (default
    ARG_MAPS); `extra(name)`, when given, adds fields of the library's state at the call to the configuration."""

    def __init__(self, real, maps=None, extra=None):
        self.real, self.configs, self.keys, self.called, self.source = real, [], {}, set(), ""
        self.maps, self.extra = ARG_MAPS if maps is None else maps, extra

    def _add(self, name, args):
        spec = [tuple(a.split(":")) for a in self.maps[name].split()]
        assert len(args) == len(spec), (name, len(args))
        cfg = {"fn": name}
        if self.extra is not None:
            cfg.update(self.extra(name))
        for (arg, kind), v in zip(spec, args):
            if arg == "stream":
                continue
            if kind == "P":
                cfg[arg] = v is not None and v != 0
            elif kind == "F":
                cfg[arg] = float(np.float32(v))                # the value the kernel sees
            else:
                cfg[arg] = v.value if hasattr(v, "value") else v
        key = tuple(sorted(cfg.items()))
        if key in self.keys:
            self.keys[key]["calls"] += 1
            return
        cfg["calls"], cfg["source"] = 1, self.source
        self.keys[key] = cfg
        self.configs.append(cfg)

    def proxy(self):
        rec = self

        class Proxy:
            def __getattr__(self, name):
                fn = getattr(rec.real, name)
                if not name.startswith("pnx_"):
                    return fn
                rec.called.add(name)
                if name not in rec.maps:
                    return fn

                def call(*args):
                    rec._add(name, args)
                    return fn(*args)
                return call
        return Proxy()


def _to_dev(ex, dev):
    return {k: ([e.to(dev) for e in v] if isinstance(v, list) and v and torch.is_tensor(v[0]) else
                (v.to(dev) if torch.is_tensor(v) else v)) for k, v in ex.items()}


def _record(rec, name, evaluate):
    dev = torch.device("cuda", torch.cuda.current_device())
    sel = synth.BENCH_CONFIGS[name]
    cfg = sel["cfg"]
    torch.manual_seed(0)
    model = modules.build_pillarnext_b(cfg).to(dev).train()
    ex = _to_dev(synth.make_batch(list(range(cfg["frames_per_gpu"])), sel["points"], cfg, kind="lidar", n_boxes=40,
                                  sweeps=sel["sweeps"], rings=sel["rings"]), dev)
    rec.source = name + " train"
    loss, _ = model(ex)
    loss.backward()
    if evaluate:
        rec.source = name + " eval"
        model.eval()
        with torch.no_grad():
            model._forward(ex)
    torch.cuda.synchronize()
    del model, ex, loss


@pytest.fixture(scope="module")
def launches():
    rec = Recorder(_lib.lib())
    prev = Fn.set_precision("bf16"), ops.set_deterministic(False)      # the production step
    with pytest.MonkeyPatch.context() as mp:
        proxy = rec.proxy()
        mp.setattr(_lib, "lib", lambda: proxy)
        mp.setattr(ops, "lib", lambda: proxy)
        try:
            _record(rec, "nusc", evaluate=True)
            _record(rec, "waymo180k", evaluate=False)
        finally:
            Fn.set_precision(prev[0])
            ops.set_deterministic(prev[1])
    torch.cuda.empty_cache()
    return rec


def _of(launches, fn):
    return [c for c in launches.configs if c["fn"] == fn]


# ------------------------------------------------------------------------------------------------- buffers
def _sentinel_buf(rows, ld, dtype):
    bits, s = SENT[dtype]
    return torch.full((rows + GUARD_ROWS, ld), s, dtype=bits, device="cuda").view(dtype)


def _place(t, ld):
    """A copy of [M, C] `t` inside a sentinel-filled [M + GUARD_ROWS, ld] buffer; returns (buffer, view)."""
    M, C = t.shape
    buf = _sentinel_buf(M, ld, t.dtype)
    buf[:M, :C] = t
    return buf, buf[:M, :C]


def _out(M, C, ld, dtype):
    buf = _sentinel_buf(M, ld, dtype)
    return buf, buf[:M, :C]


def _untouched(buf, M, C):
    bits, s = SENT[buf.dtype]
    b = buf.view(bits)
    return bool((b[:, C:] == s).all()) and bool((b[M:] == s).all())


def _ld(recorded, C, pad):
    return (recorded if recorded >= C else C) + pad


def _pad(wide, i):
    """Elements added to operand i's leading dimension: none in the replay at the recorded strides, 8 (i + 1) in the
    widened one, so that each operand's stride differs from every other's and a kernel indexing one operand with
    another's stride reads the wrong rows."""
    return 8 * (i + 1) if wide else 0


def _worst(t):
    """Largest entry with NaN counted as +inf (Python's max() and every `>` comparison would let a NaN through)."""
    return t.double().nan_to_num(nan=float("inf")).max().item()


def _fails(err, bound):
    """True where err is not within bound: NaN fails."""
    return ~(err <= bound)


POISON = set()     # names of kernel outputs to overwrite with one NaN after the launch (the NaN self-check)


def _poison(name, t, idx):
    if name in POISON:
        t[idx] = float("nan")


def _chunks(M, width):
    step = max(1024, CHUNK_BYTES // (8 * max(width, 1)))
    return [(m0, min(M, m0 + step)) for m0 in range(0, M, step)]


def _ulp_bf16(v):
    _, e = torch.frexp(v.abs().clamp(min=2.0 ** -126))
    return torch.ldexp(torch.ones_like(v), e - 8)


def _p(t):
    return None if t is None else t.data_ptr()


def _check(rc):
    _lib.check(rc)


def L():
    return _lib.lib()


# ------------------------------------------------------------------------------------------------- BatchNorm operands
def _large_cols(C):
    return [0, 9, C // 2 + 3, C - 1]


_BN_CACHE = {}


def _bn_data(M, C):
    """Operands of every BatchNorm replay at (M, C), one set at a time: x (bf16, with large-mean channels), dy, y, a
    residual, gamma / beta, and the batch statistics of x as the forward's finalize would give them."""
    if (M, C) in _BN_CACHE:
        return _BN_CACHE[(M, C)]
    _BN_CACHE.clear()
    torch.cuda.empty_cache()
    dev = "cuda"
    gen = torch.Generator(device=dev).manual_seed(M * 4099 + C)
    d = types.SimpleNamespace(M=M, C=C, big=_large_cols(C))
    big = torch.tensor(d.big, device=dev)
    std = torch.rand(C, generator=gen, device=dev) * 1.5 + 0.25
    mu = torch.randn(C, generator=gen, device=dev) * 0.5
    mu[big] = torch.tensor(LARGE_MEAN, device=dev) * std[big]
    d.x = torch.empty(M, C, dtype=torch.bfloat16, device=dev)
    d.x32big = torch.empty(M, len(d.big), dtype=torch.float32, device=dev)
    s1 = torch.zeros(C, dtype=torch.float64, device=dev)
    s2 = torch.zeros(C, dtype=torch.float64, device=dev)
    for m0, m1 in _chunks(M, C):
        v = torch.randn(m1 - m0, C, generator=gen, device=dev) * std + mu
        d.x[m0:m1] = v.bfloat16()
        d.x32big[m0:m1] = v[:, big]
        xd = d.x[m0:m1].double()
        s1 += xd.sum(0)
        s2 += (xd * xd).sum(0)
    d.stats = torch.cat([s1, s2])
    d.mean64 = s1 / M
    q = torch.zeros(C, dtype=torch.float64, device=dev)
    for m0, m1 in _chunks(M, C):
        q += ((d.x[m0:m1].double() - d.mean64) ** 2).sum(0)
    d.var64 = q / M
    m32 = d.x32big.double().mean(0)
    d.var32big = ((d.x32big.double() - m32) ** 2).mean(0)          # the variance before bf16 storage
    d.mean = d.mean64.float()
    d.invstd = (1.0 / torch.sqrt(d.var64 + 1e-5)).float()
    d.gamma = torch.rand(C, generator=gen, device=dev) + 0.5
    d.beta = torch.randn(C, generator=gen, device=dev) * 0.5
    d.fs = d.gamma * d.invstd                                        # forward affine: y = x * fs + fh
    d.fh = d.beta - d.mean * d.fs
    d.dy = torch.randn(M, C, generator=gen, device=dev).bfloat16()
    d.y = torch.randn(M, C, generator=gen, device=dev).bfloat16()
    d.res = torch.randn(M, C, generator=gen, device=dev).bfloat16()
    d.refs = {}
    _BN_CACHE[(M, C)] = d
    return d


def _gate(d, mode, m0, m1, xd):
    if mode == 0:
        return None
    if mode == 1:
        return d.y[m0:m1].double() > 0
    return xd * d.fs.double() + d.fh.double() > 0           # the sign of the exact x*fs + fh, as the kernel's fmaf gives it


def _reduce_ref(d, mode, drop_row=None):
    """fp64 sums of the reduce on the same bf16 inputs, their magnitudes, and for the large-mean channels the spread
    that bf16 storage of x alone causes in sum g*xhat."""
    key = (mode, drop_row)
    if key in d.refs:
        return d.refs[key]
    C = d.C
    z = lambda: torch.zeros(C, dtype=torch.float64, device="cuda")  # noqa: E731
    r = types.SimpleNamespace(sg=z(), sgx=z(), ag=z(), agx=z(), agxh=z())
    r.store2 = torch.zeros(len(d.big), dtype=torch.float64, device="cuda")
    mean, invstd = d.mean.double(), d.invstd.double()
    for m0, m1 in _chunks(d.M, C):
        xd = d.x[m0:m1].double()
        g = d.dy[m0:m1].double()
        gate = _gate(d, mode, m0, m1, xd)
        if gate is not None:
            g = torch.where(gate, g, torch.zeros((), dtype=torch.float64, device="cuda"))
        if drop_row is not None and m0 <= drop_row < m1:
            g[drop_row - m0] = 0
        xh = (xd - mean) * invstd
        r.sg += g.sum(0)
        r.sgx += (g * xh).sum(0)
        r.ag += g.abs().sum(0)
        r.agx += (g * xd).abs().sum(0)
        r.agxh += (g * xh).abs().sum(0)
        delta = (d.x32big[m0:m1].double() - xd[:, d.big]) * invstd[d.big]
        r.store2 += ((g[:, d.big] * delta) ** 2).sum(0)
    d.refs[key] = r
    return r


def _reduce_rows_per_thread(M, C):
    """Rows one thread of bn_bwd_reduce_kernel accumulates in fp32, from the launcher's grid (pnx_bn_bwd_reduce)."""
    rpb = 256 // (C // 8)
    nb = min(max(-(-M // (rpb * 8)), 1), 148 * 3)
    return -(-M // (nb * rpb)), nb, rpb


def _reduce_bounds(d, r):
    Lr = _reduce_rows_per_thread(d.M, d.C)[0]
    k = (Lr + 1) * U
    b_sg = k * r.ag + 1e-12 * r.ag + 1e-300
    b_sgx = d.invstd.double() * k * (r.agx + d.mean.double().abs() * r.ag) + 1e-12 * r.agxh + 1e-300
    return b_sg, b_sgx, Lr


# ------------------------------------------------------------------------------------------------- BatchNorm replays
def _launch_reduce(c, d, mode, wide):
    M, C = d.M, d.C
    dyb, dy = _place(d.dy, _ld(c["lddy"], C, _pad(wide, 0)))
    xb, x = _place(d.x, _ld(c["ldx"], C, _pad(wide, 1)))
    yb, y = _place(d.y, _ld(c["ldy"], C, _pad(wide, 2))) if mode == 1 else (None, None)
    red = torch.zeros(2 * C, dtype=torch.float64, device="cuda")
    _check(L().pnx_bn_bwd_reduce(_p(dy), dy.stride(0), _p(y), y.stride(0) if y is not None else 8, _p(x), x.stride(0), M, C,
                                 _p(d.mean), _p(d.invstd), 1 if mode else 0, _p(d.fs) if mode == 2 else None,
                                 _p(d.fh) if mode == 2 else None, _p(red), ops.stream()))
    torch.cuda.synchronize()
    _poison("reduce sum g", red, C - 1)
    _poison("reduce sum g*xhat", red, C + d.big[0])
    ok = _untouched(dyb, M, C) and _untouched(xb, M, C) and (yb is None or _untouched(yb, M, C))
    return red, ok


_INT_CACHE = {}


def _int_data(M, C):
    """Reduce operands on which every sum is exact: dy, x, y integers in [-4, 4], mean 0.5, invstd 2 and the forward
    affine x * 1 - 0.5 (mask x >= 1).  A thread's fp32 partials stay below 16 L < 2^24 (L <= 306 rows per thread at the
    step's shapes), the fp64 tail adds integers, and invstd (sum g x - mean sum g) is an integer: the kernel's sums must
    equal the fp64 reference exactly, so one missing or repeated row fails."""
    if (M, C) in _INT_CACHE:
        return _INT_CACHE[(M, C)]
    _INT_CACHE.clear()
    gen = torch.Generator(device="cuda").manual_seed(M * 31 + C)
    ints = lambda: torch.randint(-4, 5, (M, C), generator=gen, device="cuda").bfloat16()  # noqa: E731
    full = lambda v: torch.full((C,), v, device="cuda")  # noqa: E731
    d = types.SimpleNamespace(M=M, C=C, dy=ints(), x=ints(), y=ints(), mean=full(0.5), invstd=full(2.0), fs=full(1.0),
                              fh=full(-0.5), big=_large_cols(C))
    _INT_CACHE[(M, C)] = d
    return d


def _reduce_exact_ref(d, mode, drop_row=None):
    C = d.C
    ref = torch.zeros(2 * C, dtype=torch.float64, device="cuda")
    for m0, m1 in _chunks(d.M, C):
        xd = d.x[m0:m1].double()
        g = d.dy[m0:m1].double()
        gate = _gate(d, mode, m0, m1, xd)
        if gate is not None:
            g = torch.where(gate, g, torch.zeros((), dtype=torch.float64, device="cuda"))
        if drop_row is not None and m0 <= drop_row < m1:
            g[drop_row - m0] = 0
        ref[:C] += g.sum(0)
        ref[C:] += (g * (xd - 0.5) * 2).sum(0)
    return ref


def _compare_reduce(d, red, r):
    """(failures, worst err / bound, worst sum-g*xhat error in units of sum|g*x|, large-mean rows)."""
    C = d.C
    b_sg, b_sgx, _ = _reduce_bounds(d, r)
    e_sg, e_sgx = (red[:C] - r.sg).abs(), (red[C:] - r.sgx).abs()
    worst = max(_worst(e_sg / b_sg), _worst(e_sgx / b_sgx))
    bad = [] if worst <= 1.0 else ["reduce sums exceed their bound (x%.3g)" % worst]
    in_gx = _worst(e_sgx / (d.invstd.double() * r.agx + 1e-300))
    big = d.big
    rel = e_sgx[big] / r.agxh[big]
    store = r.store2.sqrt() / r.agxh[big]
    for i in _fails(rel, store).nonzero().flatten().tolist():
        bad.append("dgamma of large-mean channel %d: error %.3g of the centred sum exceeds the bf16 storage spread %.3g"
                   % (big[i], rel[i].item(), store[i].item()))
    return bad, worst, in_gx, list(zip(big, rel.tolist(), store.tolist()))


def _apply_ref_chunk(d, m0, m1, sc, sh, res, relu):
    xd = d.x[m0:m1].double()
    o = xd * sc + sh
    floor = (xd * sc).abs() + sh.abs()
    if res is not None:
        rd = res[m0:m1].double()
        o = o + rd
        floor = floor + rd.abs()
    if relu:
        o = o.clamp(min=0)
    return o, _ulp_bf16(o) + 2.0 ** -22 * floor


def _replay_bn_apply(c, d):
    M, C = d.M, d.C
    sc, sh = d.fs.double(), d.fh.double()
    res_t = d.res if c["res"] else None
    bad, worst, neq, big_ulps = [], 0.0, 0, 0.0
    for wide in (False, True):
        xb, x = _place(d.x, _ld(c["ldx"], C, _pad(wide, 0)))
        rb, r = _place(res_t, _ld(c["ldr"], C, _pad(wide, 1))) if res_t is not None else (None, None)
        yb, y = _out(M, C, _ld(c["ldy"], C, _pad(wide, 2)), torch.bfloat16)
        _check(L().pnx_bn_apply(_p(x), x.stride(0), M, C, _p(d.fs), _p(d.fh), _p(r), r.stride(0) if r is not None else 8,
                                c["relu"], _p(y), y.stride(0), ops.stream()))
        _poison("bn_apply y", y, (M - 1, C - 1))
        for m0, m1 in _chunks(M, C):
            ref, bound = _apply_ref_chunk(d, m0, m1, sc, sh, res_t, c["relu"])
            err = (y[m0:m1].double() - ref).abs()
            worst = max(worst, _worst(err / bound))
            neq += 0 if wide else int((y[m0:m1] != ref.float().bfloat16()).sum())
            big_ulps = max(big_ulps, _worst(err[:, d.big] / _ulp_bf16(ref[:, d.big])))
        if not (_untouched(yb, M, C) and _untouched(xb, M, C) and (rb is None or _untouched(rb, M, C))):
            bad.append("sentinel changed (%s strides)" % ("widened" if wide else "recorded"))
        del xb, rb, yb
    frac = neq / (M * C)
    if not worst <= 1.0:
        bad.append("y off by %.3g x its bound (1 bf16 ulp + fp32 floor)" % worst)
    if frac > 1e-3:
        bad.append("%.3g of y is not the fp64 result rounded to bf16" % frac)
    return bad, "err/bound %.3f, not bit-equal %.2e, large-mean channels %.2f ulp" % (worst, frac, big_ulps)


def _replay_bn_reduce(c, d, di, modes):
    """Exact sums on the integer operands di; the bound and the large-mean channels on the bf16 Gaussian operands d."""
    bad, notes = [], []
    for mode in modes:
        exact = _reduce_exact_ref(di, mode)
        r = _reduce_ref(d, mode)
        for wide in (False, True):
            what = "mask %d, %s strides" % (mode, "widened" if wide else "recorded")
            red, ok = _launch_reduce(c, di, mode, wide)
            _poison("reduce exact", red, 2 * di.C - 1)
            if not torch.equal(red, exact):
                n = int((red != exact).sum())
                bad.append("%s: %d integer sums differ from the exact reference" % (what, n))
            red, ok2 = _launch_reduce(c, d, mode, wide)
            b, worst, in_gx, big = _compare_reduce(d, red, r)
            bad += ["%s: %s" % (what, s) for s in b] + ([] if ok and ok2 else ["%s: sentinel changed" % what])
        Lr = _reduce_bounds(d, r)[2]
        notes.append("mask %d: integer sums exact; L %d, err/bound %.2e (sum g*xhat err %.2e of sum|g*x|); large-mean dgamma "
                     "err/centred [%s] vs bf16 storage [%s]" % (mode, Lr, worst, in_gx, " ".join("%.1e" % e for _, e, _ in big),
                                                                " ".join("%.1e" % s for _, _, s in big)))
    return bad, "; ".join(notes)


def _bwd_apply_ref_chunk(d, m0, m1, mode, red, n):
    C = d.C
    xd = d.x[m0:m1].double()
    g = d.dy[m0:m1].double()
    gate = _gate(d, mode, m0, m1, xd)
    if gate is not None:
        g = torch.where(gate, g, torch.zeros((), dtype=torch.float64, device="cuda"))
    mean, invstd = d.mean.double(), d.invstd.double()
    A = d.gamma.double() * invstd
    sgn, sgxn = red[:C] / n, red[C:] / n
    B = -A * invstd * sgxn
    dx = A * (g - sgn - (xd - mean) * invstd * sgxn)
    floor = (A * g).abs() + (B * xd).abs() + (A * sgn).abs() + (B * mean).abs()
    return dx, _ulp_bf16(dx) + 2.0 ** -20 * floor, g


def _replay_bn_bwd_apply(c, d, mode, accumulate):
    M, C = d.M, d.C
    r = _reduce_ref(d, mode)
    red = torch.cat([r.sg, r.sgx])
    n = c["count"]
    count_dev = torch.tensor([int(round(n))], dtype=torch.int32, device="cuda") if c["count_dev"] else None
    dres0 = d.res if accumulate else None
    bad, worst, neq, big_ulps = [], 0.0, 0, 0.0
    for wide in (False, True):
        strides = "widened" if wide else "recorded"
        dyb, dy = _place(d.dy, _ld(c["lddy"], C, _pad(wide, 0)))
        xb, x = _place(d.x, _ld(c["ldx"], C, _pad(wide, 1)))
        yb, y = _place(d.y, _ld(c["ldy"], C, _pad(wide, 2))) if mode == 1 else (None, None)
        dxb, dx = _out(M, C, _ld(c["lddx"], C, _pad(wide, 3)), torch.bfloat16)
        if c["dres"]:
            ld = _ld(c["lddres"], C, _pad(wide, 4))
            drb, dr = _place(dres0, ld) if accumulate else _out(M, C, ld, torch.bfloat16)
        else:
            drb, dr = None, None
        _check(L().pnx_bn_bwd_apply(_p(dy), dy.stride(0), _p(y), y.stride(0) if y is not None else 8, _p(x), x.stride(0), M, C,
                                    _p(d.mean), _p(d.invstd), _p(d.gamma), _p(red), float(n), _p(count_dev), 1 if mode else 0,
                                    _p(d.fs) if mode == 2 else None, _p(d.fh) if mode == 2 else None, _p(dx), dx.stride(0),
                                    _p(dr), dr.stride(0) if dr is not None else 8, 1 if accumulate else 0, ops.stream()))
        _poison("bn_bwd_apply dx", dx, (M - 1, C - 1))
        if dr is not None:
            _poison("bn_bwd_apply dres", dr, (M - 1, C - 1))
        for m0, m1 in _chunks(M, C):
            ref, bound, g = _bwd_apply_ref_chunk(d, m0, m1, mode, red, n)
            err = (dx[m0:m1].double() - ref).abs()
            worst = max(worst, _worst(err / bound))
            neq += 0 if wide else int((dx[m0:m1] != ref.float().bfloat16()).sum())
            big_ulps = max(big_ulps, _worst(err[:, d.big] / _ulp_bf16(ref[:, d.big])))
            if dr is not None:
                want = (g.float() + dres0[m0:m1].float()).bfloat16() if accumulate else g.bfloat16()
                if not torch.equal(dr[m0:m1], want):
                    bad.append("dres differs from g%s in rows %d..%d (%s strides)" % (" + dres" if accumulate else "", m0, m1,
                                                                                     strides))
                    break
        bufs = [b for b in (dyb, xb, yb, dxb, drb) if b is not None]
        if not all(_untouched(b, M, C) for b in bufs):
            bad.append("sentinel changed (%s strides)" % strides)
        del dyb, xb, yb, dxb, drb, bufs
    frac = neq / (M * C)
    if not worst <= 1.0:
        bad.append("dx off by %.3g x its bound (1 bf16 ulp + fp32 coefficient floor)" % worst)
    if frac > 1e-3:
        bad.append("%.3g of dx is not the fp64 result rounded to bf16" % frac)
    return bad, "mask %d%s: dx err/bound %.3f, not bit-equal %.2e, large-mean channels %.2f ulp" % (
        mode, " dres+=" if accumulate else "", worst, frac, big_ulps)


def _describe(c):
    keys = [k for k in c if k not in ("fn", "calls", "source")]
    return " ".join("%s=%s" % (k, ("%.4g" % c[k]) if isinstance(c[k], float) else c[k]) for k in keys)


def _run(configs, replay, title):
    failures = []
    print("\n%s: %d configurations" % (title, len(configs)))
    for i, c in enumerate(configs):
        bad, note = replay(c)
        print("[%2d] %-16s x%-4d %s\n       %s %s" % (i, c["source"], c["calls"], _describe(c), note,
                                                      "ok" if not bad else "FAIL: " + "; ".join(bad)))
        if bad:
            failures.append("%s %s: %s" % (c["source"], _describe(c), "; ".join(bad)))
        torch.cuda.empty_cache()
    return failures


def _mode(c):
    return 0 if not c["relu"] else (1 if c["y"] else 2)


def _by_size(configs):
    return sorted(configs, key=lambda c: (c["M"], c["C"]))


def test_bn_apply_matches_fp64(launches):
    cfgs = _by_size(_of(launches, "pnx_bn_apply"))
    assert any(c["M"] == 6 * 336 * 336 and c["C"] == 384 for c in cfgs), "no 677,376 x 384 sibling-head BatchNorm"
    assert any(c["C"] == 448 for c in cfgs), "no 448-channel Waymo sibling-head BatchNorm"
    failures = _run(cfgs, lambda c: _replay_bn_apply(c, _bn_data(c["M"], c["C"])), "pnx_bn_apply")
    assert not failures, "\n".join(failures)


def _reduce_configs(launches):
    """The recorded reduce configurations, plus one per BatchNorm shape whose reduce the step runs in the epilogue of
    the GEMM that produces dy (contiguous rows, mask recomputed from x): the stand-alone kernel runs there whenever
    that fusion does not apply."""
    cfgs = _of(launches, "pnx_bn_bwd_reduce")
    have = {(c["M"], c["C"]) for c in cfgs}
    for c in _of(launches, "pnx_bn_apply"):
        if (c["M"], c["C"]) not in have and c["source"].endswith("train"):
            have.add((c["M"], c["C"]))
            cfgs.append(dict(fn="pnx_bn_bwd_reduce", dy=True, lddy=c["C"], y=False, ldy=8, x=True, ldx=c["C"], M=c["M"],
                             C=c["C"], mean=True, invstd=True, relu=1, fscale=True, fshift=True, red=True, calls=0,
                             source="derived"))
    return _by_size(cfgs)


def test_bn_backward_reduce_matches_fp64(launches):
    """Each configuration in its recorded ReLU-mask mode; the largest one in all three (none, stored y, recomputed
    from x with the forward affine)."""
    cfgs = _reduce_configs(launches)
    largest = max(cfgs, key=lambda c: c["M"] * c["C"])
    assert largest["M"] * largest["C"] >= 6 * 336 * 336 * 384
    assert all(16 * _reduce_rows_per_thread(c["M"], c["C"])[0] < 2 ** 24 for c in cfgs), "integer sums no longer exact"
    failures = _run(cfgs, lambda c: _replay_bn_reduce(c, _bn_data(c["M"], c["C"]), _int_data(c["M"], c["C"]),
                                                      (0, 1, 2) if c is largest else (_mode(c),)), "pnx_bn_bwd_reduce")
    assert not failures, "\n".join(failures)


def test_bn_backward_apply_matches_fp64(launches):
    """Each configuration in its recorded mask mode, and with dres accumulating when it writes dres; the largest one in
    all three mask modes."""
    cfgs = _by_size(_of(launches, "pnx_bn_bwd_apply"))
    largest = max(cfgs, key=lambda c: c["M"] * c["C"])

    def replay(c):
        d = _bn_data(c["M"], c["C"])
        runs = [(m, c["dres_accumulate"]) for m in ((0, 1, 2) if c is largest else (_mode(c),))]
        if c["dres"] and not c["dres_accumulate"]:
            runs.append((_mode(c), 1))
        bad, notes = [], []
        for mode, acc in runs:
            b, n = _replay_bn_bwd_apply(c, d, mode, acc)
            bad += b
            notes.append(n)
        return bad, "; ".join(notes)
    failures = _run(cfgs, replay, "pnx_bn_bwd_apply")
    assert any(c["dres"] for c in cfgs), "no BatchNorm backward with a residual gradient"
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------- statistics
def _bn_formulas(stats, n, gamma, beta, eps, momentum, rm0, rv0, var=None):
    C = gamma.shape[0]
    mean = stats[:C] / n
    if var is None:
        var = (stats[C:] / n - mean * mean).clamp(min=0)
    invstd = 1.0 / torch.sqrt(var + eps)
    g, b = gamma.double(), beta.double()
    unb = var * (n / (n - 1.0)) if n > 1 else var
    return dict(mean=mean, invstd=invstd, scale=g * invstd, shift=b - mean * g * invstd,
                rm=(1 - momentum) * rm0.double() + momentum * mean, rv=(1 - momentum) * rv0.double() + momentum * unb,
                var=var)


DEVICE_COUNT = 40000     # population held on the device (count_ptr) in the replay of such configurations


def _finalize_population(c):
    return DEVICE_COUNT * c["count_mult"] if c["count_ptr"] else c["count_mult"]


def _replay_finalize(c, d, n_one):
    """n = *count_ptr * count_mult when the configuration reads its population from the device, else count_mult."""
    C, eps, mom = c["channels"], c["eps"], c["momentum"]
    gen = torch.Generator(device="cuda").manual_seed(C + 7)
    if n_one:
        x0 = d.x[0].double()
        stats, n, var = torch.cat([x0, x0 * x0]), 1, torch.zeros(C, dtype=torch.float64, device="cuda")
        dev_n, mult = 1, 1
    else:
        stats, n, var = d.stats, _finalize_population(c), d.var64
        dev_n, mult = DEVICE_COUNT, c["count_mult"]
    count_ptr = torch.tensor([dev_n], dtype=torch.int32, device="cuda") if c["count_ptr"] else None
    if count_ptr is None:
        mult = n
    rm0 = torch.randn(C, generator=gen, device="cuda")
    rv0 = torch.rand(C, generator=gen, device="cuda") + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    outs = [torch.full((C,), float("nan"), device="cuda") for _ in range(4)]
    _check(L().pnx_bn_finalize(_p(stats), C, _p(count_ptr), mult, _p(d.gamma), _p(d.beta), eps, mom,
                               _p(rm) if c["running_mean"] else None, _p(rv) if c["running_var"] else None, _p(outs[0]),
                               _p(outs[1]), _p(outs[2]) if c["mean_out"] else None, _p(outs[3]) if c["invstd_out"] else None,
                               ops.stream()))
    for name, t in (("scale", outs[0]), ("shift", outs[1]), ("mean", outs[2]), ("invstd", outs[3]), ("running_mean", rm),
                    ("running_var", rv)):
        _poison("finalize " + name, t, C - 1)
    want = _bn_formulas(stats, float(n), d.gamma, d.beta, eps, mom, rm0, rv0, var)
    cancel = 2.0 ** -46 * (want["mean"] ** 2 + want["var"]) / (want["var"] + eps)
    g = d.gamma.double()
    checks = [("scale", outs[0], want["scale"], want["scale"].abs() * (2.0 ** -21 + cancel)),
              ("shift", outs[1], want["shift"], 2.0 ** -20 * (d.beta.double().abs() + (want["mean"] * g * want["invstd"]).abs())
               * (1 + cancel)),
              ("running_mean", rm, want["rm"], 2.0 ** -20 * ((1 - mom) * rm0.double().abs() + mom * want["mean"].abs()) + 1e-30),
              ("running_var", rv, want["rv"], 2.0 ** -20 * ((1 - mom) * rv0.double().abs() + mom * want["var"] * 2) + 1e-30)]
    if c["mean_out"]:
        checks.append(("mean", outs[2], want["mean"], 2.0 ** -23 * want["mean"].abs() + 1e-30))
    if c["invstd_out"]:
        checks.append(("invstd", outs[3], want["invstd"], want["invstd"] * (2.0 ** -22 + cancel)))
    bad, worst = [], 0.0
    for name, got, ref, bound in checks:
        if name.startswith("running") and not c[name]:
            continue
        r = _worst((got.double() - ref).abs() / bound)
        worst = max(worst, r)
        if not r <= 1.0:
            bad.append("%s off by %.3g x its bound" % (name, r))
    note = "n = %d: err/bound %.3f" % (n, worst)
    if not n_one and c["invstd_out"]:
        big = d.big
        var_err = 2 * (outs[3].double()[big] - want["invstd"][big]).abs() / want["invstd"][big]
        store = (d.var32big - d.var64[big]).abs() / d.var64[big]
        note += "; large-mean variance rel. err [%s] vs bf16 storage [%s]" % (
            " ".join("%.1e" % e for e in var_err.tolist()), " ".join("%.1e" % s for s in store.tolist()))
        bad += ["variance of large-mean channel %d: %.3g exceeds the bf16 storage cost %.3g" % (big[i], var_err[i], store[i])
                for i in _fails(var_err, store).nonzero().flatten().tolist()]
    return bad, note


def _replay_eval_affine(c):
    C, eps = c["channels"], c["eps"]
    gen = torch.Generator(device="cuda").manual_seed(C)
    gamma = torch.rand(C, generator=gen, device="cuda") + 0.5
    beta = torch.randn(C, generator=gen, device="cuda")
    std = torch.rand(C, generator=gen, device="cuda") + 0.1
    rm = torch.randn(C, generator=gen, device="cuda")
    rm[_large_cols(C)] = torch.tensor(LARGE_MEAN, device="cuda") * std[_large_cols(C)]
    rv = std * std
    scale, shift = torch.full((C,), float("nan"), device="cuda"), torch.full((C,), float("nan"), device="cuda")
    _check(L().pnx_bn_eval_affine(C, _p(gamma), _p(beta), _p(rm), _p(rv), eps, _p(scale), _p(shift), ops.stream()))
    _poison("eval scale", scale, C - 1)
    _poison("eval shift", shift, C - 1)
    invstd = 1.0 / torch.sqrt(rv.double() + eps)
    ws = gamma.double() * invstd
    wh = beta.double() - rm.double() * ws
    e1 = _worst((scale.double() - ws).abs() / (2.0 ** -21 * ws.abs()))
    e2 = _worst((shift.double() - wh).abs() / (2.0 ** -20 * (beta.double().abs() + (rm.double() * ws).abs())))
    bad = [] if max(e1, e2) <= 1.0 else ["scale / shift off by %.3g / %.3g x their bounds" % (e1, e2)]
    return bad, "err/bound scale %.3f shift %.3f" % (e1, e2)


def test_bn_statistics_match_torch_formulas(launches):
    """pnx_bn_finalize at each recorded (C, count, eps, momentum) on the statistics of data with large-mean channels,
    and again with n = 1; pnx_bn_eval_affine at each recorded (C, eps)."""
    fin = _of(launches, "pnx_bn_finalize")
    families = {(c["eps"], c["momentum"]) for c in fin}
    assert len(families) >= 2, "both BatchNorm families (eps 1e-3 / momentum 0.01 and the torch defaults): %s" % families

    def replay(c):
        d = _bn_data(_finalize_population(c), c["channels"])
        b1, n1 = _replay_finalize(c, d, False)
        b2, n2 = _replay_finalize(c, d, True)
        return b1 + b2, n1 + "; " + n2
    failures = _run(sorted(fin, key=lambda c: (_finalize_population(c), c["channels"])), replay, "pnx_bn_finalize")

    failures += _run(_of(launches, "pnx_bn_eval_affine"), _replay_eval_affine, "pnx_bn_eval_affine")
    assert _of(launches, "pnx_bn_eval_affine"), "the eval forward launched no pnx_bn_eval_affine"
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------- exact row kernels
def _rand_rows(M, C, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(M, C, generator=gen, device="cuda").bfloat16()


def _replay_exact(c):
    fn, M, C = c["fn"], c["M"], c["C"]
    a, b = _rand_rows(M, C, M + C), _rand_rows(M, C, M + C + 1)
    bad = []
    for wide in (False, True):
        strides = "widened" if wide else "recorded"
        if fn == "pnx_add_relu":
            ab, av = _place(a, _ld(c["lda"], C, _pad(wide, 0)))
            bb, bv = _place(b, _ld(c["ldb"], C, _pad(wide, 1)))
            yb, y = _out(M, C, _ld(c["ldy"], C, _pad(wide, 2)), torch.bfloat16)
            _check(L().pnx_add_relu(_p(av), av.stride(0), _p(bv), bv.stride(0), M, C, _p(y), y.stride(0), ops.stream()))
            ref = lambda m0, m1: F.relu(a[m0:m1].float() + b[m0:m1].float()).bfloat16()  # noqa: E731
            bufs = (ab, bb, yb)
        elif fn == "pnx_relu_bwd":
            g0 = _rand_rows(M, C, M + C + 2)
            db, dv = _place(a, _ld(c["lddy"], C, _pad(wide, 0)))
            yb, yv = _place(b, _ld(c["ldy"], C, _pad(wide, 1)))
            ldg = _ld(c["ldg"], C, _pad(wide, 2))
            gb, y = _place(g0, ldg) if c["accumulate"] else _out(M, C, ldg, torch.bfloat16)
            _check(L().pnx_relu_bwd(_p(dv), dv.stride(0), _p(yv), yv.stride(0), M, C, _p(y), y.stride(0), c["accumulate"],
                                    ops.stream()))
            zero = torch.zeros((), device="cuda")

            def ref(m0, m1):
                v = torch.where(b[m0:m1].float() > 0, a[m0:m1].float(), zero)
                return (v + g0[m0:m1].float() if c["accumulate"] else v).bfloat16()
            bufs = (db, yb, gb)
        else:                                             # pnx_add_rows: a += b in place
            yb, y = _place(a, _ld(c["lda"], C, _pad(wide, 0)))
            bb, bv = _place(b, _ld(c["ldb"], C, _pad(wide, 1)))
            _check(L().pnx_add_rows(_p(y), y.stride(0), _p(bv), bv.stride(0), M, C, ops.stream()))
            ref = lambda m0, m1: (a[m0:m1].float() + b[m0:m1].float()).bfloat16()  # noqa: E731
            bufs = (yb, bb)
        _poison("exact " + fn, y, (M - 1, C - 1))
        for m0, m1 in _chunks(M, C):
            if not torch.equal(y[m0:m1], ref(m0, m1)):
                bad.append("rows %d..%d differ from torch (%s strides)" % (m0, m1, strides))
                break
        if not all(_untouched(t, M, C) for t in bufs):
            bad.append("sentinel changed (%s strides)" % strides)
    return bad, "bit-exact" if not bad else ""


def test_add_relu_relu_bwd_add_rows_bit_exact(launches):
    """The recorded add_relu / relu_bwd configurations, relu_bwd also accumulating, and add_rows (a += b; the step
    itself does not call it) at the largest add_relu shape."""
    adds = _of(launches, "pnx_add_relu")
    bwds = _of(launches, "pnx_relu_bwd")
    assert adds and bwds
    derived = [dict(c, accumulate=1, calls=0, source="derived") for c in bwds if not c["accumulate"]]
    big = max(adds, key=lambda c: c["M"] * c["C"])
    derived.append(dict(fn="pnx_add_rows", a=True, lda=big["ldy"], b=True, ldb=big["ldb"], M=big["M"], C=big["C"],
                        calls=0, source="derived"))
    failures = _run(adds + bwds + _of(launches, "pnx_add_rows") + derived, _replay_exact, "add_relu / relu_bwd / add_rows")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------- stencil
def _stencil_gather_ref(Z, bias, B, H, W, cpt, drop=None):
    """out[m, j] = bias[j] + sum over in-image taps (r, s) of Z[(y + r - 1, x + s - 1), (3r + s) cpt + j]  (j < cpt)."""
    M = B * H * W
    out = bias.view(1, 16).repeat(M, 1)
    for b in range(B):
        Zb = Z[b * H * W:(b + 1) * H * W, :9 * cpt].reshape(H, W, 9, cpt).permute(2, 3, 0, 1)
        Zp = F.pad(Zb, (1, 1, 1, 1))
        acc = torch.zeros(cpt, H, W, device=Z.device)
        for t in range(9):
            term = Zp[t, :, t // 3:t // 3 + H, t % 3:t % 3 + W]
            if drop is not None and drop[0] == b and drop[3] == t:
                term = term.clone()
                term[:, drop[1], drop[2]] = 0
            acc += term
        out[b * H * W:(b + 1) * H * W, :cpt] += acc.permute(1, 2, 0).reshape(H * W, cpt)
    return out


def _stencil_scatter_ref(dout, B, H, W, nz, cpt, dtype=torch.bfloat16):
    """dZ[m, (3r + s) cpt + j] = bf16(dout[(y - r + 1, x - s + 1), j]) inside the image, else 0; columns >= 9 cpt zero.
    dtype = torch.float32: the values before the rounding."""
    M = B * H * W
    dZ = torch.zeros(M, nz, dtype=dtype, device=dout.device)
    for b in range(B):
        Dp = F.pad(dout[b * H * W:(b + 1) * H * W, :cpt].reshape(H, W, cpt).permute(2, 0, 1), (1, 1, 1, 1))
        rows = dZ[b * H * W:(b + 1) * H * W]
        for t in range(9):
            r, s = t // 3, t % 3
            rows[:, t * cpt:(t + 1) * cpt] = Dp[:, 2 - r:2 - r + H, 2 - s:2 - s + W].permute(1, 2, 0).reshape(H * W, cpt).to(dtype)
    return dZ


def _gather_operands(c, seed):
    B, H, W, cpt = c["B"], c["H"], c["W"], c["cpt"]
    M = B * H * W
    gen = torch.Generator(device="cuda").manual_seed(seed)
    Z = torch.randint(-4, 5, (M, 9 * cpt), generator=gen, device="cuda").float()
    bias = torch.randint(-4, 5, (16,), generator=gen, device="cuda").float()
    return Z, bias


def _launch_gather(c, Z, bias, wide):
    B, H, W, cpt = c["B"], c["H"], c["W"], c["cpt"]
    M = B * H * W
    zb, zv = _place(Z, c["ldz"] + _pad(wide, 0))          # columns 9 cpt .. ldz: NaN sentinel
    ob, out = _out(M, 16, 16, torch.float32)
    _check(L().pnx_tap_gather_sum(_p(zv), zv.stride(0), cpt, _p(bias), B, H, W, _p(out), ops.stream()))
    torch.cuda.synchronize()
    _poison("gather out", out, (M - 1, 0))
    return out, _untouched(zb, M, 9 * cpt) and _untouched(ob, M, 16)


def _replay_stencil(c):
    B, H, W, cpt = c["B"], c["H"], c["W"], c["cpt"]
    M = B * H * W
    bad = []
    if c["fn"] == "pnx_tap_gather_sum":
        Z, bias = _gather_operands(c, M + cpt)
        ref = _stencil_gather_ref(Z, bias, B, H, W, cpt)
        for wide in (False, True):
            out, ok = _launch_gather(c, Z, bias, wide)
            if not torch.equal(out, ref):
                bad.append("%d outputs differ (%s ldz)" % (int((out != ref).sum()), "widened" if wide else "recorded"))
            if not ok:
                bad.append("sentinel changed (%s ldz)" % ("widened" if wide else "recorded"))
        return bad, "cpt %d, ldz %d: bit-exact" % (cpt, c["ldz"]) if not bad else ""
    assert c["lo_off"] == 0, "the bf16 step writes one piece"
    nz = c["nz"]
    gen = torch.Generator(device="cuda").manual_seed(M + nz)
    dout = torch.randn(M, cpt, generator=gen, device="cuda") * 3
    ref = _stencil_scatter_ref(dout, B, H, W, nz, cpt)
    for wide in (False, True):
        db, dv = _place(dout, 16)                         # dout rows are 16 floats; columns cpt..15 hold the sentinel
        zb, dZ = _out(M, nz, c["ldz"] + _pad(wide, 0), torch.bfloat16)
        _check(L().pnx_tap_scatter(_p(dv), B, H, W, _p(dZ), dZ.stride(0), nz, cpt, 0, ops.stream()))
        _poison("scatter dZ", dZ, (M - 1, 0))
        if not torch.equal(dZ, ref):
            bad.append("%d dZ entries differ (%s ldz)" % (int((dZ != ref).sum()), "widened" if wide else "recorded"))
        if not (_untouched(zb, M, nz) and _untouched(db, M, cpt)):
            bad.append("sentinel changed (%s ldz)" % ("widened" if wide else "recorded"))
    return bad, "cpt %d, NZ %d, slots_log2 %d: bit-exact" % (cpt, nz, 4 if nz // 8 <= 16 else 5) if not bad else ""


def test_head_stencil_bit_exact(launches):
    gs, sc = _of(launches, "pnx_tap_gather_sum"), _of(launches, "pnx_tap_scatter")
    assert {c["cpt"] for c in gs} >= {12, 16} and {c["nz"] for c in sc} >= {128, 192}, "both head final-conv geometries"
    failures = _run(gs + sc, _replay_stencil, "pnx_tap_gather_sum / pnx_tap_scatter")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------- loss
COLS = (("reg", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))
ANNO_COL = ("reg", 0), ("reg", 1), ("height", 0), ("dim", 0), ("dim", 1), ("dim", 2), ("vel", 0), ("vel", 1), ("rot", 0), ("rot", 1)


def _loss_case(c):
    """Head matrix and labels for one recorded pnx_center_loss_task configuration, with the edge cases injected."""
    name = c["source"].split()[0]
    cfg = synth.BENCH_CONFIGS[name]["cfg"]
    B, H, W, C, Mo, npad = c["B"], c["H"], c["W"], c["C"], c["M"], c["npad"]
    g = ops.grid_size_xy(cfg["voxel_size"], cfg["pc_range"])
    t = next(i for i, task in enumerate(cfg["tasks"]) if len(task) == C and int(g[0]) // cfg["out_size_factor"][i] == W)
    boxes, cls = synth.make_gt_batch(list(range(B)), 600, cfg)
    lab = ops.assign_labels(boxes.cuda(), cls.cuda(), cfg["tasks"], cfg["voxel_size"], cfg["pc_range"], cfg["out_size_factor"],
                            max_objs=Mo)
    k = types.SimpleNamespace(**{n: lab[n][t].clone() for n in ("hm", "anno_box", "ind", "mask", "cat", "gt_boxes")})
    k.cfg, k.B, k.H, k.W, k.C, k.Mo, k.npad = cfg, B, H, W, C, Mo, npad
    k.off = dict(reg=c["off_reg"], height=c["off_height"], dim=c["off_dim"], rot=c["off_rot"], vel=c["off_vel"], hm=c["off_hm"])
    npix = B * H * W
    gen = torch.Generator(device="cuda").manual_seed(npix + C)
    out = torch.randn(npix, npad, generator=gen, device="cuda")
    used = torch.zeros(npad, dtype=torch.bool)
    for n, w in COLS + (("hm", C),):
        used[k.off[n]:k.off[n] + w] = True
    o = k.off
    out[:, o["reg"]:o["reg"] + 2] = torch.rand(npix, 2, generator=gen, device="cuda")
    out[:, o["dim"]:o["dim"] + 3] = out[:, o["dim"]:o["dim"] + 3] * 0.3 + 0.3
    out[:, o["vel"]:o["vel"] + 2] *= 2
    out[:, o["hm"]:o["hm"] + C] = (out[:, o["hm"]:o["hm"] + C] * 1.5 - 2).clamp(-8, 8)
    mask = k.mask.cpu()
    ind = k.ind.cpu()
    pos0 = [j for j in range(Mo) if mask[0, j]]
    assert len(pos0) >= 8 and int(mask.sum()) >= 8 * B, "too few objects for the edge cases"
    j0, j1, j2, j3, j4, j5, j6 = pos0[:7]
    k.shared = (j0, j1)
    k.ind[0, j1] = ind[0, j0]                                             # two slots on one pixel
    hm = o["hm"]
    out[int(ind[0, j2]), hm + int(k.cat[0, j2])] = 12.0                   # sigmoid clamp at positive pixels
    out[int(ind[0, j3]), hm + int(k.cat[0, j3])] = -12.0
    taken = set((b * H * W + int(ind[b, j])) for b in range(B) for j in range(Mo) if mask[b, j])
    free = [p for p in range(npix - 1, npix - 4 * W, -1) if p not in taken][:2]
    out[free[0], hm:hm + C] = 12.0                                        # ... and at negative pixels
    out[free[1], hm:hm + C] = -12.0
    out[int(ind[0, j4]), o["dim"]:o["dim"] + 3] = torch.tensor([6.0, -6.5, 5.5], device="cuda")   # dim clamp at +-5
    # a predicted box equal to its ground truth, exact in fp32 and fp64: pixel 0 with reg 0 decodes to (ox, oy), the
    # dimension logits 0 to exp(0) = 1; every min / max of the DIoU ties
    k.ind[0, j5] = 0
    assert 0 not in taken
    out[0, o["reg"]:o["reg"] + 2] = 0.0
    out[0, o["height"]] = 0.25
    out[0, o["dim"]:o["dim"] + 3] = 0.0
    k.gt_boxes[0, j5, :6] = torch.tensor([c["ox"], c["oy"], 0.25, 1.0, 1.0, 1.0], device="cuda")
    k.anno_box[0, j6, 6:8] = float("nan")                                 # NaN velocity targets
    assert torch.isnan(k.anno_box[..., 6]).any()
    off_slots = ~k.mask.bool()                                            # masked-off slots hold garbage
    k.ind_clean = k.ind.clone()
    k.ind[off_slots] = torch.randint(-10 ** 9, 10 ** 9, (int(off_slots.sum()),), generator=gen, device="cuda")
    k.cat_clean = k.cat.clone()
    k.cat[off_slots] = torch.randint(-50, 50, (int(off_slots.sum()),), generator=gen, device="cuda")
    k.out_buf, k.out = _place(out, npad)                                  # guard rows: NaN sentinel
    k.out[:, ~used.cuda()] = float("nan")                                 # columns the loss does not own
    _untie(k, c, (0, j5))
    return k


def _untie(k, c, keep):
    """Moves the predicted boxes that lie within 1e-4 m of a DIoU min / max tie or of the clamp at 0 (all but the
    deliberate tie `keep`): there the fp32 kernel and the fp64 oracle could take different branches."""
    HW, o = k.H * k.W, k.off
    for _ in range(8):
        b, j = k.mask.nonzero(as_tuple=True)
        sel = ~((b == keep[0]) & (j == keep[1]))
        b, j = b[sel], j[sel]
        ind = k.ind_clean[b, j]
        pix = b * HW + ind
        r = k.out[pix].double()
        p = torch.stack([((ind % k.W).double() + r[:, o["reg"]]) * c["sx"] + c["ox"],
                         (torch.div(ind, k.W, rounding_mode="floor").double() + r[:, o["reg"] + 1]) * c["sy"] + c["oy"],
                         r[:, o["height"]]], 1)
        half = torch.exp(r[:, o["dim"]:o["dim"] + 3].clamp(-5, 5)) / 2
        gb = k.gt_boxes[b, j].double()
        ph, pl, gh, gl = p + half, p - half, gb[:, :3] + gb[:, 3:6] / 2, gb[:, :3] - gb[:, 3:6] / 2
        gaps = torch.cat([ph - gh, pl - gl, torch.minimum(ph, gh) - torch.maximum(pl, gl)], 1)
        near = (gaps.abs() < 1e-4).any(1)
        if not near.any():
            return
        for col in (o["reg"], o["reg"] + 1, o["height"]):
            k.out[pix[near], col] += 1e-3
    raise AssertionError("predicted boxes keep landing on DIoU ties")


def _launch_loss(c, k, ind=None, cat=None, mask=None, which="loss"):
    npix = k.B * k.H * k.W
    db, dout = _out(npix, k.npad, k.npad, torch.float32)
    acc = torch.zeros(16, dtype=torch.float64, device="cuda")
    cw = (ctypes.c_float * 10)(*k.cfg["code_weights"])
    o = k.off
    _check(L().pnx_center_loss_task(_p(k.out), _p(dout), _p(k.hm), _p(k.anno_box), _p(k.ind if ind is None else ind),
                                    _p(k.mask if mask is None else mask), _p(k.cat if cat is None else cat), _p(k.gt_boxes),
                                    k.B, k.H, k.W, k.npad, k.C, k.Mo, o["reg"], o["height"], o["dim"], o["rot"], o["vel"], o["hm"],
                                    c["sx"], c["sy"], c["ox"], c["oy"], c["weight"], ctypes.cast(cw, ctypes.c_void_p),
                                    c["with_iou"], _p(acc), ops.stream()))
    res = torch.full((16,), float("nan"), device="cuda")
    total = torch.empty(1, device="cuda")
    wdev = torch.tensor([c["weight"]], device="cuda")
    cwdev = torch.tensor(k.cfg["code_weights"], dtype=torch.float32, device="cuda")
    idev = torch.tensor([c["with_iou"]], dtype=torch.int32, device="cuda")
    _check(L().pnx_center_loss_finalize(_p(acc), 1, _p(wdev), _p(cwdev), _p(idev), _p(res), _p(total), ops.stream()))
    torch.cuda.synchronize()
    res = res.cpu()
    for i in range(16):
        _poison("%s res[%d]" % (which, i), res, i)
    _poison(which + " dout", dout, (npix - 1, k.off["hm"]))
    return dout, res, db


_ORACLE_CACHE = {}


def _loss_oracle(c, k):
    """oracle.center_loss in float64 on the same numbers (masked-off slots' ind / cat replaced by 0: the oracle
    gathers every slot).  The decode uses the kernel's fp32 sx / sy / ox / oy.  _loss_case is deterministic, so the
    result is kept per configuration."""
    from oracle import pillarnext_oracle as O
    if _describe(c) in _ORACLE_CACHE:
        return _ORACLE_CACHE[_describe(c)]
    npix = k.B * k.H * k.W
    out4 = k.out.detach().double().cpu().view(k.B, k.H, k.W, k.npad).clone().requires_grad_()
    pd = {n: out4[..., k.off[n]:k.off[n] + w].permute(0, 3, 1, 2) for n, w in COLS}
    pd["hm"] = out4[..., k.off["hm"]:k.off["hm"] + k.C].permute(0, 3, 1, 2)
    mask = k.mask.cpu()
    ex = {"hm": [k.hm.double().cpu()], "anno_box": [k.anno_box.double().cpu()], "mask": [mask],
          "ind": [torch.where(mask.bool(), k.ind_clean.cpu(), torch.zeros((), dtype=torch.int64))],
          "cat": [torch.where(mask.bool(), k.cat_clean.cpu(), torch.zeros((), dtype=torch.int64))],
          "gt_boxes": [k.gt_boxes.double().cpu()]}
    total, rets = O.center_loss(ex, [pd], c["weight"], k.cfg["code_weights"], bool(c["with_iou"]), [c["sx"], c["sy"]],
                                [c["ox"], c["oy"]], [1])
    (grad,) = torch.autograd.grad(total, [out4])
    _ORACLE_CACHE[_describe(c)] = rets[0], grad.view(npix, k.npad).cuda()
    return _ORACLE_CACHE[_describe(c)]


def _compare_loss(res, dout, ret, go):
    bad = []
    for i, key in ((0, "loss"), (1, "hm_loss"), (2, "loc_loss"), (3, "iou_reg_loss"), (4, "num_positive")):
        if key not in ret:
            continue
        want = float(ret[key].detach())
        if not abs(float(res[i]) - want) <= 1e-4 * max(1.0, abs(want)):
            bad.append("%s %.7g, fp64 %.7g" % (key, float(res[i]), want))
    e = (res[5:15].double() - ret["loc_loss_elem"].double()).abs()
    if _fails(e, 1e-4 * ret["loc_loss_elem"].double().abs() + 1e-7).any():
        bad.append("loc_loss_elem differs by up to %.3g" % _worst(e))
    scale = go.abs().max().item()
    err = _worst((dout.double() - go).abs())
    if not err <= 1e-4 * scale:
        bad.append("d(loss)/d(out) off by %.3g (max |grad| %.3g)" % (err, scale))
    return bad, err / scale


def _drop_shared_l1(k, c, go):
    """The fp64 gradient with the second shared-pixel slot's L1 regression gradient left out (counted once)."""
    j0, j1 = k.shared
    pix = int(k.ind_clean[0, j0])
    npos = float(k.mask.sum())
    g = go.clone()
    for code, (n, i) in enumerate(ANNO_COL):
        col = k.off[n] + i
        tg = float(k.anno_box[0, j1, code])
        if tg != tg:
            continue
        d = float(k.out[pix, col]) - tg
        g[pix, col] -= np.sign(d) * k.cfg["code_weights"][code] * c["weight"] / (npos + 1e-4)
    return g


def _replay_loss(c):
    k = _loss_case(c)
    npix = k.B * k.H * k.W
    dout, res, db = _launch_loss(c, k)
    ret, go = _loss_oracle(c, k)
    bad, rel = _compare_loss(res, dout, ret, go)
    if not _untouched(db, npix, k.npad):
        bad.append("dout guard rows written")
    if float(res[15]) != 0:
        bad.append("res[15] = %g bad slots on valid labels" % float(res[15]))
    # one out-of-range ind (last frame: one past the map) and one out-of-range cat: counted in res[15], nothing written;
    # every other gradient is the first launch's with npos two larger
    mask, ind, cat = k.mask.clone(), k.ind.clone(), k.cat.clone()
    jb = k.Mo - 1
    assert not mask[k.B - 1, jb] and not mask[0, jb]
    mask[k.B - 1, jb], ind[k.B - 1, jb], cat[k.B - 1, jb] = 1, k.H * k.W, 0
    mask[0, jb], ind[0, jb], cat[0, jb] = 1, int(k.ind_clean[0, k.shared[0]]), k.C
    dout2, res2, db2 = _launch_loss(c, k, ind=ind, cat=cat, mask=mask, which="bad-slot")
    npg, npb = float(k.mask.sum()), float(mask.sum())
    want = dout.double() * ((npg + 1e-4) / (npb + 1e-4))
    hm = slice(k.off["hm"], k.off["hm"] + k.C)
    want[:, hm] = dout[:, hm].double() * (npg / npb)
    e2 = (dout2.double() - want).abs()
    if float(res2[15]) != 2 or float(res2[4]) != npb:
        bad.append("bad slots: res[15] = %g, npos %g (want 2, %g)" % (float(res2[15]), float(res2[4]), npb))
    if _fails(e2, 1e-5 * want.abs() + 1e-6 * want.abs().max()).any() or not _untouched(db2, npix, k.npad):
        bad.append("bad slots changed the gradient beyond the npos rescale (%.3g) or wrote past the map" % _worst(e2))
    note = "%d positives, CTAs %d dense / %d slots; loss %.6f (fp64 %.6f); grad err %.2e of max" % (
        int(npg), min(-(-npix // 256), 1184), -(-(k.B * k.Mo) // 128), float(res[0]), float(ret["loss"].detach()), rel)
    return bad, note, (k, dout, res, ret, go)


def test_center_loss_matches_fp64_oracle_at_production_shape(launches):
    cfgs = _of(launches, "pnx_center_loss_task")
    assert any(c["B"] == 6 and c["H"] == 336 and c["W"] == 336 for c in cfgs), "no 6 x 336^2 loss"
    failures = _run(cfgs, lambda c: _replay_loss(c)[:2], "pnx_center_loss_task")
    assert not failures, "\n".join(failures)


def _replay_loss_finalize(c):
    n = c["n_tasks"]
    gen = torch.Generator().manual_seed(n)
    acc = torch.rand(n, 16, generator=gen, dtype=torch.float64) * 50
    acc[:, 0:2] *= -20
    acc[:, 2] = torch.randint(0, 400, (n,), generator=gen).double()
    acc[0, 2] = 0                                                     # a task without objects
    acc[:, 15] = torch.randint(0, 3, (n,), generator=gen).double()
    w = torch.rand(n, generator=gen) + 0.2
    cw = torch.rand(10, generator=gen) + 0.1
    wi = torch.tensor([i % 2 for i in range(n)], dtype=torch.int32)
    res = torch.full((n, 16), float("nan"), device="cuda")
    total = torch.empty(1, device="cuda")
    a, wd, cwd, wid = acc.cuda(), w.cuda(), cw.cuda(), wi.cuda()
    _check(L().pnx_center_loss_finalize(_p(a), n, _p(wd), _p(cwd), _p(wid), _p(res), _p(total), ops.stream()))
    _poison("loss finalize res", res, (n - 1, 11))
    _poison("loss finalize total", total, 0)
    res = res.cpu().double()
    npos = acc[:, 2]
    hm = -(acc[:, 1] + acc[:, 0]) / npos.clamp(min=1)
    el = acc[:, 3:13] / (npos + 1e-4).unsqueeze(1)
    loc = (el * cw.double()).sum(1)
    iou = torch.where(wi.bool(), acc[:, 13] / (npos + 1e-4), torch.zeros(n, dtype=torch.float64))
    loss = hm + w.double() * loc + w.double() * iou
    want = torch.cat([torch.stack([loss, hm, loc, iou, npos], 1), el, acc[:, 15:16]], 1)
    err = _worst((res - want).abs() / (want.abs() + 1e-6))
    terr = _worst((total.cpu().double() - loss.sum()).abs() / loss.sum().abs())
    bad = [] if max(err, terr) < 1e-5 else ["res off by %.3g relative, total by %.3g" % (err, terr)]
    return bad, "rel err %.2e, total %.2e" % (err, terr)


def test_center_loss_finalize_matches_formula(launches):
    failures = _run(_of(launches, "pnx_center_loss_finalize"), _replay_loss_finalize, "pnx_center_loss_finalize")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------- self-checks
def test_self_check_reduce_comparison_catches_a_dropped_tail_row(launches):
    """On the largest BatchNorm backward, in each mask mode, the exact integer comparison of the reduce fails when the
    reference leaves out row M - 1, which lies past the last full unroll group of rows."""
    c = max(_reduce_configs(launches), key=lambda c: c["M"] * c["C"])
    d = _int_data(c["M"], c["C"])
    M, C = d.M, d.C
    _, _, rpb = _reduce_rows_per_thread(M, C)
    assert M % (rpb * 4) != 0, "M fills its last unroll group: pick another row"
    for mode in (0, 1, 2):
        red, ok = _launch_reduce(c, d, mode, False)
        assert ok and torch.equal(red, _reduce_exact_ref(d, mode))
        dropped = _reduce_exact_ref(d, mode, drop_row=M - 1)
        print("reduce M %d C %d mask %d without row %d: %d sums differ" % (M, C, mode, M - 1, int((red != dropped).sum())))
        assert not torch.equal(red, dropped), "the reduce comparison does not notice a reference without row M - 1"


def test_self_check_stencil_comparison_catches_a_dropped_border_tap(launches):
    """On the largest tap_gather_sum configuration, the exact comparison fails when the reference leaves out tap (0, 1)
    (the row above) of the bottom-left pixel of the last frame, a tap that is inside the image at that border pixel."""
    c = max(_of(launches, "pnx_tap_gather_sum"), key=lambda c: c["B"] * c["H"] * c["W"] * c["cpt"])
    B, H, W, cpt = c["B"], c["H"], c["W"], c["cpt"]
    Z, bias = _gather_operands(c, 5)
    src = ((B - 1) * H + H - 2) * W + 0                                 # the pixel tap (0, 1) of (H - 1, 0) reads
    Z[src, 1 * cpt:2 * cpt] = 3.0
    out, ok = _launch_gather(c, Z, bias, False)
    assert ok and torch.equal(out, _stencil_gather_ref(Z, bias, B, H, W, cpt))
    assert not torch.equal(out, _stencil_gather_ref(Z, bias, B, H, W, cpt, drop=(B - 1, H - 1, 0, 1))), \
        "a dropped border tap goes unnoticed"


def test_self_check_loss_comparison_catches_a_shared_pixel_counted_once(launches):
    """On the largest loss configuration, the comparison fails when the reference counts the L1 regression gradient of
    only one of the two slots that share a pixel."""
    c = max(_of(launches, "pnx_center_loss_task"), key=lambda c: c["B"] * c["H"] * c["W"])
    bad, _, (k, dout, res, ret, go) = _replay_loss(c)
    assert not bad, bad
    found, _ = _compare_loss(res, dout, ret, _drop_shared_l1(k, c, go))
    print("loss with one shared-pixel slot counted once: %s" % found)
    assert found, "a shared-pixel slot counted once goes unnoticed"


NAN_CASES = [      # (kernel output overwritten with one NaN, entry point, failure messages the replay must report)
    ("bn_apply y", "pnx_bn_apply", ("y off by",)),
    ("bn_bwd_apply dx", "pnx_bn_bwd_apply", ("dx off by",)),
    ("bn_bwd_apply dres", "pnx_bn_bwd_apply", ("dres differs",)),
    ("reduce exact", "pnx_bn_bwd_reduce", ("integer sums differ",)),
    ("reduce sum g", "pnx_bn_bwd_reduce", ("integer sums differ", "exceed their bound")),
    ("reduce sum g*xhat", "pnx_bn_bwd_reduce", ("exceed their bound", "large-mean channel 0")),
    ("finalize scale", "pnx_bn_finalize", ("scale off by",)),
    ("finalize shift", "pnx_bn_finalize", ("shift off by",)),
    ("finalize mean", "pnx_bn_finalize", ("mean off by",)),
    ("finalize invstd", "pnx_bn_finalize", ("invstd off by", "variance of large-mean channel")),
    ("finalize running_mean", "pnx_bn_finalize", ("running_mean off by",)),
    ("finalize running_var", "pnx_bn_finalize", ("running_var off by",)),
    ("eval scale", "pnx_bn_eval_affine", ("scale / shift off by",)),
    ("eval shift", "pnx_bn_eval_affine", ("scale / shift off by",)),
    ("exact pnx_add_relu", "pnx_add_relu", ("differ from torch",)),
    ("exact pnx_relu_bwd", "pnx_relu_bwd", ("differ from torch",)),
    ("gather out", "pnx_tap_gather_sum", ("outputs differ",)),
    ("scatter dZ", "pnx_tap_scatter", ("dZ entries differ",)),
    ("loss res[0]", "pnx_center_loss_task", ("loss nan",)),
    ("loss res[1]", "pnx_center_loss_task", ("hm_loss nan",)),
    ("loss res[2]", "pnx_center_loss_task", ("loc_loss nan",)),
    ("loss res[3]", "pnx_center_loss_task", ("iou_reg_loss nan",)),
    ("loss res[4]", "pnx_center_loss_task", ("num_positive nan",)),
    ("loss res[11]", "pnx_center_loss_task", ("loc_loss_elem differs",)),
    ("loss res[15]", "pnx_center_loss_task", ("bad slots on valid labels",)),
    ("loss dout", "pnx_center_loss_task", ("d(loss)/d(out) off",)),
    ("bad-slot res[15]", "pnx_center_loss_task", ("bad slots: res[15] = nan",)),
    ("bad-slot dout", "pnx_center_loss_task", ("beyond the npos rescale",)),
    ("loss finalize res", "pnx_center_loss_finalize", ("res off by",)),
    ("loss finalize total", "pnx_center_loss_finalize", ("res off by",)),
]


def _smallest_replay(launches, fn, name):
    """Failures of the replay of the smallest configuration of `fn` (one that writes the poisoned output)."""
    if fn == "pnx_bn_bwd_reduce":
        c = min(_reduce_configs(launches), key=lambda c: c["M"] * c["C"])
        return _replay_bn_reduce(c, _bn_data(c["M"], c["C"]), _int_data(c["M"], c["C"]), (_mode(c),))[0]
    if fn == "pnx_bn_finalize":
        c = min([c for c in _of(launches, fn) if not c["count_ptr"]], key=lambda c: c["count_mult"] * c["channels"])
        return _replay_finalize(c, _bn_data(c["count_mult"], c["channels"]), False)[0]
    cfgs = _of(launches, fn)
    if fn == "pnx_bn_bwd_apply":
        c = min([c for c in cfgs if c["dres"] or "dres" not in name], key=lambda c: c["M"] * c["C"])
        return _replay_bn_bwd_apply(c, _bn_data(c["M"], c["C"]), _mode(c), c["dres_accumulate"])[0]
    if fn == "pnx_bn_apply":
        c = min(cfgs, key=lambda c: c["M"] * c["C"])
        return _replay_bn_apply(c, _bn_data(c["M"], c["C"]))[0]
    if fn in ("pnx_add_relu", "pnx_relu_bwd"):
        return _replay_exact(min(cfgs, key=lambda c: c["M"] * c["C"]))[0]
    if fn in ("pnx_tap_gather_sum", "pnx_tap_scatter"):
        return _replay_stencil(min(cfgs, key=lambda c: c["B"] * c["H"] * c["W"]))[0]
    if fn == "pnx_center_loss_task":
        return _replay_loss(min(cfgs, key=lambda c: c["B"] * c["H"] * c["W"]))[0]
    if fn == "pnx_bn_eval_affine":
        return _replay_eval_affine(min(cfgs, key=lambda c: c["channels"]))[0]
    return _replay_loss_finalize(cfgs[0])[0]


@pytest.mark.parametrize("name,fn,expect", NAN_CASES, ids=[c[0] for c in NAN_CASES])
def test_self_check_a_nan_in_a_kernel_output_fails_its_comparison(launches, name, fn, expect):
    """One kernel output element overwritten with NaN (in Python, after the launch) fails the comparison meant to
    catch it: no check lets a NaN through."""
    POISON.add(name)
    try:
        bad = _smallest_replay(launches, fn, name)
    finally:
        POISON.discard(name)
    print("%s: %s" % (name, bad))
    for e in expect:
        assert any(e in b for b in bad), "%s: no failure mentioning %r in %s" % (name, e, bad)


# ------------------------------------------------------------------------------------------------- completeness
def test_every_entry_point_of_the_step_is_covered(launches):
    """Every pnx_* entry point the step called is replayed here, replayed by tests/test_production_gemms_gpu.py, or on
    EXCLUDED with its reason."""
    print("\nentry points called: %s" % ", ".join(sorted(launches.called)))
    missing = sorted(n for n in launches.called if n not in ARG_MAPS and n not in GEMM_REPLAYED and n not in EXCLUDED)
    assert not missing, "entry points the step calls that no production replay covers: %s" % missing
    recorded = {c["fn"] for c in launches.configs}
    assert recorded >= set(ARG_MAPS) - {"pnx_add_rows"}, sorted(set(ARG_MAPS) - recorded)
