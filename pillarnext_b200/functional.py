"""torch.autograd glue: every differentiable op of the hot path as an autograd.Function whose forward AND
backward call libpnx kernels (pillarnext_b200/ops.py).  Activations between ops are bf16 row matrices
[rows, channels] (rows = active sites or channels-last pixels); parameters stay fp32 in the reference's
own layouts (state-dict compatible) and are repacked to the kernels' bf16 [tap, Cout, Cin] layout on the fly.
"""
import weakref

import torch
import torch.distributed as dist

from . import ops


# ------------------------------------------------------------------------------------------- precision mode
# "bf16"  : production path -- bf16 tensor-core operands and stored activations, fp32 accumulation.
# "split" : fp32-grade parity mode -- every activation is a (hi, lo) bf16 pair ([M, 2C] rows, include/pnx.h "split
#           rows"), the same wgmma kernels run over the hi/lo segments, raw conv outputs / BatchNorm / gradient sums
#           are fp32.  ~3x the tensor work and ~3x the bytes: used to demonstrate the north-star tolerance (1e-3 abs
#           vs the fp32 reference), not for throughput.
_PRECISION = "bf16"


PIECES = 3   # bf16 pieces per value in "split" mode: 2 = 16 mantissa bits, 3 = 24 bits (an exact fp32)


def set_precision(mode):
    global _PRECISION
    assert mode in ("bf16", "split")
    prev, _PRECISION = _PRECISION, mode
    if mode == "split":
        ops.split_pieces(PIECES)
    return prev


def get_precision():
    return _PRECISION


class precision:
    """with precision("split"): ...   (the mode is read at forward time and remembered for the backward)"""

    def __init__(self, mode):
        self.mode = mode

    def __enter__(self):
        self.prev = set_precision(self.mode)

    def __exit__(self, *a):
        set_precision(self.prev)


def _split():
    return _PRECISION == "split"


def set_deterministic(on):
    """Opt-in reproducible reductions for the bf16 path (debugging / regression hunting; slower):
      * BatchNorm statistics of the conv epilogues accumulate in fp64 (order effects 1e-16 instead of 1e-7), the fused
        BatchNorm-backward reduce is switched off in favour of the separate pass (fixed order inside a CTA, fp64 across CTAs);
    With it two runs of the same step give a bit-identical forward and bit-identical parameter gradients
    (tests/test_precision_gpu.py::test_run_to_run_spread_of_the_gradients; "bit-identical" up to the 1e-16 order effects
    of the remaining fp64 atomics, which vanish in the rounding to fp32).  Not covered: three or more positives of one
    class colliding on one heat-map cell (fp32 atomics in the loss gradient).  Returns the previous setting."""
    return ops.set_deterministic(on)


def _P():
    return ops.split_pieces()


_to_hilo = ops.to_pieces    # fp32 packed weights [..., K] -> bf16 [..., P*K] = [piece 0 | piece 1 | ...]


# ------------------------------------------------------------------------------------------- weights
class WLayout:
    """Packing between a parameter's native layout and the kernels' [taps, Cout, Cin] layout.
    kind: 'dense' nn.Conv2d [Cout,Cin,kh,kw] | 'sp' spconv [Cout,kH(y),kW(x),Cin] (tap = kx*3+ky, rulebook order)
          | 'convT' nn.ConvTranspose2d [Cin,Cout,2,2] (n = (dy*2+dx)*Cout + co)."""

    def __init__(self, kind):
        self.kind = kind

    def pack_fwd(self, w, split=False):
        if self.kind == "dense":
            co, ci, kh, kw = w.shape
            p = w.permute(2, 3, 0, 1).reshape(kh * kw, co, ci)
        elif self.kind == "sp":
            co, kh, kw, ci = w.shape
            p = w.permute(2, 1, 0, 3).reshape(kh * kw, co, ci)
        else:
            ci, co, kh, kw = w.shape
            p = w.permute(2, 3, 1, 0).reshape(1, kh * kw * co, ci)
        return _to_hilo(p.float()) if split else p.to(torch.bfloat16).contiguous()

    def pack_dgrad(self, w, flip, split=False):
        """[taps_d, Cin, Cout] bf16 for the data-gradient GEMM (split: [taps_d, Cin, 2*Cout] = hi | lo)."""
        if self.kind == "convT":
            ci, co, kh, kw = w.shape
            p = w.permute(2, 3, 0, 1).reshape(kh * kw, ci, co)
        else:
            if self.kind == "dense":
                co, ci, kh, kw = w.shape
                p = w.permute(2, 3, 0, 1).reshape(kh * kw, co, ci)
            else:
                co, kh, kw, ci = w.shape
                p = w.permute(2, 1, 0, 3).reshape(kh * kw, co, ci)
            if flip:
                p = p.flip(0)
            p = p.transpose(1, 2)
        return _to_hilo(p.float()) if split else p.to(torch.bfloat16).contiguous()

    def gather_desc(self, shape, which, flip):
        """The bf16 packed operand as a 4-D gather-copy of the fp32 parameter (pnx_pack_weights, csrc/pack.cu):
        (dims, element strides into the parameter, base offset) with dst contiguous over dims."""
        if self.kind == "sp":
            co, kh, kw, ci = shape
            if which == "fwd":
                return (kw, kh, co, ci), (ci, kw * ci, kh * kw * ci, 1), 0
            sg = -1 if flip else 1
            return (kw, kh, ci, co), (sg * ci, sg * kw * ci, 1, kh * kw * ci), ((kw - 1) * ci + (kh - 1) * kw * ci) if flip else 0
        if self.kind == "dense":
            co, ci, kh, kw = shape
            T = kh * kw
            if which == "fwd":
                return (1, T, co, ci), (0, 1, ci * T, T), 0
            return (1, T, ci, co), (0, -1 if flip else 1, T, ci * T), (T - 1) if flip else 0
        ci, co, kh, kw = shape
        T = kh * kw
        if which == "fwd":
            return (1, T, co, ci), (0, 1, T, co * T), 0
        return (1, T, ci, co), (0, 1, co * T, T), 0

    def unpack_grad(self, g, shape):
        """g fp32 [taps, Cout, Cin] (convT: [4, Cin, Cout]) -> gradient in the parameter's layout (always a fresh
        tensor: the accumulator may live in the per-step zero arena)."""
        if self.kind == "dense":
            co, ci, kh, kw = shape
            out = g.view(kh, kw, co, ci).permute(2, 3, 0, 1)
        elif self.kind == "sp":
            co, kh, kw, ci = shape
            out = g.view(kw, kh, co, ci).permute(2, 1, 0, 3)
        else:
            ci, co, kh, kw = shape
            out = g.view(kh, kw, ci, co).permute(2, 3, 0, 1)
        return out.clone(memory_format=torch.contiguous_format)


_pack_cache = {}
# Cache validity = (parameter version, optimizer generation).  The version counter alone is NOT enough: torch's fused
# optimizers (AdamW(fused=True), the reference-scale default here) update the parameters through kernels that do not bump
# `p._version` (measured on torch 2.11: version 0 -> 0 across step()), so a version-keyed cache would keep serving the
# initial bf16 weights for the whole training run.  A global post-step hook on every torch optimizer advances the
# generation; load_state_dict / manual in-place edits advance the version.
_OPT_GENERATION = [0]


def _on_optimizer_step(*_args, **_kwargs):
    _OPT_GENERATION[0] += 1


from torch.optim.optimizer import register_optimizer_step_post_hook as _register_post_step  # noqa: E402
_register_post_step(_on_optimizer_step)


def weights_changed():
    """For optimizers that bypass torch.optim (none in this repo): invalidate every packed weight."""
    _OPT_GENERATION[0] += 1



def packed(w, layout, which, flip=False, split=False):
    """Cache of bf16 packed weights keyed by parameter identity + version (repacked after optimizer steps).
    Only real parameters are cached: transient tensors (e.g. a torch.cat of sibling-head weights, a leaf under
    no_grad) have no stable identity and would only grow the cache."""
    if not isinstance(w, torch.nn.Parameter):
        with torch.no_grad():
            return layout.pack_fwd(w, split) if which == "fwd" else layout.pack_dgrad(w, flip, split)
    key = (id(w), which, flip, layout.kind, _P() if split else 0)
    ent = _pack_cache.get(key)
    ver = (w._version, _OPT_GENERATION[0])
    if ent is not None and ent[1]() is w and ent[3] == w.data_ptr():
        if ent[0] == ver:
            return ent[2]
        if not split and w.is_cuda and w.dtype == torch.float32 and w.is_contiguous():
            _repack_all(w.device)                      # every stale bf16 operand of the model in one launch
            ent = _pack_cache.get(key)
            if ent is not None and ent[0] == ver:
                return ent[2]
    with torch.no_grad():
        p = layout.pack_fwd(w, split) if which == "fwd" else layout.pack_dgrad(w, flip, split)
    if len(_pack_cache) > 4096:      # ids of dead tensors: drop everything rather than grow without bound
        _pack_cache.clear()
    _pack_cache[key] = (ver, weakref.ref(w), p, w.data_ptr())
    if not split:
        _pack_table["dirty"] = True
    return p


# One descriptor table for all cached bf16 operands (rebuilt when the set of entries changes -- the first two steps).
_pack_table = {"dirty": True, "chunks": [], "keys": [], "rebuilds": 0}


def _repack_all(device):
    """After an optimizer step (or any in-place parameter edit) rewrite EVERY cached bf16 operand on `device` in place with
    one pnx_pack_weights launch per 256 entries -- instead of ~2 torch kernels per (weight, layout) request."""
    import struct
    tb = _pack_table
    alive = all((e := _pack_cache.get(k)) is not None and (w := e[1]()) is not None and w.data_ptr() == e[3] for k in tb["keys"])
    if tb["dirty"] or not alive or tb.get("device") != device:
        keys, chunks, blob, start = [], [], bytearray(), 0
        for k, e in list(_pack_cache.items()):
            w = e[1]()
            if w is None or w.data_ptr() != e[3]:
                del _pack_cache[k]
                continue
            if k[4] != 0 or w.device != device or w.dtype != torch.float32 or not w.is_contiguous():
                continue
            dims, strides, base = WLayout(k[3]).gather_desc(tuple(w.shape), k[1], k[2])
            blob += struct.pack("<QQqq4q4i", w.data_ptr(), e[2].data_ptr(), start, base, *strides, *dims)
            start += e[2].numel()
            keys.append(k)
            if len(keys) % 256 == 0:
                chunks.append((blob, 256, start))
                blob, start = bytearray(), 0
        if len(keys) % 256:
            chunks.append((blob, len(keys) % 256, start))
        # pinned staging + async copy: a pageable .to(device) would block the host until the stream drains
        tb["host"] = [torch.frombuffer(b, dtype=torch.uint8).clone().pin_memory() for b, _, _ in chunks]
        tb["chunks"] = [(h.to(device, non_blocking=True), n, tot) for h, (_, n, tot) in zip(tb["host"], chunks)]
        tb["keys"], tb["dirty"], tb["device"] = keys, False, device
        tb["rebuilds"] += 1
    for table, n, tot in tb["chunks"]:
        ops.pack_weights(table, n, tot)
    gen = _OPT_GENERATION[0]
    for k in tb["keys"]:
        e = _pack_cache[k]
        _pack_cache[k] = ((e[1]()._version, gen), e[1], e[2], e[3])


class ConvSpec:
    """Row space and neighbour map of one convolution application.
       fwd: (nbr table | dense geometry | identity) over M_out output rows, reading M_in input rows.
       bwd: table / geometry of the data-gradient GEMM (+ whether taps are flipped)."""

    def __init__(self, M_out, M_in, taps, nbr=None, dense=None, d_nbr=None, d_dense=None, d_flip=False, d_taps=None,
                 shuffle=False):
        self.M_out, self.M_in, self.taps = M_out, M_in, taps
        self.nbr, self.dense = nbr, dense
        self.d_nbr, self.d_dense, self.d_flip = d_nbr, d_dense, d_flip
        self.d_taps = taps if d_taps is None else d_taps
        self.shuffle = shuffle


def dense_spec(B, H, W, k, dil=1):
    """Stride-1 'same' convolution on a channels-last image (zero padding = absent neighbour)."""
    pad = dil * (k // 2)
    geo = (H, W, H, W, k, 1, dil, pad)
    M = B * H * W
    return ConvSpec(M, M, k * k, dense=geo if k > 1 else None, d_dense=geo if k > 1 else None, d_flip=True)


def convT_spec(B, H, W):
    """ConvTranspose2d k2 s2: rows = input pixels, output image 2H x 2W."""
    return ConvSpec(B * H * W, B * H * W, 1, dense=(H, W, H, W, 1, 1, 1, 0), d_dense=(H, W, 2 * H, 2 * W, 2, 2, 1, 0),
                    d_taps=4, shuffle=True)


# ------------------------------------------------------------------------------------------- fused BN-backward reduce
class BNInfo:
    """Link between a BatchNorm(+ReLU) layer and the GEMM that produces the gradient of its output.  BNActFn.forward
    fills the forward quantities; the consumer's backward passes them to the GEMM epilogue (pnx_igemm / pnx_conv3x3_win
    `bnr_*` arguments), which gates dy with the ReLU mask and accumulates the two per-channel sums into `red`;
    BNActFn.backward then only runs the apply pass."""
    __slots__ = ("raw", "scale", "shift", "mean", "invstd", "C", "M", "red", "fused")

    def __init__(self):
        self.raw = self.red = None
        self.fused = False


# The fused reduce adds ~7 instructions per output element to the GEMM epilogue.  For the 3x3 convolutions (K = 9 * C >=
# 576 MMA steps per tile) that is small against the MMA loop and it removes a full sweep over dy and raw; for the thin
# GEMMs (the head's final-conv data gradient, K = 192, and the ConvTranspose2d one, K = 256) the epilogue is already the
# larger part of the kernel -- so it is applied only above this K.
FUSE_BN_REDUCE_MIN_K = 512


def _claim_bn_reduce(info, M, C, k_total):
    """The BNInfo to hand to the GEMM producing a [M, C] gradient (K = k_total), or None when the fused path does not
    apply.  All consumers of one BatchNorm output must make the same decision: they share the shape, so they do."""
    if info is None or info.raw is None or info.C != C or info.M != M or not ops.bnr_eligible(C) or k_total < FUSE_BN_REDUCE_MIN_K:
        return None
    if ops.DETERMINISTIC:          # the fused reduce goes through fp32 shared-memory partials in arrival order
        return None
    if info.red is None:
        info.red = ops.zeros(2 * C, torch.float64, info.raw.device)
    info.fused = True
    return info


# ------------------------------------------------------------------------------------------- conv
class ConvFn(torch.autograd.Function):
    """out = conv(x; w) (+bias) (relu) through pnx_igemm; optional BatchNorm statistics of the output.
    x bf16 [M_in, >=Cin]; returns (out [M_out(*4 if shuffle), Cout], stats fp64 [2*Cs] or empty)."""

    @staticmethod
    def forward(ctx, x, w, bias, spec, layout, want_stats, out_fp32, relu, bias_feeds_bn, bn_src=None):
        shape = tuple(w.shape)
        if layout.kind == "dense":
            cout, cin = shape[0], shape[1]
        elif layout.kind == "sp":
            cout, cin = shape[0], shape[3]
        else:
            cin, cout = shape[0], shape[1]
        split = _split()
        wp = packed(w, layout, "fwd", split=split)
        n_cols = wp.shape[1]
        rows = spec.M_out * (4 if spec.shuffle else 1)
        out_c = cout
        if split:
            out_fp32 = True      # raw convolution outputs stay fp32 in the fp32-grade mode
            assert not relu and x.shape[1] % _P() == 0 and x.shape[1] // _P() >= cin
        out = torch.empty(rows, out_c, dtype=torch.float32 if out_fp32 else torch.bfloat16, device=x.device)
        stats = ops.zeros(2 * cout if want_stats else 0, torch.float64, x.device)
        if split:
            ops.igemm(x, spec.M_out, wp, wp.shape[0], cin, n_cols, out, lda=x.stride(0), ldc=out_c, nbr=spec.nbr,
                      dense=spec.dense, bias=bias, stats=stats if want_stats else None,
                      stats_mod=cout if want_stats else None, shuffle=spec.shuffle, segs=ops.split_segments(), a_lo_off=x.shape[1] // _P())
        elif layout.kind == "dense" and spec.nbr is None and ops.win_eligible(spec.dense, n_cols, cin, out_fp32, spec.shuffle):
            H_, W_ = spec.dense[0], spec.dense[1]
            ops.conv3x3_win(x, spec.M_out // (H_ * W_), H_, W_, wp, cin, n_cols, out, bias=bias,
                            stats=stats if want_stats else None, relu=relu)          # im2col folded into TMA
        else:
            ops.igemm(x, spec.M_out, wp, wp.shape[0], cin, n_cols, out, lda=x.stride(0), ldc=out_c, nbr=spec.nbr,
                      dense=spec.dense, bias=bias, stats=stats if want_stats else None,
                      stats_mod=cout if want_stats else None, shuffle=spec.shuffle, relu=relu)
        ctx.save_for_backward(x, w, out if relu else None)
        ctx.spec, ctx.layout, ctx.dims = spec, layout, (cin, cout, shape)
        ctx.has_bias, ctx.relu, ctx.out_fp32 = bias is not None, relu, out_fp32
        ctx.bias_feeds_bn = bool(bias_feeds_bn)
        ctx.split = split
        ctx.bn_src = bn_src if (bn_src is not None and not split) else None
        ctx.mark_non_differentiable(stats)
        return out, stats

    @staticmethod
    def _backward_split(ctx, dout):
        """fp32-grade mode: dout = split rows [rows, 2*cout]; data gradient = hi/lo-segment GEMM -> fp32 -> split rows,
        weight gradient = three launches (hi*hi, lo*hi, hi*lo) into the same fp32 accumulator."""
        x, w, _ = ctx.saved_tensors
        spec, layout = ctx.spec, ctx.layout
        cin, cout, shape = ctx.dims
        rows = dout.shape[0]
        assert dout.dtype == torch.float32 and dout.shape[1] == cout and cout % 64 == 0, "split mode: fp32 gradient rows [M, Cout]"
        dy = ops.rows_split(dout.contiguous())                          # the conv output is fp32, so is its gradient
        xlo = x.shape[1] // _P()
        dbias = None
        if ctx.has_bias:
            dbias = torch.zeros(cout, dtype=torch.float32, device=dy.device) if ctx.bias_feeds_bn else \
                dout.sum(0)
        dx = None
        if ctx.needs_input_grad[0]:
            wd = packed(w, layout, "dgrad", spec.d_flip, split=True)        # [taps_d, Cin, P*Cout]
            d32 = torch.empty(spec.M_in, cin, dtype=torch.float32, device=dy.device)
            ops.igemm(dy, spec.M_in, wd, wd.shape[0], cout, cin, d32, nbr=spec.d_nbr, dense=spec.d_dense, segs=ops.split_segments(), a_lo_off=cout)
            dx = torch.zeros(x.shape[0], x.shape[1], dtype=torch.bfloat16, device=dy.device) if xlo != cin else \
                torch.empty(x.shape[0], x.shape[1], dtype=torch.bfloat16, device=dy.device)
            ops.rows_split(d32, cin, out=dx, lo=xlo)
        dw = None
        if ctx.needs_input_grad[1]:
            if layout.kind == "convT":
                g = torch.zeros(4, cin, cout, dtype=torch.float32, device=dy.device)
                ops.wgrad_split(x, xlo, cin, dy, cout, cout, spec.M_out, 4, g, dense=spec.d_dense, shuffle=True)
            else:
                g = torch.zeros(spec.taps, cout, cin, dtype=torch.float32, device=dy.device)
                ops.wgrad_split(dy, cout, cout, x, xlo, cin, spec.M_out, spec.taps, g, nbr=spec.nbr, dense=spec.dense)
            dw = layout.unpack_grad(g, shape)
        return dx, dw, dbias, None, None, None, None, None, None, None

    @staticmethod
    def backward(ctx, dout, _dstats):
        if ctx.split:
            return ConvFn._backward_split(ctx, dout)
        x, w, out = ctx.saved_tensors
        spec, layout = ctx.spec, ctx.layout
        cin, cout, shape = ctx.dims
        rows = dout.shape[0]
        # gradient rows as bf16, channel count padded to a multiple of 64 for the tensor-core kernels
        cpad = (cout + 63) // 64 * 64
        if dout.dtype != torch.bfloat16 or cpad != cout or not dout.is_contiguous():
            dy = torch.zeros(rows, cpad, dtype=torch.bfloat16, device=dout.device) if cpad != cout else \
                torch.empty(rows, cpad, dtype=torch.bfloat16, device=dout.device)
            dy[:, :cout] = dout
        else:
            dy = dout
        if ctx.relu:
            g = torch.empty_like(dy)
            ops.relu_bwd(dy, out, rows, cout, g)
            dy = g
        if not ctx.has_bias:
            dbias = None
        elif ctx.bias_feeds_bn:
            # conv bias in front of a training-mode BatchNorm: BN's input gradient sums to zero per channel, so the
            # bias gradient is exactly 0 (the reference's autograd produces ~1e-7 rounding noise there)
            dbias = torch.zeros(cout, dtype=torch.float32, device=dy.device)
        else:
            dbias = torch.sum(dy[:, :cout], dim=0, dtype=torch.float32)   # fp32 accumulate, no fp32 copy
        dx = None
        if ctx.needs_input_grad[0]:
            wd = packed(w, layout, "dgrad", spec.d_flip)            # [taps_d, Cin, Cout]
            if cpad != cout:
                wd = torch.nn.functional.pad(wd, (0, cpad - cout))
            dx = torch.empty(spec.M_in, cin, dtype=torch.bfloat16, device=dy.device)
            bnr = _claim_bn_reduce(ctx.bn_src, spec.M_in, cin, wd.shape[0] * cpad) if x.shape[1] == cin else None
            if layout.kind == "dense" and spec.d_nbr is None and ops.win_eligible(spec.d_dense, cin, cpad):
                H_, W_ = spec.d_dense[0], spec.d_dense[1]
                ops.conv3x3_win(dy, spec.M_in // (H_ * W_), H_, W_, wd, cpad, cin, dx, bnr=bnr)
            else:
                ops.igemm(dy, spec.M_in, wd, wd.shape[0], cpad, cin, dx, nbr=spec.d_nbr, dense=spec.d_dense, bnr=bnr)
            if x.shape[1] != cin:                                   # x was a column slice of a wider buffer
                full = torch.zeros(x.shape[0], x.shape[1], dtype=torch.bfloat16, device=dy.device)
                full[:, :cin] = dx
                dx = full
        dw = None
        if ctx.needs_input_grad[1]:
            if layout.kind == "convT":
                g = ops.zeros((4, cin, cout), torch.float32, dy.device)
                ops.wgrad(x, cin, dy, cout, spec.M_out, 4, g, dense=spec.d_dense, shuffle=True)
            else:
                # X = output gradient (direct), Y = layer input (gathered): result is [tap, Cout(pad), Cin]
                g = ops.zeros((spec.taps, cpad, cin), torch.float32, dy.device)
                ops.wgrad(dy, cpad, x, cin, spec.M_out, spec.taps, g, nbr=spec.nbr, dense=spec.dense)
                if cpad != cout:
                    g = g[:, :cout].contiguous()
            dw = layout.unpack_grad(g, shape)
        return dx, dw, dbias, None, None, None, None, None, None, None


def conv(x, w, bias, spec, layout, want_stats=False, out_fp32=False, relu=False, bias_feeds_bn=False, bn_src=None):
    """bn_src: the BNInfo of `x` when x = relu(bn(.)) is consumed by this convolution ONLY (or only by convolutions that
    all pass it): the data-gradient GEMM then also performs the reduce pass of that BatchNorm's backward."""
    return ConvFn.apply(x, w, bias, spec, layout, want_stats, out_fp32, relu, bias_feeds_bn, bn_src)


# ------------------------------------------------------------------------------------------- batch norm
def wants_sync(bn):
    """SyncBatchNorm semantics requested for this BN holder: either through enable_sync_batchnorm() (`pnx_sync`) or
    because tools/train.py:55-56 replaced it with torch.nn.SyncBatchNorm (`convert_sync_batchnorm` copies parameters
    and buffers into a new module whose forward this package never calls -- only its type carries the request)."""
    return bool(getattr(bn, "pnx_sync", False)) or isinstance(bn, torch.nn.SyncBatchNorm)


NBT_PENDING = None     # when a list: num_batches_tracked buffers to bump with ONE foreach add at the end of the forward


def bump_batches_tracked(bn):
    if bn.num_batches_tracked is None:
        return
    if NBT_PENDING is not None:
        NBT_PENDING.append(bn.num_batches_tracked)
    else:
        bn.num_batches_tracked += 1


def _sync_enabled(bn):
    return wants_sync(bn) and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1


class BNActFn(torch.autograd.Function):
    """y = relu?(BatchNorm(x_raw) (+ residual)), batch statistics taken from the conv epilogue (`stats`).
    Training: biased batch variance, running stats updated in place (momentum/eps of `bn`).
    pnx_sync (SyncBatchNorm semantics, reference tools/train.py:55-56): statistics all-reduced over ranks."""

    @staticmethod
    def forward(ctx, x_raw, stats, gamma, beta, residual, bn, relu, count, info=None):
        M, C = x_raw.shape
        count_dev = None
        if bn.training:
            if _sync_enabled(bn):
                # SyncBatchNorm (reference tools/train.py:55-56): sums and population of all ranks in one small all-reduce;
                # the global count stays on the device (no host synchronisation)
                pack = torch.cat([stats, torch.full((1,), float(count), dtype=torch.float64, device=stats.device)])
                dist.all_reduce(pack)
                stats, count_dev = pack[:-1], pack[-1:].round().to(torch.int32)
            mom = bn.momentum if bn.momentum is not None else 0.1
            scale, shift, mean, invstd = ops.bn_finalize(stats, C, count_dev, 1 if count_dev is not None else int(count), gamma, beta,
                                                         bn.eps, mom, bn.running_mean, bn.running_var)
            bump_batches_tracked(bn)
        else:
            scale, shift = ops.bn_eval_affine(gamma, beta, bn.running_mean, bn.running_var, bn.eps)
            mean = invstd = None
        ctx.split = x_raw.dtype == torch.float32
        if ctx.split:            # fp32-grade mode: fp32 raw conv output -> split rows
            y = torch.empty(M, _P() * C, dtype=torch.bfloat16, device=x_raw.device)
            ops.bn_apply_split(x_raw, M, C, scale, shift, y, C, res=residual, res_lo=C, relu=relu)
        else:
            y = torch.empty(M, C, dtype=torch.bfloat16, device=x_raw.device)
            ops.bn_apply(x_raw, M, C, scale, shift, y, res=residual, relu=relu)
        ctx.save_for_backward(x_raw, y, gamma, mean, invstd, scale, shift)
        ctx.relu, ctx.count, ctx.has_res, ctx.sync, ctx.training = relu, count, residual is not None, _sync_enabled(bn), bn.training
        ctx.count_dev = count_dev if bn.training else None
        ctx.info = None
        if info is not None and bn.training and relu and residual is None and not ctx.split:
            info.raw, info.scale, info.shift, info.mean, info.invstd, info.C, info.M = x_raw, scale, shift, mean, invstd, C, M
            info.red, info.fused = None, False
            ctx.info = info
        return y

    @staticmethod
    def _backward_split(ctx, dy):
        x_raw, y, gamma, mean, invstd, scale, shift = ctx.saved_tensors
        M, C = x_raw.shape
        dy = dy.contiguous()
        P = _P()
        assert dy.shape[1] == P * C
        ysrc = y if ctx.has_res else None
        red = ops.bn_bwd_reduce_split(dy, C, ysrc, C, x_raw, M, C, mean, invstd, ctx.relu, (scale, shift))
        local = red
        if ctx.sync:
            raise NotImplementedError("SyncBatchNorm backward is not available in the fp32-grade split mode (single-GPU parity tool)")
        dxs = torch.empty(M, P * C, dtype=torch.bfloat16, device=dy.device)
        dres = torch.empty(M, P * C, dtype=torch.bfloat16, device=dy.device) if ctx.has_res else None
        ops.bn_bwd_apply_split(dy, C, ysrc, C, x_raw, M, C, mean, invstd, gamma, red, ctx.count, ctx.relu, (scale, shift),
                               dxs, C, dres=dres, dres_lo=C)
        dx = ops.rows_merge(dxs, C, C)          # x_raw is an fp32 [M, C] tensor: its gradient has the same shape / dtype
        r = local.float()
        return dx, None, r[C:], r[:C], dres, None, None, None, None

    @staticmethod
    def backward(ctx, dy):
        if not ctx.training:
            raise RuntimeError("pillarnext_b200: backward through eval-mode BatchNorm is not supported")
        if ctx.split:
            return BNActFn._backward_split(ctx, dy)
        x_raw, y, gamma, mean, invstd, scale, shift = ctx.saved_tensors
        M, C = x_raw.shape
        dy = dy.contiguous()
        dx = torch.empty(M, C, dtype=torch.bfloat16, device=dy.device)
        dres = torch.empty(M, C, dtype=torch.bfloat16, device=dy.device) if ctx.has_res else None
        from ._lib import check, lib, ptr, stream
        info = ctx.info
        fused = info is not None and info.fused
        # without a residual the ReLU mask is recomputed from x_raw (one row-matrix read less per pass)
        ysrc = y if ctx.has_res else None
        yp, ys = (ptr(ysrc), ysrc.stride(0)) if ysrc is not None else (None, 8)
        if fused:
            local = info.red          # the reduce pass ran in the epilogue of the GEMM that produced dy (= gated g)
            info.red, info.fused = None, False
        else:
            local = ops.zeros(2 * C, torch.float64, dy.device)
            ops._count(1)
            check(lib().pnx_bn_bwd_reduce(ptr(dy), dy.stride(0), yp, ys, ptr(x_raw), x_raw.stride(0), M, C, ptr(mean), ptr(invstd),
                                          1 if ctx.relu else 0, ptr(scale), ptr(shift), ptr(local), stream()))
        red = local
        if ctx.sync:                  # SyncBatchNorm: the two sums over all ranks (dgamma / dbeta stay local, DDP averages them)
            red = local.clone()
            dist.all_reduce(red)
        ops._count(1)
        check(lib().pnx_bn_bwd_apply(ptr(dy), dy.stride(0), yp, ys, ptr(x_raw), x_raw.stride(0), M, C, ptr(mean), ptr(invstd),
                                     ptr(gamma), ptr(red), float(max(ctx.count, 1)), ptr(ctx.count_dev) if ctx.count_dev is not None else None,
                                     1 if (ctx.relu and not fused) else 0,
                                     ptr(scale), ptr(shift), ptr(dx), dx.stride(0), ptr(dres) if dres is not None else None,
                                     dres.stride(0) if dres is not None else 8, 0, stream()))
        r = local.float()
        return dx, None, r[C:], r[:C], dres, None, None, None, None


def bn_info():
    return BNInfo()


def bn_act(x_raw, stats, bn, relu=True, residual=None, count=None, info=None):
    """info: a BNInfo to fill (see conv(bn_src=...)): pass it when the output has a single, convolution consumer."""
    return BNActFn.apply(x_raw, stats, bn.weight, bn.bias, residual, bn, relu, x_raw.shape[0] if count is None else count, info)


# ------------------------------------------------------------------------------------------- fp32 <-> split rows
class SplitFn(torch.autograd.Function):
    """fp32 rows [M, C] -> split rows [M, P*C] (fp32-grade mode); backward merges the gradient pieces."""

    @staticmethod
    def forward(ctx, x):
        ctx.C = x.shape[1]
        return ops.rows_split(x.contiguous())

    @staticmethod
    def backward(ctx, d):
        return ops.rows_merge(d.contiguous(), ctx.C, ctx.C)


class MergeFn(torch.autograd.Function):
    """split rows [M, 2C] -> fp32 rows [M, C]; backward splits the fp32 gradient."""

    @staticmethod
    def forward(ctx, x):
        C = x.shape[1] // _P()
        return ops.rows_merge(x.contiguous(), C, C)

    @staticmethod
    def backward(ctx, d):
        return ops.rows_split(d.contiguous())


class FanOutFn(torch.autograd.Function):
    """A split activation with several consumers: autograd would add the consumers' gradients piece by piece in bf16
    (each piece sum rounded to 8 bits -- bf16-level error at every residual junction); this node hands every consumer
    its own copy and accumulates the incoming gradients in fp32 before splitting the sum again."""

    @staticmethod
    def forward(ctx, x, n):
        ctx.C = x.shape[1] // _P()
        return tuple(x.clone() for _ in range(n))

    @staticmethod
    def backward(ctx, *ds):
        acc = None
        for d in ds:
            if d is None:
                continue
            d = d.contiguous()
            if acc is None:
                acc = ops.rows_merge(d, ctx.C, ctx.C)
            else:
                ops.rows_merge(d, ctx.C, ctx.C, out=acc, accumulate=True)
        return (ops.rows_split(acc) if acc is not None else None), None


def fanout(x, n=2):
    """n handles of an activation that has n consumers (identity in the bf16 mode, FanOutFn in the split mode)."""
    if _split() and torch.is_grad_enabled() and x.requires_grad:
        return FanOutFn.apply(x, n)
    return (x,) * n


# ------------------------------------------------------------------------------------------- dense()
class DensifyFn(torch.autograd.Function):
    """SparseConvTensor.dense() (sparse_resnet.py:68) into channels-last rows [B*H*W, C]; backward gathers."""

    @staticmethod
    def forward(ctx, feat, level):
        C = feat.shape[1]
        canvas = ops.scatter_dense(feat, level, C)
        ctx.level, ctx.C = level, C
        return canvas.view(-1, C)

    @staticmethod
    def backward(ctx, dcanvas):
        lv, C = ctx.level, ctx.C
        d = torch.empty(max(lv.n, 1), C, dtype=torch.bfloat16, device=dcanvas.device)[:lv.n]
        g = dcanvas.contiguous().view(lv.batch, lv.V, lv.U, C)
        if lv.n:
            ops.scatter_dense(d, lv, C, canvas=g, gather=True)
        return d, None


# ------------------------------------------------------------------------------------------- ASPP branches
class ASPPBranchesFn(torch.autograd.Function):
    """x = relu(o + idt) (BasicBlock tail, conv.py:48-50) written straight into slot 0 of the concat buffer, then
    cat(x, conv1x1(x), W(*)x d=1, d=6, d=12, d=18) (aspp.py:21-31): five GEMMs writing the other column slots of
    the one [M, 6C] buffer.  Backward: five data-gradient GEMMs chained through the epilogue addend, weight
    gradients of the four dilations accumulated into the one shared tensor, then the ReLU mask."""
    DILS = (1, 6, 12, 18)

    @staticmethod
    def _forward_split(ctx, o, idt, w1x1, wshared, B, H, W):
        """fp32-grade mode: cat buffer [M, P*6C] = six piece-0 slots, six piece-1 slots, ... (a split matrix, lo = 6C)."""
        M, C = o.shape[0], o.shape[1] // _P()
        C6, ld = 6 * C, _P() * 6 * C
        cat_buf = torch.empty(M, ld, dtype=torch.bfloat16, device=o.device)
        l = WLayout("dense")
        ops.add_relu_split(o, C, idt, C, M, C, cat_buf, C6)
        tmp = torch.empty(M, C, dtype=torch.float32, device=o.device)
        ops.igemm(cat_buf, M, packed(w1x1, l, "fwd", split=True), 1, C, C, tmp, lda=ld, segs=ops.split_segments(), a_lo_off=C6)
        ops.rows_split(tmp, C, out=cat_buf[:, C:], lo=C6)
        wp = packed(wshared, l, "fwd", split=True)
        for j, d in enumerate(ASPPBranchesFn.DILS):
            ops.igemm(cat_buf, M, wp, 9, C, C, tmp, lda=ld, dense=(H, W, H, W, 3, 1, d, d), segs=ops.split_segments(), a_lo_off=C6)
            ops.rows_split(tmp, C, out=cat_buf[:, (2 + j) * C:], lo=C6)
        ctx.save_for_backward(cat_buf, w1x1, wshared)
        ctx.geo = (B, H, W, C)
        ctx.split = True
        return cat_buf

    @staticmethod
    def _backward_split(ctx, dcat):
        cat_buf, w1x1, wshared = ctx.saved_tensors
        B, H, W, C = ctx.geo
        M = cat_buf.shape[0]
        C6, ld = 6 * C, _P() * 6 * C
        l = WLayout("dense")
        dcat = dcat.contiguous()
        dx = ops.rows_merge(dcat, C, C6)                                   # fp32 accumulator of the five branches
        nxt = torch.empty_like(dx)
        ops.igemm(dcat[:, C:], M, packed(w1x1, l, "dgrad", True, split=True), 1, C, C, nxt, lda=ld, addend=dx, segs=ops.split_segments(), a_lo_off=C6)
        dx, nxt = nxt, dx
        wd = packed(wshared, l, "dgrad", True, split=True)
        for j, d in enumerate(ASPPBranchesFn.DILS):
            ops.igemm(dcat[:, (2 + j) * C:], M, wd, 9, C, C, nxt, lda=ld, dense=(H, W, H, W, 3, 1, d, d), addend=dx, segs=ops.split_segments(), a_lo_off=C6)
            dx, nxt = nxt, dx
        g1 = torch.zeros(1, C, C, dtype=torch.float32, device=dcat.device)
        ops.wgrad_split(dcat[:, C:], C6, C, cat_buf, C6, C, M, 1, g1)
        gs = torch.zeros(9, C, C, dtype=torch.float32, device=dcat.device)
        for j, d in enumerate(ASPPBranchesFn.DILS):
            ops.wgrad_split(dcat[:, (2 + j) * C:], C6, C, cat_buf, C6, C, M, 9, gs, dense=(H, W, H, W, 3, 1, d, d))
        g = torch.empty(M, _P() * C, dtype=torch.bfloat16, device=dcat.device)
        ops.relu_bwd_split(dx, cat_buf, C6, M, C, g, C)
        return g, g, l.unpack_grad(g1, tuple(w1x1.shape)), l.unpack_grad(gs, tuple(wshared.shape)), None, None, None

    @staticmethod
    def forward(ctx, o, idt, w1x1, wshared, B, H, W):
        if _split():
            return ASPPBranchesFn._forward_split(ctx, o, idt, w1x1, wshared, B, H, W)
        ctx.split = False
        M, C = o.shape
        C6 = 6 * C
        cat_buf = torch.empty(M, C6, dtype=torch.bfloat16, device=o.device)
        l = WLayout("dense")
        x = cat_buf[:, :C]
        ops.add_relu(o, idt, M, C, x)
        ops.igemm(x, M, packed(w1x1, l, "fwd"), 1, C, C, cat_buf[:, C:2 * C], lda=C6, ldc=C6)
        wp = packed(wshared, l, "fwd")
        for j, d in enumerate(ASPPBranchesFn.DILS):
            ops.igemm(x, M, wp, 9, C, C, cat_buf[:, (2 + j) * C:(3 + j) * C], lda=C6, ldc=C6, dense=(H, W, H, W, 3, 1, d, d))
        ctx.save_for_backward(cat_buf, w1x1, wshared)
        ctx.geo = (B, H, W, C)
        return cat_buf

    @staticmethod
    def backward(ctx, dcat):
        if ctx.split:
            return ASPPBranchesFn._backward_split(ctx, dcat)
        cat_buf, w1x1, wshared = ctx.saved_tensors
        B, H, W, C = ctx.geo
        M, C6 = cat_buf.shape
        l = WLayout("dense")
        dcat = dcat.contiguous()
        x = cat_buf[:, :C]
        # dx = dcat[:, 0:C] + dgrad_1x1(dcat[:, C:2C]) + sum_d dgrad_d(dcat[:, slot d])
        dx = torch.empty(M, C, dtype=torch.bfloat16, device=dcat.device)
        ops.igemm(dcat[:, C:2 * C], M, packed(w1x1, l, "dgrad", True), 1, C, C, dx, lda=C6, addend=dcat[:, :C])
        wd = packed(wshared, l, "dgrad", True)
        for j, d in enumerate(ASPPBranchesFn.DILS):
            nxt = torch.empty_like(dx)
            ops.igemm(dcat[:, (2 + j) * C:(3 + j) * C], M, wd, 9, C, C, nxt, lda=C6, dense=(H, W, H, W, 3, 1, d, d), addend=dx)
            dx = nxt
        g1 = ops.zeros((1, C, C), torch.float32, dcat.device)
        ops.wgrad(dcat[:, C:2 * C], C, x, C, M, 1, g1)
        gs = ops.zeros((9, C, C), torch.float32, dcat.device)
        for j, d in enumerate(ASPPBranchesFn.DILS):
            ops.wgrad(dcat[:, (2 + j) * C:(3 + j) * C], C, x, C, M, 9, gs, dense=(H, W, H, W, 3, 1, d, d))
        g = torch.empty(M, C, dtype=torch.bfloat16, device=dcat.device)
        ops.relu_bwd(dx, x, M, C, g)
        return g, g, l.unpack_grad(g1, tuple(w1x1.shape)), l.unpack_grad(gs, tuple(wshared.shape)), None, None, None


# ------------------------------------------------------------------------------------------- reader
class PFNFn(torch.autograd.Function):
    """PillarFeatureNet on pre-voxelized points: returns feat fp32 [P, 64] (pillar_encoder.py:174-182)."""

    @staticmethod
    def forward(ctx, w0, g0, b0, w1, g1, b1, voxels, bn0, bn1, training):
        P, _ = voxels.sync_counts()
        fwd = ops.pfn_forward(voxels, w0, (g0, b0, bn0.running_mean, bn0.running_var), w1,
                              (g1, b1, bn1.running_mean, bn1.running_var), training, eps=bn0.eps, momentum=bn0.momentum,
                              sync=_sync_enabled(bn0) or _sync_enabled(bn1))
        if training:
            for bn in (bn0, bn1):
                bump_batches_tracked(bn)
        ctx.voxels, ctx.fwd, ctx.training = voxels, fwd, training
        ctx.save_for_backward(w1, g0, g1)
        voxels.feat_bf16 = fwd["feat_bf16"]
        return fwd["feat"][:P]

    @staticmethod
    def backward(ctx, dfeat):
        if not ctx.training:
            raise RuntimeError("pillarnext_b200: backward through an eval-mode reader is not supported")
        w1, g0, g1 = ctx.saved_tensors
        dW0, dW1, dg0, db0, dg1, db1 = ops.pfn_backward(ctx.voxels, ctx.fwd, dfeat.contiguous().float(), w1, g0, g1)
        return dW0, dg0, db0, dW1, dg1, db1, None, None, None, None


class ToBF16RowsFn(torch.autograd.Function):
    """fp32 [P,64] reader output -> the bf16 copy the PFN kernel already wrote (identity for autograd)."""

    @staticmethod
    def forward(ctx, feat, feat_bf16):
        return feat_bf16[:feat.shape[0]]

    @staticmethod
    def backward(ctx, d):
        return d.float(), None


# ------------------------------------------------------------------------------------------- fused loss
class CenterLossFn(torch.autograd.Function):
    """CenterHead.loss (centerhead.py:142-229) for all tasks: value and d(loss)/d(head output) from libpnx
    (pnx_center_loss_task / _finalize).  Inputs: one channels-last fp32 head matrix [B*H*W, npad] per task."""

    @staticmethod
    def forward(ctx, meta, *outs):
        import ctypes
        from ._lib import check, lib, ptr, stream
        T = len(outs)
        dev = outs[0].device
        acc = ops.zeros((T, 16), torch.float64, dev)
        res = torch.empty(T, 16, dtype=torch.float32, device=dev)
        total = torch.empty(1, dtype=torch.float32, device=dev)
        douts = []
        cw = (ctypes.c_float * 10)(*meta["code_weights"])
        for t, out in enumerate(outs):
            m = meta["tasks"][t]
            ex = m["labels"]
            dout = torch.empty_like(out)
            ops._count(2)
            check(lib().pnx_center_loss_task(ptr(out), ptr(dout), ptr(ex["hm"]), ptr(ex["anno_box"]), ptr(ex["ind"]),
                                             ptr(ex["mask"]), ptr(ex["cat"]), ptr(ex["gt_boxes"]), m["B"], m["H"], m["W"],
                                             m["npad"], m["C"], m["M"], m["off"]["reg"], m["off"]["height"], m["off"]["dim"],
                                             m["off"]["rot"], m["off"]["vel"], m["off"]["hm"], m["sx"], m["sy"], m["ox"], m["oy"],
                                             meta["weight"], ctypes.cast(cw, ctypes.c_void_p), 1 if meta["with_reg_iou"] else 0,
                                             ptr(acc[t]), stream()))
            douts.append(dout)
        ops._count(1)
        check(lib().pnx_center_loss_finalize(ptr(acc), T, ptr(meta["weights_dev"]), ptr(meta["code_w_dev"]),
                                             ptr(meta["with_iou_dev"]), ptr(res), ptr(total), stream()))
        ctx.douts = douts
        ctx.mark_non_differentiable(res)
        return total[0], res

    @staticmethod
    def backward(ctx, g_total, _g_res):
        # out of place: the cached gradients stay valid for a second backward (retain_graph) and are never aliased
        return (None,) + tuple(d * g_total for d in ctx.douts)


# ------------------------------------------------------------------------------------------- head final convs
class HeadFinalConvFn(torch.autograd.Function):
    """The sibling heads' final Conv2d(64, c, 3) (centerhead.py:44-46) as ONE 1x1 tensor-core GEMM (N = 9 taps x cpt
    outputs, no gather) + a 9-point stencil sum (stencil.cu), instead of a gather-bound 3x3 implicit GEMM.
    y bf16 [M, Cin]; wb fp32 [16, Cin, 3, 3] (block-diagonal over the heads, zero rows as padding, `n_used` real rows);
    bias fp32 [16].  cpt = n_used rounded up to 4 channels per tap: the reference's heads have 11-13 outputs per task ->
    cpt = 12 (16 for 13) -> 108 (144) GEMM columns padded to NZ = 128 (192).  Returns fp32 [M, 16]."""

    @staticmethod
    def geometry(n_used):
        cpt = max(4, (int(n_used) + 3) // 4 * 4)
        return cpt, (128 if 9 * cpt <= 128 else 192)

    @staticmethod
    def forward(ctx, y, wb, bias, B, H, W, bn_src=None, n_used=16):
        from ._lib import check, lib, ptr, stream
        split = _split()
        ctx.bn_src = bn_src if not split else None
        M, cin = y.shape[0], y.shape[1] // (_P() if split else 1)
        assert wb.shape[0] == 16 and wb.shape[2] == 3
        cpt, NZ = HeadFinalConvFn.geometry(n_used)
        with torch.no_grad():
            wz = torch.zeros(1, NZ, cin, dtype=torch.float32, device=y.device)
            wz[0, :9 * cpt] = wb.permute(2, 3, 0, 1)[:, :, :cpt].reshape(9 * cpt, cin)            # row = tap*cpt + j
            wz = _to_hilo(wz) if split else wz.to(torch.bfloat16)
        Z = torch.empty(M, NZ, dtype=torch.float32, device=y.device)
        ops.igemm(y, M, wz, 1, cin, NZ, Z, block_n=NZ, segs=ops.split_segments() if split else None, a_lo_off=cin if split else 0)
        ctx.split = split
        out = torch.empty(M, 16, dtype=torch.float32, device=y.device)
        ops._count(1)
        check(lib().pnx_tap_gather_sum(ptr(Z), NZ, cpt, ptr(bias.detach().float().contiguous()), B, H, W, ptr(out), stream()))
        ctx.save_for_backward(y, wz)
        ctx.geo = (B, H, W, cin, cpt, NZ)
        return out

    @staticmethod
    def backward(ctx, dout):
        from ._lib import check, lib, ptr, stream
        y, wz = ctx.saved_tensors
        B, H, W, cin, cpt, NZ = ctx.geo
        M = y.shape[0]
        dout = dout.contiguous().float()
        dbias = dout.sum(0)

        def to_wb(g):       # [1, Cin, NZ] -> gradient of wb [16, Cin, 3, 3]
            d = g[0, :, :9 * cpt].reshape(cin, 3, 3, cpt).permute(3, 0, 1, 2)
            return torch.nn.functional.pad(d, (0, 0, 0, 0, 0, 0, 0, 16 - cpt)).contiguous()

        if ctx.split:
            P = _P()
            dZ = torch.empty(M, P * NZ, dtype=torch.bfloat16, device=dout.device)
            ops._count(1)
            check(lib().pnx_tap_scatter(ptr(dout), B, H, W, ptr(dZ), P * NZ, NZ, cpt, NZ, stream()))
            wzf = sum(wz[0, :, q * cin:(q + 1) * cin].float() for q in reversed(range(P)))  # [NZ, cin] (sum of the pieces)
            d32 = torch.empty(M, cin, dtype=torch.float32, device=dout.device)
            ops.igemm(dZ, M, _to_hilo(wzf.t().contiguous().unsqueeze(0)), 1, NZ, cin, d32, segs=ops.split_segments(), a_lo_off=NZ)
            dy = ops.rows_split(d32)
            g = torch.zeros(1, cin, NZ, dtype=torch.float32, device=dout.device)
            ops.wgrad_split(y, cin, cin, dZ, NZ, NZ, M, 1, g)
            return dy, to_wb(g), dbias, None, None, None, None, None
        dZ = torch.empty(M, NZ, dtype=torch.bfloat16, device=dout.device)
        ops._count(1)
        check(lib().pnx_tap_scatter(ptr(dout), B, H, W, ptr(dZ), NZ, NZ, cpt, 0, stream()))
        dy = torch.empty(M, cin, dtype=torch.bfloat16, device=dout.device)
        ops.igemm(dZ, M, wz.transpose(1, 2).contiguous(), 1, NZ, cin, dy,         # dy = dZ . Wz (+ the sibling BN's reduce pass)
                  bnr=_claim_bn_reduce(ctx.bn_src, M, cin, NZ))
        g = ops.zeros((1, cin, NZ), torch.float32, dout.device)
        ops.wgrad(y, cin, dZ, NZ, M, 1, g)                                        # [1, Cin, NZ] = y^T . dZ
        return dy, to_wb(g), dbias, None, None, None, None, None
