"""Every tensor-core GEMM launch of a production training step, replayed at its production shape against an exact reference.

One bf16 training step of the bench model (nusc: 6 frames, waymo180k: 3 frames) and one eval-mode forward (nusc) run with
ops.igemm, ops.conv3x3_win and ops.wgrad wrapped: each wrapper passes the call through and keeps its configuration (the
scalars, the shape / strides / dtype of every operand, which epilogue inputs are present, a clone of the neighbour table),
never an activation.  The unique configurations are then replayed on fresh operands holding small integers, bounded so
that every product and every fp32 partial sum is exact in any summation order: fp32 outputs and weight gradients must
equal the fp64 reference, bf16 outputs the fp64 reference rounded to bf16, bit for bit.  At these shapes a CTA walks
tens to hundreds of tiles, which the kernel tests' small shapes never make it do.  Everything else a launch writes is
checked too: guard columns and rows past M keep a sentinel, BatchNorm statistics (both accumulation modes) and the fused
BatchNorm-backward reduce match fp64 sums.  A configuration the replay cannot reproduce fails the test.  The split
mode's configurations (segments over bf16 pieces) are replayed through the same functions by
tests/test_production_split_gpu.py."""
import types

import pytest
import torch

from pillarnext_b200 import functional as Fn
from pillarnext_b200 import modules, ops, synth

pytestmark = pytest.mark.gpu

SENTINEL = 7.0          # exact in bf16 and fp32; never a value the integer operands produce at a guard position
GUARD_ROWS = 64         # rows past M in every output buffer
EXACT = 1 << 24         # fp32 sums of integers below this are exact whatever the order
CHUNK_BYTES = 1 << 28   # fp64 reference temporaries per row chunk


class Unreproducible(Exception):
    pass


# ------------------------------------------------------------------------------------------------- recording
def _desc(t):
    return None if t is None else (tuple(t.shape), tuple(t.stride()), t.dtype)


def _span(t, rows, cols):
    """(storage, first byte, row pitch in bytes, bytes per row, rows) of the elements [0, rows) x [0, cols) of a row-major view."""
    es = t.element_size()
    return (t.untyped_storage().data_ptr(), t.storage_offset() * es, t.stride(0) * es, cols * es, rows)


def _intersect(a, b):
    if a is None or b is None or a[0] != b[0]:
        return False
    (_, oa, lda, wa, ra), (_, ob, ldb, wb, rb) = a, b
    if lda == ldb and oa % lda + wa <= lda and ob % ldb + wb <= ldb:
        rows = max(oa // lda, ob // ldb) < min(oa // lda + ra, ob // ldb + rb)
        return rows and max(oa % lda, ob % ldb) < min(oa % lda + wa, ob % ldb + wb)
    return max(oa, ob) < min(oa + (ra - 1) * lda + wa, ob + (rb - 1) * ldb + wb)


def _any_intersect(spans):
    spans = [s for s in spans if s is not None]
    return any(_intersect(spans[i], spans[j]) for i in range(len(spans)) for j in range(i + 1, len(spans)))


class Recorder:
    """Wraps ops.igemm / ops.conv3x3_win / ops.wgrad; keeps one record per unique configuration."""

    def __init__(self):
        self.configs, self.keys, self.tables, self.nested = [], {}, {}, []
        self.source = ""

    def _table(self, nbr):
        if nbr is None:
            return None
        if id(nbr) not in self.tables:         # identity; the original is held until recording ends so ids stay unique
            self.tables[id(nbr)] = (nbr, len(self.tables), nbr.clone())
        return self.tables[id(nbr)][1]

    def _add(self, cfg):
        key = tuple(sorted((k, v) for k, v in cfg.items() if k not in ("tag", "source")))
        if key in self.keys:
            self.keys[key]["calls"] += 1
            return
        cfg["calls"], cfg["source"] = 1, self.source
        self.keys[key] = cfg
        self.configs.append(cfg)

    def _tag(self):
        tag = ops.PROFILE[-1][5] if ops.PROFILE else ""
        ops.PROFILE.clear()
        return tag

    def wrap(self, monkeypatch):
        igemm, win, wgrad = ops.igemm, ops.conv3x3_win, ops.wgrad
        rec = self

        def igemm_rec(A, M, w_packed, taps, cin, cout, out, *, lda=None, ldc=None, nbr=None, dense=None, bias=None, stats=None,
                      stats_mod=None, shuffle=False, relu=False, block_n=None, addend=None, segs=None, a_lo_off=0, bnr=None):
            res = igemm(A, M, w_packed, taps, cin, cout, out, lda=lda, ldc=ldc, nbr=nbr, dense=dense, bias=bias, stats=stats,
                        stats_mod=stats_mod, shuffle=shuffle, relu=relu, block_n=block_n, addend=addend, segs=segs,
                        a_lo_off=a_lo_off, bnr=bnr)
            rows = M * (4 if shuffle else 1)
            n_st = cout // 4 if shuffle else cout
            spans = [_span(A, A.shape[0], cin), _span(out, rows, n_st), _span(addend, M, cout) if addend is not None else None,
                     _span(bnr.raw, M, cout) if bnr is not None else None]
            rec._add(dict(kind="igemm", tag=rec._tag(), M=M, taps=taps, cin=cin, cout=cout, A=_desc(A), W=tuple(w_packed.shape),
                          out=_desc(out), lda=A.stride(0) if lda is None else lda, ldc=out.stride(-2) if ldc is None else ldc,
                          table=rec._table(nbr), dense=tuple(dense) if dense else None, bias=bias is not None,
                          stats=stats.numel() // 2 if stats is not None else 0, stats_mod=stats_mod, shuffle=bool(shuffle),
                          relu=bool(relu), bn=block_n or ops.pick_block_n(cout), addend=_desc(addend),
                          segs=tuple(segs) if segs else None, a_lo_off=a_lo_off, bnr=_desc(bnr.raw) if bnr is not None else None,
                          overlap=_any_intersect(spans)))
            return res

        def win_rec(A, B, H, W, w_packed, cin, cout, out, *, bias=None, stats=None, relu=False, block_n=None, base_off=None, bnr=None):
            res = win(A, B, H, W, w_packed, cin, cout, out, bias=bias, stats=stats, relu=relu, block_n=block_n, base_off=base_off,
                      bnr=bnr)
            tag = rec._tag()
            M = B * H * W
            spans = [_span(A, A.shape[0], cin), _span(out, M, cout), _span(bnr.raw, M, cout) if bnr is not None else None]
            rec._add(dict(kind="win", tag=tag, B=B, H=H, W=W, M=M, cin=cin, cout=cout, A=_desc(A), W_=tuple(w_packed.shape),
                          out=_desc(out), bias=bias is not None, stats=stats.numel() // 2 if stats is not None else 0, relu=bool(relu),
                          bn=int(tag.rsplit("_bn", 1)[1]), block_n=block_n, base_off=base_off,
                          bnr=_desc(bnr.raw) if bnr is not None else None, overlap=_any_intersect(spans)))
            return res

        def wgrad_rec(X, x_channels, Y, y_channels, M, taps, dW, *, nbr=None, dense=None, shuffle=False, gathered=None):
            rec.nested.append(False)
            try:
                res = wgrad(X, x_channels, Y, y_channels, M, taps, dW, nbr=nbr, dense=dense, shuffle=shuffle, gathered=gathered)
            finally:
                split = rec.nested.pop()
            if rec.nested:
                rec.nested[-1] = True
            if split:          # split into column slices of X: those calls reached the library and were recorded
                return res
            g = (nbr is not None or dense is not None or shuffle) if gathered is None else bool(gathered)
            spans = [_span(X, M, x_channels), _span(Y, Y.shape[0], y_channels), _span(dW.view(-1, y_channels), taps * x_channels, y_channels)]
            rec._add(dict(kind="wgrad", tag=rec._tag(), M=M, taps=taps, cx=x_channels, cy=y_channels, X=_desc(X), Y=_desc(Y),
                          dW=_desc(dW), table=rec._table(nbr), dense=tuple(dense) if dense else None, shuffle=bool(shuffle),
                          gathered=g, overlap=_any_intersect(spans)))
            return res

        monkeypatch.setattr(ops, "igemm", igemm_rec)
        monkeypatch.setattr(ops, "conv3x3_win", win_rec)
        monkeypatch.setattr(ops, "wgrad", wgrad_rec)


def _to_dev(ex, dev):
    return {k: ([e.to(dev) for e in v] if isinstance(v, list) and v and torch.is_tensor(v[0]) else
                (v.to(dev) if torch.is_tensor(v) else v)) for k, v in ex.items()}


def _record(rec, name, evaluate):
    dev = torch.device("cuda", torch.cuda.current_device())
    sel = synth.BENCH_CONFIGS[name]
    cfg = sel["cfg"]
    frames = cfg["frames_per_gpu"]
    torch.manual_seed(0)
    model = modules.build_pillarnext_b(cfg).to(dev).train()
    ex = _to_dev(synth.make_batch(list(range(frames)), sel["points"], cfg, kind="lidar", n_boxes=40, sweeps=sel["sweeps"],
                                  rings=sel["rings"]), dev)
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
    rec = Recorder()
    prev = ops.PROFILE, Fn.set_precision("bf16"), ops.set_deterministic(False)      # the production step
    with pytest.MonkeyPatch.context() as mp:
        rec.wrap(mp)
        ops.PROFILE = []
        try:
            _record(rec, "nusc", evaluate=True)
            _record(rec, "waymo180k", evaluate=False)
        finally:
            ops.PROFILE = prev[0]
            Fn.set_precision(prev[1])
            ops.set_deterministic(prev[2])
    rec.table_list = {i: c for _, i, c in rec.tables.values()}
    rec.tables = None                          # release the step's own tables; the replay reads the clones
    torch.cuda.empty_cache()
    return rec


# ------------------------------------------------------------------------------------------------- operands
def _ints(shape, amp, dtype, gen):
    return torch.randint(-amp, amp + 1, shape, generator=gen, device="cuda").to(dtype)


def _rows_buffer(desc, used_cols, amp, gen):
    """A fresh [rows, >= cols] view with the recorded shape and row stride: integers in the used columns, NaN in the rest of
    each row (a read outside the operand's columns shows in the result)."""
    shape, stride, dtype = desc
    if len(shape) != 2 or stride[1] != 1 or stride[0] < shape[1] or used_cols > shape[1]:
        raise Unreproducible("operand layout %s" % (desc,))
    buf = torch.full((shape[0], stride[0]), float("nan"), dtype=dtype, device="cuda")
    buf[:, :used_cols] = _ints((shape[0], used_cols), amp, dtype, gen)
    return buf[:, :shape[1]]


def _slot_out(desc, rows, cols, ldc):
    """The output view with the recorded shape inside a sentinel-filled [rows + GUARD_ROWS, ldc] buffer, centred in the
    row (16-byte aligned) when ldc leaves room; returns (buffer, view, column offset)."""
    shape, stride, dtype = desc
    if len(shape) != 2 or stride != (ldc, 1) or shape[0] < rows or shape[1] < cols or ldc < shape[1]:
        raise Unreproducible("output layout %s for %d x %d, ldc %d" % (desc, rows, cols, ldc))
    buf = torch.full((shape[0] + GUARD_ROWS, ldc), SENTINEL, dtype=dtype, device="cuda")
    off = (ldc - shape[1]) // 2 // 8 * 8
    return buf, buf[:shape[0], off:off + shape[1]], off


def _bnr_operands(desc, C, gen):
    shape, stride, dtype = desc
    if dtype != torch.bfloat16 or len(shape) != 2 or stride[1] != 1 or shape[1] != C:
        raise Unreproducible("bnr raw layout %s" % (desc,))
    raw = torch.full((shape[0], stride[0]), float("nan"), dtype=dtype, device="cuda")
    raw[:, :C] = torch.randn(shape[0], C, generator=gen, device="cuda").bfloat16()
    return types.SimpleNamespace(raw=raw[:, :C], scale=torch.rand(C, generator=gen, device="cuda") + 0.5,
                                 shift=torch.randn(C, generator=gen, device="cuda") * 0.5,
                                 mean=torch.randn(C, generator=gen, device="cuda") * 0.1,
                                 invstd=torch.rand(C, generator=gen, device="cuda") + 0.5, C=C,
                                 red=torch.zeros(2 * C, dtype=torch.float64, device="cuda"))


# ------------------------------------------------------------------------------------------------- gathers
def _gather_index(m0, m1, t, table, dense, dev):
    """Row of the gathered operand read for output rows [m0, m1) at tap t (-1: absent), as the kernels compute it."""
    if table is not None:
        return table[m0:m1, t].long()
    m = torch.arange(m0, m1, device=dev)
    if dense is None:
        assert t == 0
        return m
    Ho, Wo, Hi, Wi, kw, mul, dil, pad = dense
    b, rem = m // (Ho * Wo), m % (Ho * Wo)
    y, x = rem // Wo, rem % Wo
    yi = y * mul + (t // kw) * dil - pad
    xi = x * mul + (t % kw) * dil - pad
    ok = (yi >= 0) & (yi < Hi) & (xi >= 0) & (xi < Wi)
    return torch.where(ok, (b * Hi + yi) * Wi + xi, torch.full_like(m, -1))


def _shuffle_index(m0, m1, t, dense, dev):
    """ConvTranspose2d k2s2: tap q of input pixel (b, y, x) is output pixel (2y + q / 2, 2x + q % 2)."""
    H, W = dense[0], dense[1]
    m = torch.arange(m0, m1, device=dev)
    b, rem = m // (H * W), m % (H * W)
    y, x = rem // W, rem % W
    return (b * 2 * H + 2 * y + t // 2) * (2 * W) + 2 * x + t % 2


def _gather(src, idx, cols):
    rows = src[idx.clamp(min=0), :cols].double()
    return torch.where((idx >= 0).unsqueeze(1), rows, torch.zeros((), dtype=torch.float64, device=src.device))


def _chunk_rows(width):
    return max(1024, CHUNK_BYTES // (8 * max(width, 1)))


# ------------------------------------------------------------------------------------------------- igemm / window: run + reference
def _gemm_view(c):
    """The fields the igemm reference needs, for an igemm or a window-kernel configuration."""
    if c["kind"] == "win":
        return dict(M=c["M"], taps=9, cin=c["cin"], cout=c["cout"], dense=(c["H"], c["W"], c["H"], c["W"], 3, 1, 1, 1),
                    table=None, shuffle=False, stats_mod=None, addend=None, ldc=c["out"][1][0])
    return dict(M=c["M"], taps=c["taps"], cin=c["cin"], cout=c["cout"], dense=c["dense"], table=c["table"], shuffle=c["shuffle"],
                stats_mod=c["stats_mod"], addend=c["addend"], ldc=c["ldc"])


def _amplitudes(c):
    """(A, W, bias, addend) integer amplitudes; the largest possible |partial sum| must stay below 2^24.  A split-mode
    GEMM accumulates its nseg segments into one accumulator: K counts every segment."""
    k = (c["taps"] * c["cin"] if c["kind"] == "igemm" else 9 * c["cin"]) * len(c.get("segs") or (None,))
    for a, w in ((3, 2), (2, 2), (1, 2), (1, 1)):
        bound = k * a * w + 4 + 8
        if bound < EXACT:
            return (a, w, 4, 8), bound
    raise Unreproducible("K = %d: no integer range keeps the sums exact" % k)


def seg_pieces(c):
    """(A pieces, W pieces) a configuration reads: 1, 1 for a plain GEMM, 3, 3 for a 3-piece split-mode one."""
    segs = c.get("segs") or ((0, 0),)
    return max(a for a, _ in segs) + 1, max(w for _, w in segs) + 1


def pieces_buffer(desc, cols, lo, pieces, amp, gen):
    """_rows_buffer for split rows: its own integers in the columns [q lo, q lo + cols) of every piece q, NaN between
    the pieces and past the last (a piece offset that is off reads NaN or another piece's integers).  One NaN row past
    the view, so a reference taken at a shifted piece offset stays inside the storage."""
    shape, stride, dt = desc
    if len(shape) != 2 or stride[1] != 1 or stride[0] < shape[1] or lo < cols or (pieces - 1) * lo + cols > shape[1]:
        raise Unreproducible("split operand layout %s for %d pieces of %d columns at %d" % (desc, pieces, cols, lo))
    buf = torch.full((shape[0] + 1, stride[0]), float("nan"), dtype=dt, device="cuda")
    for q in range(pieces):
        buf[:shape[0], q * lo:q * lo + cols] = _ints((shape[0], cols), amp, buf.dtype, gen)
    return buf[:shape[0], :shape[1]]


def piece(t, off, cols):
    """Columns [off, off + cols) of every row of the row-major view t, read through its storage (off may pass the view)."""
    return t.as_strided((t.shape[0], cols), (t.stride(0), 1), t.storage_offset() + off)


def _gemm_operands(c, gen, tables):
    if c["kind"] == "igemm" and c["a_lo_off"] and not c["segs"]:
        raise Unreproducible("a piece offset without segments")
    if c["overlap"]:
        raise Unreproducible("operands share elements")
    g = _gemm_view(c)
    (aa, aw, ab, ad), bound = _amplitudes(c)
    assert bound < EXACT
    o = types.SimpleNamespace(bound=bound)
    a_pieces, w_pieces = seg_pieces(c)
    # split mode: no valid split (its low pieces would be zero, and a wrong piece offset would go unnoticed); every
    # piece of A and of W holds its own integers
    o.A = _rows_buffer(c["A"], g["cin"], aa, gen) if a_pieces == 1 else \
        pieces_buffer(c["A"], g["cin"], c["a_lo_off"], a_pieces, aa, gen)
    wshape = c["W"] if c["kind"] == "igemm" else c["W_"]
    if tuple(wshape) != (g["taps"], g["cout"], w_pieces * g["cin"]):
        raise Unreproducible("packed weight shape %s" % (wshape,))
    o.W = _ints(wshape, aw, torch.bfloat16, gen)
    o.bias = _ints((g["cout"],), ab, torch.float32, gen) if c["bias"] else None
    o.addend = _rows_buffer(g["addend"], g["cout"], ad, gen) if g["addend"] is not None else None
    if o.addend is not None and o.addend.shape[0] < g["M"]:
        raise Unreproducible("addend rows")
    o.table = tables[g["table"]] if g["table"] is not None else None
    o.rows = g["M"] * (4 if g["shuffle"] else 1)
    o.n_st = g["cout"] // 4 if g["shuffle"] else g["cout"]
    if g["shuffle"] and (g["cout"] % 256 or g["addend"] is not None):
        raise Unreproducible("pixel-shuffle store of %d columns" % g["cout"])
    o.buf, o.out, o.off = _slot_out(c["out"], o.rows, o.n_st, g["ldc"])
    o.out_dtype = o.out.dtype
    o.bnr = _bnr_operands(c["bnr"], g["cout"], gen) if c["bnr"] is not None else None
    return o


def _launch_gemm(c, o):
    """One launch on the operands; returns (output copy, stats, bnr red)."""
    o.buf[:] = SENTINEL
    stats = torch.zeros(2 * c["stats"], dtype=torch.float64, device="cuda") if c["stats"] else None
    if o.bnr is not None:
        o.bnr.red.zero_()
    if c["kind"] == "igemm":
        ops.igemm(o.A, c["M"], o.W, c["taps"], c["cin"], c["cout"], o.out, lda=c["lda"], ldc=c["ldc"], nbr=o.table, dense=c["dense"],
                  bias=o.bias, stats=stats, stats_mod=c["stats_mod"], shuffle=c["shuffle"], relu=c["relu"], block_n=c["bn"],
                  addend=o.addend, segs=c["segs"], a_lo_off=c["a_lo_off"], bnr=o.bnr)
    else:
        ops.conv3x3_win(o.A, c["B"], c["H"], c["W"], o.W, c["cin"], c["cout"], o.out, bias=o.bias, stats=stats, relu=c["relu"],
                        block_n=c["bn"], base_off=c["base_off"], bnr=o.bnr)
    return stats, (o.bnr.red.clone() if o.bnr is not None else None)


def _gemm_reference(c, o, drop=None, bias_delta=None, skip_tile=None, segs=None, a_lo_off=None):
    """fp64 reference of the stored output (in the output dtype), the stats sums and the bnr sums.  A split-mode
    configuration sums, over its segments (A piece ap, W piece wp), gathered piece ap of A times piece wp of W.  The
    mutations exist to show that the comparison notices them: drop = (row, tap) whose gather is left out, bias_delta =
    (column, delta), skip_tile = a 128-row tile left out of the statistics, segs / a_lo_off in place of the recorded ones."""
    g = _gemm_view(c)
    M, taps, cin, cout = g["M"], g["taps"], g["cin"], g["cout"]
    dev = o.A.device
    segs = c.get("segs") if segs is None else segs
    lo = c.get("a_lo_off", 0) if a_lo_off is None else a_lo_off
    Wd = o.W.double()
    if segs:               # the W pieces each A piece meets, summed (exact: small integers)
        groups = {}
        for ap, wp in segs:
            groups[ap] = groups.get(ap, 0) + Wd[:, :, wp * cin:(wp + 1) * cin]
        terms = [(piece(o.A, ap * lo, cin), w) for ap, w in sorted(groups.items())]
    else:
        terms = [(o.A, Wd)]
    bias = o.bias.double() if o.bias is not None else None
    if bias is not None and bias_delta is not None:
        bias = bias.clone()
        bias[bias_delta[0]] += bias_delta[1]
    exp = torch.empty(o.rows, o.n_st, dtype=o.out_dtype, device=dev)
    ns = c["stats"]
    mod = g["stats_mod"] or (ns if ns else 1)
    ssum = torch.zeros(2, ns, dtype=torch.float64, device=dev) if ns else None
    smag = torch.zeros(ns, dtype=torch.float64, device=dev) if ns else None
    chan = torch.arange(cout, device=dev) % mod if ns else None
    red = torch.zeros(4, cout, dtype=torch.float64, device=dev) if o.bnr is not None else None
    step = _chunk_rows(max(cin, cout)) // 128 * 128
    for m0 in range(0, M, step):
        m1 = min(M, m0 + step)
        v = torch.zeros(m1 - m0, cout, dtype=torch.float64, device=dev)
        for t in range(taps):
            idx = _gather_index(m0, m1, t, o.table, g["dense"], dev)
            if drop is not None and m0 <= drop[0] < m1 and t == drop[1]:
                idx = idx.clone()
                idx[drop[0] - m0] = -1
            for src, w in terms:
                v += _gather(src, idx, cin) @ w[t].t()
        if bias is not None:
            v += bias
        if o.addend is not None:
            v += o.addend[m0:m1, :cout].double()
        if c["relu"]:
            v.clamp_(min=0)
        q = v.to(o.out_dtype)
        if o.bnr is not None:
            raw = o.bnr.raw[m0:m1].double()
            gate = raw * o.bnr.scale.double() + o.bnr.shift.double() > 0
            q = torch.where(gate, q, torch.zeros_like(q))
            gd = q.double()
            xhat = (raw - o.bnr.mean.double()) * o.bnr.invstd.double()
            red += torch.stack([gd.sum(0), (gd * xhat).sum(0), gd.abs().sum(0), (gd * xhat).abs().sum(0)])
        if g["shuffle"]:
            for qd in range(4):
                exp[_shuffle_index(m0, m1, qd, g["dense"], dev)] = q[:, qd * 64:(qd + 1) * 64]
        else:
            exp[m0:m1] = q
        if ns:
            qd = q.double()
            if skip_tile is not None and m0 <= skip_tile * 128 < m1:
                qd = qd.clone()
                qd[skip_tile * 128 - m0:skip_tile * 128 - m0 + 128] = 0
            ssum[0].index_add_(0, chan, qd.sum(0))
            ssum[1].index_add_(0, chan, (qd * qd).sum(0))
            smag.index_add_(0, chan, qd.abs().sum(0))
    return types.SimpleNamespace(out=exp, stats=ssum, stats_mag=smag, red=red)


def _compare_gemm(c, o, stats, red, ref):
    """Failures (strings) of one launch against the reference; empty when it matches."""
    bad = []
    got = o.out[:o.rows, :o.n_st]
    if not torch.equal(got, ref.out):
        diff = got.double() != ref.out.double()
        rows = diff.any(1).nonzero()
        bad.append("%d outputs differ (first row %d)" % (int(diff.sum()), int(rows[0]) if rows.numel() else -1))
    if not (o.buf[o.out.shape[0]:] == SENTINEL).all() or not (o.buf[:, :o.off] == SENTINEL).all() or \
            not (o.buf[:, o.off + o.out.shape[1]:] == SENTINEL).all() or not (o.out[o.rows:] == SENTINEL).all() or \
            not (o.out[:, o.n_st:] == SENTINEL).all():
        bad.append("sentinel overwritten outside the output")
    if stats is not None:
        ns = c["stats"]
        for i, (mag, name) in enumerate(((ref.stats_mag, "sums"), (ref.stats[1], "sums of squares"))):
            err = (stats[i * ns:(i + 1) * ns] - ref.stats[i]).abs()
            if (err > 1e-5 * mag + 1e-6).any():
                bad.append("stats %s differ by up to %.3g (|v| sum %.3g)" % (name, err.max().item(), mag.max().item()))
    if red is not None:
        C = c["cout"]
        for i, name in ((0, "sum g"), (1, "sum g*xhat")):
            err = (red[i * C:(i + 1) * C] - ref.red[i]).abs().max().item()
            if err > 1e-5 * ref.red[2 + i].max().item() + 1e-6:
                bad.append("bnr %s differs by %.3g" % (name, err))
    return bad


# ------------------------------------------------------------------------------------------------- wgrad: run + reference
def _wgrad_operands(c, gen, tables):
    if c["overlap"]:
        raise Unreproducible("operands share elements")
    M, T, cx, cy = c["M"], c["taps"], c["cx"], c["cy"]
    for ax, ay in ((3, 2), (2, 2), (2, 1), (1, 1)):
        bound = M * ax * ay + 4
        if bound < EXACT:
            break
    else:
        raise Unreproducible("M = %d: no integer range keeps the sums exact" % M)
    if c["dW"][0] != (T, cx, cy) or c["dW"][2] != torch.float32:
        raise Unreproducible("dW layout %s" % (c["dW"],))
    o = types.SimpleNamespace(bound=bound)
    o.X = _rows_buffer(c["X"], cx, ax, gen)
    o.Y = _rows_buffer(c["Y"], cy, ay, gen)
    if o.X.shape[0] < M:
        raise Unreproducible("X rows")
    o.dW0 = _ints((T, cx, cy), 4, torch.float32, gen)        # the launch accumulates into dW
    o.table = tables[c["table"]] if c["table"] is not None else None
    return o


def _launch_wgrad(c, o):
    dW = o.dW0.clone()
    ops.wgrad(o.X, c["cx"], o.Y, c["cy"], c["M"], c["taps"], dW, nbr=o.table, dense=c["dense"], shuffle=c["shuffle"],
              gathered=c["gathered"])
    return dW


def _wgrad_reference(c, o, drop=None):
    M, T, cx, cy = c["M"], c["taps"], c["cx"], c["cy"]
    dev = o.X.device
    ref = o.dW0.double()
    step = _chunk_rows(cx + cy)
    for m0 in range(0, M, step):
        m1 = min(M, m0 + step)
        Xc = o.X[m0:m1, :cx].double()
        for t in range(T):
            if not c["gathered"]:
                idx = torch.arange(m0, m1, device=dev)
            elif c["shuffle"]:
                idx = _shuffle_index(m0, m1, t, c["dense"], dev)
            else:
                idx = _gather_index(m0, m1, t, o.table, c["dense"], dev)
            if drop is not None and m0 <= drop[0] < m1 and t == drop[1]:
                idx = idx.clone()
                idx[drop[0] - m0] = -1
            ref[t] += Xc.t() @ _gather(o.Y, idx, cy)
    return ref.float()


# ------------------------------------------------------------------------------------------------- the replay
def _grid(c):
    sms = ops.sm_count()
    if c["kind"] == "wgrad":
        s = ops.lib().pnx_wgrad_splits(c["cx"], c["cy"], c["taps"], c["M"], sms)
        return "%d splits x %d rows" % (s, -(-c["M"] // s)), None
    tiles = -(-c["M"] // 128) if c["kind"] == "igemm" else c["B"] * c["H"] * -(-c["W"] // 128)
    n_blocks = c["cout"] // c["bn"]
    gx = max(1, min(sms // n_blocks, tiles))
    return "%d tiles on %d x %d CTAs, %d per CTA" % (tiles, gx, n_blocks, -(-tiles // gx)), -(-tiles // gx)


def _replay(c, tables, gen):
    """Failures of one configuration (empty: every launch matched)."""
    if c["kind"] == "wgrad":
        o = _wgrad_operands(c, gen, tables)
        ref = _wgrad_reference(c, o)
        bad = []
        for det in (False, True):
            prev = ops.set_deterministic(det)
            try:
                dW = _launch_wgrad(c, o)
            finally:
                ops.set_deterministic(prev)
            if not torch.equal(dW, ref):
                bad.append("dW differs in %d entries (deterministic=%s)" % (int((dW != ref).sum()), det))
        return bad, o, ref
    o = _gemm_operands(c, gen, tables)
    ref = _gemm_reference(c, o)
    bad = []
    for det in ((False, True) if c["stats"] else (False,)):
        prev = ops.set_deterministic(det)
        try:
            stats, red = _launch_gemm(c, o)
        finally:
            ops.set_deterministic(prev)
        bad += ["%s (deterministic=%s)" % (b, det) for b in _compare_gemm(c, o, stats, red, ref)]
    return bad, o, ref


def _label(c):
    if c["kind"] == "wgrad":
        extra = ("table" if c["table"] is not None else "shuffle" if c["shuffle"] else
                 "dense s%d d%d" % c["dense"][5:7] if c["dense"] else "gathered" if c["gathered"] else "direct")
        return "wgrad %-22s %s ldx %d ldy %d" % (c["tag"], extra, c["X"][1][0], c["Y"][1][0])
    epi = [k for k in ("bias", "relu", "shuffle") if c.get(k)] + (["stats"] if c["stats"] else []) + \
        (["addend"] if c.get("addend") else []) + (["bnr"] if c["bnr"] else [])
    ld = "lda %d ldc %d" % (c["A"][1][0], c["out"][1][0])
    if c["kind"] == "igemm":
        gather = "table" if c["table"] is not None else ("dense s%d d%d" % c["dense"][5:7] if c["dense"] else "rows")
        return "igemm %-30s %s %s %s %s" % (c["tag"], gather, "fp32" if c["out"][2] == torch.float32 else "bf16", ld, "+".join(epi))
    return "win   %-30s %s %s" % (c["tag"], ld, "+".join(epi))


def test_production_gemms_match_exact_reference(launches):
    """Every unique igemm / window / wgrad configuration of the nusc and waymo180k steps (and the nusc eval forward)
    reproduces its exact integer reference."""
    kinds = {k: [c for c in launches.configs if c["kind"] == k] for k in ("igemm", "win", "wgrad")}
    assert all(kinds.values()), {k: len(v) for k, v in kinds.items()}
    for src in ("nusc train", "nusc eval", "waymo180k train"):
        assert any(c["source"] == src for c in launches.configs), src
    gen = torch.Generator(device="cuda").manual_seed(1234)
    failures, most = [], 0
    print()
    for i, c in enumerate(launches.configs):
        grid, per_cta = _grid(c)
        most = max(most, per_cta or 0)
        try:
            bad, o, ref = _replay(c, launches.table_list, gen)
            del o, ref
        except Unreproducible as e:
            bad = ["cannot be replayed: %s" % e]
        print("[%3d] %-16s %-100s %-40s x%-3d %s" % (i, c["source"], _label(c), grid, c["calls"], "ok" if not bad else "; ".join(bad)))
        if bad:
            failures.append("%s %s: %s" % (c["source"], _label(c), "; ".join(bad)))
        torch.cuda.empty_cache()
    print("peak GPU memory: %.2f GB" % (torch.cuda.max_memory_allocated() / 2 ** 30))
    assert not failures, "\n".join(failures)
    if ops.sm_count() >= 132:
        assert most >= 40, "the largest launch gives only %d tiles per CTA" % most


def _pick(configs, kind, want):
    cands = [c for c in configs if c["kind"] == kind and all(c.get(k) for k in want) and not c.get("overlap")]
    assert cands, "no %s configuration with %s" % (kind, want)
    return max(cands, key=lambda c: c["M"] * (c.get("taps", 9)))


def _gemm_tiles(c):
    return -(-c["M"] // 128) if c["kind"] == "igemm" else c["B"] * c["H"] * -(-c["W"] // 128)


def _late_row(c, o):
    """An output row in the third tile of the second CTA, and a tap whose gather reads a real row there."""
    per_cta = _grid(c)[1]
    assert per_cta >= 3, "%s: the self-check needs CTAs with three tiles or more" % c["tag"]
    gx = -(-_gemm_tiles(c) // per_cta)
    tile = 2 * gx + 1
    if c["kind"] == "igemm":
        first = tile * 128
    else:                                   # window tiles: (frame, image row) outer, 128-pixel chunk of the row inner
        xc = -(-c["W"] // 128)
        first = (tile // xc) * c["W"] + (tile % xc) * 128
    g = _gemm_view(c)
    for row in range(first + 37, first + 128):
        taps = [t for t in range(g["taps"]) if int(_gather_index(row, row + 1, t, o.table, g["dense"], o.A.device)[0]) >= 0]
        if taps:
            return row, taps[len(taps) // 2]
    raise AssertionError("%s: tile %d gathers nothing" % (c["tag"], tile))


@pytest.mark.parametrize("kind", ["igemm", "win"])
def test_self_check_gemm_comparison_catches_small_errors(launches, kind):
    """On the largest configurations of the kind, the comparison fails when the reference (a) leaves out one (row, tap)
    gather in a tile that is not its CTA's first, (b) leaves one 128-row tile out of the statistics, (c) has one bias
    entry off by 1."""
    gen = torch.Generator(device="cuda").manual_seed(99)
    runs = {}
    for name, want in (("gather", ()), ("stats", ("stats",)), ("bias", ("bias",))):
        c = _pick(launches.configs, kind, want)
        if id(c) not in runs:
            bad, o, _ = _replay(c, launches.table_list, gen)
            assert not bad, bad
            runs[id(c)] = (o, _launch_gemm(c, o))
        o, (stats, red) = runs[id(c)]
        if name == "gather":
            row, tap = _late_row(c, o)
            kw, what = dict(drop=(row, tap)), "the gather of (row %d, tap %d)" % (row, tap)
        elif name == "stats":
            tile = -(-c["M"] // 128) // 2
            kw, what = dict(skip_tile=tile), "rows %d..%d of the statistics" % (tile * 128, tile * 128 + 127)
        else:
            kw, what = dict(bias_delta=(5, 1.0)), "bias[5] + 1"
        found = _compare_gemm(c, o, stats, red, _gemm_reference(c, o, **kw))
        print("%s %s without %s: %s" % (kind, c["tag"], what, found))
        assert found, "%s: the comparison does not notice a reference without %s" % (c["tag"], what)


def test_self_check_wgrad_comparison_catches_small_errors(launches):
    """On the largest gathered wgrad configuration, the comparison fails when the reference leaves out one (row, tap)
    gather in the middle of the last K split."""
    gen = torch.Generator(device="cuda").manual_seed(98)
    c = _pick(launches.configs, "wgrad", ("gathered",))
    bad, o, ref = _replay(c, launches.table_list, gen)
    assert not bad, bad
    dW = _launch_wgrad(c, o)
    assert torch.equal(dW, ref)
    splits = ops.lib().pnx_wgrad_splits(c["cx"], c["cy"], c["taps"], c["M"], ops.sm_count())
    assert splits >= 2
    for row in range(c["M"] - c["M"] // splits // 2, c["M"]):
        taps = [t for t in range(c["taps"]) if int((_shuffle_index(row, row + 1, t, c["dense"], o.X.device) if c["shuffle"] else
                                                     _gather_index(row, row + 1, t, o.table, c["dense"], o.X.device))[0]) >= 0]
        if taps:
            break
    assert taps
    print("wgrad %s without the gather of (row %d, tap %d)" % (c["tag"], row, taps[0]))
    assert not torch.equal(dW, _wgrad_reference(c, o, drop=(row, taps[0]))), "wgrad %s: a dropped gather goes unnoticed" % c["tag"]
