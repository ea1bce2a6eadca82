"""Every launch of the fp32-grade split mode (`functional.set_precision("split")`, three bf16 pieces per value) at its
production configuration, against exact and float64 references.

The split mode is what the parity checks measure (1e-3 of the fp32 oracle, the mAP / NDS / Waymo gates, SyncBatchNorm),
and at production shapes it runs code the bf16 step never reaches: every dense 3x3 convolution through igemm's dense
gather, K loops nseg = 6 times longer with the A and W pieces addressed through the segment code and a_lo_off, fp32
addends, weight gradients as six launches into one dW, the two-stage BatchNorm-backward reduce, the fan-out's
accumulating merge and the head stencil's piece-writing scatter.  A piece-addressing or accumulation error there would
move the one-frame forward check by less than its tolerance.

One training step of the `nusc` (6 frames) and `waymo180k` (3 frames) bench models and one `nusc` eval forward run in
split mode with ops.igemm / ops.wgrad wrapped by the GEMM sibling's Recorder (tests/test_production_gemms_gpu.py), with
ops.wgrad_split wrapped as a unit (one group of segment launches into one dW = one configuration), and with the library
handle replaced by the row-wise sibling's proxy (tests/test_production_rowwise_gpu.py) extended by SPLIT_MAPS.  The same
steps run once more in bf16 through a proxy that keeps the scalar arguments of every call, so that entry points shared
with the bf16 step can be told apart by configuration.  Then:

- igemm with segments, bit for bit: every piece of A and of the packed W holds its own small integers (not a valid
  split, whose low pieces would be zero), bounded so that nseg K a w + bias + addend < 2^24; every output must equal the
  fp64 sum over the recorded segments, guard rows / columns keep their sentinel, statistics match in both accumulation
  modes.  The single wgrad launches of the groups are replayed by the sibling as well.
- wgrad_split groups, bit for bit: split buffers of the recorded ld with distinct integers in every piece, dW zeroed
  once, the recorded launches in order, against the fp64 sum over segments of X_xp^T gather(Y_yp).
- the row-wise split kernels at the recorded M, C, ld and lo, again with ld widened and lo > C (NaN between the pieces),
  with NaN guard rows, at 3 pieces and at 2: rows_split bit for bit against a bit-level round-to-nearest-even split, edge
  values included; rows_merge, add_relu_split, relu_bwd_split and tap_scatter (lo_off > 0) bit for bit against fp32
  emulations in the kernels' order; bn_apply_split within one fp32 ulp (two with the residual) of fp64, its pieces the
  exact split of the merged value; bn_bwd_reduce_split bit for bit on small integers and within (L+1) u sum|.| on
  Gaussian data, bit-identical across launches, with both ReLU gate sources; bn_bwd_apply_split's dx within the
  first-order bound of its fp32 evaluation, dres bit for bit.
- shared entry points that the split step calls with a configuration the bf16 step never produces are replayed through
  the siblings' functions; every other entry point is replayed here, by a sibling for configurations the bf16 step has
  too, or launches nothing.
- self-checks: a dropped or swapped segment, a_lo_off off by 64, a group whose last launch overwrites dW, one missing
  partial block of the reduce and a NaN in any output each fail their comparison."""
import contextlib
import os
import sys
import time
import types

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_production_gemms_gpu as G  # noqa: E402
import test_production_rowwise_gpu as R  # noqa: E402
from pillarnext_b200 import _lib, ops  # noqa: E402
from pillarnext_b200 import functional as Fn  # noqa: E402

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
PIECE_COUNTS = (3, 2)            # functional.PIECES, and the library's own default (split.cu g_pieces)

# Argument names and ctypes kinds of the split entry points, in the order of include/pnx.h
# (tests/test_split_recorder_cpu.py checks them against _lib._SIGS and the header).
SPLIT_MAPS = {
    "pnx_rows_split": "x:P ldx:L M:L C:I y:P ldy:L lo_y:L stream:P",
    "pnx_rows_merge": "x:P ldx:L lo_x:L M:L C:I y:P ldy:L accumulate:I stream:P",
    "pnx_bn_apply_split": "x:P ldx:L M:L C:I scale:P shift:P res:P ldr:L lo_r:L relu:I y:P ldy:L lo_y:L stream:P",
    "pnx_bn_bwd_reduce_split": "dy:P lddy:L lo_dy:L y:P ldy:L lo_y:L x:P ldx:L M:L C:I mean:P invstd:P relu:I fscale:P "
                               "fshift:P part:P red:P stream:P",
    "pnx_bn_bwd_apply_split": "dy:P lddy:L lo_dy:L y:P ldy:L lo_y:L x:P ldx:L M:L C:I mean:P invstd:P gamma:P red:P "
                              "count:D relu:I fscale:P fshift:P dx:P lddx:L lo_dx:L dres:P lddres:L lo_dres:L stream:P",
    "pnx_add_relu_split": "a:P lda:L lo_a:L b:P ldb:L lo_b:L M:L C:I y:P ldy:L lo_y:L stream:P",
    "pnx_relu_bwd_split": "dy:P lddy:L y:P ldy:L lo_y:L M:L C:I g:P ldg:L lo_g:L stream:P",
}
ROW_MAPS = {**R.ARG_MAPS, **SPLIT_MAPS}
PIECE_FNS = set(SPLIT_MAPS) | {"pnx_tap_scatter"}    # entry points whose layout depends on the piece count

REPLAYED_HERE = set(SPLIT_MAPS) | {"pnx_igemm", "pnx_wgrad", "pnx_tap_scatter", "pnx_scatter_dense"}
LAUNCH_NOTHING = {
    **{k: v for k, v in R.EXCLUDED.items() if "launches nothing" in v or k == "pnx_last_error"},
    "pnx_split_set_pieces": "mode switch of the split path; launches nothing",
    "pnx_bn_bwd_reduce_split_scratch": "host-side size query of the reduce's scratch; launches nothing",
}
SHARED_ROW = {    # entry points of the row-wise sibling the split step shares with the bf16 step, and their replays
    "pnx_bn_finalize": lambda c: _both(R._replay_finalize(c, R._bn_data(R._finalize_population(c), c["channels"]), False),
                                       R._replay_finalize(c, R._bn_data(R._finalize_population(c), c["channels"]), True)),
    "pnx_bn_eval_affine": R._replay_eval_affine,
    "pnx_tap_gather_sum": R._replay_stencil,
    "pnx_center_loss_task": lambda c: R._replay_loss(c)[:2],
    "pnx_center_loss_finalize": R._replay_loss_finalize,
}


def _both(a, b):
    return a[0] + b[0], a[1] + "; " + b[1]


def L():
    return _lib.lib()


def _check(rc):
    _lib.check(rc)


# ------------------------------------------------------------------------------------------------- recording
class SplitGemmRecorder(G.Recorder):
    """The GEMM sibling's recorder, plus ops.wgrad_split as a unit: each group of segment launches into one dW is one
    configuration (segments, both views' layouts and piece offsets, the table); its single launches still reach
    ops.wgrad and are recorded there."""

    def __init__(self):
        super().__init__()
        self.groups, self.group_keys = [], {}

    def wrap(self, monkeypatch):
        super().wrap(monkeypatch)
        real, rec = ops.wgrad_split, self

        def wgrad_split_rec(X, x_lo, x_channels, Y, y_lo, y_channels, M, taps, dW, **kw):
            segs = tuple(tuple(s) for s in ops.split_segments())
            res = real(X, x_lo, x_channels, Y, y_lo, y_channels, M, taps, dW, **kw)
            nbr, dense = kw.get("nbr"), kw.get("dense")
            cfg = dict(kind="wgrad_split", segs=segs, pieces=ops.split_pieces(), X=G._desc(X), x_lo=int(x_lo), cx=x_channels,
                       Y=G._desc(Y), y_lo=int(y_lo), cy=y_channels, M=M, taps=taps, dW=G._desc(dW), table=rec._table(nbr),
                       dense=tuple(dense) if dense else None, shuffle=bool(kw.get("shuffle", False)))
            key = tuple(sorted(cfg.items()))
            if key in rec.group_keys:
                rec.group_keys[key]["calls"] += 1
            else:
                cfg["calls"], cfg["source"] = 1, rec.source
                rec.group_keys[key] = cfg
                rec.groups.append(cfg)
            return res
        monkeypatch.setattr(ops, "wgrad_split", wgrad_split_rec)


def _scalar_key(kinds, args):
    """The scalar arguments of one call, pointers reduced to null / not null (streams included)."""
    return tuple((v is not None and v != 0) if k is _lib.P else (v.value if hasattr(v, "value") else v)
                 for k, v in zip(kinds, args))


class ScalarRecorder:
    """Proxy of a library handle: the scalar key of every pnx_* call, per entry point."""

    def __init__(self, inner):
        self.inner, self.keys = inner, {}

    def proxy(self):
        rec = self

        class Proxy:
            def __getattr__(self, name):
                fn = getattr(rec.inner, name)
                if not name.startswith("pnx_"):
                    return fn
                kinds = _lib._SIGS[name]

                def call(*args):
                    rec.keys.setdefault(name, set()).add(_scalar_key(kinds, args))
                    return fn(*args)
                return call
        return Proxy()


class _Sources:
    """Sets `source` on every recorder at once (the siblings' _record names the run it is in)."""

    def __init__(self, *recs):
        object.__setattr__(self, "recs", recs)

    def __setattr__(self, k, v):
        for r in self.recs:
            setattr(r, k, v)


def _row_key(c):
    return tuple(sorted((k, v) for k, v in c.items() if k not in ("calls", "source", "pieces")))


def _steps(precision, recs, mp, dense=None):
    """The three runs in `precision` with the library handle replaced by recs' proxy; returns the peak per run."""
    peaks = {}
    proxy = recs[-1].proxy()
    mp.setattr(_lib, "lib", lambda: proxy)
    mp.setattr(ops, "lib", lambda: proxy)
    if dense is not None:
        real = ops.scatter_dense

        def scatter_dense(feat, lv, channels, canvas=None, gather=False):
            out = real(feat, lv, channels, canvas=canvas, gather=gather)
            dense.append((lv, channels, gather, feat.clone(), out.clone()))     # the frontend sibling's record
            return out
        mp.setattr(ops, "scatter_dense", scatter_dense)
    with Fn.precision(precision):
        for name, evaluate in (("nusc", True), ("waymo180k", False)):
            torch.cuda.reset_peak_memory_stats()
            G._record(_Sources(*recs), name, evaluate)
            peaks[name] = torch.cuda.max_memory_allocated()
    return peaks


@pytest.fixture(scope="module")
def runs():
    t0 = time.perf_counter()
    real = _lib.lib()
    out = types.SimpleNamespace(t0=t0, gemm=SplitGemmRecorder(), dense=[])
    out.rows = R.Recorder(real, maps=ROW_MAPS,
                          extra=lambda n: {"pieces": real.pnx_split_get_pieces()} if n in PIECE_FNS else {})
    out.split_keys = ScalarRecorder(out.rows.proxy())
    prev = ops.PROFILE, Fn.get_precision(), ops.set_deterministic(False), ops.split_pieces()
    try:
        with pytest.MonkeyPatch.context() as mp:
            out.gemm.wrap(mp)
            ops.PROFILE = []
            out.peaks = _steps("split", [out.gemm, out.rows, out.split_keys], mp, out.dense)
        out.gemm.table_list = {i: c for _, i, c in out.gemm.tables.values()}
        out.gemm.tables = None
        torch.cuda.empty_cache()
        # the same runs in bf16: which configurations of the shared entry points only the split step produces
        out.bf16_rows = R.Recorder(real, maps=ROW_MAPS)
        out.bf16_keys = ScalarRecorder(out.bf16_rows.proxy())
        with pytest.MonkeyPatch.context() as mp:
            out.bf16_peaks = _steps("bf16", [out.bf16_rows, out.bf16_keys], mp)
    finally:
        ops.PROFILE = prev[0]
        Fn.set_precision(prev[1])
        ops.set_deterministic(prev[2])
        ops.split_pieces(prev[3])
    torch.cuda.empty_cache()
    for name, p in out.peaks.items():
        print("\nsplit %s step: peak %.2f GB (bf16: %.2f GB)" % (name, p / 2 ** 30, out.bf16_peaks[name] / 2 ** 30))
    torch.cuda.reset_peak_memory_stats()
    return out


@contextlib.contextmanager
def _pieces(P):
    prev = ops.split_pieces(P)
    try:
        yield P
    finally:
        ops.split_pieces(prev)


def _of(runs, fn):
    return [c for c in runs.rows.configs if c["fn"] == fn]


# ------------------------------------------------------------------------------------------------- split references
def rne_bf16(x):
    """fp32 -> fp32 holding bf16(x), round to nearest even, computed on the bits (no float arithmetic, so subnormals
    survive whatever the device's denormal mode).  x finite."""
    b = x.contiguous().view(torch.int32).long() & 0xFFFFFFFF
    r = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return (r - ((r >> 31) << 32)).int().view(torch.float32).view(x.shape)


def split_ref(x, P):
    """The P pieces (fp32 tensors holding bf16 values) of fp32 x: p0 = bf16(x), p1 = bf16(x - p0), ...  The residuals
    are exact (taken in fp64)."""
    out, rem = [], x.float()
    for _ in range(P):
        p = rne_bf16(rem)
        out.append(p)
        rem = (rem.double() - p.double()).float()
    return out


def merge_ref(pieces):
    """fp32 sum of the pieces in the kernels' order: smallest piece first; a zero sum takes the sign of piece 0."""
    f = pieces[-1].float()
    for p in reversed(pieces[:-1]):
        f = f + p.float()
    return torch.where(f == 0, torch.copysign(torch.zeros_like(f), pieces[0].float()), f)


def ulp32(v):
    """fp32 ulp at |v| (2^-149 at zero / subnormals)."""
    _, e = torch.frexp(v.double().abs().clamp(min=2.0 ** -126))
    return torch.ldexp(torch.ones_like(v, dtype=torch.float64), e - 24)


def edge_values():
    """fp32 values where a split goes wrong first: signed zeros, exact bf16 ties (even and odd), carries into the next
    binade, fp32 subnormals (ties among them too), the smallest normals, values whose low pieces are subnormal, and
    the largest values that stay finite in bf16."""
    bits = [0x00000000, 0x80000000, 0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000, 0x3F80C000, 0x3F80FFFF,
            0x3FFFFFFF, 0x3FFF8000, 0xBFFFFFFF, 0x3FFF7FFF, 0x477FFFFF, 0x4B7F8000,
            0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00008000, 0x00018000, 0x00400000, 0x00010001,
            0x00800000, 0x80800000, 0x00808001, 0x00FFFFFF, 0x0C812345, 0x8C812345, 0x09000001, 0x0A7FFFFF,
            0x7F7F7FFF, 0xFF7F7FFF, 0x7F7F0000, 0x7F7F7F00, 0x3DCCCCCD, 0x40490FDB, 0xC2F6E979, 0x3A83126F]
    t = torch.tensor([b - (1 << 32) if b >= 1 << 31 else b for b in bits], dtype=torch.int32)
    return t.view(torch.float32)


def _with_edges(x):
    """x with the edge values in its first and last row (repeated to fill them)."""
    e = edge_values().to(x.device)
    C = x.shape[1]
    row = e.repeat(-(-C // e.numel()))[:C]
    x[0], x[-1] = row, row.flip(0)
    return x


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------- split buffers
def _layout(ld, lo, C, P, wide, i):
    """(ld, lo) of a split operand: the recorded ones (ld at least what P pieces need), or widened: lo past C by
    8 (i + 1) elements, ld past the last piece by as many (a different gap per operand)."""
    lo = max(lo, C)
    if wide:
        lo += 8 * (i + 1)
        return (P - 1) * lo + C + 8 * (i + 1), lo
    return max(ld, (P - 1) * lo + C), lo


def _put(pieces, ld, lo):
    """A NaN-sentinel bf16 buffer [M + GUARD_ROWS, ld] with piece q in the columns [q lo, q lo + C)."""
    M, C = pieces[0].shape
    buf = R._sentinel_buf(M, ld, torch.bfloat16)
    for q, p in enumerate(pieces):
        buf[:M, q * lo:q * lo + C] = p
    return buf


def _get(buf, M, C, lo, P):
    return [buf[:M, q * lo:q * lo + C] for q in range(P)]


def _untouched_split(buf, M, C, lo, P):
    """Every element of buf outside the P pieces of rows [0, M) still holds the sentinel."""
    bits, s = R.SENT[torch.bfloat16]
    b = buf.view(bits)
    keep = torch.ones(b.shape[1], dtype=torch.bool, device=b.device)
    for q in range(P):
        keep[q * lo:q * lo + C] = False
    return bool((b[M:] == s).all()) and bool((b[:M][:, keep] == s).all())


POISON = set()       # names of kernel outputs to overwrite with one NaN after the launch (the NaN self-check)


def _poison(name, t, idx):
    if name in POISON:
        if isinstance(idx, tuple):
            t[idx] = float("nan")
        else:
            t.view(-1)[idx] = float("nan")


def _gauss(M, C, seed, scale=1.0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(M, C, generator=gen, device="cuda") * scale


def _loose_pieces(M, C, seed, P=3):
    """P bf16 pieces that are not a valid split: piece q ~ N(0, 2^-7q), so that their fp32 sums round."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return [(torch.randn(M, C, generator=gen, device="cuda") * 2.0 ** (-7 * q)).bfloat16() for q in range(P)]


# ------------------------------------------------------------------------------------------------- igemm with segments
def _seg_desc(c):
    a, w = G.seg_pieces(c)
    return "%d segs, A %d / W %d pieces, a_lo_off %d" % (len(c["segs"] or ()), a, w, c["a_lo_off"]) if c.get("segs") else ""


def test_split_gemms_match_exact_reference(runs):
    """Every unique igemm configuration (segments and all) and every single wgrad launch of the split runs reproduces
    its exact integer reference (the sibling's replay, extended to segments)."""
    cfgs = runs.gemm.configs
    segd = [c for c in cfgs if c["kind"] == "igemm" and c["segs"]]
    assert segd and any(c["addend"] and c["addend"][2] == torch.float32 for c in segd), "no split GEMM with an fp32 addend"
    assert any(c["dense"] and c["dense"][4] == 3 and c["taps"] == 9 for c in segd), "no dense 3x3 split convolution"
    for src in ("nusc train", "nusc eval", "waymo180k train"):
        assert any(c["source"] == src for c in cfgs), src
    gen = torch.Generator(device="cuda").manual_seed(4321)
    failures = []
    print("\n%d unique GEMM configurations (%d igemm with segments)" % (len(cfgs), len(segd)))
    for i, c in enumerate(cfgs):
        grid, _ = G._grid(c)
        try:
            bad, o, ref = G._replay(c, runs.gemm.table_list, gen)
            del o, ref
        except G.Unreproducible as e:
            bad = ["cannot be replayed: %s" % e]
        print("[%3d] %-16s %-100s %-40s x%-3d %s %s" % (i, c["source"], G._label(c), grid, c["calls"], _seg_desc(c),
                                                        "ok" if not bad else "; ".join(bad)))
        if bad:
            failures.append("%s %s: %s" % (c["source"], G._label(c), "; ".join(bad)))
        torch.cuda.empty_cache()
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------- wgrad_split groups
def _group_operands(c, gen, tables):
    nseg = len(c["segs"])
    for ax, ay in ((3, 2), (2, 2), (2, 1), (1, 1)):
        bound = nseg * c["M"] * ax * ay
        if bound < G.EXACT:
            break
    else:
        raise G.Unreproducible("M = %d, %d segments: no integer range keeps the sums exact" % (c["M"], nseg))
    if c["dW"][0] != (c["taps"], c["cx"], c["cy"]) or c["dW"][2] != torch.float32:
        raise G.Unreproducible("dW layout %s" % (c["dW"],))
    xp = max(a for a, _ in c["segs"]) + 1
    yp = max(b for _, b in c["segs"]) + 1
    o = types.SimpleNamespace(bound=bound)
    o.X = G.pieces_buffer(c["X"], c["cx"], c["x_lo"], xp, ax, gen)
    o.Y = G.pieces_buffer(c["Y"], c["cy"], c["y_lo"], yp, ay, gen)
    if o.X.shape[0] < c["M"]:
        raise G.Unreproducible("X rows")
    o.table = tables[c["table"]] if c["table"] is not None else None
    return o


def _launch_group(c, o, overwrite_last=False):
    """dW zeroed once, then the recorded launches in order (overwrite_last: the last one writes a fresh buffer that
    replaces dW, the error the self-check must catch)."""
    dW = torch.zeros(c["dW"][0], dtype=torch.float32, device="cuda")
    for i, (xp, yp) in enumerate(c["segs"]):
        dst = torch.zeros_like(dW) if overwrite_last and i == len(c["segs"]) - 1 else dW
        ops.wgrad(G.piece(o.X, xp * c["x_lo"], c["cx"]), c["cx"], G.piece(o.Y, yp * c["y_lo"], c["cy"]), c["cy"], c["M"],
                  c["taps"], dst, nbr=o.table, dense=c["dense"], shuffle=c["shuffle"])
        if dst is not dW:
            dW = dst
    _poison("wgrad_split dW", dW, dW.numel() - 1)
    return dW


def _group_reference(c, o):
    M, T, cx, cy = c["M"], c["taps"], c["cx"], c["cy"]
    dev = o.X.device
    ref = torch.zeros(T, cx, cy, dtype=torch.float64, device=dev)
    gathered = c["table"] is not None or c["dense"] is not None or c["shuffle"]
    step = G._chunk_rows(cx + cy)
    for m0 in range(0, M, step):
        m1 = min(M, m0 + step)
        for t in range(T):
            if not gathered:
                idx = torch.arange(m0, m1, device=dev)
            elif c["shuffle"]:
                idx = G._shuffle_index(m0, m1, t, c["dense"], dev)
            else:
                idx = G._gather_index(m0, m1, t, o.table, c["dense"], dev)
            for xp, yp in c["segs"]:
                Xc = G.piece(o.X, xp * c["x_lo"], cx)[m0:m1].double()
                ref[t] += Xc.t() @ G._gather(G.piece(o.Y, yp * c["y_lo"], cy), idx, cy)
    return ref.float()


def _group_label(c):
    g = "table" if c["table"] is not None else "shuffle" if c["shuffle"] else \
        "dense d%d" % c["dense"][6] if c["dense"] else "direct"
    return "wgrad_split M %d T %d X %d (ld %d lo %d) Y %d (ld %d lo %d) %s, %d segs, %d pieces" % (
        c["M"], c["taps"], c["cx"], c["X"][1][0], c["x_lo"], c["cy"], c["Y"][1][0], c["y_lo"], g, len(c["segs"]), c["pieces"])


def _replay_group(c, tables, gen):
    o = _group_operands(c, gen, tables)
    ref = _group_reference(c, o)
    dW = _launch_group(c, o)
    bad = [] if torch.equal(dW, ref) else ["dW differs in %d entries" % int((dW != ref).sum())]
    return bad, o, ref


def test_wgrad_split_groups_match_exact_reference(runs):
    groups = runs.gemm.groups
    assert groups and any(c["shuffle"] for c in groups) and any(c["table"] is not None for c in groups)
    assert any(c["X"][1][0] != c["cx"] * c["pieces"] for c in groups), "no group on column-slice views (the ASPP's)"
    gen = torch.Generator(device="cuda").manual_seed(77)
    failures = []
    print("\n%d wgrad_split groups" % len(groups))
    for i, c in enumerate(groups):
        try:
            bad, o, ref = _replay_group(c, runs.gemm.table_list, gen)
            del o, ref
        except G.Unreproducible as e:
            bad = ["cannot be replayed: %s" % e]
        print("[%2d] %-16s %-110s x%-3d %s" % (i, c["source"], _group_label(c), c["calls"], "ok" if not bad else "; ".join(bad)))
        if bad:
            failures.append("%s %s: %s" % (c["source"], _group_label(c), "; ".join(bad)))
        torch.cuda.empty_cache()
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------- row-wise: exact kernels
def _replay_rows_split(c):
    M, C = c["M"], c["C"]
    x = _with_edges(_gauss(M, C, M + C, 8.0))
    bad, notes = [], []
    for P in PIECE_COUNTS:
        with _pieces(P):
            ref = [p.bfloat16() for p in split_ref(x, P)]
            for wide in (False, True):
                what = "%d pieces, %s strides" % (P, "widened" if wide else "recorded")
                xb, xv = R._place(x, R._ld(c["ldx"], C, R._pad(wide, 0)))
                ldy, lo = _layout(c["ldy"], c["lo_y"], C, P, wide, 1)
                yb = R._sentinel_buf(M, ldy, torch.bfloat16)
                _check(L().pnx_rows_split(R._p(xv), xv.stride(0), M, C, R._p(yb), ldy, lo, ops.stream()))
                got = _get(yb, M, C, lo, P)
                _poison("rows_split y", got[P - 1], (M - 1, C - 1))
                for q in range(P):
                    if not _same_bits(got[q], ref[q]):
                        n = int((_bits(got[q]) != _bits(ref[q])).sum())
                        bad.append("%s: piece %d differs from the bit-level split in %d entries (edge rows %s)" % (
                            what, q, n, "differ" if not (_same_bits(got[q][0], ref[q][0]) and
                                                         _same_bits(got[q][-1], ref[q][-1])) else "match"))
                if not (_untouched_split(yb, M, C, lo, P) and R._untouched(xb, M, C)):
                    bad.append("%s: sentinel changed" % what)
                if P == 3 and not wide:
                    back = torch.full((M, C), float("nan"), device="cuda")
                    _check(L().pnx_rows_merge(R._p(yb), ldy, lo, M, C, R._p(back), C, 0, ops.stream()))
                    _poison("round trip", back, M * C - 1)
                    # three pieces hold every bit of an fp32 that is a multiple of 2^-133 (bf16's subnormal step):
                    # every |x| >= 2^-110; below, the low bits of subnormal residuals are lost (at most 2^-134)
                    full = (x.abs() >= 2.0 ** -110) | (x == 0)
                    exact = torch.equal(_bits(back)[full], _bits(x)[full])
                    err = (back.double() - x.double()).abs()
                    small = R._worst(err[~full]) if (~full).any() else 0.0
                    if not exact or not small <= 2.0 ** -134:
                        bad.append("rows_merge(rows_split(x)) is not x (%s; error below 2^-110: %.3g)" % (
                            "exact" if exact else "differs", small))
                    notes.append("round trip exact for |x| >= 2^-110 (%d tiny edge values within %.1e)" % (
                        int((~full).sum()), small))
                del xb, yb
    return bad, "; ".join(notes) or "bit-exact"


def _replay_rows_merge(c):
    M, C = c["M"], c["C"]
    pcs = _loose_pieces(M, C, M + C + 1)
    y0 = _gauss(M, C, M + C + 2)
    bad = []
    for P in PIECE_COUNTS:
        with _pieces(P):
            ref = merge_ref(pcs[:P])
            if c["accumulate"]:
                ref = ref + y0
            for wide in (False, True):
                what = "%d pieces, %s strides" % (P, "widened" if wide else "recorded")
                ldx, lo = _layout(c["ldx"], c["lo_x"], C, P, wide, 0)
                xb = _put(pcs[:P], ldx, lo)
                ldy = R._ld(c["ldy"], C, R._pad(wide, 1))
                yb, y = R._place(y0, ldy) if c["accumulate"] else R._out(M, C, ldy, torch.float32)
                _check(L().pnx_rows_merge(R._p(xb), ldx, lo, M, C, R._p(y), ldy, c["accumulate"], ops.stream()))
                _poison("rows_merge y", y, (M - 1, C - 1))
                if not _same_bits(y, ref):
                    bad.append("%s: %d entries differ from the fp32 emulation" % (what, int((_bits(y) != _bits(ref)).sum())))
                if not (_untouched_split(xb, M, C, lo, P) and R._untouched(yb, M, C)):
                    bad.append("%s: sentinel changed" % what)
                del xb, yb
    return bad, "bit-exact" if not bad else ""


def _replay_add_relu_split(c):
    M, C = c["M"], c["C"]
    a, b = _loose_pieces(M, C, M + C + 3), _loose_pieces(M, C, M + C + 4)
    bad = []
    for P in PIECE_COUNTS:
        with _pieces(P):
            ref = [p.bfloat16() for p in split_ref((merge_ref(a[:P]) + merge_ref(b[:P])).clamp_min(0), P)]
            for wide in (False, True):
                what = "%d pieces, %s strides" % (P, "widened" if wide else "recorded")
                lda, loa = _layout(c["lda"], c["lo_a"], C, P, wide, 0)
                ldb, lob = _layout(c["ldb"], c["lo_b"], C, P, wide, 1)
                ldy, loy = _layout(c["ldy"], c["lo_y"], C, P, wide, 2)
                ab, bb, yb = _put(a[:P], lda, loa), _put(b[:P], ldb, lob), R._sentinel_buf(M, ldy, torch.bfloat16)
                _check(L().pnx_add_relu_split(R._p(ab), lda, loa, R._p(bb), ldb, lob, M, C, R._p(yb), ldy, loy, ops.stream()))
                got = _get(yb, M, C, loy, P)
                _poison("add_relu_split y", got[0], (M - 1, C - 1))
                if not all(_same_bits(g, r) for g, r in zip(got, ref)):
                    bad.append("%s: pieces differ from the fp32 emulation" % what)
                if not (_untouched_split(ab, M, C, loa, P) and _untouched_split(bb, M, C, lob, P) and
                        _untouched_split(yb, M, C, loy, P)):
                    bad.append("%s: sentinel changed" % what)
                del ab, bb, yb
    return bad, "bit-exact" if not bad else ""


def _replay_relu_bwd_split(c):
    M, C = c["M"], c["C"]
    dy = _gauss(M, C, M + C + 5)
    y = _loose_pieces(M, C, M + C + 6)
    bad = []
    for P in PIECE_COUNTS:
        with _pieces(P):
            g = torch.where(merge_ref(y[:P]) > 0, dy, torch.zeros((), device="cuda"))
            ref = [p.bfloat16() for p in split_ref(g, P)]
            for wide in (False, True):
                what = "%d pieces, %s strides" % (P, "widened" if wide else "recorded")
                db, dv = R._place(dy, R._ld(c["lddy"], C, R._pad(wide, 0)))
                ldy, loy = _layout(c["ldy"], c["lo_y"], C, P, wide, 1)
                ldg, log_ = _layout(c["ldg"], c["lo_g"], C, P, wide, 2)
                yb, gb = _put(y[:P], ldy, loy), R._sentinel_buf(M, ldg, torch.bfloat16)
                _check(L().pnx_relu_bwd_split(R._p(dv), dv.stride(0), R._p(yb), ldy, loy, M, C, R._p(gb), ldg, log_,
                                              ops.stream()))
                got = _get(gb, M, C, log_, P)
                _poison("relu_bwd_split g", got[0], (M - 1, C - 1))
                if not all(_same_bits(a, r) for a, r in zip(got, ref)):
                    bad.append("%s: pieces differ from the fp32 emulation" % what)
                if not (R._untouched(db, M, C) and _untouched_split(yb, M, C, loy, P) and _untouched_split(gb, M, C, log_, P)):
                    bad.append("%s: sentinel changed" % what)
                del db, yb, gb
    return bad, "bit-exact" if not bad else ""


def _replay_tap_scatter(c):
    B, H, W, cpt, nz = c["B"], c["H"], c["W"], c["cpt"], c["nz"]
    M = B * H * W
    assert c["lo_off"] > 0
    dout = _gauss(M, cpt, M + nz, 3.0)
    full = R._stencil_scatter_ref(dout, B, H, W, nz, cpt, torch.float32)
    bad = []
    for P in PIECE_COUNTS:
        with _pieces(P):
            ref = [p.bfloat16() for p in split_ref(full, P)]
            for wide in (False, True):
                what = "%d pieces, %s strides" % (P, "widened" if wide else "recorded")
                db, dv = R._place(dout, 16)
                ldz, lo = _layout(c["ldz"], c["lo_off"], nz, P, wide, 0)
                zb = R._sentinel_buf(M, ldz, torch.bfloat16)
                _check(L().pnx_tap_scatter(R._p(dv), B, H, W, R._p(zb), ldz, nz, cpt, lo, ops.stream()))
                got = _get(zb, M, nz, lo, P)
                _poison("tap_scatter dZ", got[P - 1], (M - 1, 0))
                if not all(_same_bits(a, r) for a, r in zip(got, ref)):
                    bad.append("%s: dZ pieces differ from the split of the gathered dout" % what)
                if not (_untouched_split(zb, M, nz, lo, P) and R._untouched(db, M, cpt)):
                    bad.append("%s: sentinel changed" % what)
                del db, zb
    return bad, "cpt %d, NZ %d, lo_off %d: bit-exact" % (cpt, nz, c["lo_off"]) if not bad else ""


def _run(configs, replay, title):
    return R._run(R._by_size(configs) if configs and "M" in configs[0] else configs, replay, title)


def test_rows_split_bit_exact_with_edge_values(runs):
    failures = _run(_of(runs, "pnx_rows_split"), _replay_rows_split, "pnx_rows_split")
    assert _of(runs, "pnx_rows_split") and not failures, "\n".join(failures)


def test_rows_merge_bit_exact(runs):
    cfgs = _of(runs, "pnx_rows_merge")
    assert any(c["accumulate"] for c in cfgs), "no accumulating rows_merge (the fan-out's)"
    failures = _run(cfgs, _replay_rows_merge, "pnx_rows_merge")
    assert not failures, "\n".join(failures)


def test_add_relu_relu_bwd_tap_scatter_split_bit_exact(runs):
    sc = [c for c in _of(runs, "pnx_tap_scatter") if c["lo_off"] > 0]
    assert sc, "no tap_scatter writing split pieces"
    failures = _run(_of(runs, "pnx_add_relu_split"), _replay_add_relu_split, "pnx_add_relu_split")
    failures += _run(_of(runs, "pnx_relu_bwd_split"), _replay_relu_bwd_split, "pnx_relu_bwd_split")
    failures += _run(sc, _replay_tap_scatter, "pnx_tap_scatter (lo_off > 0)")
    assert _of(runs, "pnx_add_relu_split") and _of(runs, "pnx_relu_bwd_split")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------- row-wise: BatchNorm
def _replay_bn_apply_split(c):
    M, C = c["M"], c["C"]
    gen = torch.Generator(device="cuda").manual_seed(M + 3 * C)
    x = _gauss(M, C, M + C + 7, 3.0)
    scale = torch.rand(C, generator=gen, device="cuda") + 0.5
    shift = torch.randn(C, generator=gen, device="cuda")
    res32 = _gauss(M, C, M + C + 8) if c["res"] else None
    bad, worst = [], dict.fromkeys(PIECE_COUNTS, 0.0)
    for P in PIECE_COUNTS:
        with _pieces(P):
            res = [p.bfloat16() for p in split_ref(res32, P)] if res32 is not None else None
            t = x.double() * scale.double() + shift.double()
            o = t + merge_ref(res).double() if res is not None else t      # the P-piece residual's value is exact
            if c["relu"]:
                o = o.clamp(min=0)
            k = 2.0 if res is not None else 1.0
            bound = k * ulp32(torch.maximum(t.abs(), o.abs())) + (2.0 ** -16 * o.abs() if P == 2 else 0.0)
            for wide in (False, True):
                what = "%d pieces, %s strides" % (P, "widened" if wide else "recorded")
                xb, xv = R._place(x, R._ld(c["ldx"], C, R._pad(wide, 0)))
                if res is not None:
                    ldr, lor = _layout(c["ldr"], c["lo_r"], C, P, wide, 1)
                    rb = _put(res, ldr, lor)
                else:
                    ldr, lor, rb = 16, 16, None
                ldy, loy = _layout(c["ldy"], c["lo_y"], C, P, wide, 2)
                yb = R._sentinel_buf(M, ldy, torch.bfloat16)
                _check(L().pnx_bn_apply_split(R._p(xv), xv.stride(0), M, C, R._p(scale), R._p(shift), R._p(rb), ldr, lor,
                                              c["relu"], R._p(yb), ldy, loy, ops.stream()))
                got = _get(yb, M, C, loy, P)
                _poison("bn_apply_split y", got[0], (M - 1, C - 1))
                merged = merge_ref(got)
                r = R._worst((merged.double() - o).abs() / bound)
                worst[P] = max(worst[P], r)
                if not r <= 1.0:
                    bad.append("%s: merged y off by %.3g x its bound (%d fp32 ulp)" % (what, r, k))
                if P == 3 and not all(_same_bits(a, b.bfloat16()) for a, b in zip(got, split_ref(merged, P))):
                    bad.append("%s: the pieces are not the exact split of their merged value" % what)
                if not (R._untouched(xb, M, C) and _untouched_split(yb, M, C, loy, P) and
                        (rb is None or _untouched_split(rb, M, C, lor, P))):
                    bad.append("%s: sentinel changed" % what)
                del xb, rb, yb
    return bad, "err/bound " + ", ".join("%.3f at %d pieces" % (worst[P], P) for P in PIECE_COUNTS)


def _reduce_grid(M, C):
    """(rows per thread L, blocks, rows per block) of pnx_bn_bwd_reduce_split's first stage."""
    rpb = 256 // (C // 8)
    nb = min(296, max(1, -(-M // rpb)))
    return -(-M // (nb * rpb)), nb, rpb


_RED_CACHE = {}


def _red_data(M, C, exact):
    """Reduce operands: exact = small integers (3 dy pieces and 3 y pieces of their own, x in [-4, 4], mean 1, invstd
    2, forward affine x - 0.5: every fp32 partial and fp64 sum is an exact integer); else Gaussian dy (a valid split),
    x with per-channel means, its statistics, and loose y pieces."""
    key = (M, C, exact)
    if key in _RED_CACHE:
        return _RED_CACHE[key]
    if any(k[:2] != (M, C) for k in _RED_CACHE):
        _RED_CACHE.clear()
        torch.cuda.empty_cache()
    gen = torch.Generator(device="cuda").manual_seed(M * 13 + C + exact)
    d = types.SimpleNamespace(M=M, C=C)
    if exact:
        ints = lambda: torch.randint(-4, 5, (M, C), generator=gen, device="cuda")  # noqa: E731
        d.dy, d.y = [ints().bfloat16() for _ in range(3)], [ints().bfloat16() for _ in range(3)]
        d.x = ints().float()
        full = lambda v: torch.full((C,), v, device="cuda")  # noqa: E731
        d.mean, d.invstd, d.fs, d.fh = full(1.0), full(2.0), full(1.0), full(-0.5)
    else:
        d.dy = [p.bfloat16() for p in split_ref(torch.randn(M, C, generator=gen, device="cuda"), 3)]
        d.y = _loose_pieces(M, C, M + C + 9)
        mu = torch.randn(C, generator=gen, device="cuda")
        d.x = torch.randn(M, C, generator=gen, device="cuda") * (torch.rand(C, generator=gen, device="cuda") + 0.5) + mu
        d.mean = d.x.double().mean(0).float()
        d.invstd = (1.0 / d.x.double().var(0, unbiased=False).add(1e-5).sqrt()).float()
        d.fs = torch.rand(C, generator=gen, device="cuda") + 0.5
        d.fh = -d.mean * d.fs
    d.gamma = torch.rand(C, generator=gen, device="cuda") + 0.5
    _RED_CACHE[key] = d
    return d


def _gate(d, mode, P):
    if mode == 0:
        return None
    if mode == 1:
        return merge_ref(d.y[:P]) > 0
    return d.x.double() * d.fs.double() + d.fh.double() > 0     # the sign of the exact x*fs + fh, as fmaf gives it


def _gated(d, mode, P):
    g = merge_ref(d.dy[:P])
    gate = _gate(d, mode, P)
    return g if gate is None else torch.where(gate, g, torch.zeros((), device="cuda"))


def _reduce_ref(d, mode, P, drop_block=None):
    """fp64 sums of g and g (x - mean) invstd and of their magnitudes; drop_block = a first-stage block whose rows are
    left out (the self-check)."""
    g = _gated(d, mode, P).double()
    t = g * (d.x.double() - d.mean.double()) * d.invstd.double()
    if drop_block is not None:
        _, nb, rpb = _reduce_grid(d.M, d.C)
        keep = (torch.arange(d.M, device="cuda") // rpb) % nb != drop_block
        g, t = g[keep], t[keep]
    return torch.cat([g.sum(0), t.sum(0)]), torch.cat([g.abs().sum(0), t.abs().sum(0)])


def _launch_reduce_split(c, d, mode, P, wide):
    M, C = d.M, d.C
    lddy, lody = _layout(c["lddy"], c["lo_dy"], C, P, wide, 0)
    dyb = _put(d.dy[:P], lddy, lody)
    xb, xv = R._place(d.x, R._ld(c["ldx"], C, R._pad(wide, 1)))
    if mode == 1:
        ldy, loy = _layout(c["ldy"] if c["y"] else P * C, c["lo_y"] if c["y"] else C, C, P, wide, 2)
        yb = _put(d.y[:P], ldy, loy)
    else:
        ldy, loy, yb = 16, 16, None
    part = torch.full((L().pnx_bn_bwd_reduce_split_scratch(C),), float("nan"), dtype=torch.float64, device="cuda")
    red = torch.full((2 * C,), float("nan"), dtype=torch.float64, device="cuda")
    _check(L().pnx_bn_bwd_reduce_split(R._p(dyb), lddy, lody, R._p(yb), ldy, loy, R._p(xv), xv.stride(0), M, C, R._p(d.mean),
                                       R._p(d.invstd), 1 if mode else 0, R._p(d.fs) if mode == 2 else None,
                                       R._p(d.fh) if mode == 2 else None, R._p(part), R._p(red), ops.stream()))
    ok = _untouched_split(dyb, M, C, lody, P) and R._untouched(xb, M, C) and (yb is None or _untouched_split(yb, M, C, loy, P))
    _poison("reduce_split red", red, 2 * C - 1)
    return red, ok


def _mode(c):
    return 0 if not c["relu"] else (1 if c["y"] else 2)


def _replay_reduce_split(c, modes):
    M, C = c["M"], c["C"]
    Lr, nb, rpb = _reduce_grid(M, C)
    assert 12 * 5 * 2 * Lr < 2 ** 24, "integer partials no longer exact"     # |g| <= 12, |x - mean| <= 5, invstd 2
    bad, worst = [], 0.0
    for P in PIECE_COUNTS:
        with _pieces(P):
            for mode in modes:
                di = _red_data(M, C, True)
                exact, _ = _reduce_ref(di, mode, P)
                for wide in (False, True):
                    what = "%d pieces, gate %s, %s strides" % (P, ("none", "y", "x")[mode], "widened" if wide else "recorded")
                    red, ok = _launch_reduce_split(c, di, mode, P, wide)
                    if not torch.equal(red, exact):
                        bad.append("%s: %d integer sums differ from fp64" % (what, int((red != exact).sum())))
                    dg = _red_data(M, C, False)
                    ref, mag = _reduce_ref(dg, mode, P)
                    red1, ok1 = _launch_reduce_split(c, dg, mode, P, wide)
                    red2, _ = _launch_reduce_split(c, dg, mode, P, wide)
                    k = torch.cat([torch.full((C,), Lr + 1.0), torch.full((C,), Lr + 4.0)]).to(mag)
                    r = R._worst((red1 - ref).abs() / (k * U * mag + 1e-300))
                    worst = max(worst, r)
                    if not r <= 1.0:
                        bad.append("%s: Gaussian sums off by %.3g x (L+1) u sum|.|" % (what, r))
                    if not torch.equal(red1.view(torch.int64), red2.view(torch.int64)):
                        bad.append("%s: two launches differ" % what)
                    if not (ok and ok1):
                        bad.append("%s: sentinel changed" % what)
    return bad, "L %d (%d blocks x %d rows), Gaussian err/bound %.3g" % (Lr, nb, rpb, worst)


def _bwd_apply_ref(d, mode, P, red, n):
    """fp64 evaluation of dx on the kernel's fp32 inputs (the sums scaled and rounded to fp32 as the kernel does), and
    its first-order bound 8 u |A| (|g| + |s1| + |xhat s2|)."""
    C = d.C
    g = _gated(d, mode, P)
    A = d.gamma.double() * d.invstd.double()
    s1 = (red[:C] * (1.0 / n)).float().double()
    s2 = (red[C:] * (1.0 / n)).float().double()
    xh = (d.x.double() - d.mean.double()) * d.invstd.double()
    gd = g.double()
    dx = A * (gd - s1 - xh * s2)
    bound = 8 * U * A.abs() * (gd.abs() + s1.abs() + (xh * s2).abs()) + 2.0 ** -140
    if P == 2:
        bound = bound + 2.0 ** -16 * dx.abs()
    return dx, bound, g


def _replay_bwd_apply_split(c, modes):
    M, C = c["M"], c["C"]
    n = c["count"]
    bad, worst = [], dict.fromkeys(PIECE_COUNTS, 0.0)
    d = _red_data(M, C, False)
    for P in PIECE_COUNTS:
        with _pieces(P):
            for mode in modes:
                red, _ = _reduce_ref(d, mode, P)
                ref, bound, g = _bwd_apply_ref(d, mode, P, red, n)
                dres_ref = [p.bfloat16() for p in split_ref(g, P)]
                for wide in (False, True):
                    what = "%d pieces, gate %s, %s strides" % (P, ("none", "y", "x")[mode], "widened" if wide else "recorded")
                    lddy, lody = _layout(c["lddy"], c["lo_dy"], C, P, wide, 0)
                    dyb = _put(d.dy[:P], lddy, lody)
                    xb, xv = R._place(d.x, R._ld(c["ldx"], C, R._pad(wide, 1)))
                    if mode == 1:
                        ldy, loy = _layout(c["ldy"] if c["y"] else P * C, c["lo_y"] if c["y"] else C, C, P, wide, 2)
                        yb = _put(d.y[:P], ldy, loy)
                    else:
                        ldy, loy, yb = 16, 16, None
                    lddx, lodx = _layout(c["lddx"], c["lo_dx"], C, P, wide, 3)
                    dxb = R._sentinel_buf(M, lddx, torch.bfloat16)
                    if c["dres"]:
                        ldr, lor = _layout(c["lddres"], c["lo_dres"], C, P, wide, 4)
                        drb = R._sentinel_buf(M, ldr, torch.bfloat16)
                    else:
                        ldr, lor, drb = 16, 16, None
                    _check(L().pnx_bn_bwd_apply_split(R._p(dyb), lddy, lody, R._p(yb), ldy, loy, R._p(xv), xv.stride(0), M, C,
                                                      R._p(d.mean), R._p(d.invstd), R._p(d.gamma), R._p(red), float(n),
                                                      1 if mode else 0, R._p(d.fs) if mode == 2 else None,
                                                      R._p(d.fh) if mode == 2 else None, R._p(dxb), lddx, lodx, R._p(drb),
                                                      ldr, lor, ops.stream()))
                    got = _get(dxb, M, C, lodx, P)
                    _poison("bwd_apply_split dx", got[0], (M - 1, C - 1))
                    r = R._worst((merge_ref(got).double() - ref).abs() / bound)
                    worst[P] = max(worst[P], r)
                    if not r <= 1.0:
                        bad.append("%s: dx off by %.3g x its first-order bound" % (what, r))
                    if drb is not None:
                        dres = _get(drb, M, C, lor, P)
                        _poison("bwd_apply_split dres", dres[0], (M - 1, C - 1))
                        if not all(_same_bits(a, b) for a, b in zip(dres, dres_ref)):
                            bad.append("%s: dres differs from the split of g" % what)
                    bufs = [(dyb, lody), (dxb, lodx)] + ([(yb, loy)] if yb is not None else []) + \
                        ([(drb, lor)] if drb is not None else [])
                    if not (all(_untouched_split(b, M, C, lo, P) for b, lo in bufs) and R._untouched(xb, M, C)):
                        bad.append("%s: sentinel changed" % what)
                    del dyb, xb, yb, dxb, drb, bufs
    return bad, "dx err/bound " + ", ".join("%.3f at %d pieces" % (worst[P], P) for P in PIECE_COUNTS)


def test_bn_apply_split_matches_fp64(runs):
    cfgs = _of(runs, "pnx_bn_apply_split")
    assert any(c["res"] for c in cfgs) and any(not c["res"] for c in cfgs)
    failures = _run(cfgs, _replay_bn_apply_split, "pnx_bn_apply_split")
    assert not failures, "\n".join(failures)


def test_bn_bwd_reduce_split_exact_and_bounded(runs):
    """Each configuration in its recorded gate mode; the largest one with no gate, the gate from y and the gate
    recomputed from x."""
    cfgs = _of(runs, "pnx_bn_bwd_reduce_split")
    assert {_mode(c) for c in cfgs} >= {1, 2}, "both gate sources"
    largest = max(cfgs, key=lambda c: c["M"] * c["C"])
    failures = _run(cfgs, lambda c: _replay_reduce_split(c, (0, 1, 2) if c is largest else (_mode(c),)),
                    "pnx_bn_bwd_reduce_split")
    assert not failures, "\n".join(failures)


def test_bn_bwd_apply_split_matches_fp64(runs):
    cfgs = _of(runs, "pnx_bn_bwd_apply_split")
    assert any(c["dres"] for c in cfgs)
    largest = max(cfgs, key=lambda c: c["M"] * c["C"])
    failures = _run(cfgs, lambda c: _replay_bwd_apply_split(c, (0, 1, 2) if c is largest else (_mode(c),)),
                    "pnx_bn_bwd_apply_split")
    assert not failures, "\n".join(failures)


# ------------------------------------------------------------------------------------------------- completeness
def _split_only(runs, fn):
    have = {_row_key(c) for c in runs.bf16_rows.configs if c["fn"] == fn}
    return [c for c in _of(runs, fn) if _row_key(c) not in have]


def test_shared_entry_points_with_split_only_configurations_replayed(runs):
    """Row-wise entry points the bf16 step shares (BatchNorm statistics, the stencil sum, the loss) at the
    configurations only the split step produces, through the row-wise sibling's replays; the split step's densify
    calls (split rows of P * 256 channels) through the front-end sibling's check."""
    failures = []
    for fn, replay in SHARED_ROW.items():
        cfgs = _split_only(runs, fn)
        if cfgs:
            failures += R._run(cfgs, replay, fn + " (split-only configurations)")
    import test_production_frontend_gpu as FE
    assert runs.dense and any(g for _, _, g, _, _ in runs.dense)
    bad = FE._dense_fails(types.SimpleNamespace(dense=runs.dense), None)
    print("\npnx_scatter_dense: %d split-mode calls (channels %s): %s" % (
        len(runs.dense), sorted({c for _, c, _, _, _ in runs.dense}), "exact" if not bad else "; ".join(bad)))
    assert not failures + bad, "\n".join(failures + bad)


def test_every_entry_point_of_the_split_runs_is_covered(runs):
    """Every pnx_* entry point the split runs call is replayed here, replayed by a sibling production test at a
    configuration the bf16 step also produces, or launches nothing."""
    called = runs.split_keys.keys
    print("\nentry points called in split mode: %s" % ", ".join(sorted(called)))
    sibling = set(R.ARG_MAPS) | set(R.GEMM_REPLAYED) | {k for k in R.EXCLUDED if k not in LAUNCH_NOTHING}
    missing, split_only = [], []
    for fn, keys in sorted(called.items()):
        if fn in REPLAYED_HERE or fn in LAUNCH_NOTHING or fn in SHARED_ROW:
            continue
        if fn not in sibling:
            missing.append(fn)
        elif not keys <= runs.bf16_keys.keys.get(fn, set()):
            split_only.append("%s (%d configurations)" % (fn, len(keys - runs.bf16_keys.keys.get(fn, set()))))
    assert not missing, "entry points of the split runs no production replay covers: %s" % missing
    assert not split_only, "shared entry points with configurations only the split runs produce: %s" % split_only
    recorded = {c["fn"] for c in runs.rows.configs}
    assert recorded >= set(SPLIT_MAPS), sorted(set(SPLIT_MAPS) - recorded)
    assert all(c["pieces"] == Fn.PIECES for c in runs.rows.configs if c["fn"] in PIECE_FNS)
    assert all(c["pieces"] == Fn.PIECES for c in runs.gemm.groups)


# ------------------------------------------------------------------------------------------------- self-checks
def _largest_seg(runs, want=lambda c: True):
    cands = [c for c in runs.gemm.configs if c["kind"] == "igemm" and c["segs"] and not c["overlap"] and want(c)]
    assert cands
    return max(cands, key=lambda c: c["M"] * c["taps"] * c["cin"])


def test_self_check_segment_comparison_catches_dropped_swapped_and_shifted_pieces(runs):
    """On the largest split GEMM (and the largest whose A pieces are adjacent), the exact comparison fails when the
    reference drops one segment, swaps (ap, wp) of one segment, or reads A at a_lo_off + 64; it still passes with
    the segments reversed (exact integers: the order of the sum does not matter)."""
    gen = torch.Generator(device="cuda").manual_seed(55)
    for c in {id(c): c for c in (_largest_seg(runs), _largest_seg(runs, lambda c: c["a_lo_off"] == c["cin"]))}.values():
        bad, o, _ = G._replay(c, runs.gemm.table_list, gen)
        assert not bad, bad
        stats, red = G._launch_gemm(c, o)
        segs = list(c["segs"])
        i = next(j for j, (a, w) in enumerate(segs) if a != w)
        swapped = segs[:i] + [(segs[i][1], segs[i][0])] + segs[i + 1:]
        cases = [("segment %s dropped" % (segs[-1],), dict(segs=segs[:-1])),
                 ("segment %s swapped to %s" % (segs[i], swapped[i]), dict(segs=swapped)),
                 ("a_lo_off + 64", dict(a_lo_off=c["a_lo_off"] + 64))]
        for what, kw in cases:
            found = G._compare_gemm(c, o, stats, red, G._gemm_reference(c, o, **kw))
            print("%s (%s) with %s: %s" % (c["tag"], _seg_desc(c), what, found))
            assert found, "%s: a reference with %s goes unnoticed" % (c["tag"], what)
        assert not G._compare_gemm(c, o, stats, red, G._gemm_reference(c, o, segs=segs[::-1]))
        del o


def test_self_check_group_comparison_catches_an_overwriting_launch(runs):
    c = max(runs.gemm.groups, key=lambda c: c["M"] * c["taps"])
    gen = torch.Generator(device="cuda").manual_seed(56)
    bad, o, ref = _replay_group(c, runs.gemm.table_list, gen)
    assert not bad, bad
    dW = _launch_group(c, o, overwrite_last=True)
    print("%s, last launch overwriting dW: %d entries differ" % (_group_label(c), int((dW != ref).sum())))
    assert not torch.equal(dW, ref), "a group whose last launch overwrites dW goes unnoticed"


def test_self_check_reduce_comparison_catches_a_missing_partial_block(runs):
    c = max(_of(runs, "pnx_bn_bwd_reduce_split"), key=lambda c: c["M"] * c["C"])
    _, nb, _ = _reduce_grid(c["M"], c["C"])
    d = _red_data(c["M"], c["C"], True)
    with _pieces(3):
        red, ok = _launch_reduce_split(c, d, _mode(c), 3, False)
        assert ok and torch.equal(red, _reduce_ref(d, _mode(c), 3)[0])
        for blk in (0, nb // 2, nb - 1):
            dropped = _reduce_ref(d, _mode(c), 3, drop_block=blk)[0]
            print("reduce M %d C %d without block %d of %d: %d sums differ" % (c["M"], c["C"], blk, nb, int((red != dropped).sum())))
            assert not torch.equal(red, dropped), "a missing partial block goes unnoticed"


def test_self_check_row_replay_catches_a_piece_offset_off_by_8(runs):
    """rows_split at its recorded layout, its pieces read back at lo + 8: the bit-exact comparison fails."""
    c = _smallest(runs, "pnx_rows_split")
    M, C = c["M"], c["C"]
    x = _gauss(M, C, 5)
    ref = [p.bfloat16() for p in split_ref(x, 3)]
    with _pieces(3):
        xb, xv = R._place(x, R._ld(c["ldx"], C, 0))
        ldy, lo = _layout(c["ldy"], c["lo_y"], C, 3, False, 0)
        yb = R._sentinel_buf(M, ldy, torch.bfloat16)
        _check(L().pnx_rows_split(R._p(xv), xv.stride(0), M, C, R._p(yb), ldy, lo, ops.stream()))
        assert all(_same_bits(g, r) for g, r in zip(_get(yb, M, C, lo, 3), ref))
        shifted = [G.piece(yb[:M], q * (lo + 8), C) for q in range(3)]       # the guard rows keep it in the storage
        assert not all(_same_bits(g, r) for g, r in zip(shifted, ref)), "pieces read at lo + 8 go unnoticed"


def _smallest(runs, fn, want=lambda c: True):
    return min([c for c in _of(runs, fn) if want(c)], key=lambda c: c.get("M", 0) * c.get("C", 1) or c.get("B", 1) * c.get("H", 1))


NAN_CASES = [      # (kernel output overwritten with one NaN, its replay, failure messages the replay must report)
    ("rows_split y", lambda r: _replay_rows_split(_smallest(r, "pnx_rows_split")), ("differs from the bit-level split",)),
    ("round trip", lambda r: _replay_rows_split(_smallest(r, "pnx_rows_split")), ("is not x",)),
    ("rows_merge y", lambda r: _replay_rows_merge(_smallest(r, "pnx_rows_merge")), ("differ from the fp32 emulation",)),
    ("add_relu_split y", lambda r: _replay_add_relu_split(_smallest(r, "pnx_add_relu_split")), ("differ from the fp32",)),
    ("relu_bwd_split g", lambda r: _replay_relu_bwd_split(_smallest(r, "pnx_relu_bwd_split")), ("differ from the fp32",)),
    ("tap_scatter dZ", lambda r: _replay_tap_scatter(_smallest(r, "pnx_tap_scatter", lambda c: c["lo_off"] > 0)),
     ("dZ pieces differ",)),
    ("bn_apply_split y", lambda r: _replay_bn_apply_split(_smallest(r, "pnx_bn_apply_split")), ("merged y off by",)),
    ("reduce_split red", lambda r: _replay_reduce_split(_smallest(r, "pnx_bn_bwd_reduce_split"), (0,)),
     ("integer sums differ", "Gaussian sums off by")),
    ("bwd_apply_split dx", lambda r: _replay_bwd_apply_split(_smallest(r, "pnx_bn_bwd_apply_split"), (0,)), ("dx off by",)),
    ("bwd_apply_split dres", lambda r: _replay_bwd_apply_split(_smallest(r, "pnx_bn_bwd_apply_split", lambda c: c["dres"]),
                                                                (0,)), ("dres differs",)),
    ("wgrad_split dW", lambda r: _replay_group(min(r.gemm.groups, key=lambda c: c["M"] * c["taps"]), r.gemm.table_list,
                                               torch.Generator(device="cuda").manual_seed(3)), ("dW differs",)),
]


@pytest.mark.parametrize("name,replay,expect", NAN_CASES, ids=[c[0] for c in NAN_CASES])
def test_self_check_a_nan_in_a_kernel_output_fails_its_comparison(runs, name, replay, expect):
    POISON.add(name)
    try:
        bad = replay(runs)[0]
    finally:
        POISON.discard(name)
    print("%s: %s" % (name, bad))
    for e in expect:
        assert any(e in b for b in bad), "%s: no failure mentioning %r in %s" % (name, e, bad)


def test_self_check_a_nan_in_a_gemm_output_fails_its_comparison(runs):
    c = min([c for c in runs.gemm.configs if c["kind"] == "igemm" and c["segs"] and not c["overlap"]],
            key=lambda c: c["M"] * c["cout"])
    gen = torch.Generator(device="cuda").manual_seed(57)
    o = G._gemm_operands(c, gen, runs.gemm.table_list)
    ref = G._gemm_reference(c, o)
    stats, red = G._launch_gemm(c, o)
    assert not G._compare_gemm(c, o, stats, red, ref)
    o.out[o.rows - 1, o.n_st - 1] = float("nan")
    found = G._compare_gemm(c, o, stats, red, ref)
    print("%s with one NaN output: %s" % (c["tag"], found))
    assert found and "outputs differ" in found[0]


def test_wall_time_and_peak_memory(runs):
    """Reports the file's wall time and peak memory (the last test of the file)."""
    print("\ntest_production_split_gpu: %.1f s so far, peak %.2f GB after the recording; split steps peaked at %s" % (
        time.perf_counter() - runs.t0, torch.cuda.max_memory_allocated() / 2 ** 30,
        ", ".join("%s %.2f GB" % (k, v / 2 ** 30) for k, v in runs.peaks.items())))
