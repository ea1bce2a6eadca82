"""The evaluation path's decode, rotated NMS and double-flip merge (CenterHead.predict -> ops.det_postprocess:
pnx_det_keys, pnx_det_nms, pnx_det_gather and their _flip4 twins) at the configurations the bench runs, against a
float64 decode and against the reference's own GPU NMS.

Recording: the bench model of `nusc` (6 frames, 336^2 maps, 6 tasks, pre_max 1000, post_max 83) and of `waymo180k`
(3 frames, 376^2 maps, `iou` head and rectifier, pre_max 4096, post_max 500, thresholds 0.7 / 0.2, 0.25) runs the eval
forward plus predict, once plain and once with double flip (24 and 12 frames of head output), in two head regimes:
- init: the head as initialised (hm bias -2.19): many pixels near the 0.1 score threshold, every segment past pre_max,
  ~1 m boxes on 0.3 m cells (long suppression chains);
- confident: the final hm conv scaled, plus windows pushed past logit 17, where 1 + expf(-x) rounds to 1 and every score
  is exactly 1.0f (tied scores).
ops.det_postprocess is wrapped with pytest's MonkeyPatch and keeps each task's head output, arguments and results.  The
configs are recorded one after another and each model is freed before the next.

What is compared (the entry points are called again through ops.lib() on the recorded outputs, into the test's own
buffers prefilled with NaN / -1 sentinels):
- keys: labels, validity, score bits and per-segment counts against a float64 decode of every pixel, within error bounds
  derived from the fp32 arithmetic (u = 2^-24; expf 2 ulp, atan2f 3 ulp, powf 4 ulp: the CUDA maths library's bounds);
- order: the stable sort of the keys (segment, descending score, ties by ascending pixel index);
- candidate boxes: pnx_det_gather with an identity keep list (exactly the boxes the mask kernel decodes) against the
  float64 decode;
- NMS decisions: each segment's candidates, in the product's order, through the reference's nms_gpu
  (oracle/build_ref_nms.py: det3d/core/iou3d_nms/src/iou3d_nms_kernel.cu compiled for sm_90a by build()) with the
  class's own threshold: the keep lists must be equal;
- a synthetic head output at the production shape, ld and column offsets whose segments hold >= 500 candidate pairs
  with a reference IoU within 2 ulp of the threshold (some exactly on it);
- det_postprocess's outputs and predict's per-frame dicts against the kept candidates, bit for bit;
- the double-flip inputs (flip4_points, the voxelizer on the 4B-frame batch) bit for bit;
- eval_match / eval_match_center at 4096 boxes in one frame (the opt-in shared-memory path) against their host twins."""
import math
import time
import types

import numpy as np
import pytest
import torch

from oracle import build_ref_nms
from oracle import pillarnext_oracle as O
from pillarnext_b200 import _lib, modules, ops, synth
from pillarnext_b200 import functional as Fn

pytestmark = pytest.mark.gpu

CONFIGS = ("nusc", "waymo180k")
REGIMES = ("init", "confident")
U = 2.0 ** -24
INVALID_KEY = 0x7FFFFFFFFFFFFFFF
TIE_LOGIT = 20.0          # past 16.6: 1 + expf(-x) rounds to 1 and the score is exactly 1.0f
SLACK = 1.01              # on every derived bound: the float64 reference's own rounding

# Entry points of the eval path, and the test here that checks each one.
COVERED = {
    **dict.fromkeys(("pnx_det_keys", "pnx_det_keys_flip4"), "test_keys_and_order_match_float64_decode"),
    **dict.fromkeys(("pnx_det_nms", "pnx_det_nms_flip4"),
                    "test_nms_decisions_equal_reference_nms_gpu, test_threshold_segments_equal_reference_nms_gpu"),
    **dict.fromkeys(("pnx_det_gather", "pnx_det_gather_flip4"),
                    "test_candidate_boxes_match_float64_decode, test_outputs_are_the_kept_candidates"),
    "pnx_flip4_points": "test_double_flip_inputs_bit_exact",
    "pnx_voxelize": "test_double_flip_inputs_bit_exact (4B-frame batch, not frame-sorted)",
}


def _ref_nms():
    m = build_ref_nms.load(build=False)
    assert m is not None, ("oracle/_ref/ref_iou3d_nms.so is missing: run __graft_entry__.build() on a machine with the "
                           "reference tree (oracle/build_ref_nms.py compiles the reference's GPU NMS into it)")
    return m


# ------------------------------------------------------------------------------------------------- recording
def _push_windows(out, nF, H, W, offs, C, flip, seed):
    """Two 6 x 6 windows per frame (class w % C) pushed to TIE_LOGIT (iou head 1.0): every score in them is 1.0f.  With
    double flip each copy gets the window at its mirrored position, so the merged score is exactly 1.0f as well."""
    v = out.view(nF, H, W, out.shape[1])
    g = np.random.default_rng(seed)
    copies = 4 if flip else 1
    for f in range(nF // copies):
        for w in range(2):
            y0, x0, c = int(g.integers(20, H - 26)), int(g.integers(20, W - 26)), w % C
            for k in range(copies):
                ys = slice(H - y0 - 6, H - y0) if k & 1 else slice(y0, y0 + 6)
                xs = slice(W - x0 - 6, W - x0) if k & 2 else slice(x0, x0 + 6)
                v[copies * f + k, ys, xs, offs[5] + c] = TIE_LOGIT
                if offs[6] >= 0:
                    v[copies * f + k, ys, xs, offs[6]] = 1.0


class Recorder:
    def __init__(self, real):
        self.real, self.called, self.calls, self.run = real, set(), [], None

    def proxy(self):
        rec = self

        class Proxy:
            def __getattr__(self, name):
                if name.startswith("pnx_"):
                    rec.called.add(name)
                return getattr(rec.real, name)
        return Proxy()


def _wrappers(rec):
    real = {n: getattr(ops, n) for n in ("det_postprocess", "flip4_points", "voxelize")}

    def det_postprocess(out, B, H, W, C, offs, osf, voxel_size, pc_range, score_thr, post_center_range, rectifier,
                        nms_thr, pre_max, post_max, label_offset=0, double_flip=False):
        r = rec.run
        if r.regime == "confident":
            _push_windows(out, out.shape[0] // (H * W), H, W, offs, C, double_flip, 100 + len(r.calls))
        res = real["det_postprocess"](out, B, H, W, C, offs, osf, voxel_size, pc_range, score_thr, post_center_range,
                                      rectifier, nms_thr, pre_max, post_max, label_offset=label_offset,
                                      double_flip=double_flip)
        r.calls.append(types.SimpleNamespace(
            name=r.name, regime=r.regime, t=len(r.calls), out=out.detach().clone(), B=B, H=H, W=W, C=C, offs=list(offs),
            osf=osf, vs=list(voxel_size), pr=list(pc_range), score_thr=score_thr, pcr=list(post_center_range),
            rect=list(rectifier), nms_thr=list(nms_thr), pre_max=pre_max, post_max=post_max, label_offset=label_offset,
            flip=double_flip, res=[x.detach().clone() for x in res]))
        return res

    def flip4_points(points):
        out = real["flip4_points"](points)
        rec.run.flip_points = (points.detach().clone(), out.detach().clone())
        return out

    def voxelize(*a, **kw):
        v = real["voxelize"](*a, **kw)
        if rec.run.flip and rec.run.vox is None:
            rec.run.vox = (a, kw, v)
        return v
    return dict(det_postprocess=det_postprocess, flip4_points=flip4_points, voxelize=voxelize)


def _record(rec, name, dev):
    sel = synth.BENCH_CONFIGS[name]
    cfg = sel["cfg"]
    seeds = list(range(cfg["frames_per_gpu"]))
    ex = synth.make_batch(seeds, sel["points"], cfg, kind="lidar", n_boxes=40, sweeps=sel["sweeps"], rings=sel["rings"],
                          with_labels=False)
    ex = {"points": ex["points"].to(dev), "token": ["%s_%d" % (name, s) for s in seeds]}
    torch.manual_seed(0)
    model = modules.build_pillarnext_b(cfg).to(dev).eval()
    runs = []
    for regime in REGIMES:
        if regime == "confident":
            with torch.no_grad():
                for task in model.head.tasks:            # spread the heat-map logits: many confident peaks
                    task.hm[3].bias.fill_(-1.5)
                    task.hm[3].weight.mul_(6.0)
        for flip in (False, True):
            r = types.SimpleNamespace(name=name, cfg=cfg, regime=regime, flip=flip, calls=[], flip_points=None, vox=None,
                                      tokens=ex["token"])
            rec.run = r
            model.post_processing = dict(cfg["post_processing"], double_flip=flip)
            with torch.no_grad():
                r.dets = model(ex)
            torch.cuda.synchronize()
            runs.append(r)
    del model, ex
    torch.cuda.empty_cache()
    return runs


T0 = {}


@pytest.fixture(scope="module")
def recorded():
    T0["t"] = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    ref = _ref_nms()
    dev = "cuda:%d" % torch.cuda.current_device()
    rec = Recorder(_lib.lib())
    prev = Fn.set_precision("bf16"), ops.set_deterministic(False)      # the production eval forward
    runs = []
    with pytest.MonkeyPatch.context() as mp:
        proxy = rec.proxy()
        mp.setattr(_lib, "lib", lambda: proxy)
        mp.setattr(ops, "lib", lambda: proxy)
        for n, f in _wrappers(rec).items():
            mp.setattr(ops, n, f)
        try:
            for name in CONFIGS:
                runs += _record(rec, name, dev)
                print("\n%s: recorded, peak %.2f GB" % (name, torch.cuda.max_memory_allocated() / 2 ** 30))
        finally:
            Fn.set_precision(prev[0])
            ops.set_deterministic(prev[1])
    return types.SimpleNamespace(runs=runs, called=rec.called, ref=ref, cache={})


def _label(c):
    return "%s %s%s task %d" % (c.name, c.regime, " flip" if c.flip else "", c.t)


def _calls(recorded):
    return [c for r in recorded.runs for c in r.calls]


# ------------------------------------------------------------------------------------------------- replay
class Replay:
    """The three entry points of one recorded call, into fresh sentinel-filled buffers."""

    def __init__(self, c):
        self.c = c
        self.hold, params = ops._decode_params(c.offs, c.osf, c.vs, c.pr, c.score_thr, c.pcr, c.rect)
        self.common = (ops.ptr(c.out), c.out.stride(0), c.B, c.H, c.W, c.C) + params
        L = ops.lib()
        self.fk, self.fn, self.fg = ((L.pnx_det_keys_flip4, L.pnx_det_nms_flip4, L.pnx_det_gather_flip4) if c.flip else
                                     (L.pnx_det_keys, L.pnx_det_nms, L.pnx_det_gather))
        self.M, self.nseg = c.B * c.H * c.W, c.B * c.C

    def keys(self):
        dev = self.c.out.device
        keys = torch.full((self.M,), -1, dtype=torch.int64, device=dev)
        seg_count = torch.full((self.nseg,), -1, dtype=torch.int32, device=dev)
        ops.check(self.fk(*self.common, ops.ptr(keys), ops.ptr(seg_count), ops.stream()))
        return keys, seg_count

    def nms(self, order, seg_start, seg_count, pre_max, post_max, thr):
        dev = self.c.out.device
        nt, ntp = ops._host_floats(thr, 8)
        mask = torch.empty(self.nseg * pre_max * ((pre_max + 63) // 64), dtype=torch.int64, device=dev)
        keep = torch.full((self.nseg, post_max), -1, dtype=torch.int32, device=dev)
        keep_count = torch.full((self.nseg,), -1, dtype=torch.int32, device=dev)
        ops.check(self.fn(*self.common, ntp, ops.ptr(order), ops.ptr(seg_start), ops.ptr(seg_count), int(pre_max),
                          int(post_max), ops.ptr(mask), ops.ptr(keep), ops.ptr(keep_count), ops.stream()))
        return keep, keep_count

    def gather(self, order, seg_start, keep, keep_count, post_max, label_offset=0):
        dev = self.c.out.device
        box = torch.full((self.nseg, post_max, 9), float("nan"), device=dev)
        score = torch.full((self.nseg, post_max), float("nan"), device=dev)
        label = torch.full((self.nseg, post_max), -1, dtype=torch.int64, device=dev)
        ops.check(self.fg(*self.common, ops.ptr(order), ops.ptr(seg_start), ops.ptr(keep), ops.ptr(keep_count),
                          int(post_max), int(label_offset), ops.ptr(box), ops.ptr(score), ops.ptr(label), ops.stream()))
        return box, score, label


def _order(keys, seg_count):
    """What ops.det_postprocess does between the keys and the NMS."""
    order = torch.sort(keys, stable=True)[1]
    seg_start = (torch.cumsum(seg_count, 0, dtype=torch.int32) - seg_count).contiguous()
    return order, seg_start


def _identity(c, seg_count):
    """keep[s, k] = k for k < min(n, pre_max): the gather then returns exactly the candidates the mask kernel decodes."""
    n = torch.clamp(seg_count, max=c.pre_max)
    keep = torch.arange(c.pre_max, dtype=torch.int32, device=n.device).repeat(len(n), 1).contiguous()
    return keep, n.to(torch.int32).contiguous()


def _state(recorded, c):
    """Keys, order and identity-gathered candidates of a recorded call (cached)."""
    key = id(c)
    if key not in recorded.cache:
        rp = Replay(c)
        keys, seg_count = rp.keys()
        order, seg_start = _order(keys, seg_count)
        keep, n = _identity(c, seg_count)
        cand = rp.gather(order, seg_start, keep, n, c.pre_max)
        torch.cuda.synchronize()
        recorded.cache[key] = types.SimpleNamespace(rp=rp, keys=keys, seg_count=seg_count, order=order,
                                                    seg_start=seg_start, n=n, cand=cand)
    return recorded.cache[key]


# ------------------------------------------------------------------------------------------------- float64 decode
def _merge(vals, errs):
    """float64 value of det_merge4 ((v0 + v1) + (v2 + v3)) * 0.25 and the bound of its fp32 error given the errors of
    the four inputs: three rounded additions, the 0.25 is exact."""
    s01, s23 = vals[0] + vals[1], vals[2] + vals[3]
    tot = s01 + s23
    bound = 0.25 * (errs[0] + errs[1] + errs[2] + errs[3] + U * (s01.abs() + s23.abs() + tot.abs()))
    return 0.25 * tot, bound


def _sigmoid(l):
    """float64 sigmoid of fp32 logits and the bound of 1 / (1 + expf(-l)) in fp32: expf within 2 ulp (<= 4u e), the
    addition and the division rounded once each."""
    l = l.double()
    e = torch.exp(-l.clamp(min=-80.0))
    s = 1.0 / (1.0 + e)
    return s, s * (4.0 * U * e / (1.0 + e) + 2.0 * U)


def _decode64(recorded, c):
    """float64 decode of every output pixel of a recorded call, with the bound of each fp32 quantity (cached)."""
    key = ("d64", id(c))
    if key in recorded.cache:
        return recorded.cache[key]
    o, B, H, W, C = c.offs, c.B, c.H, c.W, c.C
    X = c.out
    dev = X.device
    M = B * H * W
    m = torch.arange(M, device=dev)
    b, rem = m // (H * W), m % (H * W)
    y, x = rem // W, rem % W
    zero = torch.zeros(M, dtype=torch.float64, device=dev)
    if c.flip:
        rows = []
        for k in range(4):
            yk = H - 1 - y if k & 1 else y
            xk = W - 1 - x if k & 2 else x
            rows.append(X[((4 * b + k) * H + yk) * W + xk])

        def col(j, sign_bit=0, one_minus=False):
            vals, errs = [], []
            for k in range(4):
                v = rows[k][:, j].double()
                flipped = bool(k & sign_bit)
                if flipped and one_minus:
                    v = 1.0 - v
                    errs.append(U * v.abs())
                else:
                    if flipped:
                        v = -v
                    errs.append(zero)
                vals.append(v)
            return _merge(vals, errs)
        sig, sig_b = [], []
        for cl in range(C):
            pairs = [_sigmoid(rows[k][:, o[5] + cl]) for k in range(4)]
            v, e = _merge([p[0] for p in pairs], [p[1] for p in pairs])
            sig.append(v)
            sig_b.append(e)
        sig, sig_b = torch.stack(sig, 1), torch.stack(sig_b, 1)
        rx, rx_b = col(o[0], 2, True)
        ry, ry_b = col(o[0] + 1, 1, True)
        z, z_b = col(o[1])
        iou_raw, iou_b = col(o[6]) if o[6] >= 0 else (zero, zero)
        dims, dims_b = [], []
        for d in range(3):
            ex = [torch.exp(rows[k][:, o[2] + d].double()) for k in range(4)]
            v, e = _merge(ex, [4.0 * U * t for t in ex])
            dims.append(v)
            dims_b.append(e)
        vx, vx_b = col(o[4], 2)
        vy, vy_b = col(o[4] + 1, 1)
        sn, sn_b = col(o[3], 1)
        cs, cs_b = col(o[3] + 1, 2)
    else:
        r = X
        sig, sig_b = _sigmoid(r[:, o[5]:o[5] + C])
        rx, ry, z = r[:, o[0]].double(), r[:, o[0] + 1].double(), r[:, o[1]].double()
        rx_b = ry_b = z_b = zero
        iou_raw, iou_b = (r[:, o[6]].double(), zero) if o[6] >= 0 else (zero, zero)
        dims = [torch.exp(r[:, o[2] + d].double()) for d in range(3)]
        dims_b = [4.0 * U * t for t in dims]
        vx, vy, vx_b, vy_b = r[:, o[4]].double(), r[:, o[4] + 1].double(), zero, zero
        sn, cs, sn_b, cs_b = r[:, o[3]].double(), r[:, o[3] + 1].double(), zero, zero
    f32 = lambda v: float(np.float32(v))  # noqa: E731  (the values the kernel receives)
    osf, vsx, vsy, pcx, pcy = f32(c.osf), f32(c.vs[0]), f32(c.vs[1]), f32(c.pr[0]), f32(c.pr[1])
    ax, ay = x.double() + rx, y.double() + ry
    xs, ys = ax * osf * vsx + pcx, ay * osf * vsy + pcy
    # x + reg, * osf, * voxel size, + pc_range: four rounded fp32 operations after the merged input's own error
    xs_b = SLACK * (rx_b * osf * vsx + U * (3.0 * (ax * osf * vsx).abs() + xs.abs()))
    ys_b = SLACK * (ry_b * osf * vsy + U * (3.0 * (ay * osf * vsy).abs() + ys.abs()))
    # score: rectified per class; powf within 4 ulp (8u relative) twice, (iou + 1) * 0.5 and the product rounded once
    rect = torch.tensor([f32(v) for v in c.rect], dtype=torch.float64, device=dev)
    iou = ((iou_raw + 1.0) * 0.5).clamp(0.0, 1.0)[:, None]
    score = torch.where(rect != 0, sig.pow(1.0 - rect) * iou.pow(rect), sig)
    score_b = torch.where(rect != 0, score * ((1.0 - rect) * sig_b / sig.clamp(min=1e-300) + rect * iou_b[:, None]
                                              / iou.clamp(min=1e-300) + 19.0 * U), sig_b) * SLACK
    yaw = torch.atan2(sn, cs)
    yaw_b = SLACK * ((cs.abs() * sn_b + sn.abs() * cs_b) / (sn * sn + cs * cs).clamp(min=1e-300) + 6.0 * U * yaw.abs())
    d = types.SimpleNamespace(sig=sig, sig_b=sig_b * SLACK, score=score, score_b=score_b, b=b,
                              box=torch.stack([xs, ys, z] + dims + [vx, vy, yaw], 1),
                              box_b=torch.stack([xs_b, ys_b, z_b * SLACK] + [t * SLACK for t in dims_b] +
                                                [vx_b * SLACK, vy_b * SLACK, yaw_b], 1),
                              sn=sn, sn_b=sn_b, cs=cs)
    # label: first maximum of the fp32 logits (plain; exact) or of the merged fp32 sigmoids (flip; near ties reported)
    d.label = c.out[:, o[5]:o[5] + C].argmax(1) if not c.flip else sig.argmax(1)
    thr = f32(c.score_thr)
    rng = [f32(v) for v in c.pcr]
    s_top = sig.gather(1, d.label[:, None])[:, 0]
    s_top_b = d.sig_b.gather(1, d.label[:, None])[:, 0]
    inside = ((xs >= rng[0]) & (ys >= rng[1]) & (z >= rng[2]) & (xs <= rng[3]) & (ys <= rng[4]) & (z <= rng[5]))
    d.valid = (s_top > thr) & inside
    near = (s_top - thr).abs() <= s_top_b
    for v, vb, lo, hi in ((xs, xs_b, rng[0], rng[3]), (ys, ys_b, rng[1], rng[4]), (z, z_b * SLACK, rng[2], rng[5])):
        near |= ((v - lo).abs() <= vb) | ((v - hi).abs() <= vb)
    d.ambiguous = near
    recorded.cache[key] = d
    return d


def _key_fields(keys):
    valid = keys != INVALID_KEY
    seg = torch.where(valid, keys >> 32, torch.full_like(keys, -1))
    bits = (0xFFFFFFFF - (keys & 0xFFFFFFFF)).to(torch.int32)
    return valid, seg, bits.view(torch.float32)


def _worst(t):
    return t.double().nan_to_num(nan=float("inf")).max().item() if t.numel() else 0.0


def _keys_fails(c, d, keys, seg_count):
    bad, C, nseg = [], c.C, c.B * c.C
    valid, seg, score = _key_fields(keys)
    if bool((keys == -1).any()):
        bad.append("a key was not written")
    amb = d.ambiguous
    wrong = (valid != d.valid) & ~amb
    if bool(wrong.any()):
        bad.append("%d pixels valid / invalid against float64 away from a bound" % int(wrong.sum()))
    lab = seg - d.b * C
    if bool(((lab < 0) | (lab >= C))[valid].any()):
        bad.append("a key's segment is not its frame's")
    lab = lab.clamp(0, C - 1)
    both = valid & d.valid
    ties = 0
    if not c.flip:
        if not torch.equal(lab[both], d.label[both]):
            bad.append("label differs from the first maximum of the fp32 logits")
    else:
        top = d.sig.max(1)[0]
        mine = d.sig.gather(1, lab[:, None])[:, 0]
        slack = d.sig_b.gather(1, lab[:, None])[:, 0] + d.sig_b.max(1)[0]
        far = both & (mine < top - slack)
        if bool(far.any()):
            bad.append("%d labels are not a (near-)first maximum of the merged sigmoids" % int(far.sum()))
        ties = int((both & (lab != d.label)).sum())
    ref = d.score.gather(1, lab[:, None])[:, 0]
    bnd = d.score_b.gather(1, lab[:, None])[:, 0]
    ratio = _worst(((score.double() - ref).abs() / bnd.clamp(min=1e-300))[valid])
    if ratio > 1.0:
        bad.append("score %.3g x its bound from float64" % ratio)
    want = torch.bincount(seg[valid], minlength=nseg)
    if not torch.equal(seg_count.long(), want):
        bad.append("seg_count differs from the number of valid keys")
    return bad, dict(ambiguous=int(amb.sum()), ambiguous_disagree=int(((valid != d.valid) & amb).sum()),
                     flip_near_ties=ties, score_ratio=ratio)


def _order_fails(keys, order, seg_start, seg_count):
    """Sorted keys ascending (segment, then descending score); equal keys in ascending pixel order; seg_start the
    exclusive prefix of seg_count; every segment's run holds its own keys."""
    bad = []
    sk = keys[order]
    if bool((sk[1:] < sk[:-1]).any()):
        bad.append("keys are not ascending in the order")
    eq = sk[1:] == sk[:-1]
    if bool((order[1:][eq] <= order[:-1][eq]).any()):
        bad.append("tied keys are not in ascending pixel order")
    if not torch.equal(seg_start.long(), torch.cumsum(seg_count.long(), 0) - seg_count.long()):
        bad.append("seg_start is not the exclusive prefix of seg_count")
    nv = int(seg_count.sum())
    seg = sk[:nv] >> 32
    want = torch.repeat_interleave(torch.arange(len(seg_count), device=keys.device), seg_count.long())
    if not torch.equal(seg, want) or bool((sk[nv:] != INVALID_KEY).any()):
        bad.append("a segment's run holds keys of another segment")
    veq = eq[:max(nv - 1, 0)]
    starts = veq & ~torch.cat([torch.zeros(1, dtype=torch.bool, device=keys.device), veq[:-1]])
    return bad, int(starts.sum())


def _tied_group(keys, order, n_valid):
    """(start, end) positions of the largest run of equal valid keys in the order."""
    sk = keys[order][:n_valid]
    eq = torch.cat([torch.zeros(1, dtype=torch.bool, device=sk.device), sk[1:] == sk[:-1]]).cpu().numpy()
    best, start, cur = (0, 0), 0, 0
    for i, e in enumerate(eq):
        if not e:
            start = i
        if i - start + 1 > best[1] - best[0]:
            best = (start, i + 1)
    return best


# ------------------------------------------------------------------------------------------------- keys and order
def test_keys_and_order_match_float64_decode(recorded):
    """Every pixel's key against the float64 decode (labels exact, validity away from the bounds, score bits within
    their derived bound, segment counts exact); the stable order; the tie rule."""
    failures = []
    for c in _calls(recorded):
        st = _state(recorded, c)
        d = _decode64(recorded, c)
        bad, info = _keys_fails(c, d, st.keys, st.seg_count)
        obad, groups = _order_fails(st.keys, st.order, st.seg_start, st.seg_count)
        failures += ["%s: %s" % (_label(c), b) for b in bad + obad]
        print("\n%s: %d segments, %d valid keys (max segment %d), %d tied groups, %d pixels within a bound of the score "
              "threshold / range (%d decided the other way), %d near-tie flip labels, worst score %.3f of its bound" % (
                  _label(c), c.B * c.C, int(st.seg_count.sum()), int(st.seg_count.max()), groups, info["ambiguous"],
                  info["ambiguous_disagree"], info["flip_near_ties"], info["score_ratio"]), end="")
    confident = [c for c in _calls(recorded) if c.regime == "confident"]
    assert any(_order_fails(_state(recorded, c).keys, _state(recorded, c).order, _state(recorded, c).seg_start,
                            _state(recorded, c).seg_count)[1] > 0 for c in confident), "no tied scores recorded"
    assert all(int(_state(recorded, c).seg_count.max()) > c.pre_max for c in _calls(recorded)
               if c.regime == "init" and c.name == "nusc"), "the init regime no longer saturates pre_max"
    assert not failures, "\n".join(failures)


def test_self_check_order_comparison_catches_a_reversed_tied_group(recorded):
    c = next(c for c in _calls(recorded) if c.regime == "confident" and c.name == "nusc" and not c.flip)
    st = _state(recorded, c)
    assert not _order_fails(st.keys, st.order, st.seg_start, st.seg_count)[0]
    a, b = _tied_group(st.keys, st.order, int(st.seg_count.sum()))
    assert b - a > 1, "no tied group"
    order = st.order.clone()
    order[a:b] = order[a:b].flip(0)
    bad, _ = _order_fails(st.keys, order, st.seg_start, st.seg_count)
    assert any("tied keys" in x for x in bad), bad


# ------------------------------------------------------------------------------------------------- candidates
def _gather_fails(c, d, st, drop=None):
    """Identity-gathered candidates against the float64 decode of their pixels; rows past n keep the sentinel.
    drop=k: the reference skips candidate k of every segment with more than pre_max valid keys (self-check)."""
    bad = []
    box, score, label = st.cand
    n = st.n.long()
    nseg = len(n)
    dev = box.device
    sid = torch.repeat_interleave(torch.arange(nseg, device=dev), n)
    k = torch.arange(int(n.sum()), device=dev) - torch.repeat_interleave(torch.cumsum(n, 0) - n, n)
    pos = st.seg_start.long()[sid] + k
    if drop is not None:
        pos = pos + ((k >= drop) & (st.seg_count.long()[sid] > c.pre_max)).long()
    m = st.order[pos]
    got = box[sid, k].double()
    want, bnd = d.box[m], d.box_b[m]
    err = (got - want).abs()
    wrap = (d.sn[m].abs() <= d.sn_b[m]) & (d.cs[m] < 0)      # flip: the merged sin may round across 0 at yaw = +-pi
    err[:, 8] = torch.where(wrap, torch.minimum(err[:, 8], (err[:, 8] - 2 * math.pi).abs()), err[:, 8])
    ratio = err / bnd.clamp(min=1e-300)
    worst = _worst(ratio)
    if worst > 1.0:
        col = int(ratio.nan_to_num(nan=float("inf")).max(0)[0].argmax())
        bad.append("candidate box column %d is %.3g x its bound from float64" % (col, worst))
    lab = label[sid, k]
    valid, seg, kscore = _key_fields(st.keys[m])
    if not torch.equal(lab, seg - d.b[m] * c.C):
        bad.append("candidate label differs from its key's")
    if not torch.equal(score[sid, k].view(torch.int32), kscore.view(torch.int32)):
        bad.append("candidate score differs from its key's score bits")
    tail = torch.arange(box.shape[1], device=dev)[None, :] >= n[:, None]
    if not bool(box[tail].isnan().all()) or not bool((label[tail] == -1).all()):
        bad.append("rows past min(n, pre_max) were written")
    return bad, worst


def test_candidate_boxes_match_float64_decode(recorded):
    """pnx_det_gather with an identity keep list: the boxes the mask kernel decodes, within bounds derived from the
    arithmetic (three rounded operations for the centre, expf for the sizes, atan2f for the yaw, the merge for flip)."""
    failures, lines = [], []
    for c in _calls(recorded):
        bad, worst = _gather_fails(c, _decode64(recorded, c), _state(recorded, c))
        failures += ["%s: %s" % (_label(c), b) for b in bad]
        lines.append("%s: %d candidates, worst box error %.3f of its bound" % (_label(c), int(_state(recorded, c).n.sum()),
                                                                               worst))
    print("\n" + "\n".join(lines))
    assert not failures, "\n".join(failures)


def test_self_check_gather_comparison_catches_a_dropped_last_candidate(recorded):
    """The reference skipping candidate pre_max - 1 = 999, the last one of the partial 64-candidate block."""
    c = next(c for c in _calls(recorded) if c.regime == "init" and c.name == "nusc" and not c.flip)
    assert c.pre_max == 1000
    st = _state(recorded, c)
    d = _decode64(recorded, c)
    assert not _gather_fails(c, d, st)[0]
    bad, _ = _gather_fails(c, d, st, drop=999)
    assert any("bound from float64" in b for b in bad), bad


# ------------------------------------------------------------------------------------------------- NMS decisions
def _near_pairs(ref, b7, thr, ulps, chunk=1024):
    """Pairs i < j whose reference IoU (boxes_iou_bev_gpu) lies within `ulps` ulp of thr; and exactly on it."""
    n = len(b7)
    spacing = float(np.spacing(np.float32(thr)))
    near = exact = 0
    for i0 in range(0, n, chunk):
        i1 = min(n, i0 + chunk)
        iou = torch.zeros(i1 - i0, n, device=b7.device)
        ref.boxes_iou_bev_gpu(b7[i0:i1].contiguous(), b7, iou)
        upper = torch.arange(n, device=b7.device)[None, :] > torch.arange(i0, i1, device=b7.device)[:, None]
        dv = (iou.double() - float(np.float32(thr))).abs()
        near += int(((dv <= ulps * spacing) & upper).sum())
        exact += int(((dv == 0) & upper).sum())
    return near, exact


def _nms_fails(ref, c, st, thr_of=None, count_near=True):
    """The product's keep lists against the reference's nms_gpu on the same candidates in the same order."""
    bad = []
    keep, kc = st.rp.nms(st.order, st.seg_start, st.seg_count, c.pre_max, c.post_max, c.nms_thr)
    keep, kc = keep.cpu(), kc.cpu()
    box = st.cand[0]
    n = st.n.cpu()
    stats = dict(segments=len(n), candidates=int(n.sum()), suppressed=0, near=0, exact=0)
    for s in range(len(n)):
        ns = int(n[s])
        thr = float(np.float32(c.nms_thr[s % c.C] if thr_of is None else thr_of(s)))
        b7 = box[s, :ns][:, [0, 1, 2, 3, 4, 5, 8]].contiguous()
        rk = torch.zeros(ns, dtype=torch.int64)
        nk = ref.nms_gpu(b7, rk, thr) if ns else 0
        rk = rk[:nk]
        stats["suppressed"] += ns - nk
        want = min(nk, c.post_max)
        if int(kc[s]) != want:
            bad.append("segment %d: keep_count %d, reference %d (of %d kept)" % (s, int(kc[s]), want, nk))
        elif not torch.equal(keep[s, :want].long(), rk[:want]):
            j = int((keep[s, :want].long() != rk[:want]).nonzero()[0])
            bad.append("segment %d: keep lists differ first at position %d (%d vs reference %d)" % (
                s, j, int(keep[s, j]), int(rk[j])))
        if not bool((keep[s, max(int(kc[s]), 0):] == -1).all()):
            bad.append("segment %d: keep entries past keep_count were written" % s)
        if count_near and ns > 1:
            near, exact = _near_pairs(ref, b7, thr, 4)
            stats["near"] += near
            stats["exact"] += exact
    return bad, stats


def test_nms_decisions_equal_reference_nms_gpu(recorded):
    """Each segment's candidates, in the product's order, through the reference's nms_gpu with the class's threshold:
    pnx_det_nms keeps exactly ref_keep[:post_max]."""
    failures = []
    for c in _calls(recorded):
        bad, s = _nms_fails(recorded.ref, c, _state(recorded, c))
        failures += ["%s: %s" % (_label(c), b) for b in bad]
        print("\n%s: %d segments, %d candidates, %d suppressed, %d pairs within 4 ulp of the threshold (%d on it)" % (
            _label(c), s["segments"], s["candidates"], s["suppressed"], s["near"], s["exact"]), end="")
    assert not failures, "\n".join(failures[:40])


# ------------------------------------------------------------------------------------------------- threshold segments
NEIGHBOURS = ((-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 1), (1, -1), (1, 0), (1, 1))
A_SIZE, B_WIDTH = 5.0, 2.0


def _host_centre(pix, reg, osf, vs, pc):
    """The decode's centre, fp32 operation by fp32 operation (the device pins each rounding)."""
    f = np.float32
    return f(f(f(f(pix) + f(reg)) * f(osf)) * f(vs)) + f(pc)


def _threshold_head(c, per_seg):
    """A head output with c's shape, ld and column offsets holding groups of one large box A (5 m) and eight boxes B
    inside it on the neighbouring pixels.  IoU(A, B) = area(B) / area(A) up to rounding, so each B's width is walked
    through consecutive fp32 values (the host twin judging) to put the IoU within a few ulp of the class's threshold,
    on both sides of it.  Everything else is below the score threshold.  -> (head [B*H*W, ld] cuda, #groups)."""
    B, H, W, C, o = c.B, c.H, c.W, c.C, c.offs
    ld = c.out.stride(0)
    f = np.float32
    X = np.zeros((B, H, W, ld), np.float32)
    X[..., o[5]:o[5] + C] = -20.0
    if o[6] >= 0:
        X[..., o[6]] = 1.0
    cell = float(f(c.osf) * f(c.vs[0]))
    step = int(math.ceil(12.0 / cell))
    slots = [(yy, xx) for yy in range(step // 2, H - 2, step) for xx in range(step // 2, W - 2, step)]
    assert len(slots) >= C * per_seg, (len(slots), C, per_seg)
    la, lb = f(math.log(A_SIZE)), f(math.log(B_WIDTH))
    dA, dB = f(np.exp(la)), f(np.exp(lb))
    reg = (f(0.37), f(0.61))
    pa, pb = [], []
    meta = []
    for b in range(B):
        for cl in range(C):
            thr = f(c.nms_thr[cl])
            for g in range(per_seg):
                yy, xx = slots[cl * per_seg + g]
                th = f(0.3 + 0.037 * g + 0.5 * b)
                ya = [_host_centre(xx, reg[0], c.osf, c.vs[0], c.pr[0]), _host_centre(yy, reg[1], c.osf, c.vs[1], c.pr[1])]
                boxA = np.array(ya + [0.5, dA, dA, 1.7, np.arctan2(f(np.sin(th)), f(np.cos(th)))], np.float32)
                dstar = float(thr) * float(dA) * float(dA) / float(dB)
                widths = [f(dstar)]
                for _ in range(8):
                    widths = [np.nextafter(widths[0], f(0))] + widths + [np.nextafter(widths[-1], f(10))]
                for j, (dy, dx) in enumerate(NEIGHBOURS):
                    thb = f(th + 0.05)
                    cen = [_host_centre(xx + dx, reg[0], c.osf, c.vs[0], c.pr[0]),
                           _host_centre(yy + dy, reg[1], c.osf, c.vs[1], c.pr[1])]
                    for w in widths:
                        lw = f(math.log(float(w)))
                        pa.append(boxA)
                        pb.append(np.array(cen + [0.5, f(np.exp(lw)), dB, 1.7, np.arctan2(f(np.sin(thb)), f(np.cos(thb)))],
                                           np.float32))
                        meta.append((b, cl, g, j, lw, thr, yy + dy, xx + dx, thb))
                X[b, yy, xx] = 0.0
                _put(X[b, yy, xx], o, C, reg, la, la, th, cl, 6.0 - 0.02 * g)
    iou = ops.det_iou_bev_host(np.stack(pa), np.stack(pb))
    nw = 17
    for q in range(0, len(meta), nw):                      # per B: the width whose host IoU is nearest its target
        b, cl, g, j, _, thr, py, px, thb = meta[q]
        target = float(thr) + (j % 5 - 2) * float(np.spacing(thr))
        best = q + int(np.argmin(np.abs(iou[q:q + nw].astype(np.float64) - target)))
        _put(X[b, py, px], o, C, reg, meta[best][4], lb, thb, cl, 6.0 - 0.02 * g - 0.002 * (j + 1))
    return torch.from_numpy(X.reshape(B * H * W, ld)), B * C * per_seg


def _put(row, o, C, reg, lx, ly, th, cl, logit):
    row[o[0]], row[o[0] + 1] = reg
    row[o[1]] = 0.5
    row[o[2]], row[o[2] + 1], row[o[2] + 2] = lx, ly, np.float32(math.log(1.7))
    row[o[3]], row[o[3] + 1] = np.sin(th), np.cos(th)
    row[o[4]], row[o[4] + 1] = 0.0, 0.0
    row[o[5]:o[5] + C] = -20.0
    row[o[5] + cl] = logit
    if o[6] >= 0:
        row[o[6]] = 1.0


def _threshold_cases(recorded):
    key = "thr_cases"
    if key not in recorded.cache:
        cases = []
        for name, per_seg in (("nusc", 30), ("waymo180k", 60)):
            src = next(c for c in _calls(recorded) if c.name == name and c.regime == "init" and not c.flip and c.t == 1)
            out, groups = _threshold_head(src, per_seg)
            c = types.SimpleNamespace(**{**vars(src), "out": out.cuda(), "regime": "threshold", "res": None})
            st = _state(recorded, c)
            cases.append((c, st, groups))
        recorded.cache[key] = cases
    return recorded.cache[key]


def test_threshold_segments_equal_reference_nms_gpu(recorded):
    """Segments built to sit on the threshold, at the production shape: nuScenes task 1 (6 x 336^2, 0.2) and Waymo
    task 1 (376^2, 0.2 and 0.25): at least 500 candidate pairs with a reference GPU IoU within 2 ulp of the threshold,
    some exactly on it; the product's decisions equal nms_gpu's."""
    failures = []
    for c, st, groups in _threshold_cases(recorded):
        assert torch.equal(st.n.cpu(), torch.full((c.B * c.C,), groups // (c.B * c.C) * 9, dtype=torch.int32)), st.n
        bad, _ = _gather_fails(c, _decode64(recorded, c), st)
        failures += ["%s threshold: %s" % (c.name, b) for b in bad]
        bad, s = _nms_fails(recorded.ref, c, st, count_near=False)
        failures += ["%s threshold: %s" % (c.name, b) for b in bad]
        near = exact = 0
        for seg in range(c.B * c.C):
            b7 = st.cand[0][seg, :int(st.n[seg])][:, [0, 1, 2, 3, 4, 5, 8]].contiguous()
            nr, ex = _near_pairs(recorded.ref, b7, c.nms_thr[seg % c.C], 2)
            near, exact = near + nr, exact + ex
        print("\n%s threshold segments: %d segments, %d candidates, %d suppressed, %d pairs within 2 ulp of the "
              "threshold, %d exactly on it" % (c.name, s["segments"], s["candidates"], s["suppressed"], near, exact), end="")
        assert near >= 500 and exact > 0, (c.name, near, exact)
    assert not failures, "\n".join(failures[:40])


def test_self_check_threshold_moved_by_one_ulp_flips_a_decision(recorded):
    for c, st, _ in _threshold_cases(recorded):
        assert not _nms_fails(recorded.ref, c, st, count_near=False)[0]
        flipped = 0
        for to in (0.0, 1.0):
            bad, _ = _nms_fails(recorded.ref, c, st, count_near=False,
                                thr_of=lambda s: np.nextafter(np.float32(c.nms_thr[s % c.C]), np.float32(to)))
            flipped += len(bad)
        assert flipped > 0, "%s: moving the reference threshold by one ulp changed no decision" % c.name


def test_self_check_other_class_threshold_fails(recorded):
    """Waymo task 1 has thresholds 0.2 and 0.25: the reference run with the other class's threshold must disagree."""
    c, st, _ = next(x for x in _threshold_cases(recorded) if x[0].name == "waymo180k")
    assert c.nms_thr[0] != c.nms_thr[1]
    bad, _ = _nms_fails(recorded.ref, c, st, count_near=False, thr_of=lambda s: c.nms_thr[(s + 1) % c.C])
    assert bad, "the reference with swapped class thresholds agreed with the product"


# ------------------------------------------------------------------------------------------------- outputs
def test_outputs_are_the_kept_candidates(recorded):
    """det_postprocess's det_box / det_score / det_label are the identity-gather rows at the kept positions, bit for
    bit, with label_offset applied; predict's per-frame dicts are the per-task results in task and class order."""
    failures = []
    for r in recorded.runs:
        per_frame = [([], [], []) for _ in r.tokens]
        for c in r.calls:
            st = _state(recorded, c)
            keep, kc = st.rp.nms(st.order, st.seg_start, st.seg_count, c.pre_max, c.post_max, c.nms_thr)
            det_box, det_score, det_label, count = c.res
            if not torch.equal(count, kc):
                failures.append("%s: keep_count differs from the replay" % _label(c))
                continue
            for s in range(c.B * c.C):
                k = int(kc[s])
                pos = keep[s, :k].long()
                ok = (torch.equal(det_box[s, :k].view(torch.int32), st.cand[0][s, pos].view(torch.int32)) and
                      torch.equal(det_score[s, :k].view(torch.int32), st.cand[1][s, pos].view(torch.int32)) and
                      torch.equal(det_label[s, :k], st.cand[2][s, pos] + c.label_offset))
                if not ok:
                    failures.append("%s: segment %d outputs are not the kept candidates" % (_label(c), s))
                f = s // c.C
                per_frame[f][0].append(det_box[s, :k])
                per_frame[f][1].append(det_score[s, :k])
                per_frame[f][2].append(det_label[s, :k])
        for f, tok in enumerate(r.tokens):
            got = r.dets[tok]
            want = [torch.cat(x).cpu() for x in per_frame[f]]
            if not (torch.equal(got["box3d_lidar"].view(torch.int32), want[0].view(torch.int32)) and
                    torch.equal(got["scores"].view(torch.int32), want[1].view(torch.int32)) and
                    torch.equal(got["label_preds"], want[2])):
                failures.append("%s %s%s: predict's dict for %s is not the per-task results in order" % (
                    r.name, r.regime, " flip" if r.flip else "", tok))
    assert not failures, "\n".join(failures[:40])


# ------------------------------------------------------------------------------------------------- double-flip inputs
def test_double_flip_inputs_bit_exact(recorded):
    """flip4_points at the bench point counts against torch, and the voxelizer on the 4B-frame, not frame-sorted flip
    batch against the oracle."""
    from test_production_frontend_gpu import _vox_fails
    done = set()
    for r in recorded.runs:
        if not r.flip or r.name in done:
            continue
        done.add(r.name)
        pin, pout = r.flip_points
        want = []
        for k in range(4):
            q = pin.clone()
            q[:, 0] = 4 * pin[:, 0] + k
            if k & 1:
                q[:, 2] = -q[:, 2]
            if k & 2:
                q[:, 1] = -q[:, 1]
            want.append(q)
        assert torch.equal(pout.view(torch.int32), torch.cat(want).view(torch.int32)), "%s: flip4_points" % r.name
        a, kw, v = r.vox
        assert not kw.get("frame_sorted", False)
        assert torch.equal(v.points, pout), "%s: the voxelizer did not get the flip batch" % r.name
        bad, _ = _vox_fails(v, O.voxelize(pout.cpu(), r.cfg["voxel_size"], r.cfg["pc_range"]))
        print("\n%s: flip batch of %d points, %d frames" % (r.name, pout.shape[0], 4 * len(r.tokens)), end="")
        assert not bad, "%s: %s" % (r.name, bad)
    assert done == set(CONFIGS)


# ------------------------------------------------------------------------------------------------- metric kernels
def _crowded_frame(g, M, n_det):
    """M ground-truth boxes of one class on a jittered lattice and n_det detections near some of them (duplicates
    included), scores with ties."""
    side = int(math.ceil(math.sqrt(M)))
    iy, ix = np.divmod(np.arange(M), side)
    gt = np.zeros((M, 9), np.float32)
    gt[:, 0] = (ix - side / 2) * 2.6 + g.normal(0, 0.2, M)
    gt[:, 1] = (iy - side / 2) * 2.6 + g.normal(0, 0.2, M)
    gt[:, 2] = g.normal(0, 0.3, M)
    gt[:, 3:6] = g.uniform(1.0, 2.4, (M, 3))
    gt[:, 8] = g.uniform(-math.pi, math.pi, M)
    src = g.integers(0, M, n_det)
    det = gt[src].copy()
    det[:, :3] += g.normal(0, 0.15, (n_det, 3)).astype(np.float32)
    det[:, 3:6] *= g.uniform(0.9, 1.1, (n_det, 3)).astype(np.float32)
    det[:, 8] += g.normal(0, 0.1, n_det).astype(np.float32)
    score = np.round(g.uniform(0, 1, n_det), 3).astype(np.float32)
    return gt, det, score


def test_eval_match_at_the_shared_memory_limit():
    """eval_match with 4096 boxes in one frame (kMaxBoxesPerFrame: 4096 x 53 B = 217,088 B of dynamic shared memory,
    the opt-in path above 48 KB) and eval_match_center with 4096 boxes and 8 thresholds (81,920 B), bit for bit
    against their host twins."""
    g = np.random.default_rng(17)
    M, B, C = 4096, 2, 1
    gts, dets, scores, frames = [], [], [], []
    for f, (m, nd) in enumerate(((M, 6000), (1500, 2000))):
        gt, det, sc = _crowded_frame(g, m, nd)
        gts.append(np.concatenate([gt, np.zeros((M - m, 9), np.float32)]))
        dets.append(det)
        scores.append(sc)
        frames.append(np.full(nd, f))
    gt_boxes = np.stack(gts)
    gt_classes = np.stack([np.where(np.arange(M) < m, 0, -1) for m in (M, 1500)]).astype(np.int32)
    gt_trig = np.stack([np.cos(gt_boxes[..., 8]), np.sin(gt_boxes[..., 8])], -1).astype(np.float32)
    det_boxes = np.concatenate(dets)
    det_trig = np.stack([np.cos(det_boxes[:, 8]), np.sin(det_boxes[:, 8])], -1).astype(np.float32)
    score, frame = np.concatenate(scores), np.concatenate(frames)
    order = np.lexsort((np.arange(len(score)), -score, frame)).astype(np.int64)
    seg_count = np.bincount(frame, minlength=B * C).astype(np.int32)
    seg_start = (np.cumsum(seg_count) - seg_count).astype(np.int32)
    thr = np.array([0.5], np.float32)
    host = ops.eval_match_host(det_boxes, det_trig, order, seg_start, seg_count, gt_boxes, gt_classes, gt_trig, thr)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    dev = ops.eval_match(cu(det_boxes), cu(det_trig), cu(order), cu(seg_start), cu(seg_count), cu(gt_boxes),
                         cu(gt_classes), cu(gt_trig), cu(thr))
    for name, h, d in zip(("match", "iou", "heading"), host, dev):
        d = d.cpu().numpy()
        assert np.array_equal(h.view(np.int32), d.view(np.int32)), "eval_match %s: %d of %d differ" % (
            name, int((h.view(np.int32) != d.view(np.int32)).sum()), len(h))
    assert (host[0] >= 0).sum() > 3000 and (host[0][frame == 0] >= 0).sum() > 2000
    ths = np.array([0.25, 0.5, 1.0, 2.0, 0.1, 0.75, 1.5, 4.0])
    host_c = ops.eval_match_center_host(det_boxes, order, seg_start, seg_count, gt_boxes, gt_classes, C, ths)
    dev_c = ops.eval_match_center(cu(det_boxes), cu(order), cu(seg_start), cu(seg_count), cu(gt_boxes), cu(gt_classes),
                                  C, cu(ths)).cpu().numpy()
    assert np.array_equal(host_c, dev_c), "eval_match_center: %s of %d differ per threshold" % (
        (host_c != dev_c).sum(1), host_c.shape[1])
    assert ((host_c >= 0).sum(1) > 1000).all()
    print("\neval_match: %d detections, %d matched in the 4096-box frame; eval_match_center matches per threshold %s" % (
        len(order), int((host[0][frame == 0] >= 0).sum()), (host_c >= 0).sum(1)))


# ------------------------------------------------------------------------------------------------- completeness
def test_every_eval_entry_point_is_covered(recorded):
    """Every pnx_* entry point the recorded eval forwards called is covered here or by a sibling production test."""
    from test_production_frontend_gpu import COVERED as FRONT, NO_LAUNCH
    from test_production_rowwise_gpu import ARG_MAPS, EXCLUDED, GEMM_REPLAYED
    called = recorded.called
    print("\nentry points called: %s" % ", ".join(sorted(called)))
    missing = sorted(n for n in called if n not in COVERED and n not in FRONT and n not in NO_LAUNCH and
                     n not in ARG_MAPS and n not in GEMM_REPLAYED and n not in EXCLUDED)
    assert not missing, "entry points the eval forward calls that no production test covers: %s" % missing
    assert set(COVERED) <= called, sorted(set(COVERED) - called)
    p = torch.cuda.get_device_properties(torch.cuda.current_device())
    print("wall time of the file so far %.1f s, peak GPU memory %.2f GB, on %s" % (
        time.perf_counter() - T0["t"], torch.cuda.max_memory_allocated() / 2 ** 30, p.name))
