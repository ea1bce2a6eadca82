"""fp32-grade ("split") precision mode vs the fp32 oracle -- the north-star tolerance test.

BASELINE.json north_star: "boxes/heatmaps matching the reference within 1e-3 abs on identical inputs (voxel indices
bit-exact)".  The reference is fp32 end to end; the production path stores bf16 activations and cannot meet 1e-3
through 35 conv+BN layers.  In `precision("split")` every activation is a (hi, lo) bf16 pair and the SAME wgmma
kernels (pnx_igemm / pnx_wgrad over the (piece, piece) segments of 3-piece operands) run, so the assembled detector is
compared here with the fp32 oracle at the stated tolerance: forward maps 1e-3 abs, parameter gradients 2e-3 rel-L2
(fp32 summation-order level), and the bf16 path's measured error is printed next to it.
"""
import json
import os

import pytest
import torch

from oracle import pillarnext_oracle as O
from oracle.weights import randomize_state_dict
from pillarnext_b200 import functional as Fn
from pillarnext_b200 import modules, ops, synth

pytestmark = pytest.mark.gpu
TASKS = [["car"], ["truck", "construction_vehicle"]]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def maxabs(a, b):
    return (a.detach().float().cpu() - b.detach().float().cpu()).abs().max().item()


def to_cuda(ex):
    return {k: ([e.cuda() for e in v] if isinstance(v, list) and torch.is_tensor(v[0]) else (v.cuda() if torch.is_tensor(v) else v))
            for k, v in ex.items()}


def report_to_file(name, lines):
    d = os.path.join(ROOT, "gpurun_out")
    if os.path.isdir(d):
        with open(os.path.join(d, name), "w") as fh:
            fh.write("\n".join(lines) + "\n")


# ------------------------------------------------------------------------------------------- kernel level
@pytest.fixture
def pieces(request):
    prev = ops.split_pieces()
    ops.split_pieces(request.param)
    yield request.param
    ops.split_pieces(prev)


@pytest.mark.parametrize("pieces", [2, 3], indirect=True)
@pytest.mark.parametrize("M,taps,cin,cout", [(3000, 9, 64, 64), (5000, 9, 128, 256), (4096, 1, 256, 192), (2500, 4, 64, 128)])
def test_igemm_split_matches_fp64(M, taps, cin, cout, pieces):
    """pnx_igemm over the (piece, piece) segments of 2- / 3-piece operands vs a float64 gather-GEMM of the SAME fp32
    numbers: 2 pieces ~2^-18 relative (16-bit mantissas), 3 pieces = exact fp32 operands, only the tensor core's
    truncating fp32 accumulation is left (~1e-9 per K element, tools/split_error_probe.py)."""
    g = torch.Generator(device="cuda").manual_seed(M + taps)
    a = torch.randn(M, cin, device="cuda", generator=g)
    w = torch.randn(taps, cout, cin, device="cuda", generator=g) * 0.1
    nbr = torch.randint(-1, M, (M, taps), device="cuda", generator=g, dtype=torch.int32)
    if taps == 1:
        nbr = None
    A = ops.rows_split(a)
    assert A.shape == (M, pieces * cin)
    back = ops.rows_merge(A, cin, cin)
    if pieces == 3:
        assert torch.equal(back, a)                        # three bf16 pieces hold all 24 mantissa bits
    else:
        assert (back - a).abs().max().item() <= 2.0 ** -16 * a.abs().max().item()
    out = torch.empty(M, cout, dtype=torch.float32, device="cuda")
    stats = torch.zeros(2 * cout, dtype=torch.float64, device="cuda")
    ops.igemm(A, M, Fn._to_hilo(w), taps, cin, cout, out, nbr=nbr, stats=stats, stats_mod=cout, segs=ops.split_segments(), a_lo_off=cin)
    ref = torch.zeros(M, cout, dtype=torch.float64, device="cuda")
    for t in range(taps):
        if nbr is None:
            src = a.double()
        else:
            idx = nbr[:, t].long()
            src = torch.where((idx >= 0).unsqueeze(1), a.double()[idx.clamp(min=0)], torch.zeros((), dtype=torch.float64, device="cuda"))
        ref += src @ w[t].double().t()
    e = rel(out, ref)
    print("igemm split pieces=%d M%d T%d K%d N%d: rel-L2 vs fp64 %.2e" % (pieces, M, taps, cin, cout, e))
    assert e < (6e-6 if pieces == 2 else 2e-6), e
    assert rel(stats[:cout], ref.sum(0)) < 1e-4 and rel(stats[cout:], (ref * ref).sum(0)) < 1e-4
    # the bf16 production kernel on the same numbers, for scale (8-bit mantissas)
    out16 = torch.empty(M, cout, dtype=torch.float32, device="cuda")
    ops.igemm(a.bfloat16(), M, w.bfloat16().contiguous(), taps, cin, cout, out16, nbr=nbr)
    assert rel(out16, ref) > 20 * e


@pytest.mark.parametrize("pieces", [2, 3], indirect=True)
def test_wgrad_split_matches_fp64(pieces):
    M, taps, cx, cy = 6000, 9, 128, 64
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(M, cx, device="cuda", generator=g)
    y = torch.randn(M, cy, device="cuda", generator=g)
    nbr = torch.randint(-1, M, (M, taps), device="cuda", generator=g, dtype=torch.int32)
    dW = torch.zeros(taps, cx, cy, dtype=torch.float32, device="cuda")
    ops.wgrad_split(ops.rows_split(x), cx, cx, ops.rows_split(y), cy, cy, M, taps, dW, nbr=nbr)
    ref = torch.zeros(taps, cx, cy, dtype=torch.float64, device="cuda")
    for t in range(taps):
        idx = nbr[:, t].long()
        src = torch.where((idx >= 0).unsqueeze(1), y.double()[idx.clamp(min=0)], torch.zeros((), dtype=torch.float64, device="cuda"))
        ref[t] = x.double().t() @ src
    print("wgrad split: rel-L2 vs fp64 %.2e" % rel(dW, ref))
    assert rel(dW, ref) < 1e-5


def test_split_ops_forward_backward_vs_fp64():
    """Every differentiable building block in split mode, forward AND backward, against torch float64 autograd of the
    same op on the same fp32 numbers (conv + BatchNorm + ReLU, residual BatchNorm, the head's final conv as GEMM +
    stencil, ConvTranspose2d, the fp32 gradient fan-out): 5e-6 relative -- the backward arithmetic itself is exact
    to fp32 level; what remains in the assembled test is the ReLU-gate discontinuity."""
    import torch.nn.functional as F
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    TOL = 5e-6

    def leaf(x32):
        return ops.rows_split(x32.contiguous()).requires_grad_()

    def mgrad(s, C):
        return ops.rows_merge(s.grad.contiguous(), C, C)

    def nchw(rows, B, H, W, C):
        return rows.double().view(B, H, W, C).permute(0, 3, 1, 2)

    def to_rows(x, C):
        return x.permute(0, 2, 3, 1).reshape(-1, C)

    B, H, W = 2, 24, 20
    M = B * H * W
    g = torch.Generator(device="cuda").manual_seed(0)
    with Fn.precision("split"):
        # dense 3x3 conv + BN + ReLU
        cin, cout = 64, 128
        x = torch.randn(M, cin, device="cuda", generator=g)
        w = (torch.randn(cout, cin, 3, 3, device="cuda", generator=g) * 0.05).requires_grad_()
        bn = torch.nn.BatchNorm2d(cout).cuda().train()
        R = torch.randn(M, cout, device="cuda", generator=g)
        xs = leaf(x)
        raw, stats = Fn.conv(xs, w, None, Fn.dense_spec(B, H, W, 3), Fn.WLayout("dense"), want_stats=True)
        ym = Fn.MergeFn.apply(Fn.bn_act(raw, stats, bn, relu=True))
        (ym * R).sum().backward()
        xd = nchw(x, B, H, W, cin).requires_grad_()
        wd = w.detach().double().requires_grad_()
        bnd = torch.nn.BatchNorm2d(cout).cuda().double().train()
        yd = F.relu(bnd(F.conv2d(xd, wd, padding=1)))
        (yd * nchw(R, B, H, W, cout)).sum().backward()
        for name, a, b in (("y", ym, to_rows(yd, cout)), ("dx", mgrad(xs, cin), to_rows(xd.grad, cin)), ("dw", w.grad, wd.grad),
                           ("dgamma", bn.weight.grad, bnd.weight.grad), ("dbeta", bn.bias.grad, bnd.bias.grad)):
            assert rel(a, b) < TOL, ("conv+bn+relu", name, rel(a, b))
        # BatchNorm1d + residual + ReLU
        C = 64
        xr, res, R2 = (torch.randn(M, C, device="cuda", generator=g) for _ in range(3))
        bn1 = torch.nn.BatchNorm1d(C).cuda().train()
        raw_l, rs = xr.clone().requires_grad_(), leaf(res)
        st = torch.cat([xr.double().sum(0), (xr.double() ** 2).sum(0)])
        y = Fn.MergeFn.apply(Fn.bn_act(raw_l, st, bn1, relu=True, residual=rs))
        (y * R2).sum().backward()
        bn1d = torch.nn.BatchNorm1d(C).cuda().double().train()
        rawd, resd = xr.double().requires_grad_(), res.double().requires_grad_()
        yd = F.relu(bn1d(rawd) + resd)
        (yd * R2.double()).sum().backward()
        for name, a, b in (("y", y, yd), ("draw", raw_l.grad, rawd.grad), ("dres", mgrad(rs, C), resd.grad),
                           ("dgamma", bn1.weight.grad, bn1d.weight.grad), ("dbeta", bn1.bias.grad, bn1d.bias.grad)):
            assert rel(a, b) < TOL, ("bn+res+relu", name, rel(a, b))
        # the head's final conv: 1x1 GEMM + 9-point stencil; 16 outputs (9*16 = 144 GEMM columns in 192) and the reference's
        # 11 (cpt = 12: 108 columns in 128)
        for n_used in (16, 11):
            cin = 384
            yh = torch.randn(M, cin, device="cuda", generator=g)
            wb0 = torch.randn(16, cin, 3, 3, device="cuda", generator=g) * 0.05
            wb0[n_used:] = 0
            wb = wb0.requires_grad_()
            bb = torch.randn(16, device="cuda", generator=g).requires_grad_()
            R3 = torch.randn(M, 16, device="cuda", generator=g)
            R3[:, n_used:] = 0
            ys = leaf(yh)
            out = Fn.HeadFinalConvFn.apply(ys, wb, bb, B, H, W, None, n_used)
            (out * R3).sum().backward()
            yd = nchw(yh, B, H, W, cin).requires_grad_()
            wbd, bbd = wb.detach().double().requires_grad_(), bb.detach().double().requires_grad_()
            od = F.conv2d(yd, wbd, bbd, padding=1)
            (od * nchw(R3, B, H, W, 16)).sum().backward()
            for name, a, b in (("out", out[:, :n_used], to_rows(od, 16)[:, :n_used]), ("dy", mgrad(ys, cin), to_rows(yd.grad, cin)),
                               ("dw", wb.grad, wbd.grad), ("db", bb.grad[:n_used], bbd.grad[:n_used])):
                assert rel(a, b) < TOL, ("head final conv", n_used, name, rel(a, b))
        # ConvTranspose2d k2 s2 (pixel-shuffle store), BatchNorm statistics of the fp32 output
        cin = cout = 64
        xt = torch.randn(M, cin, device="cuda", generator=g)
        wt = (torch.randn(cin, cout, 2, 2, device="cuda", generator=g) * 0.1).requires_grad_()
        R4 = torch.randn(4 * M, cout, device="cuda", generator=g)
        xs = leaf(xt)
        raw, stats = Fn.conv(xs, wt, None, Fn.convT_spec(B, H, W), Fn.WLayout("convT"), want_stats=True)
        (raw * R4).sum().backward()
        xd, wtd = nchw(xt, B, H, W, cin).requires_grad_(), wt.detach().double().requires_grad_()
        rd = F.conv_transpose2d(xd, wtd, stride=2)
        (rd * nchw(R4, B, 2 * H, 2 * W, cout)).sum().backward()
        for name, a, b in (("raw", raw, to_rows(rd, cout)), ("dx", mgrad(xs, cin), to_rows(xd.grad, cin)), ("dw", wt.grad, wtd.grad),
                           ("stats", stats[:cout], rd.sum((0, 2, 3)))):
            assert rel(a, b) < TOL, ("convT", name, rel(a, b))
        # fp32 gradient accumulation of a split activation with two consumers
        a = torch.randn(M, 64, device="cuda", generator=g)
        s = leaf(a)
        u, v = Fn.fanout(s)
        G1, G2 = torch.randn(M, 64, device="cuda", generator=g), torch.randn(M, 64, device="cuda", generator=g)
        ((Fn.MergeFn.apply(u) * G1).sum() + (Fn.MergeFn.apply(v) * G2).sum()).backward()
        assert torch.equal(mgrad(s, 64), G1 + G2)


# ------------------------------------------------------------------------------------------- assembled detector
def build(cfg, seed=3):
    model = modules.build_pillarnext_b(cfg)
    sd = randomize_state_dict(model.state_dict(), seed)
    model.load_state_dict(sd, strict=True)
    return model.cuda(), sd


def surrogate_weights(t, k, shape):
    g = torch.Generator().manual_seed(1000 * t + sum(ord(c) for c in k))
    return torch.randn(tuple(shape), generator=g)


def run_oracle(cfg, sd, ex, B, with_grads=True):
    p = {k: v.clone().requires_grad_(with_grads and v.dtype.is_floating_point and "running" not in k) for k, v in sd.items()}
    st = {}
    feat, coords, grid = O.reader_forward(ex["points"], p, cfg["voxel_size"], cfg["pc_range"], train=True, stats=st)
    f4, c4, shp = O.sparse_resnet_gather(feat, coords, grid, B, p, cfg["strides"], stats=st)
    bb = O.densify(f4, c4, shp)
    neck = O.aspp_forward(bb, p, train=True, stats=st)
    preds = O.centerhead_forward(neck, p, cfg["tasks"], cfg["common_heads"], train=True, stats=st)
    out = dict(p=p, st=st, feat=feat, coords=coords, bb=bb, neck=neck, preds=preds)
    if with_grads:
        sur = sum((v * surrogate_weights(t, k, v.shape)).sum() for t, pd in enumerate(preds) for k, v in pd.items())
        sur.backward(retain_graph=True)
        out["gsur"] = {k: v.grad.clone() for k, v in p.items() if v.grad is not None}
        for v in p.values():
            v.grad = None
        loss, rets = O.center_loss(ex, [dict(pd) for pd in preds], cfg["weight"], cfg["code_weights"], True, cfg["voxel_size"],
                                   cfg["pc_range"], cfg["out_size_factor"])
        loss.backward()
        out["loss"], out["rets"] = loss, rets
    return out


def forward_stages(model, exg, B):
    model.reader.batch_size = B
    x = model.reader(exg["points"])
    bb = model.backbone(*x)
    nk = model.neck(bb)
    preds = model.head(nk)
    return x, bb, nk, preds


@pytest.mark.parametrize("grid,npts,kind", [(128, 3000, "uniform"), (256, 4000, "lidar")])
def test_detector_split_mode_meets_north_star_tolerance(grid, npts, kind):
    cfg = synth.tiny_config(grid, TASKS)
    model, sd = build(cfg)
    model.train()
    B = 2
    ex = synth.make_batch([0, 1], npts, cfg, kind=kind, n_boxes=25, sweeps=10)
    exg = to_cuda(ex)
    of = run_oracle(cfg, sd, ex, B)
    lines = []
    with Fn.precision("split"):
        x, bb, nk, preds = forward_stages(model, exg, B)
        assert torch.equal(x[1].cpu(), of["coords"])                               # voxel indices bit-exact
        assert bb.dtype == torch.float32 and tuple(bb.shape) == tuple(of["bb"].shape)
        lines.append("backbone  max|d| %.2e rel %.2e" % (maxabs(bb, of["bb"]), rel(bb, of["bb"])))
        lines.append("neck      max|d| %.2e rel %.2e" % (maxabs(nk, of["neck"]), rel(nk, of["neck"])))
        worst = 0.0
        for t in range(len(cfg["tasks"])):
            for k in preds[t]:
                a, b = preds[t][k], of["preds"][t][k]
                d = maxabs(a, b)
                if k == "hm":
                    d_sig = maxabs(torch.sigmoid(a), torch.sigmoid(b))
                    lines.append("head %d/hm   logits max|d| %.2e  sigmoid max|d| %.2e" % (t, d, d_sig))
                else:
                    lines.append("head %d/%-6s max|d| %.2e" % (t, k, d))
                worst = max(worst, d)
        print("\n".join(lines))
        assert maxabs(bb, of["bb"]) < 1e-3 and maxabs(nk, of["neck"]) < 1e-3, "\n".join(lines)
        assert worst < 1e-3, "\n".join(lines)                                      # every head map, logits included
        # ---- backward, linear surrogate (same fixed d/dpred on both sides)
        sur = sum((v * surrogate_weights(t, k, v.shape).cuda()).sum() for t, pd in enumerate(preds) for k, v in pd.items())
        sur.backward(retain_graph=True)
        errs = []
        for k, v in model.named_parameters():
            assert v.grad is not None and torch.isfinite(v.grad).all(), k
            if k.endswith(".0.bias") and ("shared_conv" in k or ".tasks." in k):
                continue     # conv bias in front of a BatchNorm: exact gradient is zero
            errs.append((rel(v.grad, of["gsur"][k]), k))
        errs.sort(reverse=True)
        lines += ["surrogate grad rel-L2 %.2e %s" % e for e in errs[:8]]
        med = sorted(e for e, _ in errs)[len(errs) // 2]
        lines.append("surrogate grad rel-L2: median %.2e worst %.2e over %d parameters" % (med, errs[0][0], len(errs)))
        # The gradient of a ReLU network is DISCONTINUOUS in the activations: a forward difference eps flips the gate of
        # a fraction ~eps of the units (those with |pre-activation| < eps), and k flips among N units move the gradient
        # by ~sqrt(k/N) = sqrt(eps) relative.  eps ~ 5e-6 here -> ~2e-3 expected (two true-fp32 implementations would
        # see ~1e-3; the bf16 path, eps ~ 3e-2, sees ~0.2).  Each backward op alone is exact to 1e-6 on identical
        # inputs: test_split_ops_forward_backward_vs_fp64.
        assert med < 8e-3 and errs[0][0] < 8e-2, "\n".join(lines)    # worst = one small-norm BatchNorm bias, typically 2e-2
        model.zero_grad()
        # ---- the real loss (fused libpnx loss kernel on fp32 head outputs)
        loss, rets = model.head.loss(exg, [dict(pd) for pd in preds])
        lines.append("loss %.7f oracle %.7f" % (loss.item(), of["loss"].item()))
        assert abs(loss.item() - of["loss"].item()) < 1e-4 * max(1.0, abs(of["loss"].item())), "\n".join(lines)
        loss.backward()
        gerr = []
        for k, v in model.named_parameters():
            go = of["p"][k].grad
            if go is not None and go.norm() > 1e-6 and not (k.endswith(".0.bias") and ("shared_conv" in k or ".tasks." in k)):
                gerr.append((rel(v.grad, go), k))
        gerr.sort(reverse=True)
        lines += ["loss grad rel-L2 %.2e %s" % e for e in gerr[:8]]
        # same sqrt(eps) law, plus the L1 / clamp terms of the loss which are sign-discontinuous in the predictions
        assert sorted(e for e, _ in gerr)[len(gerr) // 2] < 8e-3 and gerr[0][0] < 8e-2, "\n".join(lines)
        msd = model.state_dict()
        for k, v in of["st"].items():
            assert rel(msd[k], v) < 1e-4, (k, rel(msd[k], v))
    # ---- the production bf16 path on the same inputs, for the record
    model.zero_grad()
    model2, _ = build(cfg)
    model2.train()
    _, bb16, nk16, preds16 = forward_stages(model2, exg, B)
    lines.append("bf16 path: backbone rel %.2e  neck rel %.2e" % (rel(bb16, of["bb"]), rel(nk16, of["neck"])))
    for t in range(len(cfg["tasks"])):
        lines.append("bf16 path: head %d/hm sigmoid max|d| %.2e, reg max|d| %.2e" %
                     (t, maxabs(torch.sigmoid(preds16[t]["hm"]), torch.sigmoid(of["preds"][t]["hm"])), maxabs(preds16[t]["reg"], of["preds"][t]["reg"])))
    print("\n".join(lines))
    report_to_file("parity_split_%d.txt" % grid, lines)


def test_full_size_nuscenes_frame_vs_oracle():
    """BASELINE.json configs[1] shape: one 30k-point frame, 0.075 m pillars, 1344^2 grid, 6 tasks -- the assembled
    detector (training-mode forward) against the fp32 oracle: split mode at 1e-3 abs, bf16 path reported."""
    cfg = synth.NUSC
    model, sd = build(cfg, seed=7)
    model.train()
    ex = synth.make_batch([41], 30000, cfg, kind="lidar", n_boxes=40, sweeps=10)
    exg = to_cuda(ex)
    with torch.no_grad():
        of = run_oracle(cfg, sd, ex, 1, with_grads=False)
        loss_o, _ = O.center_loss(ex, [dict(pd) for pd in of["preds"]], cfg["weight"], cfg["code_weights"], True, cfg["voxel_size"],
                                  cfg["pc_range"], cfg["out_size_factor"])
    lines = []
    with Fn.precision("split"), torch.no_grad():
        x, bb, nk, preds = forward_stages(model, exg, 1)
        assert torch.equal(x[1].cpu(), of["coords"])
        worst = 0.0
        for t in range(len(cfg["tasks"])):
            for k in preds[t]:
                worst = max(worst, maxabs(preds[t][k], of["preds"][t][k]))
        lines.append("split: backbone max|d| %.2e, neck max|d| %.2e, worst head map max|d| %.2e" % (maxabs(bb, of["bb"]), maxabs(nk, of["neck"]), worst))
        loss, _ = model.head.loss(exg, [dict(pd) for pd in preds])
        lines.append("split: loss %.6f oracle %.6f" % (loss.item(), loss_o.item()))
        print("\n".join(lines))
        assert worst < 1e-3 and maxabs(nk, of["neck"]) < 1e-3, "\n".join(lines)
        assert abs(loss.item() - loss_o.item()) < 1e-4 * max(1.0, abs(loss_o.item()))
    model2, _ = build(cfg, seed=7)
    model2.train()
    with torch.no_grad():
        _, bb16, nk16, preds16 = forward_stages(model2, exg, 1)
        w16 = max(maxabs(torch.sigmoid(preds16[t]["hm"]), torch.sigmoid(of["preds"][t]["hm"])) for t in range(len(cfg["tasks"])))
        r16 = max(rel(preds16[t][k], of["preds"][t][k]) for t in range(len(cfg["tasks"])) for k in preds16[t])
        lines.append("bf16: backbone rel %.2e, neck rel %.2e, worst head rel-L2 %.2e, heat-map (sigmoid) max|d| %.2e" %
                     (rel(bb16, of["bb"]), rel(nk16, of["neck"]), r16, w16))
        loss16, _ = model2.head.loss(exg, [dict(pd) for pd in preds16])
        lines.append("bf16: loss %.6f oracle %.6f" % (loss16.item(), loss_o.item()))
    print("\n".join(lines))
    report_to_file("parity_fullsize_nusc.txt", lines)
    assert r16 < 2e-1 and abs(loss16.item() - loss_o.item()) < 5e-2 * abs(loss_o.item()), "\n".join(lines)


def test_run_to_run_spread_of_the_gradients():
    """The cross-CTA reductions (BatchNorm statistics: fp32 shared-memory partials + fp64 global atomics; weight-gradient
    split-K: fp32 red.global.add) are ORDER-dependent, so two runs of the same step are not bit-identical.  This test
    measures the spread and pins it.
      * split (fp32-grade) mode: the BatchNorm statistics go straight to fp64 accumulators (order effects 1e-16), so the
        FORWARD is bit-identical from run to run and the gradients differ only by the fp32 split-K atomics of the weight
        gradients (3e-7, most parameters bit-identical).  Before that change the 1e-7 perturbation of the statistics
        flipped a ReLU gate / scatter_max winner in roughly one run out of three and moved a reader gradient by 2.6e-3.
      * bf16 + functional.set_deterministic(True): the same treatment for the production kernels (fp64 statistics,
        split-K slabs added in split order): forward bit-identical, every conv / BatchNorm gradient bit-identical.
      * bf16 mode: every stored activation is re-rounded to 8 mantissa bits, so ANY perturbation, however small, flips a
        few roundings in the next layer and the difference climbs to the bf16 quantisation-noise floor within a few
        layers: two identical runs differ by as much as one run differs from fp32 (3e-2 on the head maps; the ReLU-gate
        law then gives tenths on the gradients).  That is a property of bf16 storage, not a bug -- and the reason the
        parity gate of this repository is the split mode, whose assertions are tight.  (Bit-reproducible bf16 runs would
        need ordered two-stage reductions in every GEMM epilogue; only the split-mode BatchNorm backward reduce is one.)"""
    cfg = synth.tiny_config(128, TASKS)
    B = 2
    ex = to_cuda(synth.make_batch([0, 1], 3000, cfg, kind="uniform", n_boxes=25, sweeps=10))
    lines = []
    for label, tol_fwd, tol_grad in (("split", 1e-6, 1e-5), ("bf16", 1.5e-1, 1.0), ("bf16+deterministic", 0.0, 1e-5), ("split+deterministic", 0.0, 1e-5)):
        mode = label.split("+")[0]
        prev_det = Fn.set_deterministic(label.endswith("deterministic"))
        runs = []
        for _ in range(2):
            model, _ = build(cfg)
            model.train()
            with Fn.precision(mode):
                _, _, _, preds = forward_stages(model, ex, B)
                loss, _ = model.head.loss(ex, [dict(pd) for pd in preds])
                loss.backward()
            runs.append((torch.cat([v.detach().float().reshape(-1) for pd in preds for v in pd.values()]),
                         {k: v.grad.detach().clone() for k, v in model.named_parameters()}))
        Fn.set_deterministic(prev_det)
        fwd = rel(runs[0][0], runs[1][0])
        g = sorted((rel(runs[0][1][k], runs[1][1][k]), k) for k in runs[0][1] if runs[1][1][k].norm() > 1e-6)
        same = sum(1 for k in runs[0][1] if torch.equal(runs[0][1][k], runs[1][1][k]))
        lines.append("%-18s head maps rel %.2e | parameter gradients rel-L2: median %.2e worst %.2e (%s) | bit-identical %d / %d" %
                     (label, fwd, g[len(g) // 2][0], g[-1][0], g[-1][1], same, len(runs[0][1])))
        assert fwd <= tol_fwd and g[-1][0] < tol_grad, "\n".join(lines)
        if label.endswith("deterministic"):
            # functional.set_deterministic: ordered split-K in wgrad + fp64 BatchNorm statistics (+ the fp64 accumulators
            # the PillarFeatureNet backward always uses) -> the forward and EVERY parameter gradient are bit-identical
            diff = [k for k in runs[0][1] if not torch.equal(runs[0][1][k], runs[1][1][k])]
            assert torch.equal(runs[0][0], runs[1][0]), "\n".join(lines)
            assert not diff, (diff, lines)
    print("\n".join(lines))
    report_to_file("run_to_run_spread.txt", lines)
