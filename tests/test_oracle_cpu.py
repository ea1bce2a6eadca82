"""CPU tier: pins the oracle restatement against golden vectors frozen from the reference's own files
(tests/golden/ref_tiny.npz, ref_live.npz: oracle/make_golden*.py); checks the two backbone restatements against each other (spconv is absent:
parity unpinned there) and the state-dict / C-ABI contracts."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import pillarnext_oracle as O
from oracle.make_golden import golden_setup

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_tiny.npz")
GOLD_LIVE = os.path.join(os.path.dirname(__file__), "golden", "ref_live.npz")


@pytest.fixture(scope="module")
def setup():
    cfg, sd, ex, x_neck, x_head = golden_setup()
    return cfg, sd, ex, x_neck, x_head, np.load(GOLD)


def test_reader_oracle_vs_golden(setup):
    cfg, sd, ex, _, _, g = setup
    st = {}
    feat, coords, grid = O.reader_forward(ex["points"], sd, cfg["voxel_size"], cfg["pc_range"], train=True, stats=st)
    assert np.array_equal(coords.numpy(), g["reader_coords"])          # indices: bit exact
    assert np.array_equal(np.asarray(grid), g["reader_grid"])
    assert np.abs(feat.detach().numpy() - g["reader_feat"]).max() < 2e-5
    assert np.abs(st["reader.pfn_layers.0.norm.running_mean"].numpy() - g["reader_rm0"]).max() < 1e-6
    assert np.abs(st["reader.pfn_layers.1.norm.running_var"].numpy() - g["reader_rv1"]).max() < 1e-5
    # eval mode uses the running stats as updated by the training pass
    sd2 = dict(sd)
    sd2.update(st)
    feat_e, _, _ = O.reader_forward(ex["points"], sd2, cfg["voxel_size"], cfg["pc_range"], train=False)
    # the reference's layer-1 stats were also updated; only the stored ones are compared -> recompute all
    assert feat_e.shape == tuple(g["reader_feat_eval"].shape)
    assert np.abs(feat_e.detach().numpy() - g["reader_feat_eval"]).max() < 2e-4


def test_neck_head_loss_oracle_vs_golden(setup):
    cfg, sd, ex, x_neck, x_head, g = setup
    y = O.aspp_forward(x_neck, sd, train=True)
    assert np.abs(y.detach().numpy() - g["neck_out"]).max() < 1e-3 * max(1.0, np.abs(g["neck_out"]).max())
    p = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items() if k.startswith("head.")}
    xh = x_head.clone().requires_grad_()
    preds = O.centerhead_forward(xh, p, cfg["tasks"], cfg["common_heads"], train=True)
    for t, pd in enumerate(preds):
        assert list(pd.keys()) == list(cfg["common_heads"].keys()) + ["hm"]
        for k, v in pd.items():
            assert np.abs(v.detach().numpy() - g["head_t%d_%s" % (t, k)]).max() < 2e-5, (t, k)
    loss, rets = O.center_loss(ex, preds, cfg["weight"], cfg["code_weights"], True, cfg["voxel_size"], cfg["pc_range"], cfg["out_size_factor"])
    assert abs(loss.item() - float(g["loss_total"])) < 1e-4 * abs(float(g["loss_total"]))
    for t, r in enumerate(rets):
        for k in ("hm_loss", "loc_loss", "iou_reg_loss"):
            assert abs(float(r[k]) - float(g["loss_t%d_%s" % (t, k)])) < 1e-4 * max(1.0, abs(float(g["loss_t%d_%s" % (t, k)]))), (t, k)
        assert np.abs(r["loc_loss_elem"].numpy() - g["loss_t%d_loc_elem" % t]).max() < 1e-5
    loss.backward()
    for name, got in (("grad_head_x", xh.grad), ("grad_shared_conv_w", p["head.shared_conv.0.weight"].grad[:16]), ("grad_t1_hm_3_w", p["head.tasks.1.hm.3.weight"].grad)):
        ref = g[name]
        assert np.abs(got.numpy() - ref).max() < 1e-4 * max(1e-3, np.abs(ref).max()), name


def test_product_loss_matches_golden(setup):
    """pillarnext_b200.loss (sync-free variant used by the product) on CPU tensors vs the reference's numbers."""
    from pillarnext_b200 import loss as PL
    cfg, sd, ex, _, _, g = setup
    preds = [{k: torch.tensor(g["head_t%d_%s" % (t, k)]) for k in list(cfg["common_heads"].keys()) + ["hm"]} for t in range(len(cfg["tasks"]))]
    total, rets = PL.center_loss(ex, preds, cfg["tasks"], cfg["weight"], cfg["code_weights"], True, cfg["voxel_size"], cfg["pc_range"], cfg["out_size_factor"])
    assert abs(total.item() - float(g["loss_total"])) < 1e-4 * abs(float(g["loss_total"]))
    # empty-mask case: finite, equals the reference's early-out value
    ex0 = {k: [torch.zeros_like(e) for e in v] if k in ("mask",) else v for k, v in ex.items()}
    preds = [{k: torch.tensor(g["head_t%d_%s" % (t, k)]).requires_grad_() for k in list(cfg["common_heads"].keys()) + ["hm"]} for t in range(len(cfg["tasks"]))]
    t0, _ = PL.center_loss(ex0, preds, cfg["tasks"], cfg["weight"], cfg["code_weights"], True, cfg["voxel_size"], cfg["pc_range"], cfg["out_size_factor"])
    assert torch.isfinite(t0)
    t0.backward()
    assert all(torch.isfinite(v.grad).all() for pd in preds for k, v in pd.items() if v.grad is not None)


def test_backbone_restatements_agree(setup):
    cfg, sd, ex, _, _, _ = setup
    feat, coords, grid = O.reader_forward(ex["points"], sd, cfg["voxel_size"], cfg["pc_range"], train=True)
    feat = feat.detach()
    pa = {k: v.clone().requires_grad_(v.dtype.is_floating_point and "running" not in k) for k, v in sd.items() if k.startswith("backbone.")}
    pb = {k: v.clone().requires_grad_(v.dtype.is_floating_point and "running" not in k) for k, v in sd.items() if k.startswith("backbone.")}
    sa, sb = {}, {}
    dense, mask = O.sparse_resnet_dense(feat, coords, grid, 2, pa, cfg["strides"], stats=sa)
    f4, c4, shp = O.sparse_resnet_gather(feat, coords, grid, 2, pb, cfg["strides"], stats=sb)
    d2 = O.densify(f4, c4, shp)
    assert dense.shape == d2.shape == (2, 256, 8, 8)
    assert (dense - d2).abs().max().item() < 1e-4
    assert torch.equal(mask[:, 0] > 0, (d2.abs().sum(1) > 0) | (mask[:, 0] > 0))
    for k in sa:
        assert (sa[k] - sb[k]).abs().max().item() < 1e-5, k
    w = torch.randn(dense.shape, generator=torch.Generator().manual_seed(5))
    (dense * w).sum().backward()
    (d2 * w).sum().backward()
    for k in pa:
        if pa[k].grad is not None:
            e = (pa[k].grad - pb[k].grad).norm().item()
            # fp32 summation-order noise through 21 BN layers (occasional ReLU flips): relative L2 < 1e-2
            assert e < 1e-2 * max(1e-3, pb[k].grad.norm().item()), (k, e)


def test_state_dict_contract(setup):
    """Same keys and shapes as the reference modules (golden list) + the spconv-layout backbone keys of SURVEY 8b."""
    from pillarnext_b200 import modules, synth
    cfg, sd, _, _, _, g = setup
    mine = modules.build_pillarnext_b(cfg).state_dict()
    ref_names = [str(n) for n in g["sd_names"]]
    ref_shapes = {str(n): str(s) for n, s in zip(g["sd_names"], g["sd_shapes"])}
    non_backbone = [k for k in mine if not k.startswith("backbone.")]
    assert sorted(non_backbone) == sorted(ref_names)
    for k in non_backbone:
        assert ",".join(str(s) for s in mine[k].shape) == ref_shapes[k], k
    bb = [k for k in mine if k.startswith("backbone.")]
    assert mine["backbone.blocks.0.0.conv.weight"].shape == (64, 3, 3, 64)          # [Cout, kH, kW, Cin]
    assert mine["backbone.blocks.3.2.conv2.weight"].shape == (256, 3, 3, 256)
    assert mine["backbone.mapping.0.weight"].shape == (256, 1, 1, 256)
    pat = re.compile(r"backbone\.(blocks\.[0-3]\.(0\.(conv\.weight|norm\.\w+)|[12]\.(block1\.(conv\.weight|norm\.\w+)|conv2\.weight|norm2\.\w+))|mapping\.(0\.weight|1\.\w+))$")
    assert all(pat.match(k) for k in bb), [k for k in bb if not pat.match(k)]
    full = modules.build_pillarnext_b(synth.NUSC)
    assert sum(p.numel() for p in full.parameters()) == 10379782      # SURVEY 8a parameter count (nuScenes)


def test_abi_library_loads_and_exports_header_symbols():
    from pillarnext_b200 import _lib
    so = os.path.join(os.path.dirname(_lib.__file__), "libpnx.so")
    if not os.path.exists(so):
        from pillarnext_b200 import build
        build.build()
    l = ctypes.CDLL(so)
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pnx.h")).read()
    declared = set(re.findall(r"\b(pnx_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(_lib.exported_symbols()), declared ^ set(_lib.exported_symbols())
    for name in declared:
        assert hasattr(l, name), name
    l.pnx_abi_version.restype = ctypes.c_int
    assert l.pnx_abi_version() == 1
    # arity: every declaration's parameter count equals the ctypes binding's (a mismatch shifts arguments silently)
    code = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    for name, params in re.findall(r"\b(pnx_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", code):
        params = params.strip()
        n = 0 if params in ("", "void") else params.count(",") + 1
        assert n == len(_lib._SIGS[name]), (name, n, len(_lib._SIGS[name]))


def test_product_never_imports_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for d in ("pillarnext_b200", "det3d"):
        for dp, _, fs in os.walk(os.path.join(root, d)):
            for f in fs:
                if f.endswith(".py"):
                    src = open(os.path.join(dp, f)).read()
                    assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), os.path.join(dp, f)


def test_oracle_and_synth_vs_live_reference(setup):
    """The reference's AssignLabel, collate and PillarFeatureNet outputs on these inputs are stored in ref_live.npz."""
    from oracle.make_golden_live import ASSIGN_KEYS
    from pillarnext_b200 import synth
    cfg, sd, ex, _, _, _ = setup
    gold = np.load(GOLD_LIVE)
    # label assignment restatement (synth.assign_labels) vs reference AssignLabel + collate
    boxes, names = synth.make_gt(3, 25, cfg)
    mine = synth.assign_labels(boxes, names, cfg)
    for k in ASSIGN_KEYS:
        for t in range(len(cfg["tasks"])):
            want = gold["assign_%s_%d" % (k, t)]
            assert np.array_equal(np.nan_to_num(want, nan=-7.0), np.nan_to_num(np.asarray(mine[k][t]), nan=-7.0)), (k, t)
    frames = [synth.make_frame(s, 300, cfg) for s in range(2)]
    assert torch.equal(torch.from_numpy(gold["collate_points"]), synth.collate_points(frames))
    # a different seed / shape than the golden file: oracle reader vs the reference file
    pts = synth.collate_points([synth.make_frame(11, 2000, synth.NUSC, "lidar", sweeps=10)])
    f2, c2, _ = O.reader_forward(pts, sd, synth.NUSC["voxel_size"], synth.NUSC["pc_range"], train=True)
    assert torch.equal(torch.from_numpy(gold["reader_coords"]), c2)
    assert (torch.from_numpy(gold["reader_feat"]) - f2).abs().max().item() < 2e-5


def test_convert_sync_batchnorm_is_honoured():
    """tools/train.py:55-56 wraps the model with torch.nn.SyncBatchNorm.convert_sync_batchnorm: state-dict keys must
    survive and every BN holder must then ask for synchronised statistics."""
    from pillarnext_b200 import functional as Fn, modules, synth
    cfg = synth.tiny_config(64, [["car"], ["truck", "construction_vehicle"]])
    model = modules.build_pillarnext_b(cfg)
    keys = list(model.state_dict().keys())
    bns = [m for m in model.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)]
    assert bns and not any(Fn.wants_sync(m) for m in bns)
    conv = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    assert list(conv.state_dict().keys()) == keys
    bns = [m for m in conv.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)]
    assert bns and all(isinstance(m, torch.nn.SyncBatchNorm) and Fn.wants_sync(m) for m in bns)
    model2 = modules.enable_sync_batchnorm(modules.build_pillarnext_b(cfg))
    assert all(Fn.wants_sync(m) for m in model2.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm))
