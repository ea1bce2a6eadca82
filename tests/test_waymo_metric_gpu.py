"""Waymo-style AP / APH on the GPU: pnx_eval_count_points and pnx_eval_match against their host twins (bit for bit),
the match's pair skip against the full IoU routine, waymo_metrics against the sequential oracle, and the accuracy gate
of the Waymo-configured detector scored with it."""
import math
import os
import sys

import numpy as np
import pytest
import torch

from oracle import waymo_fixtures
from oracle import waymo_metric_oracle as O
from pillarnext_b200 import evaluate_waymo as EW, ops

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_match_kernel_equals_host_twin_on_crowded_frames():
    gts, det, classes = waymo_fixtures.make_frames(21, 200, n_points=100, extent=40.0)
    pk = EW.pack(gts, det, classes)
    _, m_d, i_d, h_d = EW.run_device(pk)
    _, m_h, i_h, h_h = EW.run_host(pk)
    bad = (m_d != m_h) | (i_d.view(np.int32) != i_h.view(np.int32)) | (h_d.view(np.int32) != h_h.view(np.int32))
    assert not bad.any(), "%d of %d detections differ: match %d, iou %d (max %.3g), heading %d" % (
        bad.sum(), len(bad), (m_d != m_h).sum(), (i_d != i_h).sum(), np.abs(i_d - i_h).max(), (h_d != h_h).sum())
    assert (m_d >= 0).sum() > 5000 and (i_d > 0).sum() > (m_d >= 0).sum()


def test_count_kernel_equals_host_twin():
    gts, det, classes = waymo_fixtures.make_frames(22, 24, n_points=265000)
    pk = EW.pack(gts, {}, classes)
    c_d = EW.run_device(pk)[0]
    c_h = EW.run_host(pk)[0]
    assert np.array_equal(c_d, c_h)
    assert c_d.sum() > 24 * 50000 and (c_d == 0).sum() > 0 and ((c_d >= 1) & (c_d <= 5)).sum() > 0
    for f, t in enumerate(list(gts)[:4]):                       # the point test of ground-truth sampling, summed
        g = gts[t]
        inside = ops.points_in_boxes_host(g["points"], g["boxes"], pk["count_trig"][f, :len(g["boxes"])])
        assert np.array_equal(inside.sum(0), c_d[f, :len(g["boxes"])])


def test_pair_skip_never_hides_an_overlap():
    """Touching, barely overlapping and margin-distance (within in_box2d's 1e-2) rotated pairs, one pair per frame: the
    match's IoU (device and host) must equal the full routine's wherever it is 0, and bit for bit on the device/host."""
    rng = np.random.default_rng(5)
    n = 4000
    a = np.zeros((n, 9), np.float32)
    a[:, :2] = rng.uniform(-70, 70, (n, 2))
    a[:, 2] = 0.5
    a[:, 3:6] = rng.uniform(0.5, 5.0, (n, 3))
    a[:, 8] = rng.uniform(-math.pi, math.pi, n)
    b = a.copy()
    b[:, 3:6] = rng.uniform(0.5, 5.0, (n, 3))
    b[:, 8] = rng.uniform(-math.pi, math.pi, n)
    # place b along a random direction at the distance where the footprints first touch, then move it by -5 cm .. +6 cm
    phi = rng.uniform(-math.pi, math.pi, n)
    u = np.stack([np.cos(phi), np.sin(phi)], 1)

    def support(box, dirs):                                     # half-width of a footprint along dirs
        c, s = np.cos(box[:, 8]), np.sin(box[:, 8])
        return 0.5 * (box[:, 3] * np.abs(dirs[:, 0] * c + dirs[:, 1] * s) + box[:, 4] * np.abs(-dirs[:, 0] * s + dirs[:, 1] * c))
    def full_iou(b):                                            # the full routine, host-compiled, detection first
        return ops.aligned_iou3d_host(b[:, [0, 1, 2, 3, 4, 5, 8]], a[:, [0, 1, 2, 3, 4, 5, 8]])
    lo, hi = np.zeros(n), support(a, u) + support(b, u) + 1.0
    for _ in range(40):                                         # bisect the touching distance along u
        mid = 0.5 * (lo + hi)
        b[:, :2] = a[:, :2] + mid[:, None] * u
        full = full_iou(b)
        lo, hi = np.where(full > 0, mid, lo), np.where(full > 0, hi, mid)
    b[:, :2] = a[:, :2] + (hi + rng.uniform(-0.05, 0.06, n))[:, None] * u
    gts = {i: {"boxes": a[i:i + 1], "names": ["x"], "points": np.zeros((0, 3), np.float32)} for i in range(n)}
    det = {i: {"box3d_lidar": b[i:i + 1], "scores": np.ones(1, np.float32), "label_preds": np.zeros(1, np.int64)}
           for i in range(n)}
    pk = EW.pack(gts, det, ["x"], {"x": 0.5})
    i_d, i_h = EW.run_device(pk)[2], EW.run_host(pk)[2]
    assert np.array_equal(i_d.view(np.int32), i_h.view(np.int32))
    full = full_iou(b)
    assert not ((i_d == 0) & (full != 0)).any(), "the skip hid a non-zero IoU"
    assert ((full > 0) & (full < 1e-3)).sum() > 100                 # barely overlapping pairs are covered
    assert (full == 0).sum() > 1000                                  # and disjoint ones


def test_waymo_metrics_equals_oracle():
    gts, det, classes = waymo_fixtures.make_frames(23, 4, n_points=20000, extent=40.0)
    got = EW.waymo_metrics(gts, {t: {k: torch.as_tensor(v).cuda() for k, v in d.items()} for t, d in det.items()}, classes)
    want = O.waymo_metrics(gts, det, classes)
    print(got, want)
    for k in ("mAP_L1", "mAP_L2"):
        assert abs(got[k] - want[k]) < 1e-9, (k, got[k], want[k])
    for k in ("mAPH_L1", "mAPH_L2"):
        assert abs(got[k] - want[k]) < 1e-6, (k, got[k], want[k])
    for name in classes:
        for k in ("n_gt_L1", "n_gt_L2"):
            assert got["per_class"][name][k] == want["per_class"][name][k]
    assert 5 < got["mAPH_L2"] < got["mAP_L2"] < 100


def test_train_waymo_experiment_and_gate(tmp_path):
    import importlib.util
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import train as train_tool
    from test_map_gpu import oracle_detections
    from pillarnext_b200 import functional as Fn, hydra_lite, scenes
    from pillarnext_b200.trainer import example_to_device
    spec = importlib.util.spec_from_file_location("pnx_tools_test", os.path.join(ROOT, "tools", "test.py"))
    test_tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(test_tool)
    work = str(tmp_path)
    torch.manual_seed(0)                                        # the weight initialisation, whatever ran before
    name = "synth_det_pp18_aspp_waymo"
    overrides = ["trainer.max_epochs=6", "data.train_dataset.n_frames=640", "data.val_dataset.n_frames=24",
                 "dataloader.train.num_workers=0", "dataloader.val.num_workers=0", "dataloader.train.batch_size=4"]
    tr = train_tool.main(["--config-name", name, "--work-dir", work] + overrides)
    assert tr.epoch == 6
    at_end = tr.last_eval["mAPH_L2"]
    res = test_tool.main(["--config-name", name, "--work-dir", work, "+load_from=" + os.path.join(work, "epoch_6.pth")] + overrides)
    assert abs(res["mAPH_L2"] - at_end) < 1e-6
    cfg = hydra_lite.main(os.path.join(ROOT, "configs", "experiments"), name, overrides)
    val = hydra_lite.instantiate(cfg.data.val_dataset)
    model = tr.model.eval()
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items()}
    m_oracle = val.evaluation(oracle_detections(cfg, sd, val))

    def product():
        dets = {}
        with torch.no_grad():
            for i0 in range(0, len(val), 4):
                ex = scenes.collate([val[i] for i in range(i0, min(len(val), i0 + 4))])
                dets.update(model(example_to_device(ex, torch.device("cuda"))))
        return val.evaluation(dets)

    m_bf16 = product()
    with Fn.precision("split"):
        m_split = product()
    msg = "L2 mAPH / L2 mAP / L1 mAPH on %d held-out scenes: oracle (fp32 CPU) %s | product fp32-grade %s | product bf16 %s" % (
        len(val), *["%.3f / %.3f / %.3f" % (m["mAPH_L2"], m["mAP_L2"], m["mAPH_L1"]) for m in (m_oracle, m_split, m_bf16)])
    print(msg)
    assert m_oracle["mAPH_L2"] > 5.0, "the detector did not learn the synthetic task: " + msg
    assert abs(m_split["mAPH_L2"] - m_oracle["mAPH_L2"]) <= 0.1, msg
    assert abs(m_bf16["mAPH_L2"] - m_oracle["mAPH_L2"]) <= 3.0, msg
