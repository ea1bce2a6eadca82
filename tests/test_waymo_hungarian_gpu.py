"""Waymo-style AP / APH with matching="hungarian" on the GPU: pnx_eval_pairs, pnx_eval_components and pnx_eval_assign
against their host twins (bit for bit) at the bench's scale, waymo_metrics against the sequential oracle, greedy mode
against the output recorded before the Hungarian mode existed, and the Waymo experiment scored both ways."""
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

from oracle import waymo_fixtures
from oracle import waymo_hungarian_oracle as H
from pillarnext_b200 import evaluate_waymo as EW, ops

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_waymo_hungarian_cpu import assert_greedy_equals_record, assert_same, chain  # noqa: E402


def passes(pk, device):
    """The three passes of one pack_hungarian(), on the GPU (device=True, copied back) or through the host twins."""
    if device:
        def cu(a):
            return torch.from_numpy(np.ascontiguousarray(a)).cuda()
        order = torch.sort(cu(pk["keys"]), stable=True)[1]
        pr = ops.eval_pairs(cu(pk["det_boxes"]), cu(pk["det_trig"]), order, cu(pk["seg_start"]), cu(pk["seg_count"]),
                            cu(pk["gt_boxes"]), cu(pk["gt_classes"]), cu(pk["gt_trig"]), cu(pk["thresholds"]))
        cp = ops.eval_components(pr[0], pr[1], pr[2], pk["M"], pk["C"])
        m = ops.eval_assign(cp[2], cp[0], cp[1], pr[1], pr[2], pr[3], pr[4], cu(pk["det_pass"]), cu(pk["det_range"]),
                            cu(pk["gt_range"]), pk["M"], pk["K"])
        return [t.cpu().numpy() for t in (*pr, *cp, *m)]
    order = np.argsort(pk["keys"], kind="stable").astype(np.int64)
    pr = ops.eval_pairs_host(pk["det_boxes"], pk["det_trig"], order, pk["seg_start"], pk["seg_count"], pk["gt_boxes"],
                             pk["gt_classes"], pk["gt_trig"], pk["thresholds"])
    cp = ops.eval_components_host(pr[0], pr[1], pr[2], pk["M"], pk["C"])
    m = ops.eval_assign_host(cp[2], cp[0], cp[1], pr[1], pr[2], pr[3], pr[4], pk["det_pass"], pk["det_range"],
                             pk["gt_range"], pk["M"], pk["K"])
    return [*pr, *cp, *m]


NAMES = ("edge_start", "e_det", "e_box", "e_iou", "e_head", "comp_start", "comp_nedge", "grouped", "match", "heading")


def test_kernels_equal_host_twins_at_bench_scale():
    """2000 Waymo-val-shaped frames in chunks of 200, up to 500 detections per class (the point clouds are cut to 100
    points: the three passes do not read them)."""
    n_edges = n_large = n_pairs = 0
    for c0 in range(0, 2000, 200):
        gts, det, classes = waymo_fixtures.make_frames(c0, 200, n_points=100, fp_per_class=(460, 480, 500), token0=c0)
        pk = EW.pack_hungarian(gts, det, classes)
        dev, host = passes(pk, True), passes(pk, False)
        for name, d, h in zip(NAMES, dev, host):
            assert d.dtype == h.dtype and d.shape == h.shape, name
            assert np.array_equal(d.view(np.int32), h.view(np.int32)), "chunk %d: %s: %d of %d differ" % (
                c0, name, (d != h).sum(), d.size)
        n_edges += len(dev[1])
        n_large += int((dev[6] > 32).sum())
        n_pairs += int((dev[8] >= 0).sum())
    print("\n%d feasible pairs, %d components beyond one warp, %d matches over (breakdown, cutoff)" % (
        n_edges, n_large, n_pairs))
    assert n_edges > 50000 and n_pairs > 1000000


def test_crowded_and_large_components_equal_host_twins():
    """Crowded frames (small components, many per segment) and the 40-detection tie chain (one component of 80 pairs,
    beyond the one-warp solver, solved by the CTA one)."""
    gts, det, classes = waymo_fixtures.make_frames(51, 8, n_points=100, n_labels=(40, 40, 20), fp_per_class=(60, 60, 30),
                                                   extent=6.0)
    for g, d, cl, thr in ((gts, det, classes, None), (*chain(40), ["vehicle"], {"vehicle": 0.5})):
        pk = EW.pack_hungarian(g, d, cl, thr)
        dev, host = passes(pk, True), passes(pk, False)
        assert len(dev[1]) >= 80 and (thr is None or dev[6].max() == 80)
        for name, a, b in zip(NAMES, dev, host):
            assert np.array_equal(a.view(np.int32), b.view(np.int32)), name


def test_waymo_metrics_equals_oracle_on_20_frames():
    gts, det, classes = waymo_fixtures.make_frames(5000, 20, n_points=20000, extent=60.0)
    got = EW.waymo_metrics(gts, {t: {k: torch.as_tensor(v).cuda() for k, v in d.items()} for t, d in det.items()},
                           classes, matching="hungarian")
    assert_same(got, H.waymo_metrics(gts, det, classes))
    assert 5 < got["mAPH_L2"] < got["mAP_L2"] < 100


def test_greedy_mode_equals_the_parent_output_on_the_gpu():
    rec = json.load(open(os.path.join(ROOT, "tests", "golden", "waymo_greedy_parent.json")))
    inp = rec["input"]
    gts, det, classes = waymo_fixtures.make_frames(inp["seed"], inp["n_frames"], n_points=inp["n_points"],
                                                   extent=inp["extent"])
    assert_greedy_equals_record(EW.waymo_metrics(gts, det, classes), rec["result"])
    assert_greedy_equals_record(EW.waymo_metrics(gts, det, classes, matching="greedy"), rec["result"])


def test_train_waymo_experiment_and_gate_both_matchings(tmp_path):
    """6 epochs of the Waymo synthetic experiment, scored greedy and Hungarian, by the oracle detector (fp32 CPU) and
    the fp32-grade product: each mode's two values agree to the third decimal.  No order between the modes is implied."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import train as train_tool
    from test_map_gpu import oracle_detections
    from pillarnext_b200 import functional as Fn, hydra_lite, scenes
    from pillarnext_b200.trainer import example_to_device
    work = str(tmp_path)
    torch.manual_seed(0)
    name = "synth_det_pp18_aspp_waymo_hungarian"
    overrides = ["trainer.max_epochs=6", "data.train_dataset.n_frames=640", "data.val_dataset.n_frames=24",
                 "dataloader.train.num_workers=0", "dataloader.val.num_workers=0", "dataloader.train.batch_size=4"]
    tr = train_tool.main(["--config-name", name, "--work-dir", work] + overrides)
    assert tr.epoch == 6 and "range_means" in tr.last_eval
    cfg = hydra_lite.main(os.path.join(ROOT, "configs", "experiments"), name, overrides)
    val = hydra_lite.instantiate(cfg.data.val_dataset)
    model = tr.model.eval()
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items()}
    d_oracle = oracle_detections(cfg, sd, val)
    d_split = {}
    with torch.no_grad(), Fn.precision("split"):
        for i0 in range(0, len(val), 4):
            ex = scenes.collate([val[i] for i in range(i0, min(len(val), i0 + 4))])
            d_split.update(model(example_to_device(ex, torch.device("cuda"))))
    gt = val.ground_truth()
    rows = {}
    for mode in ("greedy", "hungarian"):
        rows[mode] = [EW.waymo_metrics(gt, d, val.class_names, matching=mode) for d in (d_oracle, d_split)]
    msg = "; ".join("%s: L2 mAPH / L2 mAP / L1 mAPH oracle (fp32 CPU) %s | product fp32-grade %s" % (
        mode, *["%.3f / %.3f / %.3f" % (m["mAPH_L2"], m["mAP_L2"], m["mAPH_L1"]) for m in r]) for mode, r in rows.items())
    print("\n" + msg)
    h = rows["hungarian"][1]
    print("hungarian per range (product): " + ", ".join(
        "%s %.3f" % (r, h["range_means"][r]["mAPH_L2"]) for r in EW.RANGES))
    for mode, (o, s) in rows.items():
        assert o["mAPH_L2"] > 5.0, "the detector did not learn the synthetic task: " + msg
        for key in ("mAP_L1", "mAPH_L1", "mAP_L2", "mAPH_L2"):
            assert round(o[key], 3) == round(s[key], 3) or abs(o[key] - s[key]) < 1e-3, (mode, key, msg)
    assert all(not math.isnan(v) for v in (rows["hungarian"][0]["mAPH_L2"], rows["hungarian"][1]["mAPH_L2"]))
