"""The tracker (pnx_track_greedy) and the CLEAR-MOT pass (pnx_eval_mot) on the GPU: equal to their host twins bit for
bit on a Waymo-validation-shaped input (200 sequences x 200 frames, up to 500 detections per class and frame) and on
the hand-built cases of test_tracking_cpu.py, a sequence that fills the track capacity, and
WaymoDataset(tracking=True).evaluation() on the reader fixture."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import track_fixtures as TF
from oracle import track_oracle as O
from pillarnext_b200 import evaluate_waymo as EW, evaluate_waymo_tracking as EWT, ops
from pillarnext_b200 import track as TR

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_tracking_cpu as T  # noqa: E402

CLASSES = TF.CLASSES


def mot_device_and_host(gts, tracks, K=11):
    """pnx_eval_mot and its host twin on the same pairs and components (those of the device passes)."""
    pk = EWT.pack(gts, tracks, CLASSES, num_score_cutoffs=K)
    npts = EW.known_counts(pk, ops.eval_count_points_host(pk["points"], pk["gt_boxes"], pk["gt_classes"],
                                                           pk["count_trig"])).astype(np.int32).reshape(-1)

    def cu(a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()
    order = torch.sort(cu(pk["keys"]), stable=True)[1]
    start, e_det, e_box, e_iou, _ = ops.eval_pairs(cu(pk["det_boxes"]), cu(pk["det_trig"]), order, cu(pk["seg_start"]),
                                                   cu(pk["seg_count"]), cu(pk["gt_boxes"]), cu(pk["gt_classes"]),
                                                   cu(pk["gt_trig"]), cu(pk["thresholds"]))
    comp = ops.eval_components(start, e_det, e_box, pk["M"], pk["C"])
    args = [start, e_det, e_box, e_iou, comp[2], comp[0], comp[1], cu(pk["det_pass"]), cu(pk["det_id"]),
            cu(pk["gt_obj"].reshape(-1)), cu(npts), cu(pk["seq_start"])]
    shape = (pk["M"], pk["C"], pk["K"], pk["n_obj"])
    dev = [t.cpu().numpy() for t in ops.eval_mot(*args, *shape)]
    host = ops.eval_mot_host(*[t.cpu().numpy() for t in args], *shape)
    for a, b in zip(dev, host):
        np.testing.assert_array_equal(a, b)
    return pk, dev


@pytest.fixture(scope="module")
def waymo_val():
    return TF.waymo_val_shaped(0)


def test_kernels_equal_host_twins_on_a_waymo_val_shaped_input(waymo_val):
    dets, frames, gts = waymo_val
    pk = TR.pack(dets, frames, CLASSES)
    assert len(pk["seq_start"]) == 201 and len(pk["tokens"]) == 40000
    assert pk["seg_count"].max() == 500
    ids = TR.run_device(pk, 3, 0.1)
    np.testing.assert_array_equal(ids, TR.run_host(pk, 3, 0.1))
    assert (ids >= 0).mean() > 0.8 and ids.max() > 1000
    tracks = TR.track(dets, frames, CLASSES, min_score=0.1)
    _, (mot, dist) = mot_device_and_host(gts, tracks)
    assert mot[..., 0].sum() > 0 and mot[..., 2].sum() > 0      # matches and mismatches both occur


@pytest.mark.parametrize("case", ["birth_coast_death", "ties", "classes"])
def test_tracker_hand_built_cases_on_the_device(case):
    frames = T.frames_of(11)
    toks = list(frames)
    if case == "birth_coast_death":
        dets = {t: T.det([]) for t in toks}
        for f in (0, 1, 5, 10):
            dets[toks[f]] = T.det([(1.0 * f, 0.0, 10.0, 0.0, 0.9)])
        want = {toks[f]: [i] for f, i in ((0, 0), (1, 0), (5, 0), (10, 1))}
    elif case == "ties":
        dets = {toks[0]: T.det([(-1.0, 0.0, 0, 0, 0.8), (1.0, 0.0, 0, 0, 0.8)]),
                toks[1]: T.det([(0.0, 0.0, 0, 0, 0.5), (0.0, 0.0, 0, 0, 0.5), (20.0, 0.0, 0, 0, 0.05)])}
        want = {toks[0]: [0, 1], toks[1]: [0, 1, -1]}
    else:
        mixed = T.det([(0, 0, 0, 0, 0.9), (30, 0, 0, 0, 0.8)])
        mixed["label_preds"] = np.array([1, 0], np.int64)
        dets = {toks[0]: mixed, toks[1]: T.det([(50, 0, 0, 0, 0.9)])}
        want = {toks[0]: [1, 0], toks[1]: [2]}
    got = TR.track({k: {n: torch.from_numpy(v).cuda() for n, v in d.items()} for k, d in dets.items()}, frames,
                   CLASSES, min_score=0.1)
    host = TR.track(dets, frames, CLASSES, min_score=0.1, host=True)
    for t, ids in want.items():
        assert got[t]["tracking_id"].tolist() == ids == host[t]["tracking_id"].tolist()


def test_mot_hand_built_cases_on_the_device():
    cases = [({"s-1": T.gt_frame([(0, 0, "A", 50), (10, 0, "B", 50)], "s", 1),
               "s-2": T.gt_frame([(0, 0, "A", 50), (10, 0, "B", 50)], "s", 2)},
              {"s-1": T.tracked([(0, 0, 0.9, 0), (10, 0, 0.9, 1)]), "s-2": T.tracked([(0.1, 0, 0.9, 1)])}),
             ({"s-1": T.gt_frame([(0, 0, "A", 50)], "s", 1), "s-2": T.gt_frame([(0, 0, "A", 50)], "s", 2)},
              {"s-1": T.tracked([(0, 0, 0.9, 0)]), "s-2": T.tracked([(0.05, 0, 0.95, 7), (0.4, 0, 0.6, 0)])}),
             ({"s-1": T.gt_frame([(0, 0, "A", 50), (10, 0, "B", 3), (20, 0, "C", 0)], "s", 1)},
              {"s-1": T.tracked([(0, 0, 0.9, 0), (10, 0, 0.9, 1), (20, 0, 0.9, 2)])})]
    for gts, tracks in cases:
        mot_device_and_host(gts, tracks, K=1)
        got = EWT.waymo_tracking_metrics(gts, tracks, CLASSES, num_score_cutoffs=1)
        T.assert_metrics_close(got, O.tracking_metrics(gts, tracks, CLASSES, num_score_cutoffs=1), 1e-6)


def test_a_sequence_that_fills_the_track_capacity():
    cap = 4096
    frames = T.frames_of(3)
    toks = list(frames)
    grid = [(5.0 * (k % 64), 5.0 * (k // 64), 0.0, 0.0, 0.5) for k in range(cap)]
    dets = {toks[0]: T.det(grid, label=1), toks[1]: T.det(grid, label=1)}
    got = TR.track(dets, frames, CLASSES)
    host = TR.track(dets, frames, CLASSES, host=True)
    for t in dets:
        np.testing.assert_array_equal(got[t]["tracking_id"], host[t]["tracking_id"])
        assert sorted(got[t]["tracking_id"].tolist()) == list(range(cap))
    dets[toks[2]] = T.det(grid + [(1000.0, 0.0, 0.0, 0.0, 0.5)], label=1)
    for host_twin in (False, True):
        with pytest.raises(ValueError, match="more than 4096 live tracks"):
            TR.track(dets, frames, CLASSES, host=host_twin)


def test_waymo_dataset_evaluation_tracks_on_the_device(tmp_path):
    from det3d.datasets.waymo.waymo import WaymoDataset
    root = str(tmp_path)
    infos = T.waymo_tracking_tree(root)
    ds = WaymoDataset("waymo_infos_val.pkl", root, nsweeps=1, tracking=True)
    g = np.random.default_rng(5)
    dets = {}
    for info in infos:
        objs = info["objects"]
        b = np.array([o["box"] for o in objs], np.float32).reshape(-1, 9)
        b[:, :2] += g.normal(0, 0.1, (len(b), 2)).astype(np.float32)
        dets[info["token"]] = dict(box3d_lidar=torch.from_numpy(b).cuda(),
                                   scores=torch.from_numpy(g.uniform(0.2, 1, len(b)).astype(np.float32)).cuda(),
                                   label_preds=torch.tensor([CLASSES.index(o["label"]) for o in objs]).cuda())
    res = ds.evaluation(dets)
    assert "mAP_L1" in res
    gts = ds.ground_truth()
    host_tracks = TR.track(dets, gts, CLASSES, host=True)
    for t in dets:
        np.testing.assert_array_equal(res["tracks"][t]["tracking_id"].numpy(), host_tracks[t]["tracking_id"])
    T.assert_metrics_close(res["tracking"], O.tracking_metrics(gts, host_tracks, CLASSES), 1e-6)


def test_train_waymo_tracking_experiment_and_gate(tmp_path):
    """6 epochs of synth_det_pp18_aspp_waymo_tracking (validation: 3 sequences of 8 frames).  The oracle detector
    (fp32 CPU) tracked and scored by oracle/track_oracle.py, and the fp32-grade product detector tracked and scored by
    the product, agree on every reported tracking number to the third decimal; bf16 is reported beside them.  Six
    epochs do not teach the velocity head, so this checks agreement, not tracking quality."""
    import math
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import train as train_tool
    from test_map_gpu import oracle_detections
    from pillarnext_b200 import functional as Fn, hydra_lite, scenes
    from pillarnext_b200.trainer import example_to_device
    torch.manual_seed(0)
    name = "synth_det_pp18_aspp_waymo_tracking"
    overrides = ["trainer.max_epochs=6", "data.train_dataset.n_frames=640", "data.val_dataset.n_frames=24",
                 "dataloader.train.num_workers=0", "dataloader.val.num_workers=0", "dataloader.train.batch_size=4"]
    tr = train_tool.main(["--config-name", name, "--work-dir", str(tmp_path)] + overrides)
    assert tr.epoch == 6 and "tracking" in tr.last_eval
    cfg = hydra_lite.main(os.path.join(ROOT, "configs", "experiments"), name, overrides)
    val = hydra_lite.instantiate(cfg.data.val_dataset)
    assert val.sequence_length == 8
    model = tr.model.eval()
    sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items()}
    d_oracle = oracle_detections(cfg, sd, val)

    def product(precision):
        out = {}
        with torch.no_grad(), Fn.precision(precision):
            for i0 in range(0, len(val), 4):
                ex = scenes.collate([val[i] for i in range(i0, min(len(val), i0 + 4))])
                out.update(model(example_to_device(ex, torch.device("cuda"))))
        return out
    gt = val.ground_truth()
    ids = O.track(d_oracle, gt, val.class_names)
    o = O.tracking_metrics(gt, {t: dict(d, tracking_id=ids[t]) for t, d in d_oracle.items()}, val.class_names)
    s = EWT.track_and_score(gt, product("split"), val.class_names)[1]
    b = EWT.track_and_score(gt, product("bf16"), val.class_names)[1]
    keys = ("mMOTA_L1", "mMOTP_L1", "mMOTA_L2", "mMOTP_L2")
    msg = "; ".join("%s %s" % (who, " / ".join("%.3f" % m[k] for k in keys)) for who, m in
                    (("oracle (fp32 CPU)", o), ("product fp32-grade", s), ("product bf16", b)))
    print("\nL1 mMOTA / L1 mMOTP / L2 mMOTA / L2 mMOTP: " + msg)
    assert s["per_class"].keys() == o["per_class"].keys()
    for mo, ms in [(o, s)] + [(o["per_class"][c], s["per_class"][c]) for c in o["per_class"]]:
        for k, v in mo.items():
            if k == "per_class":
                continue
            w = ms[k]
            assert (math.isnan(v) and math.isnan(w)) or round(v, 3) == round(w, 3) or abs(v - w) < 1e-3, (k, v, w, msg)
