"""nuScenes tracking metric on the GPU: pnx_eval_pairs_center and pnx_eval_mot_center against their host twins, bit
for bit, on the nuScenes-val-shaped input of tools/bench_nusc_tracking.py (150 scenes x 40 frames: 150 x 7 x 40 =
42,000 rows in the cutoff pass), and the whole metric against the sequential oracle on a subset of scenes."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from oracle import nusc_track_fixtures as NF
from oracle import nusc_track_oracle as O
from pillarnext_b200 import evaluate_nuscenes_tracking as ENT, ops

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_nusc_tracking_cpu as T  # noqa: E402


@pytest.fixture(scope="module")
def nusc_val():
    dets, frames, gts = NF.nusc_val_shaped(0)
    tracks, metrics = ENT.track_and_score(gts, dets, NF.CLASSES)
    return gts, tracks, metrics


def test_kernels_equal_host_twins_on_a_nusc_val_shaped_input(nusc_val):
    gts, tracks, metrics = nusc_val
    pk = ENT.pack(gts, tracks, NF.CLASSES)
    dev, host = ENT.run_device(pk, gts), ENT.run_host(pk, gts)
    assert dev["counts"].shape == (150, 7, 40, 3)
    np.testing.assert_array_equal(dev["classes"], host["classes"])
    np.testing.assert_array_equal(dev["matched"], host["matched"])
    for a, b in zip(dev["cutoffs"], host["cutoffs"]):
        np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(dev["counts"], host["counts"])
    assert dev["dist"].tobytes() == host["dist"].tobytes()
    # the pairs themselves, bit for bit
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()    # noqa: E731
    args = (pk["det_boxes"], pk["order"], pk["seg_start"], pk["seg_count"], pk["gt_boxes"], host["classes"], pk["C"],
            ENT.PAIR_DIST)
    got = ops.eval_pairs_center(*[cu(a) if isinstance(a, np.ndarray) else a for a in args])
    want = ops.eval_pairs_center_host(*args)
    for g, w in zip(got, want):
        assert g.cpu().numpy().tobytes() == w.tobytes()
    assert len(want[1]) > 100000
    # every event kind occurs: matches, false positives, misses, identity switches, fragmentations
    n = dev["counts"].sum((0, 1, 2))
    assert n[0] > 0 and n[1] > 0 and n[2] > 0
    assert metrics["FP"] > 0 and metrics["FN"] > 0 and metrics["IDS"] > 0 and metrics["FRAG"] > 0
    T.same(metrics, ENT.score(pk, host))


def test_oracle_agrees_on_a_subset_of_scenes(nusc_val):
    gts, tracks, _ = nusc_val
    keep = [t for t in gts if gts[t]["sequence"] in ("scene0000", "scene0001", "scene0002", "scene0077")]
    g, tr = {t: gts[t] for t in keep}, {t: tracks[t] for t in keep}
    got = ENT.nuscenes_tracking_metrics(g, tr, NF.CLASSES)
    T.same(got, O.tracking_metrics(g, tr, NF.CLASSES))
    assert got["IDS"] > 0 and got["FRAG"] > 0


def test_hand_built_cases_on_the_device():
    for gts, tracks in (T.cardinality_case(),
                        T.scene([([(0, 0, "a", "car")], [(0.5, 0, 0.95, 7, "car")]),
                                 ([(0, 0, "a", "car")], [(1.5, 0, 0.9, 7, "car"), (0.1, 0, 0.92, 8, "car")])])):
        T.same(ENT.nuscenes_tracking_metrics(gts, tracks, T.NAMES),
               ENT.nuscenes_tracking_metrics(gts, tracks, T.NAMES, host=True), tol=0.0)


def test_nusc_dataset_evaluation_tracks_on_the_device(tmp_path):
    from det3d.datasets.nuscenes import NuScenesDataset
    info_name = "infos_train_10sweeps_withvelo_filterZero.pkl"
    root = str(tmp_path / "tree")
    os.makedirs(root)
    names, infos, dets = T.nusc_tracking_tree(root)
    dev = {t: {k: torch.from_numpy(np.asarray(v)) for k, v in d.items()} for t, d in dets.items()}
    outs = []
    for flag in (False, True):
        out = tmp_path / ("out_%d" % flag)
        out.mkdir()
        ds = NuScenesDataset(info_name, root, nsweeps=1, class_names=T.NUSC_TASKS, tracking=flag)
        outs.append((out, ds.evaluation(dev, str(out))))
    (o_off, r_off), (o_on, r_on) = outs
    # the detection JSON is byte-identical with the flag on, and the metrics are unchanged
    assert (o_off / "infos_train_10sweeps_withvelo_filterZero.json").read_bytes() == \
        (o_on / "infos_train_10sweeps_withvelo_filterZero.json").read_bytes()
    assert not (o_off / "infos_train_10sweeps_withvelo_filterZero_tracking.json").exists()
    assert "tracks" not in r_off
    T.same({k: v for k, v in r_on.items() if k != "tracks"}, r_off, tol=0.0)
    # the device tracks equal the host twin's, and the tracking JSON carries them
    ds = NuScenesDataset(info_name, root, nsweeps=1, class_names=T.NUSC_TASKS, tracking=True)
    host = ENT.track_detections(ds.frames(list(dets)), dets, names, host=True)
    js = json.load(open(o_on / "infos_train_10sweeps_withvelo_filterZero_tracking.json"))
    for t in dets:
        np.testing.assert_array_equal(np.asarray(r_on["tracks"][t]["tracking_id"]), host[t]["tracking_id"])
        assert [a["tracking_id"] for a in js["results"][t]] == [str(int(i)) for i in host[t]["tracking_id"]]


def test_train_nds_tracking_experiment_and_gate(tmp_path):
    """6 epochs of synth_det_pp18_aspp_nds_tracking (validation: 3 sequences of 8 frames 0.5 s apart).  The oracle
    detector (fp32 CPU) tracked by oracle/track_oracle.py and scored by oracle/nusc_track_oracle.py, and the fp32-grade
    product detector tracked and scored by the product, agree on every reported tracking number to the third decimal;
    bf16 is reported beside them.  Six epochs do not teach the velocity head, so this checks agreement, not tracking
    quality."""
    import math
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import train as train_tool
    from test_map_gpu import oracle_detections
    from oracle import track_oracle as TO
    from pillarnext_b200 import functional as Fn, hydra_lite, scenes
    from pillarnext_b200 import track as TR
    from pillarnext_b200.trainer import example_to_device
    torch.manual_seed(0)
    name = "synth_det_pp18_aspp_nds_tracking"
    overrides = ["trainer.max_epochs=6", "data.train_dataset.n_frames=640", "data.val_dataset.n_frames=24",
                 "dataloader.train.num_workers=0", "dataloader.val.num_workers=0", "dataloader.train.batch_size=4"]
    tr = train_tool.main(["--config-name", name, "--work-dir", str(tmp_path)] + overrides)
    assert tr.epoch == 6 and "tracking" in tr.last_eval and "NDS" in tr.last_eval
    cfg = hydra_lite.main(os.path.join(ROOT, "configs", "experiments"), name, overrides)
    val = hydra_lite.instantiate(cfg.data.val_dataset)
    assert val.sequence_length == 8 and val.sequence_step_us == 500000
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
    names = val.class_names
    tcls = ENT.tracking_classes(names)
    sub, back = {}, np.array([names.index(n) for n in tcls])
    for t, d in d_oracle.items():
        lab = np.asarray(d["label_preds"]).reshape(-1)
        keep = np.array([names[int(c)] in tcls for c in lab], bool)
        sub[t] = dict(box3d_lidar=np.asarray(d["box3d_lidar"])[keep], scores=np.asarray(d["scores"])[keep],
                      label_preds=np.array([tcls.index(names[int(c)]) for c in lab[keep]], np.int64))
    ids = TO.track(sub, gt, tcls, max_dist=TR.NUSCENES_MAX_DIST)
    o = O.tracking_metrics(gt, {t: dict(d, label_preds=back[d["label_preds"]], tracking_id=ids[t])
                                for t, d in sub.items()}, names)
    s = ENT.track_and_score(gt, product("split"), names)[1]
    b = ENT.track_and_score(gt, product("bf16"), names)[1]
    keys = ("AMOTA", "AMOTP", "MOTA", "MOTP", "recall")
    msg = "; ".join("%s %s" % (who, " / ".join("%.3f" % m[k] for k in keys)) for who, m in
                    (("oracle (fp32 CPU)", o), ("product fp32-grade", s), ("product bf16", b)))
    print("\nAMOTA / AMOTP / MOTA / MOTP / recall: " + msg)
    assert s["per_class"].keys() == o["per_class"].keys()
    for mo, ms in [(o, s)] + [(o["per_class"][c], s["per_class"][c]) for c in o["per_class"]]:
        for k, v in mo.items():
            if k == "per_class":
                continue
            w = ms[k]
            assert (isinstance(v, float) and math.isnan(v) and math.isnan(w)) or round(v, 3) == round(w, 3) or \
                abs(v - w) < 1e-3, (k, v, w, msg)
