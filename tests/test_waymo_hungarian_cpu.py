"""Waymo-style AP / APH with matching="hungarian" (pillarnext_b200/evaluate_waymo.py) without a GPU: the host twins of
pnx_eval_pairs / pnx_eval_components / pnx_eval_assign against scipy's linear_sum_assignment with the same tie rule
(oracle/waymo_hungarian_oracle.py), hand-made cases where greedy and optimal matching differ, a component larger than
the one-warp solver takes, the whole metric dict against the oracle, and self-checks of the comparison."""
import json
import math
import os

import numpy as np
import pytest

from oracle import predict_oracle as P, waymo_fixtures
from oracle import waymo_hungarian_oracle as H
from pillarnext_b200 import evaluate_waymo as EW

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def hungarian_host(gts, detections, classes, iou_thresholds=None, k=11):
    pk = EW.pack_hungarian(gts, detections, classes, iou_thresholds, k)
    counts, match, heading = EW.run_host_hungarian(pk)
    return EW.score_hungarian(pk, EW.known_counts(pk, counts), match, heading, classes), pk, match


def greedy_host(gts, detections, classes, iou_thresholds=None):
    pk = EW.pack(gts, detections, classes, iou_thresholds)
    counts, match, _, heading = EW.run_host(pk)
    return EW.score(pk, EW.known_counts(pk, counts), match, heading, classes)


def box9(rows):
    b = np.asarray(rows, np.float32).reshape(-1, 7)
    out = np.zeros((len(b), 9), np.float32)
    out[:, :6], out[:, 8] = b[:, :6], b[:, 6]
    return out


def along_x(xs, length=4.0, y=0.0):
    """Equal boxes (length x 2 x 1.7, yaw 0) at the given x: a shift s between two gives IoU (length - s) / (length + s)."""
    return [[x, y, 0.85, length, 2.0, 1.7, 0.0] for x in xs]


def scene(gt_xs, det_xs, scores, y=0.0, npts=20):
    gts = {"a": {"boxes": box9(along_x(gt_xs, y=y)), "names": ["vehicle"] * len(gt_xs),
                 "num_points": np.full(len(gt_xs), npts, np.int64)}}
    det = {"a": {"box3d_lidar": box9(along_x(det_xs, y=y)), "scores": np.asarray(scores, np.float32),
                 "label_preds": np.zeros(len(det_xs), np.int64)}}
    return gts, det


def assert_same(got, want, tol=1e-9, where=""):
    """Every value of the nested dicts within tol; APH values within 1e-5, as the product's heading accuracy is fp32 (the
    greedy match's routine) and the oracle's fp64."""
    if isinstance(want, dict):
        assert set(got) == set(want), (where, set(got) ^ set(want))
        for k in want:
            assert_same(got[k], want[k], max(tol, 1e-5) if "APH" in str(k) else tol, where + "/" + str(k))
        return
    if isinstance(want, float) and math.isnan(want):
        assert math.isnan(got), (where, got)
        return
    assert abs(got - want) <= tol, (where, got, want)


def test_optimal_matching_pairs_both_detections_where_greedy_pairs_one():
    """Boxes A (x = 0) and B (x = 1); d1 (x = 0.4, score 0.9): IoU 0.818 with A, 0.739 with B; d2 (x = -1, score 0.8):
    0.6 with A, 0.333 with B.  Greedy: d1 takes A, d2 nothing (AP 50: a TP, then an FP).  Maximum IoU: d1-B + d2-A =
    1.339 > 0.818.  Cutoffs (n = 2, K = 11): 0.8 for k < 6, 0.9 after.  At 0.8 both match: recall 1, precision 1; at 0.9
    d1 alone takes A: recall 0.5, precision 1.  AP 100."""
    gts, det = scene([0.0, 1.0], [0.4, -1.0], [0.9, 0.8])
    thr = {"vehicle": 0.5}
    r, pk, match = hungarian_host(gts, det, ["vehicle"], thr)
    assert [list(c) for c in pk["cutoffs"]] == [[np.float32(0.8)] * 6 + [np.float32(0.9)] * 5]
    assert match[0, 0].tolist() == [1, 0] and match[0, 10].tolist() == [0, -1]
    assert abs(r["mAP_L2"] - 100.0) < 1e-12 and abs(r["mAPH_L1"] - 100.0) < 1e-12
    assert abs(greedy_host(gts, det, ["vehicle"], thr)["mAP_L2"] - 50.0) < 1e-12
    assert_same(r, H.waymo_metrics(gts, det, ["vehicle"], thr))


def test_fewer_pairs_can_win_and_the_points_are_not_monotone():
    """d1 (score 0.9, x = 0.5) overlaps A (x = 0: 0.778) and B (x = 1: 0.778); d2 (score 0.5, x = 1.1) overlaps only B
    (0.951).  Optimal: d1-A + d2-B.  Add d3 (score 0.7, x = 0.05) overlapping A at 0.975 and B at 0.655: at the 0.5
    cutoff d3-A + d2-B (1.926) beats d1-A + d2-B; d1 is an FP.  By hand at K = 3 (cutoffs 0.5, 0.7, 0.9): (TP, FP) =
    (2, 1), (2, 0) -- d1-B + d3-A = 1.753 > 0.975 -- and (1, 0): recall 1, 1, 0.5 with precision 2/3, 1, 1.  Sorted by
    recall (stable): (0.5, 1), (1, 2/3), (1, 1); envelope 1, 1, 1: AP 100."""
    gts, det = scene([0.0, 1.0], [0.5, 1.1, 0.05], [0.9, 0.5, 0.7])
    r, _, match = hungarian_host(gts, det, ["vehicle"], {"vehicle": 0.5}, k=3)
    assert match[0].tolist() == [[-1, 1, 0], [1, -1, 0], [0, -1, -1]]
    assert abs(r["mAP_L2"] - 100.0) < 1e-12
    assert_same(r, H.waymo_metrics(gts, det, ["vehicle"], {"vehicle": 0.5}, 3))


def test_ties_go_to_the_higher_score_then_the_lower_box():
    """Two identical detections on one box: the higher score takes it (the other is an FP); one detection exactly
    between two equal boxes takes the lower index."""
    gts, det = scene([0.0], [0.0, 0.0], [0.6, 0.9])
    _, _, match = hungarian_host(gts, det, ["vehicle"], k=1)
    assert match[:, 0].tolist() == [[-1, 0], [-1, 0]]
    gts, det = scene([1.0, -1.0], [0.0], [0.9])
    _, _, match = hungarian_host(gts, det, ["vehicle"], {"vehicle": 0.5}, k=1)
    assert match[:, 0].tolist() == [[0], [0]]


def test_range_breakdown_splits_by_centre_distance():
    """A box at 29.9 m and its detection at 30.1 m: matched in ALL, not within a range; each range scores its own."""
    gts, det = scene([29.9, 60.0], [30.1, 60.0], [0.9, 0.8])
    r, pk, match = hungarian_host(gts, det, ["vehicle"], {"vehicle": 0.5}, k=2)
    assert pk["gt_range"][:2].tolist() == [0, 2] and pk["det_range"].tolist() == [1, 2]
    assert match[0, 0].tolist() == [0, 1] and match[1, 0].tolist() == [-1, 1]
    pr = r["per_range"]["vehicle"]
    assert (pr["0-30"]["AP_L2"], pr["0-30"]["n_gt_L2"]) == (0.0, 1) and pr["50+"]["AP_L2"] == 100.0
    assert math.isnan(pr["30-50"]["AP_L2"]) and r["range_means"]["50+"]["mAP_L2"] == 100.0
    assert r["mAP_L2"] == 100.0
    assert_same(r, H.waymo_metrics(gts, det, ["vehicle"], {"vehicle": 0.5}, 2))


def chain(n, seed=0):
    """n detections between n + 1 boxes one metre apart: each detection overlaps its two neighbours at the same IoU
    (0.778), one component of 2 n pairs in which every maximum pairs all detections -- ties everywhere."""
    rng = np.random.default_rng(seed)
    return scene(np.arange(n + 1, dtype=np.float64), np.arange(n) + 0.5, rng.permutation(n) / n + 0.01)


def test_component_larger_than_a_warp_follows_the_tie_rule():
    gts, det = chain(40)
    pk = EW.pack_hungarian(gts, det, ["vehicle"], {"vehicle": 0.5}, 4)
    from pillarnext_b200 import ops
    order = np.argsort(pk["keys"], kind="stable").astype(np.int64)
    start, e_det, e_box, e_iou, _ = ops.eval_pairs_host(pk["det_boxes"], pk["det_trig"], order, pk["seg_start"],
                                                     pk["seg_count"], pk["gt_boxes"], pk["gt_classes"], pk["gt_trig"],
                                                     pk["thresholds"])
    comp_start, comp_nedge, _ = ops.eval_components_host(start, e_det, e_box, pk["M"], pk["C"])
    assert comp_nedge.max() == 80 and (comp_nedge > 0).sum() == 1            # one component, beyond the 32-pair warp
    check_assignments(gts, det, ["vehicle"], {"vehicle": 0.5}, 4)


def check_assignments(gts, det, classes, thr=None, k=11, iou=None):
    """Every (frame, class, breakdown, cutoff) assignment of the host twins: the same total IoU and number of pairs as
    linear_sum_assignment, and the same pairs under the tie rule.  Returns (assignments compared, pairs)."""
    r, pk, match = hungarian_host(gts, det, classes, thr, k)
    thresholds = EW.class_thresholds(classes, thr)
    n_cmp = n_pairs = 0
    off = 0
    for f, t in enumerate(gts):
        g, d = gts[t], det[t]
        nd = len(d["scores"])
        b7 = g["boxes"][:, [0, 1, 2, 3, 4, 5, 8]]
        d7 = d["box3d_lidar"][:, [0, 1, 2, 3, 4, 5, 8]]
        pair = iou or (lambda i, j: P.aligned_iou3d(d7[i], b7[j]))
        for kc in range(k):
            cut = [pk["cutoffs"][c][kc] if len(pk["cutoffs"][c]) else np.float32(np.inf) for c in range(len(classes))]
            for b in (0, 1):
                got = match[b, kc, off:off + nd]
                for name, (want, best, w) in H.frame_assignments(g["boxes"], g["names"], d["box3d_lidar"], d["scores"],
                                                                d["label_preds"], classes, thresholds, cut, b,
                                                                pair).items():
                    c = classes.index(name)
                    mine = {i: int(got[i]) for i in range(nd) if d["label_preds"][i] == c and got[i] >= 0}
                    total = sum(w.get((i, j), -1e9) for i, j in mine.items())
                    assert total == best and len(mine) == len(want), (t, name, kc, b, total, best)
                    assert mine == want, (t, name, kc, b, mine, want)
                    n_cmp += 1
                    n_pairs += len(mine)
        off += nd
    return n_cmp, n_pairs


def test_host_twins_equal_linear_sum_assignment_on_crowded_scenes():
    gts, det, classes = waymo_fixtures.make_frames(41, 3, n_points=100, n_labels=(14, 10, 6), fp_per_class=(14, 10, 8),
                                                   extent=5.0)
    n_cmp, n_pairs = check_assignments(gts, det, classes)
    assert n_cmp == 3 * 3 * 2 * 11 and n_pairs > 300


def test_metric_dict_equals_the_oracle_on_20_frames():
    gts, det, classes = waymo_fixtures.make_frames(43, 20, n_points=3000, n_labels=(30, 15, 4), fp_per_class=(20, 15, 6),
                                                   extent=60.0)
    got = hungarian_host(gts, det, classes)[0]
    want = H.waymo_metrics(gts, det, classes)
    assert_same(got, want)
    assert 5 < got["mAPH_L2"] < got["mAP_L2"] < 100
    for r in EW.RANGES:
        assert got["per_range"]["vehicle"][r]["n_gt_L2"] > 0


def test_the_comparison_sees_a_dropped_pair_and_shifted_cutoffs(monkeypatch):
    gts, det, classes = waymo_fixtures.make_frames(43, 20, n_points=3000, n_labels=(30, 15, 4), fp_per_class=(20, 15, 6),
                                                   extent=60.0)
    got, pk, match = hungarian_host(gts, det, classes)
    # the feasible pair closest above its threshold among the pairs matched at the lowest cutoff
    f, lab = pk["det_frames"], pk["det_labels"]
    thr = np.array(EW.class_thresholds(classes), np.float32)
    best = None
    for i in np.nonzero(match[0, 0] >= 0)[0]:
        g = pk["gt_boxes"][f[i], match[0, 0, i]]
        v = np.float32(P.aligned_iou3d(pk["det_boxes"][i, [0, 1, 2, 3, 4, 5, 8]], g[[0, 1, 2, 3, 4, 5, 8]]))
        if best is None or v - thr[lab[i]] < best[0]:
            best = (v - thr[lab[i]], pk["det_boxes"][i, [0, 1, 2, 3, 4, 5, 8]].copy())
    assert best[0] < 0.01
    real = P.aligned_iou3d
    monkeypatch.setattr(H.P, "aligned_iou3d", lambda a, b: 0.0 if np.array_equal(np.float32(a), best[1]) else real(a, b))
    with pytest.raises(AssertionError):
        assert_same(got, H.waymo_metrics(gts, det, classes))
    monkeypatch.setattr(H.P, "aligned_iou3d", real)
    def shifted(scores, k):                                     # s_(floor(i n / K) + 1): every cutoff one score up
        s = sorted(np.float32(v) for v in scores)
        return [s[min(len(s) - 1, (i * len(s)) // k + 1)] for i in range(k)] if s else []
    monkeypatch.setattr(H, "cutoffs", shifted)
    with pytest.raises(AssertionError):
        assert_same(got, H.waymo_metrics(gts, det, classes))


def test_greedy_mode_equals_the_parent_output():
    """matching="greedy" (the default) gives what the greedy-only metric gave, to the bit: recorded from it on the
    same seeded input (tests/golden/waymo_greedy_parent.json)."""
    rec = json.load(open(os.path.join(ROOT, "tests", "golden", "waymo_greedy_parent.json")))
    inp = rec["input"]
    gts, det, classes = waymo_fixtures.make_frames(inp["seed"], inp["n_frames"], n_points=inp["n_points"],
                                                   extent=inp["extent"])
    assert_greedy_equals_record(greedy_host(gts, det, classes), rec["result"])


def assert_greedy_equals_record(got, rec, where=""):
    if isinstance(rec, dict):
        assert set(got) == set(rec), where
        for k in rec:
            assert_greedy_equals_record(got[k], rec[k], where + "/" + k)
    elif isinstance(rec, str):
        assert float(got).hex() == rec or (math.isnan(got) and rec == "nan"), (where, float(got).hex(), rec)
    else:
        assert got == rec, (where, got, rec)


def test_matching_options():
    gts, det = scene([0.0], [0.1], [0.9])
    with pytest.raises(ValueError):
        EW.waymo_metrics(gts, det, ["vehicle"], matching="optimal")
    with pytest.raises(ValueError):
        EW.pack_hungarian(gts, det, ["vehicle"], {"vehicle": 1e-6})
    with pytest.raises(ValueError):
        EW.pack_hungarian(gts, det, ["vehicle"], None, 0)


def test_hungarian_experiment_composes():
    from pillarnext_b200 import hydra_lite
    cfg = hydra_lite.main(os.path.join(ROOT, "configs", "experiments"), "synth_det_pp18_aspp_waymo_hungarian", [])
    val = hydra_lite.instantiate(cfg.data.val_dataset)
    assert val.metric == "waymo" and val.waymo_matching == "hungarian"
    train = hydra_lite.instantiate(cfg.data.train_dataset)
    assert train.waymo_matching == "greedy"


def test_heading_accuracy_is_the_greedy_match_routine():
    """Where the greedy match and the Hungarian one (lowest cutoff, ALL) pair a detection with the same box, the heading
    accuracy is the same fp32 value, bit for bit."""
    gts, det, classes = waymo_fixtures.make_frames(41, 3, n_points=100, extent=20.0)
    pk = EW.pack_hungarian(gts, det, classes)
    _, match, heading = EW.run_host_hungarian(pk)
    _, g_match, _, g_heading = EW.run_host(pk)
    same = (g_match >= 0) & (g_match == match[0, 0])
    assert same.sum() > 100
    assert np.array_equal(heading[0, 0, same].view(np.int32), g_heading[same].view(np.int32))
    assert (heading[match < 0] == 0).all() and (heading[match >= 0] < 1).any()
