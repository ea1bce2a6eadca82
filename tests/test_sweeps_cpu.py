"""Multi-sweep accumulation on the host (ops.accumulate_sweeps_host, pnx_accumulate_sweeps_host) and the moving synthetic
sweeps that feed it (scenes.make_sweep, SyntheticSceneDataset(nsweeps=...), scenes.collate).

* the host twin and the numpy oracle reproduce the reference's own nuScenes and Waymo loaders (tests/golden/
  ref_sweeps.npz) bit for bit;
* at 6 frames x 10 sweeps x 26.5k points the host twin equals the oracle except where numpy's BLAS rounds an fp64 value
  that lies next to an fp32 midpoint the other way (checked exactly with fractions);
* nsweeps = 1 datasets and batches are what they were; drop_frames draws np.random as the reference does; the sweep
  points of every box, taken into the key frame, lie in the box moved back by v * time lag."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import sweeps_oracle as O
from pillarnext_b200 import ops, scenes

OPS = ("points", "point_offsets", "sweep_points", "sweep_offsets", "transforms")
CFG = dict(tasks=[["car"], ["truck", "pedestrian"]], pc_range=[-32.0, -32.0, -5.0, 32.0, 32.0, 3.0],
           voxel_size=[0.5, 0.5, 8], intensity_max=255.0, xy_extent=34.0, z_range=[-5.0, 3.0])


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def golden(case):
    z = np.load(__file__.rsplit("/", 1)[0] + "/golden/ref_sweeps.npz")
    return [z[case + "_" + k] for k in OPS], float(z[case + "_min_distance"]), z[case + "_out"], z


@pytest.mark.parametrize("case", ["nusc", "waymo", "drop"])
def test_host_twin_and_oracle_reproduce_the_reference(case):
    a, md, want, z = golden(case)
    n, S = len(a[0]), len(a[2])
    got, count = ops.accumulate_sweeps_host(*a, md)
    assert count == len(want) and np.array_equal(bits(got[:count]), bits(want))
    assert np.all(got[count:, 0] == len(a[1]) - 1) and not got[count:, 1:].any() and len(got) == n + S
    o, oc = O.accumulate(*a, md)
    assert oc == count and np.array_equal(bits(o), bits(got))
    if case == "nusc":
        assert count < n + S                                     # some sweep points were within 1 m
        k0 = a[0][a[1][0]:a[1][1]]
        assert (np.abs(k0[:, 1:3]) < 1).all(1).any()             # ... but not the key frame's
        assert a[1][2] - a[1][1] == len(want[want[:, 0] == 1])   # frame 1: no sweeps, its key frame alone
        seg3 = slice(*a[3][2:4])                                 # sweep 3 of frame 0 loses every point
        assert (np.abs(a[2][seg3, :2]) < 1).all() and np.isnan(a[4][0, 2, 3, 3])
        assert (bits(a[2][:, :3]) == 0x80000000).any() and (bits(want[:, 1:4]) == 0x80000000).any()   # -0.0 kept
    if case == "waymo":
        assert a[3][3] - a[3][2] > 0 and a[3][4] == a[3][3]      # frame 1: one stored sweep of nsweeps - 1 = 2
    if case == "drop":
        kept = z["drop_kept"]
        assert 0 < kept.sum() < kept.size
        lens = np.diff(a[3]).reshape(kept.shape)
        assert np.array_equal(lens > 0, kept)


def fixed_order(a, md):
    """The library's arithmetic in numpy, elementwise (no BLAS): per output row its source sweep point, the exact
    operands, the "no transform" flags and the expected output rows [count, 6]; key rows get source -1."""
    pts, po, sp, so, tm = a
    B, K = tm.shape[:2]
    seg = np.repeat(np.arange(B * K), np.diff(so))
    m = tm.reshape(-1, 16)[seg]
    x, y, z = (sp[:, j].astype(np.float64) for j in range(3))
    xyz = np.stack([((m[:, 4 * r] * x + m[:, 4 * r + 1] * y) + m[:, 4 * r + 2] * z) + m[:, 4 * r + 3] for r in range(3)], 1)
    none = np.isnan(m[:, 15])
    out = np.where(none[:, None], sp[:, :3], xyz.astype(np.float32))
    keep = ~((np.abs(out[:, 0]) < md) & (np.abs(out[:, 1]) < md)) if md > 0 else np.ones(len(sp), bool)
    src, rows = [], []
    for f in range(B):
        src.append(np.full(po[f + 1] - po[f], -1))
        rows.append(pts[po[f]:po[f + 1]])
        idx = np.arange(so[f * K], so[f * K + K])
        idx = idx[keep[idx]]
        src.append(idx)
        rows.append(np.concatenate([np.full((len(idx), 1), f, np.float32), out[idx], sp[idx, 3:5]], 1))
    return np.concatenate(src), m, none, np.concatenate(rows).astype(np.float32)


def test_host_twin_equals_oracle_at_production_size_up_to_midpoint_ties():
    a = O.random_operands(6, 10, 26500, 1)
    a = [a[k] for k in OPS]
    got, count = ops.accumulate_sweeps_host(*a, 1.0)
    want, wc = O.accumulate(*a, 1.0)
    assert count == wc and 0 < len(got) - count
    assert np.array_equal(bits(got[count:]), bits(want[count:]))
    diff = np.argwhere(bits(got) != bits(want))
    src, m, none, fixed = fixed_order(a, 1.0)
    assert len(src) == count
    assert np.array_equal(bits(got[:count]), bits(fixed))       # the library's arithmetic, elementwise, no exemption
    ties = 0
    for r, c in diff:
        assert 1 <= c <= 3 and src[r] >= 0 and not none[src[r]], (r, c)
        lo, hi = sorted((float(got[r, c]), float(want[r, c])))
        assert np.nextafter(np.float32(lo), np.float32(np.inf)) == np.float32(hi)          # one ulp apart
        p, mm = a[2][src[r]], m[src[r]]
        j = c - 1
        exact = (Fraction(mm[4 * j]) * Fraction(float(p[0])) + Fraction(mm[4 * j + 1]) * Fraction(float(p[1])) +
                 Fraction(mm[4 * j + 2]) * Fraction(float(p[2])) + Fraction(mm[4 * j + 3]))
        mid = (Fraction(lo) + Fraction(hi)) / 2
        assert abs(exact - mid) <= abs(mid) * Fraction(1, 2 ** 50), (r, c, float(exact), lo, hi)
        ties += 1
    print("%d of %d coordinates differ by one ulp next to an fp32 midpoint" % (ties, 3 * count))


def test_nsweeps_1_frames_and_batches_are_unchanged():
    ds = scenes.SyntheticSceneDataset(CFG, 3, seed0=5)
    for i in range(3):
        fr = ds[i]
        pts, boxes, names = scenes.make_scene(5 + i, CFG)
        assert set(fr) == {"points", "gt_boxes_raw", "gt_classes", "token"}
        assert np.array_equal(bits(fr["points"]), bits(pts)) and np.array_equal(bits(fr["gt_boxes_raw"]), bits(boxes))
        assert fr["token"] == "scene_%d" % (5 + i)
    ex = scenes.collate([ds[i] for i in range(3)])
    assert set(ex) == {"points", "gt_boxes_raw", "gt_classes", "token"}
    want = np.concatenate([np.pad(scenes.make_scene(5 + i, CFG)[0], ((0, 0), (1, 0)), constant_values=i) for i in range(3)])
    assert np.array_equal(bits(ex["points"].numpy()), bits(want))
    multi = scenes.SyntheticSceneDataset(CFG, 3, seed0=5, nsweeps=4)
    assert multi.ground_truth().keys() == ds.ground_truth().keys()
    for i in range(3):                                           # the key frame is still make_scene's
        assert np.array_equal(bits(multi[i]["points"]), bits(ds[i]["points"]))
    exm = scenes.collate([multi[i] for i in range(3)])
    assert np.array_equal(bits(exm["points"].numpy()), bits(want))
    assert exm["sweep_transforms"].shape == (3, 3, 4, 4) and exm["sweep_offsets"].shape == (10,)
    assert exm["point_offsets"].tolist() == [0] + np.cumsum([len(ds[i]["points"]) for i in range(3)]).tolist()


def test_drop_frames_draws_np_random_in_the_reference_order():
    _, _, _, z = golden("drop")
    ds = scenes.SyntheticSceneDataset(CFG, 8, nsweeps=3, drop_frames=0.5, n_points=600)
    state = np.random.get_state()
    try:
        np.random.seed(int(z["drop_seed"]))
        kept = [ds[i]["sweeps"]["counts"] > 0 for i in range(8)]
        nxt = np.random.uniform()
    finally:
        np.random.set_state(state)
    assert np.array_equal(np.array(kept), z["drop_kept"]) and nxt == float(z["drop_next"])


def test_sweep_points_of_each_box_lie_in_the_box_moved_back_by_its_velocity():
    pts, boxes, _ = scenes.make_scene(3, CFG)
    moving = np.hypot(boxes[:, 6], boxes[:, 7]) > 0.5
    assert moving.any()
    for k in (1, 5, 9):
        sw, T, owner = scenes.make_sweep(3, k, CFG, boxes, 6000)
        lag = k * 0.05
        assert sw.dtype == np.float32 and (sw[:, 4] == np.float32(lag)).all()
        assert not np.allclose(T[:2, :2], np.eye(2)) and np.hypot(*T[:2, 3]) > 0
        key = (np.c_[sw[:, :3].astype(np.float64), np.ones(len(sw))] @ T.T)[:, :3]
        for j, b in enumerate(boxes.astype(np.float64)):
            p = key[owner == j]
            assert len(p) > 0
            c = b[:2] - b[6:8] * lag
            cs, sn = np.cos(-b[8]), np.sin(-b[8])
            lx = (p[:, 0] - c[0]) * cs - (p[:, 1] - c[1]) * sn
            ly = (p[:, 0] - c[0]) * sn + (p[:, 1] - c[1]) * cs
            tol = 0.1                                            # the 2 cm surface noise
            assert (np.abs(lx) <= b[3] / 2 + tol).all() and (np.abs(ly) <= b[4] / 2 + tol).all()
            assert (np.abs(p[:, 2] - b[2]) <= b[5] / 2 + tol).all()
            if moving[j] and k == 9:                             # ... and not where the box is at the key frame
                lx0 = (p[:, 0] - b[0]) * cs - (p[:, 1] - b[1]) * sn
                ly0 = (p[:, 0] - b[0]) * sn + (p[:, 1] - b[1]) * cs
                assert not ((np.abs(lx0) <= b[3] / 2 + tol) & (np.abs(ly0) <= b[4] / 2 + tol)).all()
        ground = key[owner < 0]
        for b in boxes.astype(np.float64):                       # no ground returns under the moved boxes
            c = b[:2] - b[6:8] * lag
            cs, sn = np.cos(-b[8]), np.sin(-b[8])
            lx = (ground[:, 0] - c[0]) * cs - (ground[:, 1] - c[1]) * sn
            ly = (ground[:, 0] - c[0]) * sn + (ground[:, 1] - c[1]) * cs
            assert not ((np.abs(lx) < b[3] / 2 - 1e-6) & (np.abs(ly) < b[4] / 2 - 1e-6)).any()


def test_host_wrapper_checks_its_operands():
    a, md, want, _ = golden("nusc")
    with pytest.raises(ValueError, match="points"):
        ops.accumulate_sweeps_host(a[0].astype(np.float64), *a[1:], md)
    with pytest.raises(ValueError, match="sweep_points"):
        ops.accumulate_sweeps_host(a[0], a[1], a[2].astype(np.float64), *a[3:], md)
    with pytest.raises(ValueError, match="points"):
        ops.accumulate_sweeps_host(a[0][:, :5], *a[1:], md)
    with pytest.raises(ValueError, match="sweep_points"):
        ops.accumulate_sweeps_host(a[0], a[1], np.c_[a[2], a[2][:, :1]], *a[3:], md)
    with pytest.raises(ValueError, match="transforms"):
        ops.accumulate_sweeps_host(*a[:4], a[4].astype(np.float32), md)
    with pytest.raises(ValueError, match="sweep_offsets"):
        ops.accumulate_sweeps_host(a[0], a[1], a[2], a[3][:-1], a[4], md)
    with pytest.raises(ValueError, match="sweep_points"):
        ops.accumulate_sweeps_host(a[0], a[1], torch.from_numpy(a[2]), *a[3:], md)
    wide = np.zeros((len(a[0]), 9), np.float32)                  # non-contiguous views are accepted
    wide[:, 2:8] = a[0]
    swide = np.zeros((len(a[2]), 7), np.float32)
    swide[:, 1:6] = a[2]
    got, count = ops.accumulate_sweeps_host(wide[:, 2:8], a[1], swide[:, 1:6], *a[3:], md)
    assert count == len(want) and np.array_equal(bits(got[:count]), bits(want))
    with pytest.raises(RuntimeError, match="min_distance"):
        ops.accumulate_sweeps_host(*a, -1.0)
