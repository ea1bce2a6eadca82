"""Global training augmentation (rotation, scaling, translation, flip), CPU only.

* the drop-in transforms (det3d/datasets/pipelines/augmentation.py), seeded like the reference, make the reference's
  np.random calls and yield its parameters (tests/golden/ref_aug.npz, frozen by oracle/make_golden_aug.py);
* the product's per-point / per-box math compiled for the host (pnx_global_aug_host) reproduces the reference's numpy
  outputs bit for bit, NaN elements, yaw wrap and far-away coordinates included; so does the numpy oracle;
* the augmentation nodes of the reference's experiments instantiate the drop-in classes with the reference's values;
* dataset and collate: test mode refuses augmentation, no `aug` key without it, one record per op with it.
"""
import json
import os

import numpy as np
import pytest
import torch
import yaml

from det3d.datasets.pipelines import augmentation as A
from oracle import aug_oracle
from pillarnext_b200 import hydra_lite, modules, scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
EXPERIMENTS = os.path.join(ROOT, "configs", "experiments")


def golden():
    return np.load(os.path.join(GOLDEN, "ref_aug.npz"))


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


@pytest.fixture
def np_random_state():
    state = np.random.get_state()
    yield
    np.random.set_state(state)


def host_aug(points, boxes, aug):
    from pillarnext_b200 import ops
    return ops.global_aug_host(np.asarray(points, np.float32), np.asarray(boxes, np.float32), np.asarray(aug, np.float64))


def test_dropin_classes_draw_the_reference_parameters(np_random_state, monkeypatch):
    g = golden()
    chains, calls = json.loads(str(g["chains"])), json.loads(str(g["calls"]))
    log = []
    for name in ("uniform", "normal", "choice"):
        fn = getattr(np.random, name)
        monkeypatch.setattr(np.random, name, lambda *a, _fn=fn, _n=name, **k: (log.append(_n), _fn(*a, **k))[1])
    for f, chain in enumerate(chains):
        np.random.seed(int(g["seeds"][f]))
        log.clear()
        res = {}
        for name, kw in chain:
            res = getattr(A, name)(**kw)(res)
        assert log == calls[f], (f, chain)
        want = [tuple(r) for r in g["aug"][f] if r[0] != 0]
        assert res["aug"] == want, (f, res["aug"], want)
        assert np.random.random_sample() == g["next_draw"][f]          # same state after the chain: nothing extra drawn
    assert {tuple(r[1:3]) for r in g["aug"].reshape(-1, 4) if r[0] == A.FLIP} == {(0.0, 0.0), (1.0, 0.0), (0.0, 1.0), (1.0, 1.0)}


def test_host_twin_reproduces_the_reference_bit_for_bit():
    g = golden()
    p_in, b_in = g["points"].copy(), g["boxes"].copy()
    p, b = host_aug(g["points"], g["boxes"], g["aug"])
    assert np.array_equal(bits(p), bits(g["out_points"]))
    assert np.array_equal(bits(b), bits(g["out_boxes"]))        # NaNs compared by bit pattern
    assert np.array_equal(bits(g["points"]), bits(p_in)) and np.array_equal(bits(g["boxes"]), bits(b_in))
    # the goldens exercise what they claim to: NaNs kept, yaws wrapped across +-pi, far-away points moved
    assert np.isnan(b).sum() == np.isnan(g["boxes"]).sum() > 0
    yaw_in, yaw_out = g["boxes"][..., 8], b[..., 8]
    assert (np.abs(yaw_in) >= np.float32(np.pi) - 1e-3).sum() >= 4 * len(b)
    assert np.nanmax(np.abs(yaw_out)) > np.pi and np.abs(p[:, 1:4]).max() > 1e4


def test_oracle_reproduces_the_reference_bit_for_bit():
    g = golden()
    p, b = aug_oracle.apply(g["points"], g["boxes"], g["aug"])
    assert np.array_equal(bits(p), bits(g["out_points"])) and np.array_equal(bits(b), bits(g["out_boxes"]))


def test_host_twin_matches_the_oracle_on_a_full_batch(np_random_state):
    """6 frames x 30k points, the reference's chain: the fp64 rotation, the roundings and the yaw wrap agree on every
    element, not only on the golden frames."""
    rng = np.random.default_rng(3)
    B, n, M = 6, 30000, 40
    pts = np.concatenate([np.concatenate([np.full((n, 1), f), rng.uniform(-60, 60, (n, 2)), rng.uniform(-4, 3, (n, 1)),
                                          rng.uniform(0, 255, (n, 1)), np.zeros((n, 1))], 1) for f in range(B)]).astype(np.float32)
    boxes = np.concatenate([rng.uniform(-60, 60, (B, M, 3)), rng.uniform(0.3, 12, (B, M, 3)), rng.normal(0, 3, (B, M, 2)),
                            rng.uniform(-np.pi, np.pi, (B, M, 1))], 2).astype(np.float32)
    boxes[:, ::7, 6:8] = np.nan
    np.random.seed(11)
    aug = np.zeros((B, 4, 4))
    ops = [A.Rotation([-0.785, 0.785]), A.Scaling([0.9, 1.1]), A.Translation(0.5), A.Flip([0.5, 0.5])]
    for f in range(B):
        res = {}
        for op in ops:
            res = op(res)
        aug[f] = res["aug"]
    p_h, b_h = host_aug(pts, boxes, aug)
    p_o, b_o = aug_oracle.apply(pts, boxes, aug)
    assert np.array_equal(bits(p_h), bits(p_o)) and np.array_equal(bits(b_h), bits(b_o))


@pytest.mark.parametrize("experiment", ["nusc_det_pp18_aspp_iou_sp", "waymo_det_pp18_aspp_iou_car_sp"])
def test_reference_augmentation_nodes_instantiate_the_dropin_classes(experiment):
    with open(os.path.join(GOLDEN, "ref_aug_configs.json")) as fh:
        node = json.load(fh)[experiment]
    assert list(node) == ["rotation", "scaling", "translation", "flip"]
    objs = hydra_lite.instantiate(node)
    assert list(objs) == list(node)
    assert isinstance(objs.rotation, A.Rotation) and list(objs.rotation.rotation) == [-0.785, 0.785]
    assert isinstance(objs.scaling, A.Scaling) and (objs.scaling.min_scale, objs.scaling.max_scale) == (0.9, 1.1)
    assert isinstance(objs.translation, A.Translation) and objs.translation.noise == 0.5
    assert isinstance(objs.flip, A.Flip) and list(objs.flip.flip_prob) == [0.5, 0.5]
    with open(os.path.join(ROOT, "configs", "dataset", "preprocess", "augmentation.yaml")) as fh:
        assert yaml.safe_load(fh) == node                      # this repo's preprocess group is the reference's


def test_flip_keeps_the_reference_assertions():
    with pytest.raises(AssertionError):
        A.Flip([1.0, 0.5])
    with pytest.raises(AssertionError):
        A.Flip([0.5, -0.1])


def test_test_mode_dataset_with_augmentation_raises():
    cfg = hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp_aug", [])
    node = dict(cfg.data.val_dataset, augmentation=cfg.data.train_dataset.augmentation)
    with pytest.raises(ValueError, match="test_mode"):
        hydra_lite.instantiate(node)


def test_collate_without_augmentation_has_no_aug_key():
    cfg = hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp", ["data.train_dataset.n_frames=2"])
    ds = hydra_lite.instantiate(cfg.data.train_dataset)
    assert ds.augmentations is None
    ex = scenes.collate([ds[0], ds[1]])
    assert "aug" not in ex and "aug" not in ds[0]


def test_augmented_collate_packs_one_record_per_op(np_random_state):
    cfg = hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp_aug", ["data.train_dataset.n_frames=3"])
    ds = hydra_lite.instantiate(cfg.data.train_dataset)
    plain = hydra_lite.instantiate(hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp", []).data.train_dataset)
    np.random.seed(5)
    items = [ds[i] for i in range(3)]
    ex = scenes.collate(items)
    assert ex["aug"].dtype == torch.float64 and tuple(ex["aug"].shape) == (3, 4, 4)
    assert ex["aug"][:, :, 0].tolist() == [[A.ROTATION, A.SCALING, A.TRANSLATION, A.FLIP]] * 3
    assert all(r[2] == np.cos(r[1]) and r[3] == np.sin(r[1]) for r in ex["aug"][:, 0].numpy())   # numpy's cos / sin
    # the scene itself is untouched on the host: the GPU applies the records
    ref = plain[0]
    assert np.array_equal(items[0]["points"], ref["points"]) and np.array_equal(items[0]["gt_boxes_raw"], ref["gt_boxes_raw"])
    with pytest.raises(ValueError, match="at most 4"):
        scenes.collate([dict(items[0], aug=items[0]["aug"] + [(A.FLIP, 1.0, 0.0, 0.0)])])


def test_augmentation_after_label_assignment_is_an_error():
    with pytest.raises(ValueError, match="assigned labels"):
        modules.SingleStageDetector.global_aug(None, {"hm": [], "aug": torch.zeros(1, 4, 4, dtype=torch.float64)})
