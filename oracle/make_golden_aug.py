"""Freeze the reference's OWN global augmentation into tests/golden/ref_aug.npz, and the augmentation nodes of its
experiments into tests/golden/ref_aug_configs.json (TEST INFRASTRUCTURE; run where the reference tree is present).

ref_aug.npz: one frame per case.  Each case seeds np.random, runs a chain of the reference's transforms
(det3d/datasets/pipelines/augmentation.py, on top of its box_np_ops) on fp32 points and boxes, and records every
np.random call the chain makes.  Cases: each op alone, both flips alone and together, the reference's chain in config
order with all four flip outcomes, and a reordered chain.  The boxes include yaws at and near +-pi, NaN velocities,
a NaN yaw, a padding row as scenes.collate writes it and coordinates far outside any pc_range.  Stored:
  points [N, 6] (frame index, x, y, z, intensity, time), boxes [B, M, 9]    inputs
  out_points, out_boxes                                                        the reference's outputs
  aug [B, 4, 4]          the records (code, p0, p1, p2) built from the reference's own draws
  seeds [B], next_draw [B]  np.random.seed per case, np.random.random_sample() right after the chain
  chains, calls          JSON: the chain per case ([class name, kwargs]) and the np.random function names it called

ref_aug_configs.json: data.train_dataset.augmentation of every reference experiment, composed and resolved with
pillarnext_b200.hydra_lite (the tests run without the reference tree).

    python -m oracle.make_golden_aug
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np

from oracle import reference_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
N_POINTS, N_BOXES = 48, 8
FULL = [("Rotation", dict(rotation=[-0.785, 0.785])), ("Scaling", dict(scale=[0.9, 1.1])),
        ("Translation", dict(noise=0.5)), ("Flip", dict(flip_prob=[0.5, 0.5]))]
# (chain, wanted (x flip, y flip) or None)
CASES = [
    ([FULL[0]], None),
    ([("Rotation", dict(rotation=[-3.2, 3.2]))], None),
    ([FULL[1]], None),
    ([FULL[2]], None),
    ([("Flip", dict(flip_prob=[0.5, 0.0]))], (True, False)),
    ([("Flip", dict(flip_prob=[0.0, 0.5]))], (False, True)),
    ([FULL[3]], (True, True)),
    ([FULL[3]], (False, False)),
    (FULL, (False, False)),
    (FULL, (True, False)),
    (FULL, (False, True)),
    (FULL, (True, True)),
    ([FULL[3], FULL[2], FULL[1], FULL[0]], (True, True)),
]


def load_reference_augmentation():
    """The reference's augmentation module, importing its own box_np_ops (this repo's `det3d` package is set aside
    while it loads)."""
    ref = reference_loader.REF_ROOT
    spec = importlib.util.spec_from_file_location("ref_box_np_ops", os.path.join(ref, "det3d", "core", "bbox", "box_np_ops.py"))
    box_np_ops = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(box_np_ops)
    names = ["det3d", "det3d.core", "det3d.core.bbox", "det3d.core.bbox.box_np_ops"]
    saved = {n: sys.modules.get(n) for n in names}
    pkgs = [types.ModuleType(n) for n in names[:3]] + [box_np_ops]
    for parent, child, attr in zip(pkgs, pkgs[1:], ("core", "bbox", "box_np_ops")):
        setattr(parent, attr, child)
    sys.modules.update(dict(zip(names, pkgs)))
    try:
        spec = importlib.util.spec_from_file_location(
            "ref_augmentation", os.path.join(ref, "det3d", "datasets", "pipelines", "augmentation.py"))
        aug = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(aug)
    finally:
        for n, m in saved.items():
            if m is None:
                sys.modules.pop(n, None)
            else:
                sys.modules[n] = m
    return aug


def frame(case):
    """Points [N_POINTS, 5] and boxes [N_BOXES, 9], fp32."""
    g = np.random.default_rng(500 + case)
    pts = np.zeros((N_POINTS, 5))
    pts[:, 0:2] = g.uniform(-60, 60, (N_POINTS, 2))
    pts[:, 2] = g.uniform(-3, 2, N_POINTS)
    pts[:, 3] = g.uniform(0, 255, N_POINTS)
    pts[:, 4] = g.uniform(0, 0.5, N_POINTS)
    pts[:4, :3] = [[1.0e3, -2.0e3, 40.0], [-2.5e4, 3.0e3, -15.0], [0.0, 0.0, 0.0], [7.5e4, 1.0e-3, 3.0e2]]
    b = np.zeros((N_BOXES, 9))
    b[:, 0:2] = g.uniform(-50, 50, (N_BOXES, 2))
    b[:, 2] = g.uniform(-2, 1, N_BOXES)
    b[:, 3:6] = g.uniform(0.5, 5, (N_BOXES, 3))
    b[:, 6:8] = g.normal(0, 3, (N_BOXES, 2))
    b[:, 8] = g.uniform(-np.pi, np.pi, N_BOXES)
    b[1, 8], b[2, 8], b[3, 8], b[4, 8] = np.pi, -np.pi, np.pi - 1e-4, -np.pi + 1e-4
    b[3, 6] = np.nan                                            # vx NaN: rotation computes vy' with vx = 0
    b[4, 7] = np.nan
    b[5, 6:8] = np.nan
    b[5, 0:2] = [500.0, -800.0]
    b[6] = [0, 0, 0, 1, 1, 1, 0, 0, 0]                          # padding row of scenes.collate
    b[7, 0:2], b[7, 8] = [-2.5e4, 3.0e3], np.nan
    return pts.astype(np.float32), b.astype(np.float32)


class DrawLog:
    """Records np.random.uniform / normal / choice calls (name, result) while active."""

    def __init__(self):
        self.calls = []

    def __enter__(self):
        self.saved = {n: getattr(np.random, n) for n in ("uniform", "normal", "choice")}
        for n, fn in self.saved.items():
            setattr(np.random, n, self._wrap(n, fn))
        return self

    def _wrap(self, name, fn):
        def call(*a, **k):
            r = fn(*a, **k)
            self.calls.append((name, r))
            return r
        return call

    def __exit__(self, *exc):
        for n, fn in self.saved.items():
            setattr(np.random, n, fn)


def records(chain, calls):
    """aug rows (code, p0, p1, p2) from the draws the reference made for `chain`."""
    it = iter(calls)
    rows = []
    for name, kw in chain:
        if name == "Rotation":
            fn, th = next(it)
            assert fn == "uniform"
            rows.append((1.0, th, np.cos(th), np.sin(th)))
        elif name == "Scaling":
            fn, s = next(it)
            assert fn == "uniform"
            rows.append((2.0, s, 0.0, 0.0))
        elif name == "Translation":
            fn, t = next(it)
            assert fn == "normal" and t.shape == (1,)
            rows.append((3.0, t[0], 0.0, 0.0))
        else:
            f = []
            for p in kw["flip_prob"]:
                if p > 0:
                    fn, e = next(it)
                    assert fn == "choice"
                    f.append(float(bool(e)))
                else:
                    f.append(0.0)
            rows.append((4.0, f[0], f[1], 0.0))
    assert next(it, None) is None
    return np.array(rows + [(0.0,) * 4] * (4 - len(rows)), dtype=np.float64)


def run_case(ref, case, chain, want):
    pts, boxes = frame(case)
    for k in range(10000):
        seed = 1000 * case + k
        np.random.seed(seed)
        res = {"points": pts.copy(), "annotations": {"gt_boxes": boxes.copy()}}
        with DrawLog() as log:
            for name, kw in chain:
                res = getattr(ref, name)(**kw)(res)
        rec = records(chain, log.calls)
        flips = [r for r in rec if r[0] == 4.0]
        if want is None or (bool(flips[0][1]), bool(flips[0][2])) == want:
            break
    else:
        raise RuntimeError("no seed gives flips %s" % (want,))
    next_draw = np.random.random_sample()
    return dict(pts=pts, boxes=boxes, out_pts=res["points"], out_boxes=res["annotations"]["gt_boxes"], aug=rec, seed=seed,
                next_draw=next_draw, calls=[c[0] for c in log.calls])


def config_nodes():
    from pillarnext_b200 import hydra_lite
    d = os.path.join(reference_loader.REF_ROOT, "configs", "experiments")
    out = {}
    for f in sorted(os.listdir(d)):
        if f.endswith(".yaml"):
            cfg = hydra_lite.resolve(hydra_lite.compose(d, f[:-5]))
            out[f[:-5]] = cfg["data"]["train_dataset"]["augmentation"]
    return out


def main():
    ref = load_reference_augmentation()
    cases = [run_case(ref, i, chain, want) for i, (chain, want) in enumerate(CASES)]
    for c in cases:
        assert c["out_pts"].dtype == np.float32 and c["out_boxes"].dtype == np.float32
    pts = np.concatenate([np.pad(c["pts"], ((0, 0), (1, 0)), constant_values=i) for i, c in enumerate(cases)])
    out_pts = np.concatenate([np.pad(c["out_pts"], ((0, 0), (1, 0)), constant_values=i) for i, c in enumerate(cases)])
    arrays = dict(points=pts, boxes=np.stack([c["boxes"] for c in cases]), out_points=out_pts,
                  out_boxes=np.stack([c["out_boxes"] for c in cases]), aug=np.stack([c["aug"] for c in cases]),
                  seeds=np.array([c["seed"] for c in cases], dtype=np.int64),
                  next_draw=np.array([c["next_draw"] for c in cases]),
                  chains=np.array(json.dumps([chain for chain, _ in CASES])),
                  calls=np.array(json.dumps([c["calls"] for c in cases])))
    out = os.path.join(GOLDEN, "ref_aug.npz")
    np.savez_compressed(out, **arrays)
    print("wrote", out, {k: v.shape for k, v in arrays.items()})
    nodes = config_nodes()
    out = os.path.join(GOLDEN, "ref_aug_configs.json")
    with open(out, "w") as fh:
        json.dump(nodes, fh, indent=1)             # key order is the order the transforms run in
        fh.write("\n")
    print("wrote", out, sorted(nodes))


if __name__ == "__main__":
    main()
