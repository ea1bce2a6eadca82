"""Freeze the reference's OWN ground-truth database sampling into tests/golden/ref_gts.npz, and the sampler nodes of its
experiments into tests/golden/ref_gts_configs.json (TEST INFRASTRUCTURE; run where the reference tree is present).

A subclass of the reference's BaseDataset (det3d/datasets/base.py) with in-memory frames runs its own __getitem__ with
its own DataBaseSamplerV2, DBFilterByMinNumPoint, box_np_ops and numba, on a small gt database written to a temporary
directory.  np.random is seeded once before the sampler is built; the frames are then read in order, so the class lists
wrap (short list, partial rest, exact fit) as they would in a data-loader worker.  Every list the sampler returns is
logged.  Cases (frame: what it covers):
  0, 4-7  random scene cars and pedestrians; trucks: A and B overlap only each other (the first drawn is rejected by
          the later one, which is accepted), C touches a scene box along a shared edge (accepted), D contains a small
          scene box (rejected by the containment test); scene points exactly on C's faces and one ulp outside
  1       no scene boxes
  2       one scene box covering everything: every candidate rejected
  3       as many scene cars as the group maximum: nothing to sample for `car`
Stored:
  db_names [K], db_boxes [K, 9], db_counts [K], db_points [sum, 5], db_paths [K]     the database (before filtering)
  points [N, 6] (frame, x, y, z, intensity, time), boxes [B, M, 9], names (JSON)      the scenes
  scene_trig [B, M, 2]          numpy's (cos, sin) of the scene yaws
  draws [B, S]                  database index of every drawn candidate in draw order (-1 = none)
  cand_trig [B, S, 4]           numpy cos, sin and libm cosf, sinf of the candidates' yaws
  out_points [N', 6], out_boxes [B, M + S, 9] (padding: class -1 rows), out_names (JSON)   the reference's output
  inside [N, K]                 box_np_ops.points_in_rbbox(every scene point, every database box), as
                                create_gt_database calls it
  seed, next_draw, groups (JSON), min_points (JSON), classes (JSON)

    python -m oracle.make_golden_gts
"""
import importlib
import json
import os
import pickle
import sys
import tempfile
import types

import numpy as np

from oracle import reference_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
CLASSES = ["car", "truck", "pedestrian"]
GROUPS = [{"car": 8}, {"truck": 4}, {"pedestrian": 3}]
MIN_POINTS = {"car": 5, "truck": 5, "pedestrian": 5}
SEED = 7
N_FRAMES = 8
F = np.float32


def load_reference():
    """The reference's sample_ops, base and box_np_ops modules (this repo's `det3d` is set aside while they load)."""
    from oracle import torch_scatter_shim
    saved = {k: v for k, v in sys.modules.items() if k == "det3d" or k.startswith("det3d.")}
    for k in saved:
        del sys.modules[k]
    had_ts = sys.modules.get("torch_scatter")
    sys.modules["torch_scatter"] = torch_scatter_shim
    sys.path.insert(0, reference_loader.REF_ROOT)
    try:
        importlib.import_module("det3d")
        sys.modules["det3d.core.iou3d_nms.iou3d_nms_cuda"] = types.ModuleType("det3d.core.iou3d_nms.iou3d_nms_cuda")
        ns = types.SimpleNamespace(sample_ops=importlib.import_module("det3d.datasets.pipelines.sample_ops"),
                                   base=importlib.import_module("det3d.datasets.base"),
                                   box_np_ops=importlib.import_module("det3d.core.bbox.box_np_ops"))
    finally:
        sys.path.remove(reference_loader.REF_ROOT)
        for k in [k for k in sys.modules if k == "det3d" or k.startswith("det3d.")]:
            del sys.modules[k]
        sys.modules.update(saved)
        if had_ts is None:
            sys.modules.pop("torch_scatter", None)
        else:
            sys.modules["torch_scatter"] = had_ts
    return ns


def box(x, y, z, dx, dy, dz, yaw, vx=0.0, vy=0.0):
    return np.array([x, y, z, dx, dy, dz, vx, vy, yaw], dtype=F)


TRUCKS = [box(45, 0, 0, 7, 2.5, 3, 0.3), box(47, 1, 0, 7, 2.5, 3, 0.2), box(50, 20, 0, 6, 2.5, 3, 0.0),
          box(50, -20, 0, 8, 8, 3, 0.1)]
ANCHORS = [box(56, 20, 0, 6, 2.5, 3, 0.0), box(50, -20, 0, 1, 1, 1, 0.7)]   # C's neighbour, the box inside D


def database(g):
    """[(name, box, points relative to the centre)]: 14 cars (2 with fewer than 5 points), trucks A-D, 2 pedestrians."""
    out = []
    for k in range(14):
        b = box(g.uniform(-40, 20), g.uniform(-40, 40), -1.0, *(np.array([4.6, 1.9, 1.7]) * g.uniform(0.9, 1.1, 3)),
                g.uniform(-np.pi, np.pi), *g.normal(0, 1, 2))
        out.append(("car", b, 3 if k in (4, 9) else int(g.integers(5, 40))))
    out += [("truck", b, int(g.integers(20, 60))) for b in TRUCKS]
    out += [("pedestrian", box(-5, 45, -1, 0.7, 0.7, 1.8, 0.4), 12), ("pedestrian", box(5, 45, -1, 0.7, 0.7, 1.8, -1.0), 9)]
    return [(n, b, (g.uniform(-0.6, 0.6, (k, 5)) * np.array([b[3], b[4], b[5], 0, 0]) +
                    np.array([0, 0, 0, 1, 0]) * g.uniform(0, 255, (k, 1))).astype(F)) for n, b, k in out]


def scene(g, case):
    """(points [n, 5], boxes [m, 9], names) of one frame."""
    boxes, names = [], []
    if case == 2:
        boxes, names = [box(0, 0, 0, 200, 200, 10, 0.0)], ["pedestrian"]
    elif case != 1:
        n_cars = 6 if case == 3 else 3
        for _ in range(n_cars):
            boxes.append(box(g.uniform(-40, 20), g.uniform(-40, 40), -1.0, 4.5, 1.9, 1.7, g.uniform(-np.pi, np.pi)))
            names.append("car")
        boxes.append(box(g.uniform(-8, 8), g.uniform(-30, 30), -1.0, 0.7, 0.7, 1.8, g.uniform(-np.pi, np.pi)))
        names.append("pedestrian")
        boxes += ANCHORS
        names += ["car", "car"]
    pts = np.zeros((400, 5), dtype=F)
    pts[:, 0] = g.uniform(-45, 62, 400)
    pts[:, 1] = g.uniform(-45, 50, 400)
    pts[:, 2] = g.uniform(-2.5, 2, 400)
    pts[:, 3] = g.uniform(0, 255, 400)
    # truck C (50, 20, 0; 6 x 2.5 x 3, yaw 0): points on its faces and one ulp outside, and inside A / B / D / pedestrians
    ties = [(47, 20, 0), (53, 20.5, 1), (50, 18.75, -1), (51, 21.25, 0.5), (49, 19, 1.5), (52, 21, -1.5), (47, 18.75, 1.5)]
    out = [(np.nextafter(F(47), F(0)), 20, 0), (np.nextafter(F(53), F(99)), 20, 0), (50, 20, np.nextafter(F(1.5), F(9))),
           (50, np.nextafter(F(18.75), F(0)), 0)]
    extra = ties + out + [(45, 0, 0), (47, 1, 0.5), (46, 0.5, -1), (50, -20, 0.2), (52, -18, -0.5), (-5, 45, -1), (5, 45, -1)]
    for k, (x, y, z) in enumerate(extra):
        pts[k, :3] = x, y, z
    pts = pts[g.permutation(len(pts))]
    return pts, (np.stack(boxes) if boxes else np.zeros((0, 9), F)), names


def config_nodes():
    from pillarnext_b200 import hydra_lite
    d = os.path.join(reference_loader.REF_ROOT, "configs", "experiments")
    out = {}
    for f in sorted(os.listdir(d)):
        if f.endswith(".yaml"):
            cfg = hydra_lite.resolve(hydra_lite.compose(d, f[:-5]))
            node = cfg["data"]["train_dataset"].get("sampler")
            if node is not None:
                out[f[:-5]] = node
    return out


def main():
    ref = load_reference()
    g = np.random.default_rng(2024)
    db = database(g)
    frames = [scene(g, c) for c in range(N_FRAMES)]
    with tempfile.TemporaryDirectory() as root:
        infos, paths = {}, []
        for k, (name, b, p) in enumerate(db):
            rel = os.path.join("gt_database_1sweeps_withvelo", name, "golden_%s_%d.bin" % (name, k))
            os.makedirs(os.path.join(root, os.path.dirname(rel)), exist_ok=True)
            p.tofile(os.path.join(root, rel))
            paths.append(rel)
            infos.setdefault(name, []).append({"name": name, "path": rel, "image_idx": "golden", "gt_idx": k,
                                               "box3d_lidar": b, "num_points_in_gt": len(p), "difficulty": 0,
                                               "group_id": k})
        with open(os.path.join(root, "dbinfos_train_1sweeps_withvelo.pkl"), "wb") as fh:
            pickle.dump(infos, fh)
        index_of = {p: k for k, p in enumerate(paths)}

        class MemDataset(ref.base.BaseDataset):
            def load_infos(self):
                self.infos = [{"token": "golden_%d" % i, "frame": fr} for i, fr in enumerate(frames)]

            def load_pointcloud(self, res, info):
                res["points"] = info["frame"][0].copy()
                return res

            def load_box3d(self, res, info):
                res["annotations"] = {"gt_boxes": info["frame"][1].copy(), "gt_names": np.array(info["frame"][2])}
                return res

        import functools
        sampler = functools.partial(
            ref.sample_ops.DataBaseSamplerV2, root_path=root, dbinfo_path="dbinfos_train_1sweeps_withvelo.pkl",
            groups=GROUPS, db_prepor={"filter_by_num": ref.sample_ops.DBFilterByMinNumPoint(dict(MIN_POINTS))},
            rate=1.0, gt_drop_percentage=0, gt_drop_max_keep_points=-1, point_dim=5)
        log = []
        orig = ref.sample_ops.BatchSampler.sample

        def logged(self, num):
            r = orig(self, num)
            log.append([index_of[i["path"]] for i in r])
            return r

        ref.sample_ops.BatchSampler.sample = logged
        try:
            np.random.seed(SEED)
            ds = MemDataset(root_path=root, info_path="unused", sampler=sampler,
                            loading_pipelines=["load_pointcloud", "load_box3d"], create_database=True)
            outs, draws = [], []
            for i in range(N_FRAMES):
                log.clear()
                res = ds[i]
                draws.append([k for call in log for k in call])
                outs.append((res["points"], res["annotations"]["gt_boxes"], list(res["annotations"]["gt_names"])))
            next_draw = np.random.random_sample()
        finally:
            ref.sample_ops.BatchSampler.sample = orig

    from det3d.datasets.pipelines.sample_ops import libm_trig, numpy_trig
    B = N_FRAMES
    M = max(1, max(len(f[2]) for f in frames))
    S = max(1, max(len(d) for d in draws))
    boxes = np.zeros((B, M, 9), F)
    boxes[:, :, 3:6] = 1
    scene_trig = np.zeros((B, M, 2), F)
    scene_trig[:, :, 0] = 1
    dr = np.full((B, S), -1, np.int64)
    cand_trig = np.zeros((B, S, 4), F)
    cand_trig[:, :, 0] = cand_trig[:, :, 2] = 1
    out_boxes = np.zeros((B, M + S, 9), F)
    out_boxes[:, :, 3:6] = 1
    for f, (p, b, n) in enumerate(frames):
        boxes[f, :len(b)] = b
        scene_trig[f, :len(b)] = numpy_trig(b) if len(b) else np.zeros((0, 2), F)
        dr[f, :len(draws[f])] = draws[f]
        if draws[f]:
            cb = np.stack([db[k][1] for k in draws[f]])
            cand_trig[f, :len(cb)] = np.concatenate([numpy_trig(cb), libm_trig(cb[:, -1])], 1)
        ob = outs[f][1]
        assert ob.dtype == F
        out_boxes[f, :len(ob)] = ob
    pts = np.concatenate([np.pad(p, ((0, 0), (1, 0)), constant_values=f) for f, (p, _, _) in enumerate(frames)])
    out_pts = np.concatenate([np.pad(o[0], ((0, 0), (1, 0)), constant_values=f) for f, o in enumerate(outs)])
    db_boxes = np.stack([d[1] for d in db])
    inside = ref.box_np_ops.points_in_rbbox(pts[:, 1:].astype(F), db_boxes[:, [0, 1, 2, 3, 4, 5, -1]])
    n_acc = [len(o[2]) - len(fr[2]) for o, fr in zip(outs, frames)]
    print("candidates per frame", [len(d) for d in draws], "accepted", n_acc)
    assert n_acc[2] == 0 and len(draws[2]) > 0                      # every candidate rejected
    assert all(db[k][0] != "car" for k in draws[3])                 # nothing to sample for car
    arrays = dict(db_names=np.array([d[0] for d in db]), db_boxes=db_boxes, inside=inside,
                  db_counts=np.array([len(d[2]) for d in db]), db_points=np.concatenate([d[2] for d in db]),
                  db_paths=np.array(paths), points=pts.astype(F), boxes=boxes, scene_trig=scene_trig,
                  names=np.array(json.dumps([f[2] for f in frames])), draws=dr, cand_trig=cand_trig,
                  out_points=out_pts.astype(F), out_boxes=out_boxes, out_names=np.array(json.dumps([o[2] for o in outs])),
                  seed=np.array(SEED), next_draw=np.array(next_draw), groups=np.array(json.dumps(GROUPS)),
                  min_points=np.array(json.dumps(MIN_POINTS)), classes=np.array(json.dumps(CLASSES)))
    out = os.path.join(GOLDEN, "ref_gts.npz")
    np.savez_compressed(out, **arrays)
    print("wrote", out, {k: v.shape for k, v in arrays.items()})
    nodes = config_nodes()
    out = os.path.join(GOLDEN, "ref_gts_configs.json")
    with open(out, "w") as fh:
        json.dump(nodes, fh, indent=1)
        fh.write("\n")
    print("wrote", out, sorted(nodes))


if __name__ == "__main__":
    main()
