"""Freeze the reference's OWN multi-sweep loading into tests/golden/ref_sweeps.npz (TEST INFRASTRUCTURE; run where the
reference tree is present).

The reference's NuScenesDataset.load_pointcloud (nusc.py: read_file, read_sweep, remove_close) and
WaymoDataset.load_pointcloud (waymo.py: read_file with its no-label-zone filter, rel_pose = inv(pose) @ sweep_pose,
drop_frames) run on .bin files written to a temporary root; the packages they import but these methods never use
(nuscenes, pyquaternion, tqdm, fire, waymo_open_dataset) are stubbed in sys.modules while they load.  Cases:
  nusc   frame 0: key-frame points inside the +-1 m square (kept: the key frame is never filtered); sweep 1 with
                  transform_matrix None: coordinates exactly at +-1.0, inside the square in x only or y only, inside in
                  both (removed), -0.0 coordinates; sweep 2 with a rotation + translation, some points landing in the
                  square; sweep 3 None, every point inside the square (the sweep loses everything)
         frame 1: no sweeps
         frame 2: two transformed sweeps of random points
  waymo  nsweeps 3: frame 0 with two stored sweeps, frame 1 with one (fewer than nsweeps - 1), frame 2 with none; some
         points in no-label zones (dropped by read_file)
  drop   nsweeps 3, drop_frames 0.5 under np.random.seed(SEED): eight frames of two stored sweeps each
Stored per case <c> (the operands of ops.accumulate_sweeps, as scenes.collate packs them, and the reference's output):
  <c>_points [n, 6], <c>_point_offsets [B + 1], <c>_sweep_points [S, 5], <c>_sweep_offsets [B K + 1],
  <c>_transforms [B, K, 4, 4] (NaN = None / dropped), <c>_min_distance, <c>_out [count, 6] (frame index prepended)
  drop_kept [B, 2] the sweeps the reference kept, drop_next = np.random.uniform() after the last frame, drop_seed

    python -m oracle.make_golden_sweeps
"""
import importlib
import os
import pickle
import sys
import tempfile
import types

import numpy as np

from oracle import reference_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
SEED = 11
F = np.float32
STUBS = ["nuscenes", "nuscenes.utils", "nuscenes.utils.splits", "nuscenes.utils.data_classes", "nuscenes.eval",
         "nuscenes.eval.detection", "nuscenes.eval.detection.config", "nuscenes.eval.detection.evaluate", "pyquaternion",
         "tqdm", "fire", "waymo_open_dataset", "waymo_open_dataset.protos"]


class _Stub(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


def load_reference():
    """The reference's NuScenesDataset and WaymoDataset classes (this repo's `det3d` is set aside while they load)."""
    saved = {k: v for k, v in sys.modules.items() if k == "det3d" or k.startswith("det3d.") or k in STUBS}
    for k in saved:
        del sys.modules[k]
    for k in STUBS:
        sys.modules[k] = _Stub(k)
    sys.path.insert(0, reference_loader.REF_ROOT)
    try:
        importlib.import_module("det3d")
        ns = types.SimpleNamespace(nusc=importlib.import_module("det3d.datasets.nuscenes.nusc").NuScenesDataset,
                                   waymo=importlib.import_module("det3d.datasets.waymo.waymo").WaymoDataset)
    finally:
        sys.path.remove(reference_loader.REF_ROOT)
        for k in [k for k in sys.modules if k == "det3d" or k.startswith("det3d.") or k in STUBS]:
            del sys.modules[k]
        sys.modules.update(saved)
    return ns


def rigid(yaw, tx, ty, tz=0.0):
    c, s = np.cos(yaw), np.sin(yaw)
    T = np.eye(4)
    T[:2, :2] = [[c, -s], [s, c]]
    T[:3, 3] = tx, ty, tz
    return T


def cloud(g, n, ext=30.0):
    return np.concatenate([g.uniform(-ext, ext, (n, 2)), g.uniform(-2, 1, (n, 1)), g.uniform(0, 255, (n, 1))], 1).astype(F)


def write(root, name, arr):
    arr.astype(F).tofile(os.path.join(root, name))
    return name


def pack(frames, K, min_distance):
    """frames: [(key [n, 4 or 5] fp32 as read, [(sweep [m, 5] fp32 as read, 4x4 or None)] * <= K)] -> operands."""
    pts, po, sp, so, tms = [], [0], [], [0], np.full((len(frames), K, 4, 4), np.nan)
    for f, (key, sweeps) in enumerate(frames):
        key5 = key if key.shape[1] == 5 else np.concatenate([key, np.zeros((len(key), 1), F)], 1)
        pts.append(np.concatenate([np.full((len(key5), 1), f, F), key5], 1))
        po.append(po[-1] + len(key5))
        for k in range(K):
            sw, T = sweeps[k] if k < len(sweeps) else (np.zeros((0, 5), F), None)
            sp.append(sw)
            so.append(so[-1] + len(sw))
            if T is not None:
                tms[f, k] = T
    return dict(points=np.concatenate(pts).astype(F), point_offsets=np.array(po, np.int32),
                sweep_points=np.concatenate(sp).astype(F).reshape(-1, 5), sweep_offsets=np.array(so, np.int32),
                transforms=tms, min_distance=np.float32(min_distance))


def with_frame(outs):
    return np.concatenate([np.concatenate([np.full((len(o), 1), f, F), o.astype(F)], 1) for f, o in enumerate(outs)])


def nusc_case(ref, root, g):
    edge = np.array([[1.0, 0.5], [-1.0, 0.5], [0.5, 1.0], [0.5, -1.0], [0.999, 0.999], [-0.5, -0.5], [0.5, 7.0],
                     [7.0, 0.5], [-0.0, -0.0], [-0.0, 3.0], [3.0, -0.0], [np.nextafter(F(1), F(0)), 0.0],
                     [np.nextafter(F(1), F(2)), 0.0]], F)
    s1 = np.concatenate([edge, np.full((len(edge), 1), -0.0, F), g.uniform(0, 255, (len(edge), 1))], 1).astype(F)
    s1 = np.concatenate([s1, cloud(g, 40)])
    T2 = rigid(0.3, 1.7, -0.4, 0.05)
    near = (np.linalg.inv(T2) @ np.c_[g.uniform(-0.9, 0.9, (12, 2)), np.zeros(12), np.ones(12)].T).T[:, :3]
    s2 = np.concatenate([cloud(g, 60), np.c_[near, g.uniform(0, 255, 12)].astype(F)])
    s3 = np.c_[g.uniform(-0.99, 0.99, (9, 2)), g.uniform(-2, 1, (9, 1)), g.uniform(0, 255, (9, 1))].astype(F)
    key0 = np.concatenate([cloud(g, 30), np.array([[0.2, -0.3, -1.0, 9.0], [-0.0, 0.0, -0.0, 1.0]], F)])
    frames = [(key0, [(s1, None, 0.050101), (s2, T2, 0.0999), (s3, None, 0.15)]),
              (cloud(g, 25), []),
              (cloud(g, 35), [(cloud(g, 50), rigid(-1.2, -3.3, 2.9), 0.05), (cloud(g, 45), rigid(2.5, 0.6, 0.25, -0.1), 0.1)])]
    infos = []
    for f, (key, sweeps) in enumerate(frames):
        name = write(root, "n%d.bin" % f, np.c_[key, np.zeros(len(key))])
        infos.append({"lidar_path": name, "token": "n%d" % f,
                      "sweeps": [{"lidar_path": write(root, "n%d_%d.bin" % (f, k), np.c_[sw, np.full(len(sw), 7.0)]),
                                  "transform_matrix": T, "time_lag": lag} for k, (sw, T, lag) in enumerate(sweeps)]})
    with open(os.path.join(root, "nusc_infos.pkl"), "wb") as fh:
        pickle.dump(infos, fh)
    ds = ref.nusc("nusc_infos.pkl", root, nsweeps=4)
    outs = [ds.load_pointcloud({}, info)["points"] for info in infos]
    ops_in = [(key, [(np.c_[sw, np.full(len(sw), F(lag))].astype(F), T) for sw, T, lag in sweeps]) for key, sweeps in frames]
    return pack(ops_in, 3, 1.0), with_frame(outs)


def waymo_frames(g, n_stored):
    out = []
    for f, m in enumerate(n_stored):
        pose = rigid(g.uniform(-np.pi, np.pi), *g.uniform(-500, 500, 2), g.uniform(-1, 1))
        sweeps = []
        for k in range(m):
            d = rigid(g.uniform(-0.05, 0.05), *g.uniform(-2, 2, 2), g.uniform(-0.02, 0.02))
            sweeps.append((cloud(g, int(g.integers(20, 60)), 60.0), pose @ d, 0.1 * (k + 1) + g.uniform(0, 1e-3)))
        out.append((cloud(g, int(g.integers(20, 60)), 60.0), pose, sweeps))
    return out


def waymo_case(ref, root, g, tag, n_stored, drop_frames):
    frames = waymo_frames(g, n_stored)

    def nlz(c):                      # 6-column .bin: x, y, z, intensity, elongation, nlz flag (-1 = not in a zone)
        flag = np.where(g.uniform(0, 1, len(c)) < 0.2, 1.0, -1.0)
        return np.c_[c, g.uniform(0, 1, len(c)), flag]
    infos = []
    for f, (key, pose, sweeps) in enumerate(frames):
        write(root, "lidar_point/%s%d.bin" % (tag, f), nlz(key))
        for k, (sw, _, _) in enumerate(sweeps):
            write(root, "lidar_point/%s%d_%d.bin" % (tag, f, k), nlz(sw))
        infos.append({"token": "%s%d" % (tag, f), "pose": pose,
                      "sweeps": [{"token": "%s%d_%d" % (tag, f, k), "pose": sp, "timestamp": ts}
                                 for k, (_, sp, ts) in enumerate(sweeps)]})
    with open(os.path.join(root, tag + "_infos.pkl"), "wb") as fh:
        pickle.dump(infos, fh)
    ds = ref.waymo(tag + "_infos.pkl", root, nsweeps=3, drop_frames=drop_frames)
    np.random.seed(SEED)
    outs, kept = [], []
    for info in infos:
        state = np.random.get_state()
        outs.append(ds.load_pointcloud({}, info)["points"])
        after = np.random.get_state()
        np.random.set_state(state)           # replay the same draws to record which sweeps were kept
        ks = [not (drop_frames > 0 and np.random.uniform() < drop_frames) for _ in range(min(2, len(info["sweeps"])))]
        assert all(a == b for a, b in zip(np.random.get_state()[1], after[1]))
        kept.append(ks + [False] * (2 - len(ks)))
    nxt = np.random.uniform()
    ops_in = []
    for f, info in enumerate(infos):
        key = ds.read_file("lidar_point/%s.bin" % info["token"])
        sweeps = []
        for k in range(min(2, len(info["sweeps"]))):
            sw = info["sweeps"][k]
            if kept[f][k]:
                sweeps.append((ds.read_file("lidar_point/%s.bin" % sw["token"], timestamp=sw["timestamp"]),
                               np.linalg.inv(info["pose"]) @ sw["pose"]))
            else:
                sweeps.append((np.zeros((0, 5), F), None))
        ops_in.append((key, sweeps))
    return pack(ops_in, 2, 0.0), with_frame(outs), np.array(kept), nxt


def main():
    ref = load_reference()
    g = np.random.default_rng(SEED)
    out = {}
    with tempfile.TemporaryDirectory() as root:
        os.makedirs(os.path.join(root, "lidar_point"))
        ops_in, res = nusc_case(ref, root, g)
        out.update({"nusc_" + k: v for k, v in ops_in.items()}, nusc_out=res)
        ops_in, res, _, _ = waymo_case(ref, root, g, "w", [2, 1, 0], 0.0)
        out.update({"waymo_" + k: v for k, v in ops_in.items()}, waymo_out=res)
        ops_in, res, kept, nxt = waymo_case(ref, root, g, "d", [2] * 8, 0.5)
        out.update({"drop_" + k: v for k, v in ops_in.items()}, drop_out=res, drop_kept=kept, drop_next=nxt,
                   drop_seed=SEED)
    path = os.path.join(GOLDEN, "ref_sweeps.npz")
    np.savez_compressed(path, **out)
    print("wrote %s: nusc %d -> %d rows, waymo %d -> %d, drop %d -> %d (kept %s)" % (
        path, len(out["nusc_points"]) + len(out["nusc_sweep_points"]), len(out["nusc_out"]),
        len(out["waymo_points"]) + len(out["waymo_sweep_points"]), len(out["waymo_out"]),
        len(out["drop_points"]) + len(out["drop_sweep_points"]), len(out["drop_out"]), kept.sum(0)))


if __name__ == "__main__":
    main()
