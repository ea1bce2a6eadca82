"""Freeze the reference's OWN box mirroring, det3d/core/bbox/box_np_ops.py:5-26 (`flip`), into tests/golden/ref_flip.npz
(TEST INFRASTRUCTURE; run in the build container, where the reference tree is present).

The double-flip undo transforms of oracle/flip_oracle.py and of the product's decode are checked against these outputs
(tests/test_double_flip_cpu.py): a box mirrored by the reference, encoded the way the head is trained (assign.py:101-105:
reg offset, height, log dims, vx, vy, sin, cos), mapped back by the undo, must decode to the original box.

    python -m oracle.make_golden_flip
"""
import importlib.util
import os

import numpy as np

from oracle import reference_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def boxes():
    """[n, 9] (x, y, z, dx, dy, dz, vx, vy, yaw): seeded boxes plus yaws at and near +-pi, 0 and +-pi/2."""
    g = np.random.default_rng(7)
    n = 24
    b = np.zeros((n, 9))
    b[:, 0:2] = g.uniform(-30, 30, (n, 2))
    b[:, 2] = g.uniform(-2, 1, n)
    b[:, 3:6] = g.uniform(0.5, 5, (n, 3))
    b[:, 6:8] = g.normal(0, 4, (n, 2))
    b[:, 8] = g.uniform(-np.pi, np.pi, n)
    b[:10, 8] = [np.pi, -np.pi, np.pi - 1e-4, -np.pi + 1e-4, 0.0, 1e-4, np.pi / 2, -np.pi / 2, np.pi - 0.3, -np.pi + 0.3]
    return b


def main():
    path = os.path.join(reference_loader.REF_ROOT, "det3d", "core", "bbox", "box_np_ops.py")
    spec = importlib.util.spec_from_file_location("ref_box_np_ops", path)
    ops = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ops)
    b = boxes()
    arrays = dict(boxes=b, flip_x=ops.flip(b.copy(), "x"), flip_y=ops.flip(b.copy(), "y"),
                  flip_xy=ops.flip(ops.flip(b.copy(), "x"), "y"))
    out = os.path.join(ROOT, "tests", "golden", "ref_flip.npz")
    np.savez_compressed(out, **arrays)
    print("wrote", out, {k: v.shape for k, v in arrays.items()})


if __name__ == "__main__":
    main()
