"""Plain-numpy restatement of the global training augmentation (TEST INFRASTRUCTURE, never imported by the product).

Applies the collated records aug [B, 4, 4] (code, p0, p1, p2; det3d/datasets/pipelines/augmentation.py) the way the
reference's numpy transforms do (det3d/datasets/pipelines/augmentation.py + box_np_ops.rotate / scaling / translate /
flip of the reference), with every dtype spelled out instead of left to numpy's scalar promotion:
  * rotation: fp32 rows @ a float64 rotation matrix, stored back into fp32; yaw += fp32(theta);
  * scaling: fp32 multiply by fp32(s) (point xyz, box columns 0-7);
  * translation: + t as a float64 array (computed in fp64, stored into fp32);
  * flip: negations, yaw -> -yaw or -yaw + fp32(pi), then the wrap by fp32(2 pi) against fp32(pi);
  * NaN box elements read as 0 by each op and restored to NaN after it.
tests/test_global_aug_cpu.py pins it to the reference's own outputs (tests/golden/ref_aug.npz); the GPU tests compare
ops.global_aug and a training step against it."""
import numpy as np

PI32, TWO_PI32 = np.float32(np.pi), np.float32(2 * np.pi)


def _rotate(v, c, s):
    rot_mat_T = np.array([[c, s, 0.0], [-s, c, 0.0], [0.0, 0.0, 1.0]], dtype=np.float64)
    return v @ rot_mat_T


def _wrap(yaw):
    yaw = np.where(yaw > PI32, yaw - TWO_PI32, yaw)
    return np.where(yaw < -PI32, yaw + TWO_PI32, yaw)


def apply_frame(points, boxes, records):
    """points [n, k >= 3] fp32 (x, y, z first), boxes [m, 9] fp32, records [4, 4] -> transformed copies."""
    p, b = np.array(points, dtype=np.float32), np.array(boxes, dtype=np.float32)
    for code, p0, p1, p2 in np.asarray(records, dtype=np.float64):
        code = int(code)
        if code not in (1, 2, 3, 4):
            continue
        nan = np.isnan(b)
        b[nan] = 0
        if code == 1:
            p[:, :3] = _rotate(p[:, :3], p1, p2)
            b[:, :3] = _rotate(b[:, :3], p1, p2)
            b[:, 6:8] = _rotate(np.hstack([b[:, 6:8], np.zeros((len(b), 1))]), p1, p2)[:, :2]
            b[:, 8] = b[:, 8] + np.float32(p0)
        elif code == 2:
            s = np.float32(p0)
            p[:, :3] = p[:, :3] * s
            b[:, :8] = b[:, :8] * s
        elif code == 3:
            t = np.array([p0], dtype=np.float64)
            p[:, :3] = p[:, :3] + t
            b[:, :3] = b[:, :3] + t
        else:
            if p0 != 0:
                p[:, 1], b[:, 1], b[:, 7] = -p[:, 1], -b[:, 1], -b[:, 7]
                b[:, 8] = _wrap(-b[:, 8])
            if p1 != 0:
                p[:, 0], b[:, 0], b[:, 6] = -p[:, 0], -b[:, 0], -b[:, 6]
                b[:, 8] = _wrap(-b[:, 8] + PI32)
        b[nan] = np.nan
    return p, b


def apply(points, boxes, aug):
    """Collated batch: points [N, 6] (frame index in column 0), boxes [B, M, 9], aug [B, 4, 4] -> (points, boxes),
    new arrays; the point order is kept."""
    points, boxes, aug = np.asarray(points, np.float32), np.asarray(boxes, np.float32), np.asarray(aug, np.float64)
    p_out, b_out = points.copy(), boxes.copy()
    for f in range(boxes.shape[0]):
        sel = points[:, 0] == f
        p_out[sel, 1:], b_out[f] = apply_frame(points[sel, 1:], boxes[f], aug[f])
    return p_out, b_out
