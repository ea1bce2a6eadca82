"""Plain-numpy restatement of ground-truth database sampling's GPU half (TEST INFRASTRUCTURE, never imported by the
product): the reference's collision test and greedy acceptance (sample_ops.sample_class_v2 on box_np_ops.
center_to_corner_box2d / box_collision_test), the removal of scene points inside accepted boxes (points_in_rbbox) and
the paste (datasets/base.py:77-96), for the candidates scenes.collate packs.  Every fp32 operation is spelled out:
  * corners: (dx, dy) * (+-0.5), x' = fl(fl(px c) + fl(py -s)) + cx, y' = fl(fl(px s) + fl(py c)) + cy, with numpy's
    (c, s) shipped by the loader;
  * collision[i, j] with the candidate i first: standup overlap, strict segment crossings, then containment either way;
  * a candidate is rejected if it collides with a scene box, an earlier accepted candidate or any later candidate of
    its class call (a run of equal class ids); a rejected candidate's column is cleared;
  * points: |z - bz| <= dz / 2, |lx| <= dx / 2, |ly| <= dy / 2 (halves in fp64) with libm's (cosf, sinf).
tests/test_gt_sampling_cpu.py pins it to the reference's own outputs (tests/golden/ref_gts.npz)."""
import numpy as np

F = np.float32
NX, NY = F([-0.5, -0.5, 0.5, 0.5]), F([-0.5, 0.5, 0.5, -0.5])


def corners(box, c, s):
    """[4, 2] BEV corners and [4] standup (min x, min y, max x, max y) of one 9-column fp32 box."""
    c, s = F(c), F(s)
    px, py = F(box[3]) * NX, F(box[4]) * NY
    x = (px * c + py * (-s)) + F(box[0])
    y = (px * s + py * c) + F(box[1])
    return np.stack([x, y], 1), np.array([x.min(), y.min(), x.max(), y.max()], dtype=F)


def _inside(b, q):
    for l in range(4):
        for k in range(4):
            v = -(b[k] - b[(k + 1) % 4])
            cross = v[1] * (b[k, 0] - q[l, 0])
            cross = cross - v[0] * (b[k, 1] - q[l, 1])
            if cross >= 0:
                return False
    return True


def collide(gb, gq):
    (b, sb), (q, sq) = gb, gq
    iw = min(sb[2], sq[2]) - max(sb[0], sq[0])
    if not iw > 0:
        return False
    ih = min(sb[3], sq[3]) - max(sb[1], sq[1])
    if not ih > 0:
        return False
    for k in range(4):
        A, B = b[k], b[(k + 1) % 4]
        for l in range(4):
            C, D = q[l], q[(l + 1) % 4]
            acd = (D[1] - A[1]) * (C[0] - A[0]) > (C[1] - A[1]) * (D[0] - A[0])
            bcd = (D[1] - B[1]) * (C[0] - B[0]) > (C[1] - B[1]) * (D[0] - B[0])
            if acd != bcd:
                abc = (C[1] - A[1]) * (B[0] - A[0]) > (B[1] - A[1]) * (C[0] - A[0])
                abd = (D[1] - A[1]) * (B[0] - A[0]) > (B[1] - A[1]) * (D[0] - A[0])
                if abc != abd:
                    return True
    return _inside(b, q) or _inside(q, b)


def select(boxes, classes, trig, cboxes, cclasses, ctrig):
    """One frame: scene boxes [M, 9] (class -1 = padding), their numpy (cos, sin) [M, 2], candidates [S, 9] / [S] /
    [S, 4] -> accepted [S] bool."""
    avoid = [corners(b, *t) for b, k, t in zip(boxes, classes, trig) if k >= 0]
    geo = [corners(b, t[0], t[1]) if k >= 0 else None for b, k, t in zip(cboxes, cclasses, ctrig)]
    acc = np.zeros(len(cclasses), dtype=bool)
    s = 0
    while s < len(cclasses):
        if cclasses[s] < 0:
            s += 1
            continue
        e = s + 1
        while e < len(cclasses) and cclasses[e] == cclasses[s]:
            e += 1
        ext = [any(collide(geo[i], g) for g in avoid) for i in range(s, e)]
        cleared = set()
        for i in range(s, e):
            hit = ext[i - s] or any(collide(geo[i], geo[j]) for j in range(s, e) if j != i and j not in cleared)
            if hit:
                cleared.add(i)
            else:
                acc[i] = True
        avoid += [geo[i] for i in range(s, e) if acc[i]]
        s = e
    return acc


def points_in_boxes(points, boxes, trig):
    """[n, >= 3] fp32 points x [m, 9] fp32 boxes with libm (cosf, sinf) [m, 2] -> [n, m] bool."""
    p = np.asarray(points, dtype=F)
    out = np.zeros((len(p), len(boxes)), dtype=bool)
    for j, (b, (c, s)) in enumerate(zip(np.asarray(boxes, F), np.asarray(trig, F))):
        zin = np.abs(p[:, 2] - b[2]).astype(np.float64) <= np.float64(b[5]) / 2.0
        sx, sy = p[:, 0] - b[0], p[:, 1] - b[1]
        lx = sx * c + sy * s
        ly = (-sx) * s + sy * c
        out[:, j] = zin & (np.abs(lx).astype(np.float64) <= np.float64(b[3]) / 2.0) & \
            (np.abs(ly).astype(np.float64) <= np.float64(b[4]) / 2.0)
    return out


def apply(points, boxes, classes, trig, cboxes, cclasses, ctrig, cpoints, coffsets):
    """A collated batch (scenes.collate's points, gt_boxes_raw, gt_classes, gt_trig and gts_* arrays) ->
    (points [count, 6] compacted, boxes [B, M + S, 9], classes [B, M + S], accepted [B, S])."""
    points, boxes, cboxes = np.asarray(points, F), np.asarray(boxes, F), np.asarray(cboxes, F)
    B, M, S = boxes.shape[0], boxes.shape[1], cboxes.shape[1]
    out_pts, out_boxes = [], np.zeros((B, M + S, 9), dtype=F)
    out_boxes[:, :, 3:6] = 1.0
    out_cls = np.full((B, M + S), -1, dtype=np.int32)
    acc_all = np.zeros((B, S), dtype=bool)
    for f in range(B):
        acc = select(boxes[f], classes[f], trig[f], cboxes[f], cclasses[f], ctrig[f])
        acc_all[f] = acc
        real = np.asarray(classes[f]) >= 0
        rows = np.concatenate([boxes[f][real], cboxes[f][acc]])
        out_boxes[f, :len(rows)] = rows
        out_cls[f, :len(rows)] = np.concatenate([np.asarray(classes[f])[real], np.asarray(cclasses[f])[acc]])
        for s in np.flatnonzero(acc):
            r = f * S + s
            q = np.array(cpoints[coffsets[r]:coffsets[r + 1]], dtype=F)
            q[:, :3] += cboxes[f, s, :3]
            out_pts.append(np.concatenate([np.full((len(q), 1), f, F), q], 1))
        sel = points[:, 0] == f
        scene = points[sel]
        if acc.any():
            inside = points_in_boxes(scene[:, 1:4], cboxes[f][acc], np.asarray(ctrig[f], F)[acc][:, 2:4])
            scene = scene[~inside.any(1)]
        out_pts.append(scene)
    pts = np.concatenate(out_pts, 0) if out_pts else np.zeros((0, 6), F)
    return pts.astype(F), out_boxes, out_cls, acc_all
