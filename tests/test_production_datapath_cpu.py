"""The edge-case launches of tests/test_production_datapath_gpu.py, CPU only.

* the builders produce what they claim: the select kernel's shared memory, computed from the layout gt_sample.cu
  documents (select_smem), lies just past the 48 KB opt-in threshold, at the 200 KB cap and one box past it; the packed
  class call has at least 65 candidates with its collisions across collision-row words 31/32 and 63/64; the inputs carry
  frame-B tail rows, zero-point candidates, a scene class equal to len(class_names), padding boxes and a frame without
  scene boxes;
* on a reduced copy of every edge case (fewer points, the same boxes) the numpy oracle chain (oracle/gts_oracle then
  oracle/aug_oracle) equals the host-twin chain (ops.gt_sample_host then ops.global_aug_host) bit for bit, so the two
  references the GPU file compares with agree before they are trusted."""
import numpy as np

from det3d.datasets.pipelines.sample_ops import libm_trig, numpy_trig
from oracle import aug_oracle, gts_oracle
from pillarnext_b200 import ops

F = np.float32
SMEM_OPT_IN = 48 * 1024          # above this the select kernel needs cudaFuncSetAttribute
SMEM_CAP = 200 * 1024            # pnx_gt_sample refuses more
N_CLASSES = 10                   # the nuScenes class list: a scene class of 10 is a name outside it
KEYS = ("points", "gt_boxes", "gt_classes", "gt_trig", "cand_boxes", "cand_classes", "cand_trig", "cand_points",
        "cand_offsets")


def select_smem(M, S):
    """Dynamic shared memory of gts_select_kernel for M scene + S candidate rows (gt_sample.cu): BEV geometry
    [M + S][12] fp32, the avoid list [M + S], ext [S] and acc [S] int32, collision rows [S][W] and valid [W] uint32,
    W = ceil(S / 32)."""
    W = (S + 31) // 32
    return (M + S) * 12 * 4 + (M + S) * 4 + S * 4 * 2 + S * W * 4 + W * 4


def boxes_around(limit, S):
    """(M at the limit, M one past it): the largest M with select_smem(M, S) <= limit, and that M + 1."""
    M = 0
    while select_smem(M + 1, S) <= limit:
        M += 1
    return M, M + 1


def _box(x, y, yaw, size=2.0, z=-1.0, vel=(0.5, -0.25)):
    return [x, y, z, size, size, 1.5, vel[0], vel[1], yaw]


def _pack(points, frames, cand_pts_per_frame):
    """frames: per frame (scene boxes [M, 9], classes [M], candidates [S, 9], classes [S]); cand_pts_per_frame: per
    frame a list of [k, 5] point arrays, one per candidate -> the operands of ops.gt_sample as numpy arrays."""
    B = len(frames)
    gb = np.stack([np.asarray(f[0], F) for f in frames])
    gc = np.stack([np.asarray(f[1], np.int32) for f in frames])
    cb = np.stack([np.asarray(f[2], F) for f in frames])
    cc = np.stack([np.asarray(f[3], np.int32) for f in frames])
    gt = np.stack([numpy_trig(b) for b in gb])
    ct = np.stack([np.concatenate([numpy_trig(b), libm_trig(b[:, 8])], 1) for b in cb])
    pts = [p for f in range(B) for p in cand_pts_per_frame[f]]
    off = np.concatenate([[0], np.cumsum([len(p) for p in pts])]).astype(np.int32)
    cp = np.concatenate(pts).astype(F).reshape(-1, 5) if pts else np.zeros((0, 5), F)
    return dict(points=np.ascontiguousarray(points, F), gt_boxes=gb, gt_classes=gc, gt_trig=gt, cand_boxes=cb,
                cand_classes=cc, cand_trig=ct, cand_points=cp, cand_offsets=off)


def _cloud(g, n, frame, lo, hi):
    xy = g.uniform(lo, hi, (n, 2))
    return np.concatenate([np.full((n, 1), frame), xy, g.uniform(-2.5, 0.5, (n, 1)), g.uniform(0, 255, (n, 1)),
                           np.zeros((n, 1))], 1).astype(F)


def _object_points(g, box, k):
    """k points inside `box`, relative to its centre (x, y, z, intensity, time)."""
    half = np.asarray(box[3:6], F) * F(0.45)
    return np.concatenate([g.uniform(-half, half, (k, 3)), g.uniform(0, 255, (k, 1)), np.zeros((k, 1))], 1).astype(F)


def _tail(n, B):
    t = np.zeros((n, 6), F)
    t[:, 0] = B
    return t


def grid_launch(M, S, n_points=60000, n_tail=700, seed=0):
    """One frame: M scene boxes (1 m squares, yaw 0 or pi/2) on a 2.5 m grid and one class call of S candidates, the even
    ones on a scene box (rejected), the odd ones in the gap between four (accepted), every eighth with no points;
    n_points scene points over the grid, then n_tail frame-B rows, as the sweeps stage leaves them."""
    g = np.random.default_rng(seed)
    side = int(np.ceil(np.sqrt(M)))
    ij = np.stack(np.divmod(np.arange(M), side), 1).astype(np.float64)
    xy = (ij - side / 2.0) * 2.5
    scene = np.array([_box(x, y, g.choice([0.0, np.pi / 2]), size=1.0) for x, y in xy], F)
    cls = np.arange(M, dtype=np.int32) % N_CLASSES
    slots = g.choice(M, S, replace=False)
    cand = np.array([_box(xy[k, 0] + (1.25 if s % 2 else 0.0), xy[k, 1] + (1.25 if s % 2 else 0.0), g.uniform(-0.3, 0.3),
                          size=1.0) for s, k in enumerate(slots)], F)
    cpts = [_object_points(g, b, 0 if s % 8 == 3 else int(g.integers(5, 60))) for s, b in enumerate(cand)]
    lo, hi = xy.min() - 2.0, xy.max() + 2.0
    points = np.concatenate([_cloud(g, n_points, 0, lo, hi), _tail(n_tail, 1)])
    return _pack(points, [(scene, cls, cand, np.zeros(S, np.int32))], [cpts])


def _word_frame0(g):
    """Frame 0 of word_launch: (scene boxes, classes, candidates, classes, expected acceptance)."""
    pos = {i: (5.0 * (i % 10), 10.0 + 5.0 * (i // 10)) for i in range(70)}
    early = [(-20.0, 0.0), (-20.0, 6.0), (-20.0, 12.0)]             # the earlier call (class 1): isolated, accepted
    len_box, pad_box = (-30.0, 20.0), (-30.0, 30.0)
    pos[32] = (pos[31][0] + 0.6, pos[31][1])                          # 31 / 32: collision row words 0 and 1
    pos[63] = (pos[62][0] + 0.6, pos[62][1])                          # 62 / 63 / 64: a chain across words 1 and 2
    pos[64] = (pos[62][0] + 1.2, pos[62][1])
    pos[69] = (pos[0][0], pos[0][1] + 0.6)                            # 0 / 69: words 0 and 2
    pos[40] = (early[1][0] + 0.3, early[1][1])                        # on an accepted box of the earlier call
    pos[45] = (len_box[0] + 0.2, len_box[1])                          # on a scene box of class len(class_names)
    pos[50] = pad_box                                                 # on a padding row: not an obstacle
    scene = [_box(-45.0 + 6.0 * k, -20.0, g.uniform(-1, 1)) for k in range(6)]
    scene += [_box(*len_box, 0.1), _box(*pad_box, 0.0)]
    scls = [0, 3, 5, 8, 9, 2, N_CLASSES, -1]
    cand = [_box(x, y, g.uniform(-0.3, 0.3)) for x, y in early] + [_box(*pos[i], g.uniform(-0.3, 0.3)) for i in range(70)]
    cand += [_box(0.0, 0.0, 0.0)] * 3                                 # trailing padding candidates
    ccls = [1] * 3 + [0] * 70 + [-1] * 3
    acc = np.zeros(76, bool)
    acc[:73] = True
    for i in (0, 31, 62, 63, 40, 45):
        acc[3 + i] = False
    acc[73:] = False
    return scene, scls, cand, ccls, acc


def word_launch(n_points=20000, n_tail=500, seed=1):
    """Three frames, S = 76 candidate slots, M = 8 scene slots:
      frame 0  an earlier class call of 3 accepted candidates, then one call of 70 packed so that its collisions cross
               the collision-row words at 31/32, 62-63/64 and 0/69, one candidate on an accepted box of the earlier
               call, one on a scene box of class len(class_names) (both rejected) and one on a padding row
               (accepted); candidates 10, 20 and 32 have no points;
      frame 1  no scene boxes (all padding) and a call of 5 with one colliding pair;
      frame 2  scene boxes and no candidates.
    n_points scene points per frame, then n_tail frame-B rows.  Returns (operands, expected acceptance [3, 76])."""
    g = np.random.default_rng(seed)
    scene0, scls0, cand0, ccls0, acc0 = _word_frame0(g)
    cand1 = [_box(-10.0 + 5.0 * k, -40.0, 0.2) for k in range(5)]
    cand1[3] = _box(cand1[2][0] + 0.5, -40.0, 0.2)                   # 2 collides with 3: 2 rejected, 3 accepted
    cand1 += [_box(0.0, 0.0, 0.0)] * 71
    acc1 = np.zeros(76, bool)
    acc1[[0, 1, 3, 4]] = True
    frames = [(scene0, scls0, cand0, ccls0),
              ([_box(0.0, 0.0, 0.0)] * 8, [-1] * 8, cand1, [7] * 5 + [-1] * 71),
              ([_box(-40.0 + 10.0 * k, 30.0, 0.5) for k in range(8)], list(range(8)), [_box(0.0, 0.0, 0.0)] * 76, [-1] * 76)]
    cpts = []
    for f, (_, _, cand, ccls) in enumerate(frames):
        empty = {3 + 10, 3 + 20, 3 + 32} if f == 0 else set()
        cpts.append([_object_points(g, b, 0 if (c < 0 or s in empty) else int(g.integers(5, 40)))
                     for s, (b, c) in enumerate(zip(cand, ccls))])
    points = np.concatenate([_cloud(g, n_points, f, -50.0, 50.0) for f in range(3)] + [_tail(n_tail, 3)])
    return _pack(points, frames, cpts), np.stack([acc0, acc1, np.zeros(76, bool)])


def aug_records(B, seed=2):
    """aug [B, 4, 4] fp64 with all four record kinds in varying order and the flips (x and y, x only, y only)."""
    g = np.random.default_rng(seed)
    out = np.zeros((B, 4, 4))
    flips = ((1.0, 1.0), (1.0, 0.0), (0.0, 1.0))
    for f in range(B):
        th = g.uniform(-0.785, 0.785)
        recs = [[1, th, np.cos(th), np.sin(th)], [2, g.uniform(0.9, 1.1), 0, 0], [3, g.normal(0, 0.5), 0, 0],
                [4, *flips[f % 3], 0]]
        out[f] = [recs[(k + f) % 4] for k in range(4)]
    return out


def aug_launch(B=3, n_per_frame=540000, M=200, n_tail=3000, seed=3):
    """Points [B n + n_tail, 6] (frames in order, then frame-B rows) and boxes [B, M, 9] with NaN elements, yaws on
    both sides of +-pi and padding rows, with aug_records(B)."""
    g = np.random.default_rng(seed)
    pts = np.concatenate([_cloud(g, n_per_frame, f, -76.8, 76.8) for f in range(B)] + [_tail(n_tail, B)])
    pts[:, 4:6] = g.uniform(0, 1, (len(pts), 2))
    pts[-n_tail:, 1:] = 0.0
    boxes = np.concatenate([g.uniform(-70, 70, (B, M, 2)), g.uniform(-2, 1, (B, M, 1)), g.uniform(0.5, 5, (B, M, 3)),
                            g.normal(0, 3, (B, M, 2)), g.uniform(-np.pi, np.pi, (B, M, 1))], 2).astype(F)
    boxes[:, :8, 8] = F([np.pi, -np.pi, 3.1415925, -3.1415925, 0.0, -0.0, 1.5707964, -1.5707964])
    nan = g.uniform(0, 1, boxes.shape) < 0.03
    boxes[nan] = np.nan
    boxes[:, -5:] = 0.0                                            # padding rows
    boxes[:, -5:, 3:6] = 1.0
    return pts, boxes, aug_records(B)


def gts_oracle_full(op):
    """oracle/gts_oracle.apply on the operands, with the point output laid out like the kernels': [n + P, 6], the rows
    past count set to (B, 0, 0, 0, 0, 0) -> (points, boxes, classes, accepted int32, count)."""
    pts, boxes, classes, acc = gts_oracle.apply(*[op[k] for k in KEYS])
    B = op["gt_boxes"].shape[0]
    out = np.zeros((len(op["points"]) + len(op["cand_points"]), 6), F)
    out[:, 0] = B
    out[:len(pts)] = pts
    return out, boxes, classes, acc.astype(np.int32), len(pts)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def gts_fails(got, want, what):
    """(points, boxes, classes, accepted, count) against the same from a reference, bit for bit -> failure strings."""
    names = ("points", "boxes", "classes", "accepted")
    bad = ["%s: %s differs" % (what, n) for n, g, w in zip(names, got[:4], want[:4]) if not same_bits(g, w)]
    gc, wc = (int(np.asarray(x).reshape(-1)[0]) for x in (got[4], want[4]))
    if gc != wc:
        bad.append("%s: count %d, want %d" % (what, gc, wc))
    return bad


def reduced(op, n_keep):
    """A copy of an edge case with the first n_keep scene points of each frame and its tail rows."""
    p = op["points"]
    keep = np.zeros(len(p), bool)
    for f in np.unique(p[:, 0]):
        idx = np.flatnonzero(p[:, 0] == f)
        keep[idx[:n_keep]] = True
    return dict(op, points=np.ascontiguousarray(p[keep]))


# ------------------------------------------------------------------------------------------------- tests
def test_builders_reach_the_select_thresholds_and_the_cap():
    S = 64
    m48, past48 = boxes_around(SMEM_OPT_IN, S)
    mcap, pastcap = boxes_around(SMEM_CAP, S)
    assert select_smem(m48, S) <= SMEM_OPT_IN < select_smem(past48, S)
    assert select_smem(mcap, S) <= SMEM_CAP < select_smem(pastcap, S)
    assert (past48 + S, mcap + S) == (926, 3918)
    for M in (past48, mcap):
        op = grid_launch(M, S, n_points=100)
        assert op["gt_boxes"].shape == (1, M, 9) and op["cand_boxes"].shape == (1, S, 9)
        assert (op["points"][:, 0] == 1).sum() == 700
        assert (np.diff(op["cand_offsets"]) == 0).any() and (np.diff(op["cand_offsets"]) > 0).any()


def test_word_launch_crosses_the_collision_row_words():
    op, acc = word_launch(n_points=200)
    cc = op["cand_classes"]
    runs = [(f, s) for f in range(cc.shape[0]) for s in range(cc.shape[1])
            if cc[f, s] >= 0 and (s == 0 or cc[f, s - 1] != cc[f, s])]
    longest = max(int(np.argmax(np.append(cc[f, s:] != cc[f, s], True))) for f, s in runs)
    assert longest >= 65 and select_smem(op["gt_boxes"].shape[1], cc.shape[1]) <= SMEM_OPT_IN
    assert (op["points"][:, 0] == 3).any()
    assert (op["gt_classes"][0] == N_CLASSES).any() and (op["gt_classes"][1] < 0).all()
    assert (op["cand_classes"][2] < 0).all()
    lens = np.diff(op["cand_offsets"]).reshape(3, -1)
    assert (lens[0][[13, 23, 35]] == 0).all() and (lens[0][3:73] > 0).sum() == 67
    # the collision rows the kernel sees cross the word boundaries: 31 | 32, 63 | 64, 0 | 69
    geo = [gts_oracle.corners(b, *t[:2]) for b, t in zip(op["cand_boxes"][0], op["cand_trig"][0])]
    for i, j in ((31, 32), (63, 64), (62, 63), (0, 69)):
        assert gts_oracle.collide(geo[3 + i], geo[3 + j]) and gts_oracle.collide(geo[3 + j], geo[3 + i])
        assert i // 32 != j // 32 or (i, j) == (62, 63)
    want = gts_oracle_full(op)
    assert same_bits(want[3], acc.astype(np.int32)), np.argwhere(want[3] != acc)


def test_oracle_chain_equals_the_host_twin_chain_on_reduced_edge_cases():
    """gt_sample then global_aug on every edge case with 3000 scene points per frame: oracle against host twins."""
    S = 64
    cases = {"past 48 KB": grid_launch(boxes_around(SMEM_OPT_IN, S)[1], S, n_points=3000),
             "at the cap": grid_launch(boxes_around(SMEM_CAP, S)[0], S, n_points=3000),
             "words": reduced(word_launch()[0], 3000)}
    bad = []
    for what, op in cases.items():
        want = gts_oracle_full(op)
        got = ops.gt_sample_host(*[op[k] for k in KEYS])
        bad += gts_fails(got, want, what)
        assert 0 < want[3].sum() < want[3].size
        aug = aug_records(op["gt_boxes"].shape[0])
        pa, ba = aug_oracle.apply(want[0], want[1], aug)
        ph, bh = ops.global_aug_host(got[0], got[1], aug)
        if not (same_bits(pa, ph) and same_bits(ba, bh)):
            bad.append("%s: global_aug differs" % what)
    pts, boxes, aug = aug_launch(n_per_frame=5000, n_tail=300)
    pa, ba = aug_oracle.apply(pts, boxes, aug)
    ph, bh = ops.global_aug_host(pts, boxes, aug)
    if not (same_bits(pa, ph) and same_bits(ba, bh)):
        bad.append("aug launch: global_aug differs")
    assert np.isnan(ba).any() and (ba.view(np.int32)[np.isnan(ba)] == 0x7fc00000).all()
    assert not bad, bad
