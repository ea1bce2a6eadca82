"""The binding boundary, CPU only.

* pillarnext_b200/ops.py is the only caller of libpnx: no other module of the package, det3d or tools imports the
  ctypes binding (_lib) or calls a function named `lib`;
* every host twin wrapper of ops.py checks its numpy operands: an fp64 array where fp32 is required and an operand with
  the wrong trailing dimension raise, and a non-contiguous operand gives the result of its contiguous copy.
"""
import ast
import os

import numpy as np
import pytest

from oracle.predict_fixtures import fake_preds, to_rows
from pillarnext_b200 import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BINDING = {os.path.join("pillarnext_b200", "ops.py"), os.path.join("pillarnext_b200", "_lib.py")}


def _violations(tree):
    for node in ast.walk(tree):
        if isinstance(node, ast.Import):
            for a in node.names:
                if "_lib" in a.name.split("."):
                    yield node.lineno, "import " + a.name
        elif isinstance(node, ast.ImportFrom):
            if "_lib" in (node.module or "").split(".") or any(a.name == "_lib" for a in node.names):
                yield node.lineno, "from %s%s import ..." % ("." * node.level, node.module or "")
        elif isinstance(node, ast.Call):
            f = node.func
            if (isinstance(f, ast.Name) and f.id == "lib") or (isinstance(f, ast.Attribute) and f.attr == "lib"):
                yield node.lineno, "call of lib()"


def test_only_ops_calls_the_library():
    bad, n_files = [], 0
    for top in ("pillarnext_b200", "det3d", "tools"):
        for d, _, files in os.walk(os.path.join(ROOT, top)):
            for f in sorted(files):
                rel = os.path.relpath(os.path.join(d, f), ROOT)
                if not f.endswith(".py") or rel in BINDING:
                    continue
                n_files += 1
                with open(os.path.join(ROOT, rel)) as fh:
                    tree = ast.parse(fh.read(), rel)
                bad += ["%s:%d: %s" % (rel, line, what) for line, what in _violations(tree)]
    assert n_files > 40
    assert not bad, "libpnx is called outside pillarnext_b200/ops.py:\n" + "\n".join(bad)


def test_the_check_sees_each_kind_of_call():
    src = "from ._lib import check\nfrom pillarnext_b200 import _lib\nimport pillarnext_b200._lib\nL = ops.lib()\nlib()\n"
    assert len(list(_violations(ast.parse(src)))) == 5
    assert not list(_violations(ast.parse("bn.pnx_sync = True\nx = ops.bitmap_words(1, 2, 3)\n")))


# ---------------------------------------------------------------------- host twin wrappers
def _boxes9(rng, *lead):
    n = int(np.prod(lead))
    b = np.concatenate([rng.uniform(-6, 6, (n, 2)), rng.uniform(-1, 1, (n, 1)), rng.uniform(1, 3, (n, 3)),
                        rng.normal(0, 1, (n, 2)), rng.uniform(-np.pi, np.pi, (n, 1))], 1)
    return b.reshape(*lead, 9).astype(np.float32)


def _trig(boxes):
    return np.stack([np.cos(boxes[..., 8]), np.sin(boxes[..., 8])], -1).astype(np.float32)


def _points(rng, n, frames, cols=4):
    p = np.concatenate([rng.integers(0, frames, (n, 1)), rng.uniform(-8, 8, (n, 2)), rng.uniform(-1, 1, (n, 1)),
                        rng.uniform(0, 1, (n, cols - 4))], 1)
    return p.astype(np.float32)


def _decode(double_flip):
    out = to_rows(fake_preds(4 if double_flip else 1, 6, 5, 2, 3)).numpy()
    args = dict(out=out, B=1, H=6, W=5, C=2, offs=[0, 2, 3, 6, 8, 10, -1], osf=4.0, voxel_size=[0.075, 0.075],
                pc_range=[-50.4, -50.4], score_thr=0.1, post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0],
                rectifier=[0.0, 0.0], double_flip=double_flip)
    return ops.det_decode_host, args, "out", 11                  # the decode reads 12 columns at these offsets


def _box_pairs(fn):
    rng = np.random.default_rng(1)
    a, b = _boxes9(rng, 12)[:, [0, 1, 2, 3, 4, 5, 8]], _boxes9(rng, 12)[:, [0, 1, 2, 3, 4, 5, 8]]
    b[:6, :2] = a[:6, :2] + 0.5                                  # half of the pairs overlap
    return fn, dict(a=a, b=b), "a", 6


def _global_aug():
    rng = np.random.default_rng(2)
    aug = np.zeros((2, 4, 4))
    aug[:, 0] = (1, 0.3, np.cos(0.3), np.sin(0.3))
    aug[1, 1] = (4, 1.0, 0.0, 0.0)
    return ops.global_aug_host, dict(points=_points(rng, 40, 2, 6), gt_boxes=_boxes9(rng, 2, 3), aug=aug), "points", 5


def _gt_sample():
    rng = np.random.default_rng(3)
    boxes, cand = _boxes9(rng, 1, 2), _boxes9(rng, 1, 2)
    cand[0, :, 0] = (-30.0, 30.0)                                # far from the scene boxes: both accepted
    args = dict(points=_points(rng, 30, 1, 6), gt_boxes=boxes, gt_classes=np.array([[0, 1]], np.int32),
                gt_trig=_trig(boxes), cand_boxes=cand, cand_classes=np.array([[0, 0]], np.int32),
                cand_trig=np.concatenate([_trig(cand), _trig(cand)], -1),
                cand_points=rng.uniform(-0.5, 0.5, (4, 5)).astype(np.float32), cand_offsets=np.array([0, 2, 4], np.int32))
    return ops.gt_sample_host, args, "points", 5


def _points_in_boxes():
    rng = np.random.default_rng(4)
    boxes = _boxes9(rng, 3)
    return ops.points_in_boxes_host, dict(points=_points(rng, 50, 1), boxes=boxes, trig=_trig(boxes)), "boxes", 8


def _count_points():
    rng = np.random.default_rng(5)
    boxes = _boxes9(rng, 2, 3)
    args = dict(points=_points(rng, 60, 2), boxes=boxes, classes=np.array([[0, 1, -1], [1, 0, 0]], np.int32),
                trig=_trig(boxes))
    return ops.eval_count_points_host, args, "boxes", 8


def _detections(rng):
    gt = _boxes9(rng, 1, 3)
    det = np.concatenate([gt[0, :2], _boxes9(rng, 2)])[[0, 2, 1, 3]]        # segment 0: dets 0, 1; segment 1: dets 2, 3
    det[:, :2] += 0.2
    return dict(det_boxes=det, order=np.arange(4, dtype=np.int64), seg_start=np.array([0, 2], np.int32),
                seg_count=np.array([2, 2], np.int32), gt_boxes=gt, gt_classes=np.array([[0, 1, 0]], np.int32))


def _eval_match():
    rng = np.random.default_rng(6)
    args = _detections(rng)
    args.update(det_trig=_trig(args["det_boxes"]), gt_trig=_trig(args["gt_boxes"]), thresholds=np.full(2, 0.1, np.float32))
    return ops.eval_match_host, args, "det_boxes", 8


def _eval_match_center():
    args = _detections(np.random.default_rng(7))
    args.update(n_classes=2, dist_ths=np.array([0.5, 1.0, 2.0, 4.0]))
    return ops.eval_match_center_host, args, "det_boxes", 8


CASES = {"det_decode_host": lambda: _decode(False), "det_decode_host[double_flip]": lambda: _decode(True),
         "det_iou_bev_host": lambda: _box_pairs(ops.det_iou_bev_host),
         "aligned_iou3d_host": lambda: _box_pairs(ops.aligned_iou3d_host), "global_aug_host": _global_aug,
         "gt_sample_host": _gt_sample, "points_in_boxes_host": _points_in_boxes, "eval_count_points_host": _count_points,
         "eval_match_host": _eval_match, "eval_match_center_host": _eval_match_center}


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_wrapper_refuses_float64(name):
    fn, args, key, _ = CASES[name]()
    with pytest.raises(ValueError, match=key):
        fn(**dict(args, **{key: args[key].astype(np.float64)}))


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_wrapper_refuses_a_wrong_trailing_dimension(name):
    fn, args, key, cols = CASES[name]()
    with pytest.raises(ValueError, match=key):
        fn(**dict(args, **{key: np.ascontiguousarray(args[key][..., :cols])}))


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_wrapper_makes_operands_contiguous(name):
    fn, args, key, _ = CASES[name]()
    a = args[key]
    wide = np.zeros(a.shape[:-1] + (a.shape[-1] + 3,), a.dtype)
    wide[..., :a.shape[-1]] = a
    view = wide[..., :a.shape[-1]]
    assert not view.flags.c_contiguous
    want, got = fn(**args), fn(**dict(args, **{key: view}))
    want, got = (want, got) if isinstance(want, tuple) else ((want,), (got,))
    assert len(got) == len(want)
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g, w)
