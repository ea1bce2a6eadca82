"""Drop-in for the reference's ground-truth database sampler (the `sampler:` node of its training datasets):
BatchSampler, DBFilterByMinNumPoint and DataBaseSamplerV2.

Import paths, constructor arguments and the dbinfos pickle format are the reference's, and so are the random draws:
one np.random.shuffle per class list when the sampler is built (in dbinfos dict order, after the db_prepor filters),
and one more each time a class list runs out.  Per group class, in config order, n = round(rate * (max - count of the
class in the scene)) objects are drawn when n > 0; a request that reaches the end of the list (idx + n >= len, so also
one that fits exactly) returns only the rest of the list and reshuffles it.  The draws never depend on which objects
are accepted.

Difference: sample_all does not decide which drawn objects are pasted.  It returns the candidate record -- every drawn
object's box, name, stored points (read from its .bin as the reference reads the accepted ones, relative to the box
centre) and two (cos, sin) pairs of its yaw: numpy's vectorised fp32 pair, which the reference's corner path
(box_np_ops.center_to_corner_box2d) uses, and libm's cosf / sinf, which its numba point test (points_in_boxes_jit)
uses.  The collision test, the removal of scene points inside accepted boxes and the paste run on the GPU
(SingleStageDetector.gt_sample, ops.gt_sample, include/pnx.h).

Not supported (ValueError): 0 < gt_drop_percentage < 1 (per-point drops drawn for accepted objects only; no reference
config uses it), infos carrying `rot_transform` (the reference's create_gt_database never writes it), boxes that are not
float32, and a class listed twice in `groups` (the GPU tells class calls apart by runs of equal class ids)."""
import ctypes
import ctypes.util
import pathlib
import pickle

import numpy as np

_libm = None


def libm_trig(yaw):
    """(cosf, sinf) of each fp32 yaw through the C library: the values numba's scalar fp32 np.cos / np.sin give."""
    global _libm
    if _libm is None:
        lib = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
        for fn in (lib.cosf, lib.sinf):
            fn.restype, fn.argtypes = ctypes.c_float, [ctypes.c_float]
        _libm = lib
    yaw = np.asarray(yaw, dtype=np.float32).reshape(-1)
    out = np.empty((len(yaw), 2), dtype=np.float32)
    for i, a in enumerate(yaw.tolist()):
        out[i] = _libm.cosf(a), _libm.sinf(a)
    return out


def numpy_trig(boxes):
    """numpy's fp32 (cos, sin) of the yaws of 9-column boxes, taken the way center_to_corner_box2d takes them."""
    yaw = np.asarray(boxes, dtype=np.float32)[:, [0, 1, 3, 4, -1]][:, -1]
    return np.stack([np.cos(yaw), np.sin(yaw)], axis=1).astype(np.float32)


class BatchSampler:
    """Walks a shuffled index list of one class's infos, `num` at a time."""

    def __init__(self, sampled_list, name=None, epoch=None, shuffle=True, drop_reminder=False):
        self._sampled_list = sampled_list
        self._example_num = len(sampled_list)
        self._indices = np.arange(self._example_num)
        self._shuffle = shuffle
        if shuffle:
            np.random.shuffle(self._indices)
        self._idx = 0
        self._name = name
        self._epoch = epoch
        self._epoch_counter = 0
        self._drop_reminder = drop_reminder

    def _sample(self, num):
        start = self._idx
        if start + num < self._example_num:
            self._idx = start + num
            return self._indices[start:start + num]
        rest = self._indices[start:].copy()       # reaching the end (even exactly) returns the rest and reshuffles
        self._reset()
        return rest

    def _reset(self):
        if self._shuffle:
            np.random.shuffle(self._indices)
        self._idx = 0

    def sample(self, num):
        return [self._sampled_list[i] for i in self._sample(num)]


class DataBasePreprocessing:
    def __call__(self, db_infos):
        return self._preprocess(db_infos)

    def _preprocess(self, db_infos):
        raise NotImplementedError


class DBFilterByMinNumPoint(DataBasePreprocessing):
    """Keeps the infos of each listed class with at least min_gt_point_dict[class] stored points (0 keeps all)."""

    def __init__(self, min_gt_point_dict, logger=None):
        self._min_gt_point_dict = min_gt_point_dict

    def _preprocess(self, db_infos):
        for name, min_num in self._min_gt_point_dict.items():
            if min_num > 0:
                db_infos[name] = [info for info in db_infos[name] if info["num_points_in_gt"] >= min_num]
        return db_infos


class DataBaseSamplerV2:
    def __init__(self, root_path, dbinfo_path, groups, db_prepor, rate, gt_drop_percentage, gt_drop_max_keep_points,
                 point_dim):
        if 0 < gt_drop_percentage < 1:
            raise ValueError("gt_drop_percentage in (0, 1) is not supported: per-point drops of the pasted objects are "
                             "not implemented (every reference config uses 0)")
        self.root_path = root_path
        with open(pathlib.Path(root_path) / dbinfo_path, "rb") as f:
            db_infos = pickle.load(f)
        for infos in db_infos.values():
            for info in infos:
                if "rot_transform" in info:
                    raise ValueError("dbinfos with rot_transform are not supported (%s)" % info.get("path"))
                if np.asarray(info["box3d_lidar"]).dtype != np.float32:
                    raise ValueError("box3d_lidar must be float32 (%s)" % info.get("path"))
        if db_prepor is not None:
            for prepor in db_prepor.values():
                db_infos = prepor(db_infos)
        self.db_infos = db_infos
        self._rate = rate
        self._groups = groups
        self._point_dim = point_dim
        self._gt_drop_rate = gt_drop_percentage
        self._gt_drop_max_keep = gt_drop_max_keep_points
        self._sample_classes, self._sample_max_nums = [], []
        for group in groups:
            self._sample_classes += list(group.keys())
            self._sample_max_nums += list(group.values())
        if len(set(self._sample_classes)) != len(self._sample_classes):
            raise ValueError("a class is listed twice in groups: %s" % (self._sample_classes,))
        self._group_db_infos = self.db_infos
        self._sampler_dict = {k: BatchSampler(v, k) for k, v in self._group_db_infos.items()}

    def sample_all(self, gt_boxes, gt_names):
        """The candidate record of one frame, or None when nothing is drawn:
            gt_names [S] str, gt_boxes [S, 9] float32, difficulty [S]   every drawn object, in draw order
            points [sum num_points, point_dim] float32                   their stored points, relative to the centre
            num_points [S] int64
            trig [S, 4] float32                                          numpy cos, numpy sin, libm cosf, sinf of the yaw
        Consecutive objects of one class form one class call of the reference's sample_class_v2."""
        names = list(gt_names)
        drawn = []
        for class_name, max_num in zip(self._sample_classes, self._sample_max_nums):
            n = int(max_num - np.sum([nm == class_name for nm in names]))
            n = np.round(self._rate * n).astype(np.int64)
            if n > 0:
                got = self._sampler_dict[class_name].sample(n)
                if not got:
                    raise ValueError("no database objects left for class %r" % class_name)
                drawn += got
        if not drawn:
            return None
        boxes = np.stack([np.asarray(s["box3d_lidar"], dtype=np.float32) for s in drawn], axis=0)
        pts = [np.fromfile(str(pathlib.Path(self.root_path) / s["path"]), dtype=np.float32).reshape(-1, self._point_dim)
               for s in drawn]
        return {
            "gt_names": np.array([s["name"] for s in drawn]),
            "difficulty": np.array([s["difficulty"] for s in drawn]),
            "gt_boxes": boxes,
            "points": np.concatenate(pts, axis=0).astype(np.float32),
            "num_points": np.array([len(p) for p in pts], dtype=np.int64),
            "trig": np.concatenate([numpy_trig(boxes), libm_trig(boxes[:, -1])], axis=1),
        }
