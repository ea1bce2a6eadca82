"""Drop-in for the reference's AssignLabel (det3d/datasets/pipelines/assign.py), the `prepare_label.centermap` node of
its training datasets.

Constructor arguments are the reference's.  __call__ does not build the heat maps and regression targets: it hands the
frame's annotations on as gt_boxes_raw [M, 9] fp32 and gt_classes [M] int32, and the detector builds the targets on
the GPU (SingleStageDetector.assign_labels, pnx_assign_labels).  A class is numbered by its position in the flattened
`tasks`.  A name outside the tasks gets len(class_names): label assignment skips it, as the reference's does, while the
box still takes part in the ground-truth sampler's collision test, as in the reference.

The GPU reads gaussian_overlap, max_objs and min_radius from SingleStageDetector.label_cfg (the values of every
reference config); other values raise ValueError here instead of being ignored.  pc_range, voxel_size and
out_size_factor are the model's own (head.pc_range / voxel_size / out_size_factor)."""
import numpy as np


class AssignLabel(object):
    def __init__(self, tasks, gaussian_overlap, max_objs, min_radius, pc_range, voxel_size, out_size_factor):
        from pillarnext_b200.modules import SingleStageDetector
        got = dict(gaussian_overlap=gaussian_overlap, max_objs=max_objs, min_radius=min_radius)
        if got != SingleStageDetector.label_cfg:
            raise ValueError("label assignment runs on the GPU with %s, got %s" % (SingleStageDetector.label_cfg, got))
        self.out_size_factor = np.array(out_size_factor)
        self.tasks = tasks
        self.gaussian_overlap = gaussian_overlap
        self._max_objs = max_objs
        self._min_radius = min_radius
        self.pc_range = np.array(pc_range)
        self.voxel_size = np.array(voxel_size)
        self.class_names = [n for t in tasks for n in t]

    def __call__(self, res):
        a = res["annotations"]
        ids = {n: i for i, n in enumerate(self.class_names)}
        res["gt_boxes_raw"] = np.asarray(a["gt_boxes"], np.float32).reshape(-1, 9)
        res["gt_classes"] = np.array([ids.get(n, len(self.class_names)) for n in a["gt_names"]], np.int32)
        return res
