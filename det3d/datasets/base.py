"""Drop-in for the reference's BaseDataset (det3d/datasets/base.py): the info-file readers' shared constructor and
__getitem__.

Constructor arguments, the info pickle at root_path / info_path and the order of the np.random draws are the
reference's: the loading_pipelines methods, then the sampler, then the augmentation transforms in dict order, then
prepare_label.  What a frame hands on differs: it is the record pillarnext_b200.scenes.SyntheticSceneDataset makes, so
scenes.collate and SingleStageDetector.training_step / validation_step take it unchanged.
  points [N, 5] fp32        the key frame (x, y, z, intensity, time), in its stored frame
  sweeps                    past sweeps, untransformed, with their fp64 transforms (accumulated on the GPU)
  gts                       the sampler's candidate objects (the collision test, removal and paste run on the GPU)
  aug                       the augmentation records (applied on the GPU)
  gt_boxes_raw [M, 9] fp32, gt_classes [M] int32   the annotations, classes as AssignLabel numbers them
The label targets themselves are built on the GPU (pnx_assign_labels).  With create_database=True the `annotations`
stay in the record, as in the reference."""
import os
import pickle
from pathlib import Path

import numpy as np
from torch.utils.data import Dataset

from pillarnext_b200 import scenes


class BaseDataset(Dataset):
    def __init__(self, root_path, info_path, sampler=None, loading_pipelines=None, augmentation=None, prepare_label=None,
                 evaluations=None, create_database=False, use_gt_sampling=True):
        self._info_path = info_path
        self._root_path = Path(root_path)
        self.loading_pipelines = loading_pipelines
        self.augmentations = augmentation
        self.prepare_label = prepare_label
        self.evaluations = evaluations
        self.create_database = create_database
        self.use_gt_sampling = use_gt_sampling
        self.load_infos()
        self.class_names = None
        for pl in (prepare_label or {}).values():
            if hasattr(pl, "class_names"):
                self.class_names = pl.class_names
        if use_gt_sampling and sampler is not None:
            if self.class_names is None:
                raise ValueError("a sampler needs prepare_label (AssignLabel) to number the sampled classes")
            self.sampler = sampler()
        else:
            self.sampler = None

    def __len__(self):
        return len(self.infos)

    def load_infos(self):
        with open(os.path.join(self._root_path, self._info_path), "rb") as f:
            self.infos = pickle.load(f)

    def load_pointcloud(self, res, info):
        raise NotImplementedError

    def load_box3d(self, res, info):
        res["annotations"] = {"gt_boxes": info["gt_boxes"].astype(np.float32).copy(),
                              "gt_names": np.array(info["gt_names"]).reshape(-1).copy()}
        return res

    def __getitem__(self, idx):
        info = self.infos[idx]
        res = {"token": info["token"]}
        for lp in self.loading_pipelines or []:
            res = getattr(self, lp)(res, info)
        if self.sampler is not None:
            a = res["annotations"]
            res["gts"] = scenes.sampling_record(self.sampler, a["gt_boxes"], a["gt_names"], self.class_names)
        for aug in (self.augmentations or {}).values():
            res = aug(res)
        for pl in (self.prepare_label or {}).values():
            res = pl(res)
        if "gt_boxes_raw" not in res:
            res["gt_boxes_raw"], res["gt_classes"] = np.zeros((0, 9), np.float32), np.zeros(0, np.int32)
        if "annotations" in res and not self.create_database:
            del res["annotations"]
        return res
