"""Drop-in check at the CONFIG level (SURVEY.md section 8b/8f-F4), CPU only.  tests/golden/ref_configs.json.gz holds the
reference's experiment files composed to the model node (pillarnext_b200/hydra_lite.py) and the state-dict shapes of its own
reader / neck / head; `instantiate(cfg.model)` (tools/train.py:53) must build this repo's modules with the same shapes.
"""
import gzip
import json
import os

import pytest

from pillarnext_b200 import hydra_lite

_instantiate = hydra_lite.instantiate
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_configs.json.gz")


@pytest.mark.parametrize("experiment,n_tasks,has_iou", [("nusc_det_pp18_aspp_iou_sp", 6, False),
                                                         ("waymo_det_pp18_aspp_iou_car_sp", 2, True)])
def test_reference_experiment_instantiates_our_modules(experiment, n_tasks, has_iou):
    with gzip.open(GOLD, "rt") as fh:
        gold = json.load(fh)[experiment]
    m = gold["model"]
    assert m["_target_"] == "det3d.models.detectors.single_stage.SingleStageDetector"
    assert m["backbone"]["num_input_features"] == 64 and len(m["head"]["tasks"]) == n_tasks      # interpolations resolved
    assert m["post_processing"]["out_size_factor"] == [4] * n_tasks
    model = _instantiate(m)                                           # tools/train.py:53 `instantiate(cfg.model)`
    from pillarnext_b200 import modules
    assert isinstance(model, modules.SingleStageDetector) and isinstance(model.head, modules.CenterHead)
    assert model.post_processing["nms"]["nms_pre_max_size"] >= model.post_processing["nms"]["nms_post_max_size"]
    assert ("iou" in model.head.tasks[0].heads) == has_iou
    assert [float(r) for r in model.head.rectifier[0]] == [float(r) for r in m["head"]["rectifier"][0]]
    # the reference's own reader / neck / head built from the same composed node: identical parameter/buffer names+shapes
    ours = model.state_dict()
    for part in ("reader", "neck", "head"):
        want = {k: tuple(v) for k, v in gold["state_dict_shapes"].items() if k.startswith(part + ".")}
        got = {k: tuple(v.shape) for k, v in ours.items() if k.startswith(part + ".")}
        assert got == want, (part, sorted(set(got) ^ set(want))[:6])
    n_params = sum(p.numel() for p in model.parameters())
    assert n_params == (10_379_782 if experiment.startswith("nusc") else n_params)             # SURVEY section 8a count
