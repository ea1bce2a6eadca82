"""Multi-sweep accumulation on the GPU (ops.accumulate_sweeps, pnx_accumulate_sweeps).

* bit-exact against the reference's own nuScenes and Waymo loaders (tests/golden/ref_sweeps.npz) and, at 6 frames x 10
  sweeps x 26.5k points and 3 frames x 3 sweeps x 180k points, against the host twin, tail rows included; the inputs
  are left untouched and the output stays frame-sorted;
* a training step fed a GPU-accumulated example gives a bit-identical loss and gradients to the same step fed the
  oracle's pre-accumulated, compacted points (both voxelizers; once more with gt sampling and augmentation in the chain),
  and validation_step returns the same detections, with and without double flip;
* a 6-epoch run of the ten-sweep experiment passes the NDS gate of tests/test_nds_metric_gpu.py (fp32-grade product
  against the fp32 oracle on oracle-accumulated points); the single-sweep run is trained beside it and both runs' NDS,
  mAP and mAVE are printed.  No velocity margin is asserted: in 6 epochs neither run learns the velocities (README).
"""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import sweeps_oracle as O
from pillarnext_b200 import functional as Fn
from pillarnext_b200 import hydra_lite, ops, scenes
from pillarnext_b200.trainer import example_to_device

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXPERIMENTS = os.path.join(ROOT, "configs", "experiments")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from test_sweeps_cpu import OPS, bits, golden  # noqa: E402


def run_gpu(a, md):
    dev = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]
    before = [t.clone() for t in dev]
    out, count = ops.accumulate_sweeps(*dev, md)
    torch.cuda.synchronize()
    assert all(torch.equal(x.view(torch.uint8), y.view(torch.uint8)) for x, y in zip(dev, before))   # inputs untouched
    return out.cpu().numpy(), int(count.item())


@pytest.mark.parametrize("case", ["nusc", "waymo", "drop"])
def test_accumulate_sweeps_matches_the_reference(case):
    a, md, want, _ = golden(case)
    got, count = run_gpu(a, md)
    assert count == len(want) and np.array_equal(bits(got[:count]), bits(want))
    assert np.array_equal(bits(got), bits(ops.accumulate_sweeps_host(*a, md)[0]))


@pytest.mark.parametrize("shape,md", [((6, 10, 26500), 1.0), ((3, 3, 180000), 1.0), ((6, 10, 26500), 0.0)])
def test_accumulate_sweeps_matches_the_host_twin_at_bench_shapes(shape, md):
    a = O.random_operands(*shape, seed=2)
    a = [a[k] for k in OPS]
    want, wc = ops.accumulate_sweeps_host(*a, md)
    got, count = run_gpu(a, md)
    assert count == wc and np.array_equal(bits(got), bits(want))          # tail rows included
    assert (count < len(got)) == (md > 0)
    assert np.all(got[count:, 0] == shape[0]) and np.all(np.diff(got[:count, 0]) >= 0)


def _model(cfg):
    torch.manual_seed(0)
    return hydra_lite.instantiate(cfg.model).cuda().train()


def _batch(ds, n=4):
    state = np.random.get_state()
    np.random.seed(3)
    try:
        return scenes.collate([ds[i] for i in range(n)])
    finally:
        np.random.set_state(state)


def _train_parity(cfg, ex, voxelizer):
    pre = O.accumulate_example(ex)
    ex_d, pre_d = example_to_device(ex, torch.device("cuda")), example_to_device(pre, torch.device("cuda"))
    prev = Fn.set_deterministic(True)
    try:
        runs = []
        for example in (ex_d, pre_d):
            model = _model(cfg)
            if voxelizer == "force":
                model.reader.frame_sorted = "force"
            loss, _ = model(example)
            loss.backward()
            torch.cuda.synchronize()
            runs.append((loss.detach().clone(), {k: v.grad.detach().clone() for k, v in model.named_parameters()}))
    finally:
        Fn.set_deterministic(prev)
    (loss_a, g_a), (loss_b, g_b) = runs
    assert torch.isfinite(loss_a) and torch.equal(loss_a, loss_b), (loss_a.item(), loss_b.item())
    assert not [k for k in g_a if not torch.equal(g_a[k], g_b[k])]
    assert "sweep_points" in ex_d                                        # the step did not consume the caller's example
    return ex_d


@pytest.mark.parametrize("voxelizer", ["default", "force"])
def test_training_step_on_gpu_accumulated_example_matches_preaccumulated_oracle(voxelizer):
    cfg = hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp_nds_sweeps", ["data.train_dataset.n_frames=4"])
    ex = _batch(hydra_lite.instantiate(cfg.data.train_dataset))
    assert len(ex["sweep_points"]) > 8 * len(ex["points"])
    _train_parity(cfg, ex, voxelizer)


def test_training_step_with_sweeps_sampling_and_augmentation_matches_preaccumulated_oracle(tmp_path):
    from test_gt_sampling_cpu import _gts_db
    _gts_db(tmp_path)
    cfg = hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp_gts", ["data.train_dataset.root_path=%s" % tmp_path,
                                                                    "data.train_dataset.n_frames=4",
                                                                    "+data.train_dataset.nsweeps=10"])
    ex = _batch(hydra_lite.instantiate(cfg.data.train_dataset))
    assert "gts_boxes" in ex and "aug" in ex and "sweep_points" in ex
    ex_d = _train_parity(cfg, ex, "default")
    assert "gts_boxes" in ex_d and "aug" in ex_d


@pytest.mark.parametrize("double_flip", [False, True])
def test_validation_step_on_sweeps_matches_preaccumulated_points(double_flip):
    ov = ["data.val_dataset.n_frames=3"] + (["+model.post_processing.double_flip=True"] if double_flip else [])
    cfg = hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp_nds_sweeps", ov)
    ex = scenes.collate([hydra_lite.instantiate(cfg.data.val_dataset)[i] for i in range(3)])
    pre = O.accumulate_example(ex)
    model = _model(cfg).eval()
    with torch.no_grad():
        for task in model.head.tasks:                                   # spread the heat-map logits so boxes pass
            task.hm[3].bias.fill_(-1.5)
            task.hm[3].weight.mul_(6.0)
    a = model(example_to_device(ex, torch.device("cuda")))
    b = model(example_to_device(pre, torch.device("cuda")))
    assert a.keys() == b.keys() and sum(len(d["scores"]) for d in a.values()) > 0
    for t in a:
        assert a[t].keys() == b[t].keys()
        for k, v in a[t].items():
            assert torch.equal(v, b[t][k]) if torch.is_tensor(v) else v == b[t][k], (t, k)


class _Accumulated:
    """A sweeps dataset whose frames carry the oracle's accumulated points instead of their sweeps."""

    def __init__(self, ds):
        self.ds = ds

    def __len__(self):
        return len(self.ds)

    def __getitem__(self, i):
        fr = dict(self.ds[i])
        sw = fr.pop("sweeps")
        key = np.c_[np.zeros(len(fr["points"]), np.float32), fr["points"]]
        off = np.concatenate([[0], np.cumsum(sw["counts"])]).astype(np.int32)
        out, count = O.accumulate(key, np.array([0, len(key)], np.int32), sw["points"], off, sw["transforms"][None],
                                  sw["min_distance"])
        fr["points"] = out[:count, 1:].copy()
        return fr


def test_train_sweeps_experiment_gate(tmp_path):
    import train as train_tool
    from test_map_gpu import oracle_detections
    overrides = ["trainer.max_epochs=6", "data.train_dataset.n_frames=640", "data.val_dataset.n_frames=24",
                 "dataloader.train.num_workers=0", "dataloader.val.num_workers=0", "dataloader.train.batch_size=4"]
    results = {}
    for name in ("synth_det_pp18_aspp_nds_sweeps", "synth_det_pp18_aspp_nds"):
        work = str(tmp_path / name)
        torch.manual_seed(0)
        tr = train_tool.main(["--config-name", name, "--work-dir", work] + overrides)
        assert tr.epoch == 6
        cfg = hydra_lite.main(EXPERIMENTS, name, overrides)
        val = hydra_lite.instantiate(cfg.data.val_dataset)
        model = tr.model.eval()
        dets = {}
        with torch.no_grad():
            for i0 in range(0, len(val), 4):
                ex = scenes.collate([val[i] for i in range(i0, min(len(val), i0 + 4))])
                dets.update(model(example_to_device(ex, torch.device("cuda"))))
        m = {"bf16": val.evaluation(dets)}
        if name.endswith("sweeps"):
            dets = {}
            with Fn.precision("split"), torch.no_grad():
                for i0 in range(0, len(val), 4):
                    ex = scenes.collate([val[i] for i in range(i0, min(len(val), i0 + 4))])
                    dets.update(model(example_to_device(ex, torch.device("cuda"))))
            m["split"] = val.evaluation(dets)
            sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items()}
            m["oracle"] = val.evaluation(oracle_detections(cfg, sd, _Accumulated(val)))
        results[name] = m
    sw = results["synth_det_pp18_aspp_nds_sweeps"]
    msg = "NDS / mAP / mAVE on 24 held-out scenes: " + " | ".join(
        "%s %s %.3f / %.3f / %.3f" % (name[len("synth_det_pp18_aspp_"):], k, v["NDS"], v["mAP"], v["mAVE"])
        for name, m in results.items() for k, v in m.items())
    print(msg)
    assert sw["oracle"]["mAP"] > 5.0, msg
    assert abs(sw["split"]["NDS"] - sw["oracle"]["NDS"]) <= 0.1 and abs(sw["split"]["mAP"] - sw["oracle"]["mAP"]) <= 0.1, msg
    assert abs(sw["bf16"]["NDS"] - sw["oracle"]["NDS"]) <= 1.5, msg
