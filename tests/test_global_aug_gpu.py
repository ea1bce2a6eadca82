"""Global training augmentation on the GPU (ops.global_aug, pnx_global_aug).

* bit-exact against the reference's own outputs (tests/golden/ref_aug.npz) and, at 6 frames x 30k points, against the
  host twin; the inputs are left untouched;
* a training step fed an augmented example (records applied on the GPU) gives a bit-identical loss and bit-identical
  gradients to the same step fed the oracle's pre-augmented points and boxes;
* a short tools/train.py run of the `_aug` experiment passes the mAP gate of tests/test_map_gpu.py: the fp32-grade
  product against the fp32 oracle on the same weights, within 0.1 mAP.
"""
import os
import sys

import numpy as np
import pytest
import torch

from det3d.datasets.pipelines import augmentation as A
from oracle import aug_oracle
from pillarnext_b200 import functional as Fn
from pillarnext_b200 import hydra_lite, ops, scenes
from pillarnext_b200.trainer import example_to_device

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXPERIMENTS = os.path.join(ROOT, "configs", "experiments")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from test_global_aug_cpu import host_aug  # noqa: E402


def bits(t):
    return t.contiguous().view(torch.int32)


def test_global_aug_matches_the_reference_goldens():
    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_aug.npz"))
    pts, boxes, aug = (torch.from_numpy(g[k]).cuda() for k in ("points", "boxes", "aug"))
    p_in, b_in = pts.clone(), boxes.clone()
    p, b = ops.global_aug(pts, boxes, aug)
    torch.cuda.synchronize()
    assert torch.equal(bits(p.cpu()), bits(torch.from_numpy(g["out_points"])))
    assert torch.equal(bits(b.cpu()), bits(torch.from_numpy(g["out_boxes"])))
    assert torch.equal(bits(pts), bits(p_in)) and torch.equal(bits(boxes), bits(b_in))


def test_global_aug_matches_the_host_twin_at_6x30k():
    rng = np.random.default_rng(8)
    B, n, M = 6, 30000, 60
    pts = np.concatenate([np.concatenate([np.full((n, 1), f), rng.uniform(-80, 80, (n, 2)), rng.uniform(-5, 3, (n, 1)),
                                          rng.uniform(0, 255, (n, 1)), rng.uniform(0, 0.5, (n, 1))], 1)
                          for f in range(B)]).astype(np.float32)
    boxes = np.concatenate([rng.uniform(-80, 80, (B, M, 3)), rng.uniform(0.3, 12, (B, M, 3)), rng.normal(0, 3, (B, M, 2)),
                            rng.uniform(-np.pi, np.pi, (B, M, 1))], 2).astype(np.float32)
    boxes[:, ::5, 6] = np.nan
    boxes[:, 1::5, 8] = np.float32(np.pi)
    boxes[:, -3:] = [0, 0, 0, 1, 1, 1, 0, 0, 0]                      # padding rows
    state = np.random.get_state()
    np.random.seed(21)
    chain = [A.Rotation([-0.785, 0.785]), A.Scaling([0.9, 1.1]), A.Translation(0.5), A.Flip([0.5, 0.5])]
    aug = np.zeros((B, 4, 4))
    for f in range(B):
        res = {}
        for op in chain:
            res = op(res)
        aug[f] = res["aug"]
    np.random.set_state(state)
    aug[5, 1:] = 0                                                   # a frame with one record only
    p_h, b_h = host_aug(pts, boxes, aug)
    pts_d, boxes_d, aug_d = torch.from_numpy(pts).cuda(), torch.from_numpy(boxes).cuda(), torch.from_numpy(aug).cuda()
    p_in, b_in = pts_d.clone(), boxes_d.clone()
    p, b = ops.global_aug(pts_d, boxes_d, aug_d)
    torch.cuda.synchronize()
    assert torch.equal(bits(p.cpu()), bits(torch.from_numpy(p_h)))
    assert torch.equal(bits(b.cpu()), bits(torch.from_numpy(b_h)))
    assert torch.equal(bits(pts_d), bits(p_in)) and torch.equal(bits(boxes_d), bits(b_in))
    assert not torch.equal(p, pts_d)


def _model(cfg):
    torch.manual_seed(0)
    return hydra_lite.instantiate(cfg.model).cuda().train()


def test_training_step_on_gpu_augmented_example_matches_preaugmented_oracle():
    cfg = hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp_aug", ["data.train_dataset.n_frames=4"])
    ds = hydra_lite.instantiate(cfg.data.train_dataset)
    state = np.random.get_state()
    np.random.seed(3)
    ex = scenes.collate([ds[i] for i in range(4)])
    np.random.set_state(state)
    assert ex["aug"][:, 3, 1:3].sum() > 0                            # some frame is flipped
    p_o, b_o = aug_oracle.apply(ex["points"].numpy(), ex["gt_boxes_raw"].numpy(), ex["aug"].numpy())
    pre = {k: v for k, v in ex.items() if k != "aug"}
    pre["points"], pre["gt_boxes_raw"] = torch.from_numpy(p_o), torch.from_numpy(b_o)
    ex_d, pre_d = example_to_device(ex, torch.device("cuda")), example_to_device(pre, torch.device("cuda"))
    p, b = ops.global_aug(ex_d["points"], ex_d["gt_boxes_raw"], ex_d["aug"])
    assert torch.equal(bits(p), bits(pre_d["points"])) and torch.equal(bits(b), bits(pre_d["gt_boxes_raw"]))
    prev = Fn.set_deterministic(True)
    try:
        runs = []
        for example in (ex_d, pre_d):
            model = _model(cfg)
            loss, _ = model(example)
            loss.backward()
            torch.cuda.synchronize()
            runs.append((loss.detach().clone(), {k: v.grad.detach().clone() for k, v in model.named_parameters()}))
    finally:
        Fn.set_deterministic(prev)
    (loss_a, g_a), (loss_b, g_b) = runs
    assert torch.isfinite(loss_a) and torch.equal(loss_a, loss_b), (loss_a.item(), loss_b.item())
    assert not [k for k in g_a if not torch.equal(g_a[k], g_b[k])]
    assert "aug" in ex_d                                             # the step did not consume the caller's example


def test_aug_experiment_passes_the_map_gate(tmp_path):
    import train as train_tool
    from test_map_gpu import oracle_detections
    overrides = ["trainer.max_epochs=6", "data.train_dataset.n_frames=640", "data.val_dataset.n_frames=24",
                 "dataloader.train.num_workers=0", "dataloader.val.num_workers=0", "dataloader.train.batch_size=4"]
    maps = {}
    for name in ("synth_det_pp18_aspp_aug", "synth_det_pp18_aspp"):
        state = np.random.get_state()
        np.random.seed(0)
        tr = train_tool.main(["--config-name", name, "--work-dir", str(tmp_path / name)] + overrides)
        np.random.set_state(state)
        cfg = hydra_lite.main(EXPERIMENTS, name, overrides)
        val = hydra_lite.instantiate(cfg.data.val_dataset)
        model = tr.model.eval()
        sd = {k: v.detach().float().cpu() for k, v in model.state_dict().items()}
        m_oracle = val.evaluation(oracle_detections(cfg, sd, val))["mAP"]
        dets = {}
        with torch.no_grad(), Fn.precision("split"):
            for i0 in range(0, len(val), 4):
                batch = scenes.collate([val[i] for i in range(i0, min(len(val), i0 + 4))])
                dets.update(model(example_to_device(batch, torch.device("cuda"))))
        maps[name] = (m_oracle, val.evaluation(dets)["mAP"])
    (o_aug, s_aug), (o_plain, s_plain) = maps["synth_det_pp18_aspp_aug"], maps["synth_det_pp18_aspp"]
    msg = ("mAP on 24 held-out scenes after 6 epochs | augmented training: oracle (fp32 CPU) %.3f, product fp32-grade %.3f"
           " | unaugmented training: oracle %.3f, product fp32-grade %.3f" % (o_aug, s_aug, o_plain, s_plain))
    print(msg)                                                       # reported with `pytest -s` (or -rP)
    assert o_aug > 5.0, "the augmented run did not learn the synthetic task: " + msg
    assert abs(s_aug - o_aug) <= 0.1, msg
