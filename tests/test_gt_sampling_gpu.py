"""Ground-truth database sampling on the GPU (ops.gt_sample, pnx_gt_sample).

* bit-exact against the reference's own outputs (tests/golden/ref_gts.npz) and, at 6 frames x 30k points with about
  40 candidates per frame in the nuScenes groups' ten class calls, against the host twin; the inputs are left untouched
  and the unused tail rows carry frame index B;
* a training step fed a GPU-sampled and augmented example gives a bit-identical loss and bit-identical gradients to the
  same step fed the oracle's pre-sampled, compacted points, with the default voxelizer and the frame-tiled one;
* a 6-epoch tools/train.py run of the `_gts` experiment passes the mAP gate of tests/test_map_gpu.py: the fp32-grade
  product against the fp32 oracle on the same weights, within 0.1 mAP; the unsampled `_aug` run is reported beside it.
"""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import gts_oracle
from pillarnext_b200 import functional as Fn
from pillarnext_b200 import hydra_lite, ops, scenes
from pillarnext_b200.trainer import example_to_device

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXPERIMENTS = os.path.join(ROOT, "configs", "experiments")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from test_gt_sampling_cpu import _gts_db, bits, golden, golden_batch, golden_expected, host_gts  # noqa: E402

ORDER = ("points", "boxes", "classes", "trig", "cboxes", "cclasses", "ctrig", "cpoints", "coffsets")


def run_gpu(batch):
    dt = {"classes": torch.int32, "cclasses": torch.int32, "coffsets": torch.int32}
    dev = [torch.from_numpy(np.ascontiguousarray(batch[k])).to(dt.get(k, torch.float32)).cuda() for k in ORDER]
    before = [t.clone() for t in dev]
    out = ops.gt_sample(*dev)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(dev, before))            # inputs untouched
    return [t.cpu().numpy() for t in out]


def test_gt_sample_matches_the_reference_goldens():
    g = golden()
    p, b, c, acc, count = run_gpu(golden_batch(g))
    want_p, want_b, want_c = golden_expected(g)
    assert int(count[0]) == len(want_p)
    assert np.array_equal(bits(p[:len(want_p)]), bits(want_p))
    assert np.array_equal(bits(b), bits(want_b)) and np.array_equal(c, want_c)
    B = g["boxes"].shape[0]
    assert np.all(p[len(want_p):, 0] == B) and np.all(p[len(want_p):, 1:] == 0)


NUSC_GROUPS = [2, 3, 7, 4, 6, 2, 6, 6, 2, 2]       # the reference nuScenes sampler's group maxima, 40 in all


def big_batch(rng, B=6, n=30000, M=40):
    pts = np.concatenate([np.concatenate([np.full((n, 1), f), rng.uniform(-55, 55, (n, 2)), rng.uniform(-3, 2, (n, 1)),
                                          rng.uniform(0, 255, (n, 1)), rng.uniform(0, 0.5, (n, 1))], 1)
                          for f in range(B)]).astype(np.float32)
    def boxes(k):
        b = np.concatenate([rng.uniform(-50, 50, (k, 2)), rng.uniform(-2, 0, (k, 1)), rng.uniform(0.5, 8, (k, 2)),
                            rng.uniform(1, 3, (k, 1)), rng.normal(0, 1, (k, 2)), rng.uniform(-np.pi, np.pi, (k, 1))], 1)
        return b.astype(np.float32)
    from det3d.datasets.pipelines.sample_ops import libm_trig, numpy_trig
    S = sum(NUSC_GROUPS)
    sb, scls, strig = np.zeros((B, M, 9), np.float32), np.full((B, M), -1, np.int32), np.zeros((B, M, 2), np.float32)
    cb, ccls, ctrig = np.zeros((B, S, 9), np.float32), np.full((B, S), -1, np.int32), np.zeros((B, S, 4), np.float32)
    counts = np.zeros((B, S), np.int64)
    for f in range(B):
        m = M - 3 * f
        sb[f, :m] = boxes(m)
        scls[f, :m] = rng.integers(0, 10, m)
        strig[f, :m] = numpy_trig(sb[f, :m])
        s = S - f                                      # fewer candidates on later frames; padding at the end
        cb[f, :s] = boxes(s)
        ccls[f, :s] = np.repeat(np.arange(10), NUSC_GROUPS)[:s]
        ctrig[f, :s] = np.concatenate([numpy_trig(cb[f, :s]), libm_trig(cb[f, :s, -1])], 1)
        counts[f, :s] = rng.integers(0, 400, s)
    off = np.concatenate([[0], np.cumsum(counts.reshape(-1))]).astype(np.int32)
    cpts = np.concatenate([rng.uniform(-1.5, 1.5, (off[-1], 3)), rng.uniform(0, 255, (off[-1], 1)),
                           rng.uniform(0, 0.5, (off[-1], 1))], 1).astype(np.float32)
    return dict(points=pts, boxes=sb, classes=scls, trig=strig, cboxes=cb, cclasses=ccls, ctrig=ctrig, cpoints=cpts,
                coffsets=off)


def test_gt_sample_matches_the_host_twin_at_6x30k():
    batch = big_batch(np.random.default_rng(5))
    hp, hb, hc, hacc, hcount = host_gts(**batch)
    p, b, c, acc, count = run_gpu(batch)
    assert int(count[0]) == hcount and 0 < hacc.sum() < hacc.size
    assert np.array_equal(bits(p), bits(hp))                  # tail rows included
    assert np.array_equal(bits(b), bits(hb)) and np.array_equal(c, hc) and np.array_equal(acc, hacc)
    assert np.all(p[hcount:, 0] == 6) and len(p) > hcount
    assert np.all(np.diff(p[:hcount, 0]) >= 0)                # frame-sorted input stays frame-sorted


def _model(cfg):
    torch.manual_seed(0)
    return hydra_lite.instantiate(cfg.model).cuda().train()


@pytest.mark.parametrize("voxelizer", ["default", "force"])
def test_training_step_on_gpu_sampled_example_matches_presampled_oracle(tmp_path, voxelizer, monkeypatch):
    cfg, _ = _gts_db(tmp_path)
    cfg = hydra_lite.main(EXPERIMENTS, "synth_det_pp18_aspp_gts", ["data.train_dataset.root_path=%s" % tmp_path,
                                                                    "data.train_dataset.n_frames=4"])
    ds = hydra_lite.instantiate(cfg.data.train_dataset)
    state = np.random.get_state()
    np.random.seed(3)
    ex = scenes.collate([ds[i] for i in range(4)])
    np.random.set_state(state)
    p_o, b_o, c_o, acc = gts_oracle.apply(*(ex[k].numpy() for k in ("points", "gt_boxes_raw", "gt_classes", "gt_trig",
                                                                     "gts_boxes", "gts_classes", "gts_trig",
                                                                     "gts_points", "gts_offsets")))
    assert acc.sum() > 0 and (~acc[ex["gts_classes"].numpy() >= 0]).sum() > 0
    pre = {k: v for k, v in ex.items() if not k.startswith("gts_") and k != "gt_trig"}
    pre["points"], pre["gt_boxes_raw"], pre["gt_classes"] = torch.from_numpy(p_o), torch.from_numpy(b_o), torch.from_numpy(c_o)
    ex_d, pre_d = example_to_device(ex, torch.device("cuda")), example_to_device(pre, torch.device("cuda"))
    statuses = []
    real_vox = ops.voxelize

    def vox(*a, **k):
        v = real_vox(*a, **k)
        if getattr(v, "status", None) is not None:
            statuses.append(v.status)
        return v

    monkeypatch.setattr(ops, "voxelize", vox)
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
    assert "gts_boxes" in ex_d and "aug" in ex_d                      # the step did not consume the caller's example
    if voxelizer == "force":
        assert len(statuses) >= 2 and all(int(s.item()) == 0 for s in statuses)


def test_gts_experiment_passes_the_map_gate(tmp_path):
    import train as train_tool
    from test_map_gpu import oracle_detections
    overrides = ["trainer.max_epochs=6", "data.train_dataset.n_frames=640", "data.val_dataset.n_frames=24",
                 "dataloader.train.num_workers=0", "dataloader.val.num_workers=0", "dataloader.train.batch_size=4"]
    _gts_db(tmp_path, 640)
    maps = {}
    for name in ("synth_det_pp18_aspp_gts", "synth_det_pp18_aspp_aug"):
        ov = overrides + (["data.train_dataset.root_path=%s" % tmp_path] if name.endswith("_gts") else [])
        state = np.random.get_state()
        np.random.seed(0)
        tr = train_tool.main(["--config-name", name, "--work-dir", str(tmp_path / name)] + ov)
        np.random.set_state(state)
        cfg = hydra_lite.main(EXPERIMENTS, name, ov)
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
    (o_gts, s_gts), (o_plain, s_plain) = maps["synth_det_pp18_aspp_gts"], maps["synth_det_pp18_aspp_aug"]
    msg = ("mAP on 24 held-out scenes after 6 epochs | with gt sampling: oracle (fp32 CPU) %.3f, product fp32-grade %.3f"
           " | without (augmentation only): oracle %.3f, product fp32-grade %.3f" % (o_gts, s_gts, o_plain, s_plain))
    print(msg)                                                        # reported with `pytest -s` (or -rP)
    assert o_gts > 5.0, "the sampled run did not learn the synthetic task: " + msg
    assert abs(s_gts - o_gts) <= 0.1, msg
