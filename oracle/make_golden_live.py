"""Freeze the reference's OWN outputs (CPU) on the seeded inputs of the reference-comparison tests (TEST INFRASTRUCTURE;
needs the reference tree): tests/golden/ref_live.npz (IoU, iou-head loss, AssignLabel / collate / PillarFeatureNet) and
tests/golden/ref_configs.json.gz (composed experiment model nodes + reference state-dict shapes).
    python -m oracle.make_golden_live
"""
import gzip
import json
import math
import os

import numpy as np
import torch

from oracle import build_ref_iou, predict_oracle as P, reference_loader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
EXPERIMENTS = ("nusc_det_pp18_aspp_iou_sp", "waymo_det_pp18_aspp_iou_car_sp")
ASSIGN_KEYS = ("hm", "anno_box", "ind", "mask", "cat", "gt_boxes")


def rand_boxes(n, seed, spread=6.0):
    g = torch.Generator().manual_seed(seed)
    xy = (torch.rand(n, 2, generator=g) - 0.5) * spread
    z = torch.rand(n, 1, generator=g)
    dims = torch.rand(n, 3, generator=g) * 3 + 0.5
    yaw = (torch.rand(n, 1, generator=g) - 0.5) * 2 * math.pi
    return torch.cat([xy, z, dims, yaw], 1).float()


def iou_head_loss_case():
    from pillarnext_b200 import synth
    tasks = [["vehicle"], ["pedestrian", "cyclist"]]
    cfg = synth.tiny_config(64, tasks)
    heads = dict(reg=[2, 2], height=[1, 2], dim=[3, 2], rot=[2, 2], vel=[2, 2], iou=[1, 2])
    ex = synth.make_batch([3, 4], 1500, cfg, n_boxes=12, sweeps=1)
    H = W = 64 // 8 * 2
    g = torch.Generator().manual_seed(5)
    preds = []
    for t, names in enumerate(tasks):
        pd = {k: torch.randn(2, c, H, W, generator=g) * 0.5 for k, (c, _) in heads.items()}
        pd["hm"] = torch.randn(2, len(names), H, W, generator=g) - 2.0
        preds.append(pd)
    return tasks, cfg, heads, ex, preds


def main():
    from oracle.make_golden import golden_setup
    from pillarnext_b200 import synth
    ref = reference_loader.load_reference()
    arrays = {}

    ext = build_ref_iou.load(build=True)
    a, b = rand_boxes(24, 1), rand_boxes(24, 2)
    want = torch.zeros(24, 24)
    ext.boxes_iou_bev_cpu(a.contiguous(), b.contiguous(), want)
    arrays["iou_bev"] = want.numpy()

    tasks, cfg, heads, ex, preds = iou_head_loss_case()
    head = ref.CenterHead(in_channels=256, tasks=tasks, weight=1.0, code_weights=cfg["code_weights"], common_heads=heads,
                          strides=[2, 2], with_reg_iou=True, voxel_size=cfg["voxel_size"], pc_range=cfg["pc_range"],
                          out_size_factor=[4, 4], rectifier=[[0.68], [0.71, 0.65]])
    fake = lambda x, y: torch.tensor([[float(P.aligned_iou3d(p.numpy(), q.numpy()))] for p, q in zip(x, y)],
                                     dtype=x.dtype).reshape(-1, 1)
    saved = ref.centerloss.boxes_aligned_iou3d_gpu
    ref.centerloss.boxes_aligned_iou3d_gpu = fake       # CUDA-only in the reference: the oracle's aligned IoU stands in
    try:
        loss, logs = head.loss(ex, [{k: v.clone() for k, v in pd.items()} for pd in preds])
    finally:
        ref.centerloss.boxes_aligned_iou3d_gpu = saved
    arrays["iou_head_loss"] = np.array([float(loss)], dtype=np.float64)
    arrays["iou_head_iou_loss"] = np.array([float(logs[t]["iou_loss"]) for t in range(len(tasks))], dtype=np.float64)

    gcfg = golden_setup()[0]
    boxes, names = synth.make_gt(3, 25, gcfg)
    al = ref.AssignLabel(gcfg["tasks"], 0.1, 500, 2, gcfg["pc_range"], gcfg["voxel_size"], gcfg["out_size_factor"])
    res = al({"annotations": {"gt_boxes": boxes, "gt_names": np.array(names)}})
    for k in ASSIGN_KEYS:
        for t in range(len(gcfg["tasks"])):
            arrays["assign_%s_%d" % (k, t)] = np.asarray(res[k][t])
    frames = [synth.make_frame(s, 300, gcfg) for s in range(2)]
    arrays["collate_points"] = ref.collate([{"points": f} for f in frames])["points"].numpy()
    sd = golden_setup()[1]
    r = ref.PillarFeatureNet(5, [64, 64], synth.NUSC["voxel_size"], synth.NUSC["pc_range"])
    r.load_state_dict({k[len("reader."):]: v.clone() for k, v in sd.items() if k.startswith("reader.")})
    r.train()
    f, c, _ = r(synth.collate_points([synth.make_frame(11, 2000, synth.NUSC, "lidar", sweeps=10)]))
    arrays["reader_feat"] = f.detach().numpy()
    arrays["reader_coords"] = c.numpy()
    np.savez_compressed(os.path.join(GOLDEN, "ref_live.npz"), **arrays)

    from pillarnext_b200 import hydra_lite
    cfg_root = os.path.join(reference_loader.REF_ROOT, "configs", "experiments")
    configs = {}
    for exp in EXPERIMENTS:
        out = hydra_lite.compose(cfg_root, exp, only_groups=["models/"])
        m = hydra_lite.resolve(out["model"], out)
        kw = lambda n: {k: v for k, v in m[n].items() if not k.startswith("_")}
        parts = dict(reader=ref.PillarFeatureNet(**kw("reader")), neck=ref.ASPPNeck(**kw("neck")), head=ref.CenterHead(**kw("head")))
        shapes = {part + "." + k: list(v.shape) for part, mod in parts.items() for k, v in mod.state_dict().items()}
        configs[exp] = {"model": m, "state_dict_shapes": shapes}
    with gzip.GzipFile(os.path.join(GOLDEN, "ref_configs.json.gz"), "wb", mtime=0) as fh:
        fh.write(json.dumps(configs, sort_keys=True, separators=(",", ":")).encode())
    print("wrote", {k: v.shape for k, v in arrays.items()})


if __name__ == "__main__":
    main()
