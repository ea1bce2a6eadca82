"""Freeze golden vectors from the reference's OWN files (TEST INFRASTRUCTURE; build container only).

    python -m oracle.make_golden        # writes tests/golden/ref_tiny.npz

Runs /root/reference's PillarFeatureNet, ASPPNeck, CenterHead (+ loss + backward) unmodified on CPU
(oracle/reference_loader.py) with seeded weights/inputs and stores the OUTPUTS.  Inputs and weights are
regenerated from seeds by tests (oracle/weights.py, pillarnext_b200/synth.py), so the fixture stays small.
The sparse backbone cannot be run (spconv absent) -> no golden vector for it (parity unpinned).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import reference_loader as RL  # noqa: E402
from oracle.weights import randomize_state_dict  # noqa: E402

TASKS = [["car"], ["truck", "construction_vehicle"]]


def golden_setup():
    """Everything a test needs to regenerate the inputs: config, weights, points, labels, dense inputs."""
    from pillarnext_b200 import modules, synth
    cfg = synth.tiny_config(64, tasks=TASKS)
    template = modules.build_pillarnext_b(cfg).state_dict()
    sd = randomize_state_dict(template, seed=7)
    ex = synth.make_batch([0, 1], 600, cfg, kind="uniform", n_boxes=12, sweeps=10)
    g = torch.Generator().manual_seed(99)
    x_neck = torch.randn(2, 256, 8, 8, generator=g)
    x_head = torch.randn(2, 256, 8, 8, generator=g)
    return cfg, sd, ex, x_neck, x_head


def sub(sd, prefix):
    return {k[len(prefix):]: v.clone() for k, v in sd.items() if k.startswith(prefix)}


def main():
    ref = RL.load_reference()
    cfg, sd, ex, x_neck, x_head = golden_setup()
    out = {}
    # ---- reader (pillar_encoder.py), training mode
    reader = ref.PillarFeatureNet(5, [64, 64], cfg["voxel_size"], cfg["pc_range"])
    reader.load_state_dict(sub(sd, "reader."), strict=True)
    reader.train()
    feat, coords, grid = reader(ex["points"])
    out["reader_feat"] = feat.detach().numpy()
    out["reader_coords"] = coords.numpy()
    out["reader_grid"] = np.asarray(grid)
    out["reader_rm0"] = reader.pfn_layers[0].norm.running_mean.numpy().copy()
    out["reader_rv1"] = reader.pfn_layers[1].norm.running_var.numpy().copy()
    reader.eval()
    feat_e, _, _ = reader(ex["points"])
    out["reader_feat_eval"] = feat_e.detach().numpy()
    # ---- neck (aspp.py), training mode (no grad input -> no checkpoint path)
    neck = ref.ASPPNeck(256)
    neck.load_state_dict(sub(sd, "neck."), strict=True)
    neck.train()
    out["neck_out"] = neck(x_neck).detach().numpy()
    # ---- head (centerhead.py) + loss + backward
    head = ref.CenterHead(256, cfg["tasks"], cfg["weight"], cfg["code_weights"], dict(cfg["common_heads"]),
                          cfg["head_strides"], with_reg_iou=True, voxel_size=cfg["voxel_size"], pc_range=cfg["pc_range"],
                          out_size_factor=cfg["out_size_factor"])
    head.load_state_dict(sub(sd, "head."), strict=True)
    head.train()
    xh = x_head.clone().requires_grad_()
    preds = head(xh)
    for t, pd in enumerate(preds):
        for k, v in pd.items():
            out["head_t%d_%s" % (t, k)] = v.detach().numpy().copy()
    example = {k: [e.clone() for e in ex[k]] for k in ("hm", "anno_box", "ind", "mask", "cat", "gt_boxes")}
    loss, rets = head.loss(example, preds)
    loss.backward()
    out["loss_total"] = np.array(loss.item())
    for t, r in enumerate(rets):
        for k in ("hm_loss", "loc_loss", "iou_reg_loss"):
            out["loss_t%d_%s" % (t, k)] = np.array(float(r[k]))
        out["loss_t%d_loc_elem" % t] = r["loc_loss_elem"].numpy()
    out["grad_head_x"] = xh.grad.numpy()
    out["grad_shared_conv_w"] = head.shared_conv[0].weight.grad.numpy()[:16].copy()   # first 16 output channels (file size)
    out["grad_t1_hm_3_w"] = head.tasks[1].hm[3].weight.grad.numpy()
    # ---- state-dict contract (names + shapes) of the reference modules
    names, shapes = [], []
    for pfx, m in (("reader.", reader), ("neck.", neck), ("head.", head)):
        for k, v in m.state_dict().items():
            names.append(pfx + k)
            shapes.append(",".join(str(s) for s in v.shape))
    out["sd_names"] = np.array(names)
    out["sd_shapes"] = np.array(shapes)
    path = os.path.join(ROOT, "tests", "golden", "ref_tiny.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes;", len(out), "arrays")


if __name__ == "__main__":
    main()
