"""CPU restatement of double-flip test-time augmentation (TEST INFRASTRUCTURE -- see oracle/__init__.py).

Frame b of a batch runs as frames 4b + k: k = 0 as is, k = 1 mirrored in y (the reference's box_np_ops.flip(axis='x')),
k = 2 mirrored in x (flip(axis='y')), k = 3 both.  Each copy's head output is mapped back onto the original frame (map
rows are y, columns x) and the four are merged as ((v0 + v1) + (v2 + v3)) * 0.25 in fp32 -- the summation order of the
product's pnx_det_*_flip4 decode -- before the unchanged score / range filter, rectifier and per-class NMS of
oracle/predict_oracle.py.

Undo of a y mirror: reg_y -> 1 - reg_y, sin -> -sin, vy -> -vy; of an x mirror: reg_x -> 1 - reg_x, cos -> -cos,
vx -> -vx.  They follow from box_np_ops.flip (y -> -y, yaw -> -yaw; x -> -x, yaw -> pi - yaw) and the rot = (sin, cos)
encoding of assign.py:101-105; tests/golden/ref_flip.npz holds the reference's flip outputs they are checked against.
"""
import torch

from oracle import predict_oracle as P


def flip4_points(points):
    """[N, 6] (b, x, y, z, i, t) -> [4N, 6]: copy k of point i at row k*N + i, batch index 4b + k."""
    out = []
    for k in range(4):
        q = points.clone()
        q[:, 0] = points[:, 0] * 4 + k
        if k & 2:
            q[:, 1] = -points[:, 1]
        if k & 1:
            q[:, 2] = -points[:, 2]
        out.append(q)
    return torch.cat(out)


def undo_flip(pd, flip_y, flip_x):
    """One copy's head maps ([B, c, H, W] raw) mapped back onto the original frame: pixel mirror + raw-value undo."""
    dims = ([2] if flip_y else []) + ([3] if flip_x else [])
    out = {k: (torch.flip(v, dims) if dims else v.clone()) for k, v in pd.items()}
    if flip_y:
        out["reg"][:, 1] = 1 - out["reg"][:, 1]
        out["rot"][:, 0] = -out["rot"][:, 0]
        out["vel"][:, 1] = -out["vel"][:, 1]
    if flip_x:
        out["reg"][:, 0] = 1 - out["reg"][:, 0]
        out["rot"][:, 1] = -out["rot"][:, 1]
        out["vel"][:, 0] = -out["vel"][:, 0]
    return out


def merge4(v):
    return ((v[0] + v[1]) + (v[2] + v[3])) * 0.25


def merge_double_flip(pd4):
    """pd4: head name -> [4B, c, H, W] raw output of a flip4 batch.  Returns (merged raw maps, merged sigmoid(hm),
    merged exp(dim)), each [B, c, H, W]: reg / height / rot / vel / iou are merged raw after the undo, hm after the
    sigmoid and dim after exp."""
    copies = [undo_flip({k: v[k4::4] for k, v in pd4.items()}, bool(k4 & 1), bool(k4 & 2)) for k4 in range(4)]
    raw = {k: merge4([c[k] for c in copies]) for k in pd4}
    hm = merge4([torch.sigmoid(c["hm"]) for c in copies])
    dim = merge4([torch.exp(c["dim"]) for c in copies])
    return raw, hm, dim


def decode_double_flip(pd4, out_size_factor, voxel_size, pc_range):
    """P.decode on the merged maps: same outputs (boxes [B, H*W, 9], hm [B, H*W, C], iou [B, H*W]), with the score and
    the box dimensions taken from the merged sigmoid / exp instead of being recomputed from merged logits."""
    raw, hm, dim = merge_double_flip(pd4)
    boxes, _, iou = P.decode(raw, out_size_factor, voxel_size, pc_range)
    B, C, H, W = hm.shape
    boxes[:, :, 3:6] = dim.permute(0, 2, 3, 1).reshape(B, H * W, 3)
    return boxes, hm.permute(0, 2, 3, 1).reshape(B, H * W, C), iou


def predict_double_flip(preds_dicts, num_classes, test_cfg, rectifier, tokens=None):
    """P.predict for the head output of a flip4 batch (4B frames) -> detections of the B original frames."""
    rets = []
    for t, pd in enumerate(preds_dicts):
        boxes, hm, iou = decode_double_flip(pd, test_cfg["out_size_factor"][t], test_cfg["voxel_size"], test_cfg["pc_range"])
        rets.append(P.post_processing(boxes, hm, iou, rectifier[t], test_cfg["score_threshold"],
                                      test_cfg["post_center_limit_range"], test_cfg["nms"]["nms_iou_threshold"][t],
                                      test_cfg["nms"]["nms_pre_max_size"], test_cfg["nms"]["nms_post_max_size"]))
    out = []
    for i in range(len(rets[0])):
        flag, labs = 0, []
        for t, nc in enumerate(num_classes):
            labs.append(rets[t][i]["label_preds"] + flag)
            flag += nc
        out.append(dict(box3d_lidar=torch.cat([r[i]["box3d_lidar"] for r in rets]),
                        scores=torch.cat([r[i]["scores"] for r in rets]), label_preds=torch.cat(labs),
                        token=tokens[i] if tokens else None))
    return out


def mirror_copies(pd):
    """The four copies a perfectly mirror-equivariant head would output for the single-pass maps `pd` ([B, c, H, W] raw):
    copy k = the maps of the mirrored frame, interleaved as frames 4b + k ([4B, c, H, W])."""
    copies = [undo_flip(pd, bool(k & 1), bool(k & 2)) for k in range(4)]      # the undo is its own inverse
    return {k: torch.stack([c[k] for c in copies], 1).reshape(-1, *pd[k].shape[1:]) for k in pd}
