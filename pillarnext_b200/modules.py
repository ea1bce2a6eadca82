"""Host-side mirror of the reference's model classes for the PillarNeXt-B hot path.

Same class names, constructor kwargs, forward signatures and state-dict keys as the reference
(SURVEY.md section 8b) so hydra's `_target_` strings, `load_checkpoint(strict=True)`, DDP and
`tools/train.py` / `tools/test.py` work unchanged -- but every forward/backward runs in libpnx (sm_90a).
The drop-in module paths live in the top-level `det3d/` package, which re-exports these classes.

  PillarFeatureNet  <- det3d/models/readers/pillar_encoder.py:128-182
  SparseResNet      <- det3d/models/backbones/sparse_resnet.py:10-68 (+ utils/sparse_conv.py:16-63)
  ASPPNeck          <- det3d/models/necks/aspp.py:8-40 (+ utils/conv.py)
  CenterHead        <- det3d/models/heads/centerhead.py:62-136 (forward), :142-229 (loss)
  SingleStageDetector <- det3d/models/detectors/single_stage.py:5-59
"""
import copy
from collections import OrderedDict

import numpy as np
import torch
from torch import nn

from . import functional as Fn
from . import loss as L
from . import ops


def _require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError("pillarnext_b200.%s runs on CUDA (sm_90a) only -- there is no CPU path" % what)


# =========================================================================================== reader
class PFNLayer(nn.Module):
    """Parameter container with the reference's names (pillar_encoder.py:15-33): linear.weight, norm.*"""

    def __init__(self, in_channels, out_channels, norm_cfg=None, last_layer=False):
        super().__init__()
        self.last_vfe = last_layer
        if not self.last_vfe:
            out_channels = out_channels // 2
        self.units = out_channels
        self.linear = nn.Linear(in_channels, out_channels, bias=False)
        self.norm = nn.BatchNorm1d(out_channels, eps=1e-3, momentum=0.01)


class PillarNet(nn.Module):
    """Dynamic voxelizer with the reference's interface (pillar_encoder.py:53-125):
    forward(points) -> (features [Nv, 10], coords [P, 3] int32 (b, y, x), unq_inv [Nv] int64, grid_size (Gy, Gx)).
    The indices come from the CUDA voxelizer (bit-exact with torch.unique); the decorated point features are materialised
    here only for callers of THIS module -- PillarFeatureNet never builds them (pnx_pfn_lin0 fuses the decoration into the
    first linear layer).  The voxelizer result rides along as `features._pnx_vox`."""

    def __init__(self, num_input_features, voxel_size, pc_range):
        super().__init__()
        self.voxel_size = np.array(voxel_size)
        self.pc_range = np.array(pc_range)

    def voxelize(self, points, batch_size=None, frame_sorted=False):
        _require_cuda(points, "PillarNet")
        if batch_size is None:
            batch_size = int(points[:, 0].max().item()) + 1 if points.shape[0] else 1
        return ops.voxelize(points, batch_size, self.voxel_size, self.pc_range, frame_sorted=frame_sorted)

    def forward(self, points, batch_size=None):
        points = points.float()
        vox = self.voxelize(points, batch_size)
        P, _ = vox.sync_counts()
        pop = vox.pillar_of_point[:points.shape[0]]
        keep = pop >= 0                                                    # :98-103 range mask
        pts = points[keep]
        unq_inv = pop[keep].long()
        coords = vox.coords[:P]                                            # (b, y, x) = unq[:, [0, 2, 1]]
        vs = torch.tensor(self.voxel_size[:2], dtype=points.dtype, device=points.device)
        pr = torch.tensor(self.pc_range[:2], dtype=points.dtype, device=points.device)
        mean = ops.pillar_mean(vox)[:P]                                    # :113-114
        f_cluster = pts[:, 1:4] - mean[unq_inv]                            # :116
        cxy = coords[unq_inv][:, [2, 1]].to(points.dtype)                  # (xi, yi) of the point's pillar
        f_center = pts[:, 1:3] - (cxy * vs.unsqueeze(0) + vs.unsqueeze(0) / 2 + pr.unsqueeze(0))   # :119-120
        features = torch.cat([pts[:, 1:], f_cluster, f_center], dim=-1)    # :123
        features._pnx_vox = vox
        return features, coords, unq_inv, ops.grid_size_xy(self.voxel_size, self.pc_range)[[1, 0]]


class Pyramid:
    """Active-site levels + neighbour tables of the sparse backbone for one batch (built once per step)."""
    pass


def build_pyramid(vox, strides):
    """Level 0 = pillars; level s+1 = SparseConv2d(k3,p1,stride) dilation of level s.  One host sync for all
    site counts.  Returns Pyramid with levels[0..4], entry specs (regular conv) and subm specs per stage."""
    lv0 = ops.level_from_bitmap(vox.bitmap, vox.blockpref, vox.counts[0:1], vox.batch, vox.gx, vox.gy, inblk=vox.inblk)
    levels = [lv0]
    for s in strides:
        levels.append(ops.level_dilate(levels[-1], int(s)))
    status = getattr(vox, "status", None)
    counts = torch.cat([vox.counts] + [lv.count for lv in levels[1:]] + ([status] if status is not None else [])).cpu().tolist()   # the one sync
    if status is not None:
        vox.check_order(counts.pop())          # frame-tiled voxelizer: the points must have been grouped by frame
    vox.P, vox.Nv = int(counts[0]), int(counts[1])
    ns = [vox.P] + [int(c) for c in counts[2:]]
    for lv, n in zip(levels, ns):
        ops.level_coords(lv, n)
    pyr = Pyramid()
    pyr.levels, pyr.entry, pyr.subm = levels, [], []
    for s, stride in enumerate(strides):
        src, dst = levels[s], levels[s + 1]
        nbr = ops.nbr_table(dst, src, int(stride), False)
        nbr_t = ops.nbr_table(src, dst, int(stride), True)
        pyr.entry.append(Fn.ConvSpec(dst.n, src.n, 9, nbr=nbr, d_nbr=nbr_t, d_flip=False))
        sub = ops.nbr_table(dst, dst, 1, False)
        pyr.subm.append(Fn.ConvSpec(dst.n, dst.n, 9, nbr=sub, d_nbr=sub, d_flip=True))
    last = levels[-1]
    pyr.map1x1 = Fn.ConvSpec(last.n, last.n, 1)
    return pyr


class PillarFeatureNet(nn.Module):
    def __init__(self, num_input_features, num_filters, voxel_size, pc_range, norm_cfg=None):
        super().__init__()
        assert len(num_filters) > 0
        num_input_features += 5
        num_filters = [num_input_features] + list(num_filters)
        if list(num_filters) != [10, 64, 64]:
            raise NotImplementedError("pillarnext_b200 implements the PillarNeXt-B reader: 5+5 inputs, num_filters=[64,64]")
        layers = []
        for i in range(len(num_filters) - 1):
            layers.append(PFNLayer(num_filters[i], num_filters[i + 1], norm_cfg=norm_cfg, last_layer=i == len(num_filters) - 2))
        self.pfn_layers = nn.ModuleList(layers)
        self.feature_output_dim = num_filters[-1]
        self.voxel_size = np.array(voxel_size)
        self.pc_range = np.array(pc_range)
        self.voxelization = PillarNet(num_input_features, voxel_size, pc_range)
        self.pyramid_strides = None      # set by SingleStageDetector: build the backbone rulebook in the same sync
        self.batch_size = None           # frames per batch when known by the caller (else read from the points)
        # collate_kitti (loader/collate.py:17-21) concatenates the frames in order, so the points arrive grouped by frame and
        # ops.voxelize MAY pick the frame-tiled kernels (ops.FRAME_TILED_MIN_CTAS; the order is then verified on the device
        # and a violation raises at the step's one host synchronisation).  Set False for point tensors in arbitrary order.
        self.frame_sorted = True

    def forward(self, points):
        """points [N, 6] (batch_idx, x, y, z, intensity, time) -> (feat_max [P,64] fp32, coords [P,3] int32 (b,y,x),
        grid_size np.int64[2] (H, W)) exactly like pillar_encoder.py:174-182."""
        _require_cuda(points, "PillarFeatureNet")
        points = points.float()
        B = self.batch_size
        if B is None:
            B = int(points[:, 0].max().item()) + 1 if points.shape[0] else 1
        vox = ops.voxelize(points, B, self.voxel_size, self.pc_range, frame_sorted=self.frame_sorted)
        if self.pyramid_strides is not None:
            vox.pyramid = build_pyramid(vox, self.pyramid_strides)
        l0, l1 = self.pfn_layers[0], self.pfn_layers[1]
        feat = Fn.PFNFn.apply(l0.linear.weight, l0.norm.weight, l0.norm.bias, l1.linear.weight, l1.norm.weight,
                              l1.norm.bias, vox, l0.norm, l1.norm, self.training)
        coords = vox.coords[:vox.P]
        feat._pnx_vox = vox              # lets SparseResNet reuse the bitmap / rulebook (plain tensors also work)
        grid = ops.grid_size_xy(self.voxel_size, self.pc_range)
        return feat, coords, grid[[1, 0]]


# =========================================================================================== backbone
class _SpConv(nn.Module):
    """Holds `weight` in spconv's layout [Cout, kH, kW, Cin] (bias=False everywhere in the reference)."""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(cout, k, k, cin))
        nn.init.kaiming_uniform_(self.weight.view(cout, -1), a=5 ** 0.5)   # spconv default init (uniform, fan_in = k*k*cin)
        self.in_channels, self.out_channels, self.kernel_size = cin, cout, k


class SparseConvBlock(nn.Module):
    """sparse_conv.py:16-39: conv + BatchNorm1d(eps 1e-3, mom 0.01) + ReLU"""

    def __init__(self, in_channels, out_channels, kernel_size, stride, use_subm=True, bias=False):
        super().__init__()
        assert not bias
        self.conv = _SpConv(in_channels, out_channels, kernel_size)
        self.norm = nn.BatchNorm1d(out_channels, eps=1e-3, momentum=0.01)
        self.act = nn.ReLU()
        self.stride, self.subm = stride, (stride == 1 and use_subm)

    def run(self, x, spec, info=None):
        raw, stats = Fn.conv(x, self.conv.weight, None, spec, Fn.WLayout("sp"), want_stats=True)
        return Fn.bn_act(raw, stats, self.norm, relu=True, info=info)


class SparseBasicBlock(nn.Module):
    """sparse_conv.py:42-63"""

    def __init__(self, channels, kernel_size):
        super().__init__()
        self.block1 = SparseConvBlock(channels, channels, kernel_size, 1)
        self.conv2 = _SpConv(channels, channels, kernel_size)
        self.norm2 = nn.BatchNorm1d(channels, eps=1e-3, momentum=0.01)
        self.act2 = nn.ReLU()

    def run(self, x, spec):
        x, idt = Fn.fanout(x)
        info = Fn.bn_info()                     # block1's output feeds conv2 only: conv2's dgrad does block1's BN reduce
        out = self.block1.run(x, spec, info)
        raw, stats = Fn.conv(out, self.conv2.weight, None, spec, Fn.WLayout("sp"), want_stats=True, bn_src=info)
        return Fn.bn_act(raw, stats, self.norm2, relu=True, residual=idt)    # relu(bn(conv) + identity)


class _Stage(nn.Sequential):
    pass


class SparseResNet(nn.Module):
    def __init__(self, layer_nums, ds_layer_strides, ds_num_filters, num_input_features, kernel_size=[3, 3, 3, 3],
                 out_channels=256):
        super().__init__()
        self._layer_strides = [int(s) for s in ds_layer_strides]
        self._num_filters = [int(c) for c in ds_num_filters]
        self._layer_nums = [int(n) for n in layer_nums]
        self._num_input_features = int(num_input_features)
        assert len(self._layer_strides) == len(self._layer_nums) == len(self._num_filters)
        assert all(int(k) == 3 for k in kernel_size), "PillarNeXt-B uses 3x3 kernels"
        in_filters = [self._num_input_features, *self._num_filters[:-1]]
        blocks = []
        for i, n in enumerate(self._layer_nums):
            layers = [SparseConvBlock(in_filters[i], self._num_filters[i], 3, self._layer_strides[i], use_subm=False)]
            layers += [SparseBasicBlock(self._num_filters[i], 3) for _ in range(n)]
            blocks.append(_Stage(*layers))
        self.blocks = nn.ModuleList(blocks)
        self.mapping = nn.Sequential(_SpConv(self._num_filters[-1], out_channels, 1),
                                     nn.BatchNorm1d(out_channels, eps=1e-3, momentum=0.01), nn.ReLU())
        self.out_channels = out_channels

    def _pyramid_from_plain(self, feat, coors, input_shape):
        """The reference's own calling convention, `backbone(features [P, C], coors [P, 3] int (b, y, x), (H, W))`
        (sparse_resnet.py:61-64), for callers that do not come through this package's reader: the active-site bitmap,
        its rank structure and the rulebook are built from the coordinates (any row order, rows must be unique sites).
        Returns (voxel-like object, features in sorted-site order as bf16 rows (differentiable), row permutation).
        Batch size = max(b) + 1 (SURVEY Appendix A: the reference uses len(unique(b)), which breaks on an empty frame)."""
        assert coors.dim() == 2 and coors.shape[1] == 3 and feat.shape[0] == coors.shape[0]
        H, W = int(input_shape[0]), int(input_shape[1])
        dev = feat.device
        c = coors.to(dev).long()
        batch = int(c[:, 0].max().item()) + 1 if c.shape[0] else 1
        L = ops.lib()
        vwords = (H + 31) // 32
        key = (c[:, 0] * W + c[:, 2]) * (vwords * 32) + c[:, 1]          # bit index: (b, x, y) order = the reader's sort order
        order = torch.argsort(key)
        key = key[order]
        if key.numel() > 1 and bool((key[1:] == key[:-1]).any()):
            raise ValueError("SparseResNet: duplicate (b, y, x) coordinates")
        words = L.pnx_voxelize_bitmap_words(batch, W, H)
        bm = torch.zeros(words, dtype=torch.int32, device=dev)
        bits = torch.ones_like(key, dtype=torch.int32) << (key & 31).to(torch.int32)
        bm.index_add_(0, key >> 5, bits)                                   # distinct bits: the sum is the OR
        lv = ops.level_from_mask_words(bm, batch, W, H)
        vox = ops.Voxels()
        vox.bitmap, vox.blockpref, vox.inblk = lv.bm, lv.blockpref, lv.inblk
        vox.batch, vox.gx, vox.gy = batch, W, H
        vox.counts = torch.cat([lv.count, lv.count]).contiguous()
        rows = feat.index_select(0, order)
        return vox, rows, order

    def forward(self, pillar_features, coors, input_shape):
        """-> dense [B, 256, H/8, W/8] (bf16, channels-last memory) like sparse_resnet.py:61-68.
        NOTE (Appendix A): B is the collated batch size, not len(unique(coors[:,0]))."""
        _require_cuda(pillar_features, "SparseResNet")
        vox = getattr(pillar_features, "_pnx_vox", None)
        split = Fn.get_precision() == "split"
        if vox is None:
            vox, rows, _ = self._pyramid_from_plain(pillar_features, coors, input_shape)
            pyr = vox.pyramid = build_pyramid(vox, self._layer_strides)
            x = Fn.SplitFn.apply(rows.float()) if split else rows.to(torch.bfloat16)
        else:
            pyr = getattr(vox, "pyramid", None)
            if pyr is None:
                pyr = vox.pyramid = build_pyramid(vox, self._layer_strides)
            x = Fn.SplitFn.apply(pillar_features) if split else Fn.ToBF16RowsFn.apply(pillar_features, vox.feat_bf16)
        for s, stage in enumerate(self.blocks):
            x = stage[0].run(x, pyr.entry[s])
            for blk in list(stage)[1:]:
                x = blk.run(x, pyr.subm[s])
        raw, stats = Fn.conv(x, self.mapping[0].weight, None, pyr.map1x1, Fn.WLayout("sp"), want_stats=True)
        x = Fn.bn_act(raw, stats, self.mapping[1], relu=True)
        last = pyr.levels[-1]
        rows = Fn.DensifyFn.apply(x, last)
        if split:
            rows = Fn.MergeFn.apply(rows)         # fp32-grade mode: modules exchange fp32 NCHW tensors like the reference
        return rows.view(last.batch, last.V, last.U, self.out_channels).permute(0, 3, 1, 2)


# =========================================================================================== neck
class _Conv(nn.Module):
    """conv.py:3-14 `Conv`: holds .conv (nn.Conv2d / nn.ConvTranspose2d parameters only)."""

    def __init__(self, inplanes, planes, kernel_size, stride, conv_layer=nn.Conv2d, bias=False, **kwargs):
        super().__init__()
        padding = kwargs.get("padding", kernel_size // 2)
        self.conv = conv_layer(inplanes, planes, kernel_size=kernel_size, stride=stride, padding=padding, bias=bias)


class ConvBlock(nn.Module):
    """conv.py:17-34: conv(bias=False) + BatchNorm2d + ReLU on channels-last rows."""

    def __init__(self, inplanes, planes, kernel_size, stride=1, conv_layer=nn.Conv2d, norm_layer=nn.BatchNorm2d,
                 act_layer=nn.ReLU, **kwargs):
        super().__init__()
        padding = kwargs.get("padding", kernel_size // 2)
        self.conv = _Conv(inplanes, planes, kernel_size=kernel_size, stride=stride, padding=padding, bias=False,
                          conv_layer=conv_layer)
        self.norm = norm_layer(planes)
        self.act = act_layer()
        self.is_transpose = conv_layer is nn.ConvTranspose2d
        self.kernel_size = kernel_size

    def run(self, x, B, H, W, bn_src=None, info=None):
        """bn_src: BNInfo of x (this conv is the only kind of consumer of x); info: BNInfo to fill for this block's output."""
        if self.is_transpose:
            raw, stats = Fn.conv(x, self.conv.conv.weight, None, Fn.convT_spec(B, H, W), Fn.WLayout("convT"), want_stats=True,
                                 bn_src=bn_src)
        else:
            raw, stats = Fn.conv(x, self.conv.conv.weight, None, Fn.dense_spec(B, H, W, self.kernel_size),
                                 Fn.WLayout("dense"), want_stats=True, bn_src=bn_src)
        return Fn.bn_act(raw, stats, self.norm, relu=True, info=info)


class BasicBlock(nn.Module):
    """conv.py:37-51: relu(block2(block1(x)) + x), both blocks with their own ReLU."""

    def __init__(self, inplanes, kernel_size=3):
        super().__init__()
        self.block1 = ConvBlock(inplanes, inplanes, kernel_size=kernel_size)
        self.block2 = ConvBlock(inplanes, inplanes, kernel_size=kernel_size)
        self.act = nn.ReLU()


def _to_rows(x):
    """NCHW tensor (any dtype/strides) -> (rows bf16 [B*H*W, C], B, H, W); free if already channels-last bf16.
    fp32-grade mode: split rows [B*H*W, 2C] (hi | lo)."""
    B, C, H, W = x.shape
    r = x.permute(0, 2, 3, 1)
    if Fn.get_precision() == "split":
        return Fn.SplitFn.apply(r.float().contiguous().view(B * H * W, C)), B, H, W
    if r.dtype != torch.bfloat16:
        r = r.to(torch.bfloat16)
    return r.contiguous().view(B * H * W, C), B, H, W


class ASPPNeck(nn.Module):
    def __init__(self, in_channels):
        super().__init__()
        self.pre_conv = BasicBlock(in_channels)
        self.conv1x1 = nn.Conv2d(in_channels, in_channels, kernel_size=1, stride=1, bias=False, padding=0)
        self.weight = nn.Parameter(torch.randn(in_channels, in_channels, 3, 3))
        self.post_conv = ConvBlock(in_channels * 6, in_channels, kernel_size=1, stride=1)
        self.in_channels = in_channels

    def forward(self, x):
        """aspp.py:19-40 (activation checkpointing dropped: values identical, the 80 GB of an H100 hold the activations)."""
        _require_cuda(x, "ASPPNeck")
        rows, B, H, W = _to_rows(x)
        C = self.in_channels
        rows, idt = Fn.fanout(rows)
        info = Fn.bn_info()
        o = self.pre_conv.block1.run(rows, B, H, W, info=info)
        o = self.pre_conv.block2.run(o, B, H, W, bn_src=info)
        cat = Fn.ASPPBranchesFn.apply(o, idt, self.conv1x1.weight, self.weight, B, H, W)
        y = self.post_conv.run(cat, B, H, W)
        if Fn.get_precision() == "split":
            y = Fn.MergeFn.apply(y)
        return y.view(B, H, W, C).permute(0, 3, 1, 2)


# =========================================================================================== head
class SepHead(nn.Module):
    """centerhead.py:12-59.  Parameters are kept per head with the reference's names
    (`<head>.0` conv, `<head>.1` BN, `<head>.3` final conv); the forward batches all sibling heads of a task:
    one 64->(64*heads) 3x3 GEMM + one BatchNorm over the concatenated channels + one block-diagonal
    (64*heads)->sum(classes) 3x3 GEMM (same arithmetic per output channel)."""

    def __init__(self, in_channels, heads, stride=1, head_conv=64, final_kernel=1, bn=True, init_bias=-2.19, **kwargs):
        super().__init__(**kwargs)
        if stride > 1:
            self.deblock = ConvBlock(in_channels, head_conv, kernel_size=int(stride), stride=int(stride), padding=0,
                                     conv_layer=nn.ConvTranspose2d)
            in_channels = head_conv
        else:
            self.deblock = nn.Identity()
        self.stride = int(stride)
        assert self.stride in (1, 2), "CenterHead strides 1 or 2"
        self.heads = heads
        self.head_conv, self.final_kernel = head_conv, final_kernel
        for head in self.heads:
            classes, num_conv = self.heads[head]
            assert num_conv == 2 and bn and final_kernel == 3, "PillarNeXt-B heads: conv3x3+BN+ReLU+conv3x3"
            fc = nn.Sequential()
            fc.append(nn.Conv2d(in_channels, head_conv, kernel_size=final_kernel, stride=1, padding=final_kernel // 2, bias=True))
            fc.append(nn.BatchNorm2d(head_conv))
            fc.append(nn.ReLU())
            fc.append(nn.Conv2d(head_conv, classes, kernel_size=final_kernel, stride=1, padding=final_kernel // 2, bias=True))
            if "hm" in head:
                fc[-1].bias.data.fill_(init_bias)
            self.__setattr__(head, fc)
        self._bn_cat = None

    def _cat_bn(self, names):
        """One BatchNorm2d-like holder over the concatenated sibling channels.  The per-head running_mean / running_var
        buffers (the reference's state-dict entries `<head>.1.running_*`) are made VIEWS of one concatenated tensor
        each, so the fused BatchNorm updates all of them in place with no per-step copies; `.to()` / `.cuda()` give
        every buffer its own storage again, which is detected (data_ptr) and repaired here."""
        hc = self.head_conv
        members = [getattr(self, n)[1] for n in names]
        dev = members[0].running_mean.device
        cat = getattr(self, "_stat_cat", None)
        ok = cat is not None and cat[0].device == dev and all(
            m.running_mean.data_ptr() == cat[0][i * hc:].data_ptr() and m.running_var.data_ptr() == cat[1][i * hc:].data_ptr()
            for i, m in enumerate(members))
        if not ok:
            with torch.no_grad():
                rm = torch.cat([m.running_mean for m in members]).contiguous()
                rv = torch.cat([m.running_var for m in members]).contiguous()
            for i, m in enumerate(members):
                m.running_mean = rm[i * hc:(i + 1) * hc]
                m.running_var = rv[i * hc:(i + 1) * hc]
            cat = (rm, rv)
            object.__setattr__(self, "_stat_cat", cat)
        bn = self._bn_cat
        if bn is None or bn.weight.device != dev:
            bn = nn.BatchNorm2d(hc * len(names)).to(dev)
            object.__setattr__(self, "_bn_cat", bn)   # not a registered submodule: no extra state-dict keys
        bn.running_mean, bn.running_var = cat
        bn.num_batches_tracked = None                 # the members' own counters are bumped below
        bn.training = self.training
        ref = members[0]
        bn.eps, bn.momentum = ref.eps, ref.momentum
        bn.pnx_sync = Fn.wants_sync(ref)
        return bn

    def run(self, x, B, H, W, bn_src=None):
        names = list(self.heads.keys())
        hc = self.head_conv
        info_x = None
        if self.stride > 1:
            info_x = Fn.bn_info()
            x = self.deblock.run(x, B, H, W, bn_src=bn_src, info=info_x)
            H, W = 2 * H, 2 * W
        wa = torch.cat([getattr(self, n)[0].weight for n in names], 0)
        ba = torch.cat([getattr(self, n)[0].bias for n in names], 0)
        ga = torch.cat([getattr(self, n)[1].weight for n in names], 0)
        be = torch.cat([getattr(self, n)[1].bias for n in names], 0)
        bn = self._cat_bn(names)
        raw, stats = Fn.conv(x, wa, ba, Fn.dense_spec(B, H, W, 3), Fn.WLayout("dense"), want_stats=True,
                             bias_feeds_bn=self.training, bn_src=info_x)
        info_y = Fn.bn_info()
        y = Fn.BNActFn.apply(raw, stats, ga, be, None, bn, True, raw.shape[0], info_y)
        if self.training:
            for n in names:
                Fn.bump_batches_tracked(getattr(self, n)[1])
        classes = [self.heads[n][0] for n in names]
        tot = sum(classes)
        npad = (tot + 15) // 16 * 16
        wb = x.new_zeros((npad, hc * len(names), 3, 3), dtype=torch.float32)
        bb = x.new_zeros((npad,), dtype=torch.float32)
        rows_w, rows_b, o = [], [], 0
        for i, n in enumerate(names):
            w = getattr(self, n)[3].weight                                   # [c, 64, 3, 3]
            rows_w.append(torch.nn.functional.pad(w, (0, 0, 0, 0, i * hc, (len(names) - 1 - i) * hc)))
            rows_b.append(getattr(self, n)[3].bias)
            o += classes[i]
        wb = torch.cat(rows_w + ([wb[tot:]] if npad > tot else []), 0)
        bb = torch.cat(rows_b + ([bb[tot:]] if npad > tot else []), 0)
        if npad == 16:
            out = Fn.HeadFinalConvFn.apply(y, wb, bb, B, H, W, info_y, tot)  # 1x1 GEMM + stencil (gather-free)
        else:
            out, _ = Fn.conv(y, wb, bb, Fn.dense_spec(B, H, W, 3), Fn.WLayout("dense"), out_fp32=True)
        out4 = out.view(B, H, W, npad)
        ret, o, offs = dict(), 0, {}
        for i, n in enumerate(names):
            ret[n] = out4[..., o:o + classes[i]].permute(0, 3, 1, 2)
            offs[n] = o
            o += classes[i]
        # lets CenterHead.loss run the fused kernel on the channels-last matrix the GEMM wrote (no gathers/permutes)
        ret["hm"]._pnx_raw = dict(out=out, npad=npad, off=offs, B=B, H=H, W=W, C=classes[names.index("hm")])
        return ret

    def forward(self, x):
        rows, B, H, W = _to_rows(x)
        return self.run(rows, B, H, W)


class CenterHead(nn.Module):
    def __init__(self, in_channels, tasks, weight, code_weights, common_heads, strides, init_bias=-2.19,
                 share_conv_channel=64, num_hm_conv=2, with_reg_iou=False, voxel_size=None, pc_range=None,
                 out_size_factor=None, rectifier=[[0.], [0.], [0.]]):
        super().__init__()
        tasks = [list(t) for t in tasks]
        num_classes = [len(t) for t in tasks]
        self.class_names = tasks
        self.code_weights = [float(c) for c in code_weights]
        self.weight = float(weight)
        self.in_channels = in_channels
        self.num_classes = num_classes
        self.with_reg_iou = with_reg_iou
        common_heads = OrderedDict((k, (int(v[0]), int(v[1]))) for k, v in dict(common_heads).items())
        self.with_iou = "iou" in common_heads
        if self.with_iou or with_reg_iou:
            self.voxel_size = [float(v) for v in voxel_size]
            self.pc_range = [float(v) for v in pc_range]
            self.out_size_factor = [int(v) for v in out_size_factor]
        self.strides = [int(s) for s in strides]
        self.rectifier = rectifier
        self.shared_conv = nn.Sequential(
            nn.Conv2d(in_channels, share_conv_channel, kernel_size=3, padding=1, bias=True),
            nn.BatchNorm2d(share_conv_channel), nn.ReLU(inplace=True))
        self.tasks = nn.ModuleList()
        for num_cls, stride in zip(num_classes, self.strides):
            heads = copy.deepcopy(common_heads)
            heads.update(dict(hm=(num_cls, num_hm_conv)))
            self.tasks.append(SepHead(share_conv_channel, heads, stride=stride, bn=True, init_bias=init_bias, final_kernel=3))

    def forward(self, x, *kwargs):
        """centerhead.py:128-136 -> list (one per task) of dict head-name -> [B, c, H', W'] fp32."""
        _require_cuda(x, "CenterHead")
        rows, B, H, W = _to_rows(x)
        raw, stats = Fn.conv(rows, self.shared_conv[0].weight, self.shared_conv[0].bias, Fn.dense_spec(B, H, W, 3),
                             Fn.WLayout("dense"), want_stats=True, bias_feeds_bn=self.training)
        # y feeds the deblock ConvTranspose2d of every task and nothing else: each of their data-gradient GEMMs gates its
        # part of dy and accumulates into the same two sums (the reduce is linear), when all tasks have a deblock
        info = Fn.bn_info() if all(t.stride > 1 for t in self.tasks) else None
        y = Fn.bn_act(raw, stats, self.shared_conv[1], relu=True, info=info)
        return [task.run(yt, B, H, W, bn_src=info) for task, yt in zip(self.tasks, Fn.fanout(y, len(self.tasks)))]

    def loss(self, example, preds_dicts, **kwargs):
        """centerhead.py:142-229, including the Waymo `iou` head branch (:210-215) on the fused-head path."""
        raws = [getattr(pd.get("hm"), "_pnx_raw", None) for pd in preds_dicts]
        if all(r is not None for r in raws) and all(set(r["off"]) >= {"reg", "height", "dim", "rot", "vel", "hm"} for r in raws):
            total, rets = self._fused_loss(example, preds_dicts, raws)
            if self.with_iou:
                for t, r in enumerate(raws):
                    il = L.iou_head_loss(r["out"], r["off"], r["B"], r["H"], r["W"], example["ind"][t], example["mask"][t],
                                         example["gt_boxes"][t], self.out_size_factor[t], self.voxel_size, self.pc_range)
                    total = total + il
                    rets[t]["iou_loss"] = il.detach()
                    rets[t]["loss"] = rets[t]["loss"] + il.detach()
            return total, rets
        if self.with_iou:
            raise NotImplementedError("the `iou` head loss needs the fused head output (reg/height/dim/rot/vel/iou/hm)")
        return L.center_loss(example, preds_dicts, self.class_names, self.weight, self.code_weights, self.with_reg_iou,
                             getattr(self, "voxel_size", None), getattr(self, "pc_range", None),
                             getattr(self, "out_size_factor", None))

    def _fused_loss(self, example, preds_dicts, raws):
        """Same value/gradient as loss.center_loss, from the fused libpnx kernels (3 launches per task instead of ~150)."""
        dev = raws[0]["out"].device
        if getattr(self, "_loss_consts", None) is None or self._loss_consts[0].device != dev:
            self._loss_consts = (torch.full((len(raws),), self.weight, dtype=torch.float32, device=dev),
                                 torch.tensor(self.code_weights, dtype=torch.float32, device=dev),
                                 torch.full((len(raws),), 1 if self.with_reg_iou else 0, dtype=torch.int32, device=dev))
        tasks = []
        for t, r in enumerate(raws):
            labels = {k: example[k][t].contiguous() for k in ("hm", "anno_box", "ind", "mask", "cat", "gt_boxes")}
            assert labels["hm"].dtype == torch.float32 and labels["ind"].dtype == torch.int64 and labels["mask"].dtype == torch.uint8
            assert labels["cat"].dtype == torch.int64 and labels["anno_box"].dtype == torch.float32 and labels["gt_boxes"].dtype == torch.float32
            Mobj = labels["ind"].shape[1]
            assert tuple(labels["anno_box"].shape) == (r["B"], Mobj, 10) and tuple(labels["gt_boxes"].shape) == (r["B"], Mobj, 7), \
                "label tensors must be anno_box [B, M, 10] / gt_boxes [B, M, 7] (det3d/datasets/pipelines/assign.py:42-48)"
            assert tuple(labels["hm"].shape) == (r["B"], r["C"], r["H"], r["W"]), "heat-map label shape does not match the head output"
            osf = self.out_size_factor[t] if self.with_reg_iou else 1
            vs = self.voxel_size if self.with_reg_iou else [1.0, 1.0]
            pr = self.pc_range if self.with_reg_iou else [0.0, 0.0]
            tasks.append(dict(labels=labels, B=r["B"], H=r["H"], W=r["W"], npad=r["npad"], C=r["C"], M=labels["ind"].shape[1],
                              off=r["off"], sx=float(osf * vs[0]), sy=float(osf * vs[1]), ox=float(pr[0]), oy=float(pr[1])))
        meta = dict(tasks=tasks, weight=self.weight, code_weights=self.code_weights, with_reg_iou=self.with_reg_iou,
                    weights_dev=self._loss_consts[0], code_w_dev=self._loss_consts[1], with_iou_dev=self._loss_consts[2])
        total, res = Fn.CenterLossFn.apply(meta, *[r["out"] for r in raws])
        rets = []
        for t in range(len(raws)):
            ret = OrderedDict()
            ret.update({"task": self.class_names[t], "loss": res[t, 0], "hm_loss": res[t, 1], "loc_loss": res[t, 2],
                        "loc_loss_elem": res[t, 5:15], "num_positive": res[t, 4]})
            if self.with_reg_iou:
                ret.update({"iou_reg_loss": res[t, 3]})
            rets.append(ret)
        return total, rets

    @torch.no_grad()
    def predict(self, example, preds_dicts, test_cfg):
        """centerhead.py:231-330: decode, score/range filter, per-class rotated NMS, merge tasks.  test_cfg is the
        reference's `post_processing` config (attribute or mapping access): post_center_limit_range, score_threshold,
        out_size_factor (per task), voxel_size, pc_range, nms.{nms_iou_threshold (per task, per class),
        nms_pre_max_size, nms_post_max_size}.  Returns a list (one per frame) of dicts box3d_lidar [K, 9]
        (x, y, z, dx, dy, dz, vx, vy, yaw), scores [K], label_preds [K] (int64), token.  One host sync (the kept counts)."""
        def get(cfg, name):
            return cfg[name] if isinstance(cfg, dict) or hasattr(cfg, "keys") else getattr(cfg, name)

        raws = [getattr(pd.get("hm"), "_pnx_raw", None) for pd in preds_dicts]
        if any(r is None for r in raws):
            raise NotImplementedError("predict needs the fused head output (PillarNeXt-B heads: reg/height/dim/rot/vel/hm)")
        nms = get(test_cfg, "nms")
        pre_max, post_max = int(get(nms, "nms_pre_max_size")), int(get(nms, "nms_post_max_size"))
        thr_all = get(nms, "nms_iou_threshold")
        pcr = [float(v) for v in get(test_cfg, "post_center_limit_range")]
        if len(pcr) != 6:
            raise NotImplementedError("predict needs a 6-value post_center_limit_range")
        vs, pr = get(test_cfg, "voxel_size"), get(test_cfg, "pc_range")
        osf_all = get(test_cfg, "out_size_factor")
        tokens = example.get("token") if isinstance(example, dict) else None
        results, flag = [], 0
        for t, r in enumerate(raws):
            off = r["off"]
            offs = [off["reg"], off["height"], off["dim"], off["rot"], off["vel"], off["hm"], off.get("iou", -1)]
            rect = [float(v) for v in self.rectifier[t]]
            results.append(ops.det_postprocess(r["out"], r["B"], r["H"], r["W"], r["C"], offs, float(osf_all[t]), vs, pr,
                                               float(get(test_cfg, "score_threshold")), pcr, rect,
                                               [float(v) for v in thr_all[t]], pre_max, post_max, label_offset=flag))
            flag += self.num_classes[t]
        counts = torch.cat([res[3] for res in results]).cpu().tolist()       # the one host synchronisation
        B = raws[0]["B"]
        out, base = [], 0
        bases = []
        for r in raws:
            bases.append(base)
            base += r["B"] * r["C"]
        for b in range(B):
            boxes, scores, labels = [], [], []
            for t, (r, res) in enumerate(zip(raws, results)):
                for c in range(r["C"]):
                    s = b * r["C"] + c
                    k = counts[bases[t] + s]
                    boxes.append(res[0][s, :k]); scores.append(res[1][s, :k]); labels.append(res[2][s, :k])
            out.append(dict(box3d_lidar=torch.cat(boxes), scores=torch.cat(scores), label_preds=torch.cat(labels),
                            token=tokens[b] if tokens is not None and len(tokens) > b else None))
        return out


# =========================================================================================== detector
class SingleStageDetector(nn.Module):
    def __init__(self, reader, backbone=None, neck=None, head=None, post_processing=None, **kwargs):
        super().__init__()
        self.reader = reader
        self.backbone = backbone
        self.neck = neck
        self.head = head
        self.post_processing = post_processing
        if kwargs.get("sync_batchnorm", False):
            enable_sync_batchnorm(self)
        if backbone is not None and hasattr(reader, "pyramid_strides"):
            reader.pyramid_strides = list(backbone._layer_strides)

    def extract_feat(self, data):
        x = self.reader(data)
        if self.backbone is not None:
            x = self.backbone(*x)
        if self.neck is not None:
            x = self.neck(x)
        return x

    def _forward(self, example):
        points = example["points"]
        if hasattr(self.reader, "batch_size"):
            tok = example.get("token") if isinstance(example, dict) else None
            self.reader.batch_size = len(tok) if tok is not None and len(tok) > 0 else None
        x = self.extract_feat(points)
        return self.head(x)

    def forward(self, example):
        return self.training_step(example) if self.training else self.validation_step(example)

    label_cfg = dict(gaussian_overlap=0.1, max_objs=500, min_radius=2)     # configs/dataset/base/base_det_train.yaml:11-13

    def assign_labels(self, example):
        """Row F3: CenterPoint targets on the GPU.  An example that carries the raw ground truth (`gt_boxes_raw`
        [B, N, 9] fp32, `gt_classes` [B, N] int32 index into the flattened class list) instead of the dense label
        tensors gets hm / anno_box / ind / mask / cat / gt_boxes from pnx_assign_labels -- what the reference's
        data-loader workers compute in numpy (AssignLabel + collate) and ship over PCIe."""
        h = self.head
        vs = h.voxel_size if hasattr(h, "voxel_size") else self.reader.voxel_size
        pr = h.pc_range if hasattr(h, "pc_range") else self.reader.pc_range
        osf = h.out_size_factor if hasattr(h, "out_size_factor") else [4] * len(h.class_names)
        lab = ops.assign_labels(example["gt_boxes_raw"], example["gt_classes"], h.class_names, vs, pr, osf, **self.label_cfg)
        out = dict(example)
        out.update(lab)
        return out

    def training_step(self, example):
        if "hm" not in example and "gt_boxes_raw" in example:
            example = self.assign_labels(example)
        if torch.is_grad_enabled():
            ops.ARENA.begin_step(example["points"].device)        # one memset for the step's small accumulators
        Fn.NBT_PENDING = []
        try:
            preds = self._forward(example)
            out = self.head.loss(example, preds)
        finally:
            pending, Fn.NBT_PENDING = Fn.NBT_PENDING, None
        if pending:
            torch._foreach_add_(pending, 1)                        # every BatchNorm's num_batches_tracked, one launch
        return out

    @torch.no_grad()
    def validation_step(self, example):
        preds = self._forward(example)
        outputs = self.head.predict(example, preds, self.post_processing)
        detections = {}
        for output in outputs:
            token = output["token"]
            for k, v in output.items():
                if k != "token":
                    output[k] = v.to(torch.device("cpu"))
            detections.update({token: output})
        return detections


def enable_sync_batchnorm(module, enabled=True):
    """SyncBatchNorm semantics (reference tools/train.py:55-56) for this package's fused BN ops:
    statistics are all-reduced over the default process group.  Off by default (BASELINE north_star:
    gradient all-reduce only)."""
    for m in module.modules():
        if isinstance(m, nn.modules.batchnorm._BatchNorm):
            m.pnx_sync = enabled
    return module


def build_pillarnext_b(cfg, sync_batchnorm=False):
    """PillarNeXt-B (`pillarnet18_aspp`) from a synth-style config dict (what hydra would instantiate from
    configs/experiments/nusc_det_pp18_aspp_iou_sp.yaml)."""
    reader = PillarFeatureNet(5, [64, 64], cfg["voxel_size"], cfg["pc_range"])
    backbone = SparseResNet([2, 2, 2, 2], cfg["strides"], [64, 128, 256, 256], 64)
    neck = ASPPNeck(256)
    head = CenterHead(256, cfg["tasks"], cfg["weight"], cfg["code_weights"], cfg["common_heads"], cfg["head_strides"],
                      with_reg_iou=cfg["with_reg_iou"], voxel_size=cfg["voxel_size"], pc_range=cfg["pc_range"],
                      out_size_factor=cfg["out_size_factor"],
                      rectifier=cfg.get("rectifier", [[0.0] * len(t) for t in cfg["tasks"]]))
    return SingleStageDetector(reader, backbone, neck, head, post_processing=cfg.get("post_processing"),
                               sync_batchnorm=sync_batchnorm)
