"""V1-V3 parity: CUDA voxelizer (through the C-ABI) vs the oracle restatement of
pillar_encoder.py:78-125.  Index work must be BIT-EXACT."""
import numpy as np
import pytest
import torch

from oracle import pillarnext_oracle as O
from pillarnext_b200 import ops, synth

pytestmark = pytest.mark.gpu


def run_case(points, batch, cfg, frame_sorted=False):
    v = ops.voxelize(points.cuda(), batch, cfg["voxel_size"], cfg["pc_range"], frame_sorted="force" if frame_sorted else False)
    P, Nv = v.sync_counts()
    if frame_sorted and points.shape[0]:
        assert v.status is not None, "the frame-tiled kernels must be the ones that ran"
    ref = O.voxelize(points, cfg["voxel_size"], cfg["pc_range"])
    assert P == ref["coords"].shape[0]
    assert Nv == int(ref["keep"].sum())
    coords = v.coords[:P].cpu()
    assert torch.equal(coords, ref["coords"]), "pillar coords differ (must be bit exact, same order)"
    pop = v.pillar_of_point[:points.shape[0]].cpu().long()
    if points.shape[0]:
        assert torch.equal(pop, ref["pillar_of_point"]), "unq_inv differs"
    # CSR buckets: ascending point ids inside each pillar, every kept point exactly once
    off = v.bucket_off[:P + 1].cpu().long()
    pts = v.bucket_pts[:Nv].cpu().long()
    assert off[0] == 0 and off[-1] == Nv
    if Nv:
        seg = torch.repeat_interleave(torch.arange(P), off[1:] - off[:-1])
        assert torch.equal(ref["pillar_of_point"][pts], seg)
        same = seg[1:] == seg[:-1]
        assert bool((pts[1:][same] > pts[:-1][same]).all())
        assert torch.equal(torch.sort(pts)[0], torch.nonzero(ref["keep"]).flatten())
    return v, ref


@pytest.mark.parametrize("n,batch,kind", [(30000, 1, "uniform"), (30000, 2, "lidar"), (1000, 3, "uniform"), (257, 1, "uniform")])
def test_voxelize_matches_oracle(n, batch, kind):
    cfg = synth.NUSC
    pts = synth.collate_points([synth.make_frame(s, n, cfg, kind, sweeps=10) for s in range(batch)])
    run_case(pts, batch, cfg)


def test_voxelize_edge_cases():
    cfg = synth.NUSC
    # empty
    run_case(torch.zeros(0, 6), 1, cfg)
    # all out of range / NaN / inf / exactly on the borders
    p = torch.zeros(8, 6)
    p[:, 1] = torch.tensor([-50.4, 50.4, 50.399998, -50.400002, float("nan"), float("inf"), 0.0, 1e9])
    p[:, 2] = torch.tensor([-50.4, 0.0, 50.399998, 0.0, 0.0, 0.0, float("nan"), 0.0])
    p[:, 3] = 100.0  # z is never range-checked (pillar_encoder.py:98-101)
    run_case(p, 1, cfg)
    # one hot pillar with many points + duplicates
    g = torch.Generator().manual_seed(0)
    q = torch.zeros(5000, 6)
    q[:, 1:3] = torch.rand(5000, 2, generator=g) * 0.07 + 1.0
    q[:, 3] = torch.rand(5000, generator=g)
    run_case(q, 1, cfg)


def test_voxelize_waymo_shape_and_tiny():
    cfg = synth.WAYMO_BENCH
    pts = synth.collate_points([synth.make_frame(7, 180000, cfg, "uniform")])
    run_case(pts, 1, cfg)
    cfg = synth.tiny_config(40)  # V not a multiple of 32
    pts = synth.collate_points([synth.make_frame(s, 500, cfg) for s in range(2)])
    run_case(pts, 2, cfg)


def frames_supported(batch, cfg):
    g = ops.grid_size_xy(cfg["voxel_size"], cfg["pc_range"])
    return bool(ops.voxelize_frames_supported(batch, int(g[0]), int(g[1])))


@pytest.mark.parametrize("n,batch,kind", [(30000, 1, "uniform"), (30001, 2, "lidar"), (1001, 3, "uniform"), (257, 1, "uniform"),
                                          (30000, 6, "lidar"), (2999, 40, "lidar")])
def test_frame_tiled_voxelizer_matches_oracle(n, batch, kind):
    """pnx_voxelize_frames (bitmap slices in shared memory) = same bit-exact contract as pnx_voxelize; odd frame lengths
    exercise the unaligned first point (bulk copies must start at even points)."""
    cfg = synth.NUSC
    assert frames_supported(batch, cfg)
    pts = synth.collate_points([synth.make_frame(s, n + 7 * s, cfg, kind, sweeps=10) for s in range(batch)])
    v, ref = run_case(pts, batch, cfg, frame_sorted=True)
    # the occupancy bitmap / block prefixes feed the rulebook: identical to the general path's
    w = ops.voxelize(pts.cuda(), batch, cfg["voxel_size"], cfg["pc_range"], frame_sorted=False)
    assert torch.equal(v.bitmap, w.bitmap) and torch.equal(v.inblk, w.inblk) and torch.equal(v.blockpref, w.blockpref)


def test_frame_tiled_voxelizer_edge_cases():
    cfg = synth.NUSC
    g = torch.Generator().manual_seed(5)
    # an empty frame in the middle, a frame of one point, points outside the range, NaN / inf coordinates
    f0 = torch.tensor(synth.make_frame(0, 5001, cfg, "lidar", sweeps=10))
    f2 = torch.tensor(synth.make_frame(2, 1, cfg, "uniform"))
    f3 = torch.tensor(synth.make_frame(3, 4000, cfg, "uniform"))
    f3[:50, 0] = float("nan")
    f3[50:60, 1] = float("inf")
    f3[60:90, 0] = 1e6
    pts = torch.cat([torch.nn.functional.pad(f, (1, 0), value=float(b)) for b, f in ((0, f0), (2, f2), (3, f3))])
    run_case(pts, 4, cfg, frame_sorted=True)
    # batch indices outside [0, batch) sit in front of / behind the frames in sorted order: dropped like everywhere else
    lead = torch.nn.functional.pad(torch.tensor(synth.make_frame(9, 33, cfg, "uniform")), (1, 0), value=-1.0)
    tail = torch.nn.functional.pad(torch.tensor(synth.make_frame(8, 77, cfg, "uniform")), (1, 0), value=4.0)
    v = ops.voxelize(torch.cat([lead, pts, tail]).cuda(), 4, cfg["voxel_size"], cfg["pc_range"], frame_sorted="force")
    w = ops.voxelize(torch.cat([lead, pts, tail]).cuda(), 4, cfg["voxel_size"], cfg["pc_range"], frame_sorted=False)
    assert v.sync_counts() == w.sync_counts()
    assert torch.equal(v.pillar_of_point, w.pillar_of_point) and torch.equal(v.coords[:v.P], w.coords[:w.P])
    assert torch.equal(v.bucket_pts[:v.Nv], w.bucket_pts[:w.Nv]) and torch.equal(v.bucket_off[:v.P + 1], w.bucket_off[:w.P + 1])
    # one hot pillar (5000 points in one cell): every mark hits the same shared-memory word
    q = torch.zeros(5000, 6)
    q[:, 1:3] = torch.rand(5000, 2, generator=g) * 0.07 + 1.0
    run_case(q, 1, cfg, frame_sorted=True)


def test_frame_tiled_voxelizer_rejects_ungrouped_points():
    """The order is verified on the device: interleaved frames raise at the next synchronisation instead of producing
    wrong indices."""
    cfg = synth.NUSC
    pts = synth.collate_points([synth.make_frame(s, 4000, cfg, "lidar", sweeps=10) for s in range(3)])
    perm = torch.randperm(pts.shape[0], generator=torch.Generator().manual_seed(1))
    v = ops.voxelize(pts[perm].cuda(), 3, cfg["voxel_size"], cfg["pc_range"], frame_sorted="force")
    with pytest.raises(RuntimeError, match="not grouped"):
        v.sync_counts()
    # a single misplaced point is enough
    one = pts.clone()
    one[[10, 9000]] = one[[9000, 10]]
    v = ops.voxelize(one.cuda(), 3, cfg["voxel_size"], cfg["pc_range"], frame_sorted="force")
    with pytest.raises(RuntimeError, match="not grouped"):
        v.sync_counts()
    run_case(pts[perm], 3, cfg, frame_sorted=False)      # the general path takes any order


def test_frame_tiled_voxelizer_waymo_and_fallback_geometry():
    cfg = synth.WAYMO_BENCH
    assert frames_supported(2, cfg)
    pts = synth.collate_points([synth.make_frame(7 + s, 90000 + s, cfg, "uniform") for s in range(2)])
    run_case(pts, 2, cfg, frame_sorted=True)
    cfg = synth.tiny_config(40)  # 40 x 2 words per frame: not whole 32-word blocks -> the general kernels run
    assert not frames_supported(2, cfg)
    pts = synth.collate_points([synth.make_frame(s, 500, cfg) for s in range(2)])
    v = ops.voxelize(pts.cuda(), 2, cfg["voxel_size"], cfg["pc_range"], frame_sorted="force")
    assert v.status is None
    cfg = synth.tiny_config(128)
    assert frames_supported(2, cfg)
    pts = synth.collate_points([synth.make_frame(s, 3000, cfg) for s in range(2)])
    run_case(pts, 2, cfg, frame_sorted=True)


def test_pfn_forward_matches_oracle():
    cfg = synth.NUSC
    torch.manual_seed(0)
    sd = {
        "reader.pfn_layers.0.linear.weight": torch.randn(32, 10) * 0.3,
        "reader.pfn_layers.0.norm.weight": torch.rand(32) + 0.5, "reader.pfn_layers.0.norm.bias": torch.randn(32) * 0.1,
        "reader.pfn_layers.0.norm.running_mean": torch.zeros(32), "reader.pfn_layers.0.norm.running_var": torch.ones(32),
        "reader.pfn_layers.1.linear.weight": torch.randn(64, 64) * 0.1,
        "reader.pfn_layers.1.norm.weight": torch.rand(64) + 0.5, "reader.pfn_layers.1.norm.bias": torch.randn(64) * 0.1,
        "reader.pfn_layers.1.norm.running_mean": torch.zeros(64), "reader.pfn_layers.1.norm.running_var": torch.ones(64),
    }
    pts = synth.collate_points([synth.make_frame(s, 20000, cfg, "lidar", sweeps=10) for s in range(2)])
    for training in (True, False):
        st = {}
        feat_ref, coords_ref, _ = O.reader_forward(pts, sd, cfg["voxel_size"], cfg["pc_range"], train=training, stats=st)
        d = {k: v.clone().cuda() for k, v in sd.items()}
        v = ops.voxelize(pts.cuda(), 2, cfg["voxel_size"], cfg["pc_range"])
        bn = lambda i: tuple(d["reader.pfn_layers.%d.norm.%s" % (i, k)] for k in ("weight", "bias", "running_mean", "running_var"))
        out = ops.pfn_forward(v, d["reader.pfn_layers.0.linear.weight"], bn(0), d["reader.pfn_layers.1.linear.weight"], bn(1), training)
        P, _ = v.sync_counts()
        feat = out["feat"][:P].cpu()
        err = (feat - feat_ref).abs().max().item()
        assert err < 2e-4, "PFN feature max abs err %g (training=%s)" % (err, training)   # fp32, tolerance 2e-4 abs
        fb = out["feat_bf16"][:P].float().cpu()
        assert torch.equal(fb, feat.bfloat16().float())  # bf16 copy == round-to-nearest of the fp32 result
        if training:
            for i in (0, 1):
                for k in ("running_mean", "running_var"):
                    key = "reader.pfn_layers.%d.norm.%s" % (i, k)
                    e = (d[key].cpu() - st[key]).abs().max().item()
                    assert e < 1e-4, (key, e)


def test_pillarnet_module_returns_the_reference_tuple():
    """modules.PillarNet.forward = the reference's (features, coords, unq_inv, grid_size) (pillar_encoder.py:78-125)."""
    from pillarnext_b200 import modules
    cfg = synth.NUSC
    pts = synth.collate_points([synth.make_frame(s, 9000, cfg, "lidar", sweeps=10) for s in range(2)])
    net = modules.PillarNet(5, cfg["voxel_size"], cfg["pc_range"])
    feats, coords, inv, grid = net(pts.cuda())
    ref = O.voxelize(pts, cfg["voxel_size"], cfg["pc_range"])
    assert torch.equal(coords.cpu(), ref["coords"]) and torch.equal(inv.cpu(), ref["unq_inv"])
    assert list(grid) == list(ref["grid"])
    assert feats.shape == ref["features"].shape
    assert torch.equal(feats[:, :5].cpu(), ref["features"][:, :5])                       # the points themselves
    assert torch.equal(feats[:, 8:].cpu(), ref["features"][:, 8:])                       # f_center: same fp32 expression
    assert (feats[:, 5:8].cpu() - ref["features"][:, 5:8]).abs().max().item() < 2e-5     # f_cluster: mean summation order
