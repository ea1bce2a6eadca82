"""Host-side pieces of the production split-mode replay (tests/test_production_split_gpu.py), without a GPU: its argument
maps against the C ABI, the integer amplitude rule against every split GEMM the bench models can issue, and the
bit-level split reference on edge values."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import test_production_gemms_gpu as G  # noqa: E402
import test_production_split_gpu as S  # noqa: E402
import test_rowwise_recorder_cpu as RC  # noqa: E402
from pillarnext_b200 import _lib, modules, ops, synth  # noqa: E402
from pillarnext_b200 import functional as Fn  # noqa: E402


@pytest.mark.parametrize("name", sorted(S.SPLIT_MAPS))
def test_split_argument_map_matches_the_abi(name):
    spec = [tuple(a.split(":")) for a in S.SPLIT_MAPS[name].split()]
    assert name in _lib._SIGS, name
    assert [RC.KINDS[k] for _, k in spec] == _lib._SIGS[name], name
    names = [a for a, _ in spec]
    assert len(set(names)) == len(names) and names[-1] == "stream", names
    assert names == RC._declared_names(name)


def test_covered_entry_points_exist():
    for name in set(S.REPLAYED_HERE) | set(S.LAUNCH_NOTHING) | set(S.SHARED_ROW):
        assert name in _lib._SIGS, name
    assert not (set(S.REPLAYED_HERE) & set(S.LAUNCH_NOTHING))


def test_recorder_keeps_the_piece_count_with_each_configuration():
    class FakeLib:
        pieces = 3

        def pnx_rows_merge(self, *a):
            return 0

        def pnx_split_get_pieces(self):
            return self.pieces

    real = FakeLib()
    rec = S.R.Recorder(real, maps=S.ROW_MAPS, extra=lambda n: {"pieces": real.pnx_split_get_pieces()} if n in S.PIECE_FNS else {})
    lib = rec.proxy()
    for pieces in (3, 3, 2):
        real.pieces = pieces
        lib.pnx_rows_merge(1000, 192, 64, 77, 64, 2000, 64, 1, 5)
    assert [(c["pieces"], c["calls"], c["lo_x"], c["accumulate"]) for c in rec.configs] == [(3, 2, 64, 1), (2, 1, 64, 1)]


def _split_gemms(name):
    """(taps, K per tap) of every igemm the split mode issues for the bench model `name`, forward and data gradient,
    from the model's parameters: sparse / dense convolutions, the ASPP branches and post-convolution, the head's
    ConvTranspose2d, the fused sibling-head convolutions and the final 1x1 GEMM of the stencil form (HeadFinalConvFn,
    both directions, NZ up to 192)."""
    cfg = synth.BENCH_CONFIGS[name]["cfg"]
    model = modules.build_pillarnext_b(cfg)
    out = []
    for mod in model.modules():
        if isinstance(mod, modules.SepHead):
            names = list(mod.heads)
            hc = mod.head_conv * len(names)
            cin = getattr(mod, names[0])[0].weight.shape[1]
            out += [(9, cin), (9, hc)]                              # sibling 3x3: forward, data gradient
            tot = sum(mod.heads[n][0] for n in names)
            nz = Fn.HeadFinalConvFn.geometry(tot)[1]
            out += [(1, hc), (1, nz)] if (tot + 15) // 16 * 16 == 16 else [(9, hc), (9, (tot + 15) // 16 * 16)]
    for pname, p in model.named_parameters():
        if p.dim() != 4 or any(k in pname for k in ("tasks.",)):
            continue
        if ".deblock." in pname or p.shape[2:] == (2, 2):          # ConvTranspose2d [Cin, Cout, 2, 2]
            out += [(1, p.shape[0]), (4, p.shape[1])]
        elif p.shape[1] == p.shape[2] and p.shape[-1] != p.shape[-2]:   # spconv [Cout, kH, kW, Cin]
            out += [(p.shape[1] * p.shape[2], p.shape[3]), (p.shape[1] * p.shape[2], p.shape[0])]
        else:                                                      # nn.Conv2d [Cout, Cin, kh, kw]
            t = p.shape[2] * p.shape[3]
            out += [(t, p.shape[1]), (t, p.shape[0])]
    for pname, p in model.named_parameters():                      # the heads' ConvTranspose2d
        if ".deblock." in pname and p.dim() == 4:
            out += [(1, p.shape[0]), (4, p.shape[1])]
    return out


@pytest.mark.parametrize("name", ["nusc", "waymo180k"])
def test_amplitude_rule_keeps_every_split_gemm_exact(name):
    """nseg K a w + bias + addend < 2^24 for every split GEMM the bench model can issue, with the largest amplitudes
    the rule picks (so the replay never reports a shape as unreproducible)."""
    gemms = _split_gemms(name)
    assert any(t == 9 for t, _ in gemms) and any(t == 4 for t, _ in gemms)
    worst = 0
    for P, segs in ops.SEGMENTS.items():
        for taps, k in gemms:
            c = dict(kind="igemm", taps=taps, cin=k, segs=tuple(segs))
            (a, w, b, d), bound = G._amplitudes(c)
            assert bound == len(segs) * taps * k * a * w + b + d < G.EXACT, (name, P, taps, k)
            assert (a, w) == (3, 2), "the largest amplitudes fit every split GEMM of %s: (%d, %d) at K %d" % (name, a, w, taps * k)
            worst = max(worst, bound)
    print("%s: %d GEMM shapes, largest bound %d < 2^24" % (name, len(gemms), worst))


def test_split_reference_on_edge_values():
    """The bit-level split: pieces are bf16 values (ties to even, carries, subnormals kept), and three of them hold every
    bit of x down to 2^-133 (all |x| >= 2^-110); below, what is lost stays under 2^-134."""
    x = S.edge_values()
    for P in (2, 3):
        pcs = S.split_ref(x, P)
        for p in pcs:
            assert torch.equal(p.bfloat16().float().view(torch.int32), p.view(torch.int32))
        assert torch.equal(pcs[0].view(torch.int32), x.bfloat16().float().view(torch.int32))
    back = S.merge_ref([p.bfloat16() for p in S.split_ref(x, 3)])
    full = (x.abs() >= 2.0 ** -110) | (x == 0)
    assert torch.equal(back.view(torch.int32)[full], x.view(torch.int32)[full])
    assert ((back.double() - x.double()).abs()[~full] <= 2.0 ** -134).all()
    assert (~full).sum() >= 8, "the edge values include subnormals"
    ties = torch.tensor([0x3F808000, 0x3F818000, 0x00008000, 0x00018000], dtype=torch.int32).view(torch.float32)
    assert S.rne_bf16(ties).view(torch.int32).tolist() == [0x3F800000, 0x3F820000, 0x00000000, 0x00020000]
