"""MSDeformAttnPixelDecoder3D (CUDA, through the C ABI) vs the oracle port and the reference-generated golden fixture
(tests/golden/neck_small.npz, produced by oracle/gen_golden.py from the reference's own module under the shim).
Tolerance = SURVEY.md 8(d), both criteria (tests/util.py)."""
import pytest
import torch
import torch.nn.functional as F

from oracle import port
from util import assert_close, golden

pytestmark = pytest.mark.gpu


def _level_major(t_list):
    """list over levels of (B, n_l, C) -> level-major rows (sum_l B*n_l, C)"""
    return torch.cat([t.reshape(-1, t.shape[-1]) for t in t_list], 0).contiguous()


@pytest.mark.parametrize("B", [1, 2])
def test_ms_deform_attn_core_vs_port(cuda, B):
    """occ_ms_deform_attn vs port.ms_deform_attn_core_3d (= multi_scale_deformable_attn_pytorch): same value tensor, same
    offsets / logits; sampling points land inside, on the border and outside the volumes (zeros padding)."""
    from occformer_b200 import ops
    E, H, L, P = 96, 4, 3, 4
    grids = [(3, 2, 2), (6, 4, 3), (12, 8, 6)]  # coarse -> fine
    strides = [8, 4, 2]
    ns = [x * y * z for x, y, z in grids]
    Nq = sum(ns)
    g = torch.Generator().manual_seed(B)
    value = torch.randn(B, Nq, H, E // H, generator=g)
    off = torch.randn(B, Nq, H, L, P, 3, generator=g) * 1.5
    logits = torch.randn(B, Nq, H, L * P, generator=g)
    refs = [port.grid_priors_3d(gr, st) / (torch.tensor([[gr[2], gr[1], gr[0]]], dtype=torch.float32) * st)
            for gr, st in zip(grids, strides)]
    ref_pts = torch.cat(refs, 0)[None, :, None].repeat(B, 1, L, 1)
    norm = torch.tensor([[Z, Y, X] for (X, Y, Z) in grids], dtype=torch.float32)
    loc = ref_pts[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
    aw = logits.softmax(-1).view(B, Nq, H, L, P)
    want = port.ms_deform_attn_core_3d(value, grids, loc, aw)  # (B, Nq, E)
    # level-major operands
    starts = [sum(ns[:i]) for i in range(L)]
    lm = lambda t: _level_major([t[:, s:s + n] for s, n in zip(starts, ns)])  # noqa: E731
    v_rows = lm(value.reshape(B, Nq, E)).to(cuda)
    ow_rows = lm(torch.cat([off.reshape(B, Nq, -1), logits.reshape(B, Nq, -1)], -1)).to(cuda)
    got = ops.from_split(ops.ms_deform_attn(v_rows, ow_rows, grids, strides, B, E, H, P))
    assert_close(got, lm(want), 2e-5, f"ms_deform_attn core B={B}")
    # head slices padded to one 128-byte line each (the layout the neck's value_proj writes): same result, bit for bit
    hd = E // H
    v_pad = torch.zeros(v_rows.shape[0], H, 32, device=cuda)
    v_pad[:, :, :hd] = v_rows.view(-1, H, hd)
    got_p = ops.from_split(ops.ms_deform_attn(v_pad.view(-1, H * 32), ow_rows, grids, strides, B, E, H, P))
    assert torch.equal(got_p, got)


def test_token_prep_and_upsample_add(cuda):
    from occformer_b200 import ops
    g = torch.Generator().manual_seed(3)
    C, B = 96, 2
    grids = [(2, 2, 1), (4, 3, 2)]
    ns = [4, 24]
    rows = B * sum(ns)
    x = torch.randn(rows, C, generator=g)
    w, b = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    pos = torch.randn(sum(ns), C, generator=g)
    f32, s32, ps = ops.neck_token_prep(x.to(cuda), grids, B, ln=(w.to(cuda), b.to(cuda)), pos=pos.to(cuda), want_pos=True)
    ref = F.layer_norm(x, (C,), w, b, 1e-5)
    assert_close(f32, ref, 1e-5, "token_prep LayerNorm")
    assert torch.equal(ops.to_split(f32).view(torch.int32), s32.view(torch.int32))
    # level-major: rows of level l are (b, local); pos row = start_l + local
    pos_rows = torch.cat([pos[:4].repeat(B, 1), pos[4:].repeat(B, 1)], 0)
    assert_close(ops.from_split(ps), ref + pos_rows, 2e-5, "token_prep x + pos")
    # GroupNorm + trilinear x2 upsample + add
    Bc, X, Y, Z, G = 2, 6, 4, 4, 32
    cur = torch.randn(Bc, X, Y, Z, C, generator=g)
    coarse = torch.randn(Bc, X // 2, Y // 2, Z // 2, C, generator=g)
    gw, gb = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    st = ops.gn_stats(cur.view(-1, C).to(cuda), Bc, X * Y * Z, C, G)
    got = ops.from_split(ops.gn_upsample_add(cur.to(cuda), st, gw.to(cuda), gb.to(cuda), G, coarse.to(cuda)))
    cur_n = F.group_norm(cur.permute(0, 4, 1, 2, 3), G, gw, gb, 1e-5)
    up = F.interpolate(coarse.permute(0, 4, 1, 2, 3), size=(X, Y, Z), mode="trilinear", align_corners=False)
    assert_close(got.permute(0, 4, 1, 2, 3), cur_n + up, 2e-5, "gn + trilinear upsample + add")


def _neck(cuda, c, sd):
    from occformer_b200.neck import MSDeformAttnPixelDecoder3D, neck_cfg
    n = MSDeformAttnPixelDecoder3D(**neck_cfg(c["in_channels"], c["strides"], c["E"], c["layers"], c["heads"], c["levels"],
                                              c["points"], c["ffn"]))
    n.load_state_dict(sd, strict=True)
    return n.to(cuda).eval()


@pytest.mark.parametrize("B", [1, 2])
def test_neck_vs_reference_golden_and_port(cuda, B):
    c = port.NECK_CASE
    sd = port.make_neck_state(c["in_channels"], c["E"], c["layers"], c["heads"], c["levels"], c["points"], c["ffn"],
                              seed=c["wseed"])
    feats = port.neck_inputs(c, B=B)
    neck = _neck(cuda, c, sd)
    outs = neck([f.to(cuda) for f in feats])
    want = port.ms_deform_pixel_decoder_3d(feats, sd, c["strides"], c["heads"], c["layers"], c["levels"], c["points"])
    assert len(outs) == len(want) == 4
    gold = golden("neck_small.npz")
    for i, (o, r) in enumerate(zip(outs, want)):
        assert o.shape == r.shape
        assert_close(o, r, what=f"neck out[{i}] {tuple(r.shape)} vs port (B={B})")
        if B == 1:
            assert_close(o, torch.from_numpy(gold[f"out{i}"]), what=f"neck out[{i}] vs reference golden")
    # the S32 twin handed to the head equals split(mask_feature)
    from occformer_b200 import ops
    from occformer_b200.common import twin_of
    mf = outs[0].permute(0, 2, 3, 4, 1).contiguous()
    assert torch.equal(ops.to_split(mf).view(torch.int32), twin_of(outs[0]).view(torch.int32))


def test_neck_full_width_pr1_grid(cuda):
    """The reference width (E = 192, 8 heads of 24, ffn 768, in_channels 128..1024, strides 2..16) on the PR1 pyramid
    (50x50x8 .. 7x7x1: odd sizes, non-divisible up-sampling ratios), 2 encoder layers."""
    c = dict(in_channels=[128, 256, 512, 1024], strides=[2, 4, 8, 16], E=192, layers=2, heads=8, levels=3, points=4, ffn=768,
             sizes=[(50, 50, 8), (25, 25, 4), (13, 13, 2), (7, 7, 1)], wseed=5, xseed=6)
    sd = port.make_neck_state(c["in_channels"], c["E"], c["layers"], c["heads"], c["levels"], c["points"], c["ffn"], seed=5)
    feats = port.neck_inputs(c, B=1)
    neck = _neck(cuda, c, sd)
    outs = neck([f.to(cuda) for f in feats])
    want = port.ms_deform_pixel_decoder_3d(feats, sd, c["strides"], c["heads"], c["layers"], c["levels"], c["points"])
    for i, (o, r) in enumerate(zip(outs, want)):
        assert_close(o, r, what=f"full-width neck out[{i}] {tuple(r.shape)}")
