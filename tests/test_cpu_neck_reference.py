"""The fp64 reference of tests/test_gpu_neck_ops.py (tests/neck_ref.py) against oracle.port and against planted
mistakes.  Composed launch by launch with fp64 torch Linears and convolutions, it equals the port's deformable-attention
core, one encoder layer of the pixel decoder and its FPN step to fp64 round-off; and on the GPU test's own inputs, each
planted mistake moves the result by more than 10x the GPU gate.  A GPU failure then points at a kernel, and a case that
cannot tell a mistake apart fails here."""
import pytest
import torch
import torch.nn.functional as F

import neck_ref as ref
from oracle import port
from util import rel_err

BITE = 10 * ref.GATE_S32  # a planted mistake must move the result by more than this (10x the looser gate)


def _sample_major(t, grids, B):
    """level-major rows (B*Nq, ...) -> (B, Nq, ...) in the port's order (levels concatenated per sample)"""
    starts, ns = ref.level_starts(grids)
    return torch.cat([t[B * s:B * (s + n)].reshape(B, n, *t.shape[1:]) for s, n in zip(starts, ns)], 1)


def _level_major(t, grids):
    """(B, Nq, ...) -> level-major rows (B*Nq, ...)"""
    starts, ns = ref.level_starts(grids)
    return torch.cat([t[:, s:s + n].reshape(-1, *t.shape[2:]) for s, n in zip(starts, ns)])


def _port_ref_points(grids, strides):
    """the port decoder's reference points (grid_priors_3d / (size * stride)), divided in fp64: (Nq, 3)"""
    return torch.cat([port.grid_priors_3d(g, s).double() / (torch.tensor([[g[2], g[1], g[0]]], dtype=torch.float64) * s)
                      for g, s in zip(grids, strides)])


def _port_msda(value, ow, grids, strides, B, E, H, P):
    """port.ms_deform_attn_core_3d on level-major operands (fp64) -> level-major (rows, E)"""
    L = len(grids)
    Nq = sum(x * y * z for x, y, z in grids)
    v = _sample_major(value, grids, B).view(B, Nq, H, E // H)
    o = _sample_major(ow, grids, B)
    off = o[..., :H * L * P * 3].reshape(B, Nq, H, L, P, 3)
    aw = o[..., H * L * P * 3:].reshape(B, Nq, H, L * P).softmax(-1).view(B, Nq, H, L, P)
    norm = torch.tensor([[Z, Y, X] for (X, Y, Z) in grids], dtype=torch.float64)
    loc = _port_ref_points(grids, strides)[None, :, None, None, None, :] + off / norm[None, None, None, :, None, :]
    return _level_major(port.ms_deform_attn_core_3d(v, grids, loc, aw), grids)


def _ow(grids, B, H, seed):
    """ow_input in fp64 with the +-1e30 offsets brought to +-(1e4 + 50): grid_sample's int conversion is not defined
    that far out, and both are beyond every volume"""
    ow = ref.ow_input(grids, B, H, seed=seed).double()
    n = ow.shape[1] // 4 * 3
    ow[:, :n] = ow[:, :n].clamp(-1e4 - 50, 1e4 + 50)
    return ow


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("grids,strides", [
    ([(9, 6, 3)], (4,)),
    ([(3, 5, 2), (6, 10, 4)], (8, 4)),
    ([(7, 7, 1), (13, 13, 2), (25, 25, 4)], (12, 6, 3)),
    ([(2, 2, 1), (4, 3, 2), (8, 6, 4), (16, 12, 8)], (16, 8, 4, 2))])
def test_ms_deform_attn_equals_port_core(grids, strides, B):
    E, H, P = 32, 4, 4
    value = ref.value_input(grids, B, E, H, seed=len(grids) + B).double()
    ow = _ow(grids, B, H, seed=10 * len(grids) + B)
    got = ref.ms_deform_attn(value, ow, grids, strides, B, E, H, P, chunk=500)
    torch.testing.assert_close(got, _port_msda(value, ow, grids, strides, B, E, H, P), rtol=1e-12, atol=1e-12)
    # the GPU test's fp32 sampling coordinates differ from fp64 ones by rounding only
    f32 = ref.ms_deform_attn(value, ow.float(), grids, strides, B, E, H, P, chunk=500, coords="fp32")
    assert rel_err(f32, ref.ms_deform_attn(value, ow.float(), grids, strides, B, E, H, P)) < 1e-5


@pytest.mark.parametrize("B", [1, 2])
def test_encoder_layer_composes_to_port(B):
    """one encoder layer of port.NECK_CASE (E 96, 4 heads, 3 levels, ffn 192): token_prep (+ pos) -> value and
    offset / logit Linears -> ms_deform_attn -> output Linear + residual -> token_prep (norms.0) -> FFN -> token_prep
    (norms.1), against port.ms_deform_attn_3d + LayerNorm + FFN + LayerNorm"""
    c = port.NECK_CASE
    E, H, P, L = c["E"], c["heads"], c["points"], c["levels"]
    sd = {k: v.double() for k, v in port.make_neck_state(c["in_channels"], E, c["layers"], H, L, P, c["ffn"],
                                                         seed=c["wseed"]).items()}
    nin = len(c["sizes"])
    grids = [tuple(c["sizes"][nin - i - 1]) for i in range(L)]
    strides = [c["strides"][nin - i - 1] for i in range(L)]
    Nq = sum(x * y * z for x, y, z in grids)
    g = torch.Generator().manual_seed(B)
    x = torch.randn(B * Nq, E, generator=g, dtype=torch.float64)
    pos = torch.randn(Nq, E, generator=g, dtype=torch.float64)
    p = "encoder.layers.0."
    a = p + "attentions.0."
    # the port: (Nq, B, E) sample-major tokens
    xs = _sample_major(x, grids, B).transpose(0, 1)
    refp = _port_ref_points(grids, strides)[None, :, None].repeat(B, 1, L, 1)
    y = port.ms_deform_attn_3d(xs, pos[:, None].expand(Nq, B, E), refp, grids, sd, a, H, P)
    y = F.layer_norm(y, (E,), sd[p + "norms.0.weight"], sd[p + "norms.0.bias"], ref.EPS)
    y = y + F.linear(F.relu(F.linear(y, sd[p + "ffns.0.layers.0.0.weight"], sd[p + "ffns.0.layers.0.0.bias"])),
                     sd[p + "ffns.0.layers.1.weight"], sd[p + "ffns.0.layers.1.bias"])
    want = _level_major(F.layer_norm(y, (E,), sd[p + "norms.1.weight"], sd[p + "norms.1.bias"], ref.EPS).transpose(0, 1),
                        grids)
    # the library's launches
    _, xq = ref.token_prep(x, grids, B, pos=pos)
    v = F.linear(x, sd[a + "value_proj.weight"], sd[a + "value_proj.bias"])
    ow = torch.cat([F.linear(xq, sd[a + "sampling_offsets.weight"], sd[a + "sampling_offsets.bias"]),
                    F.linear(xq, sd[a + "attention_weights.weight"], sd[a + "attention_weights.bias"])], 1)
    att = ref.ms_deform_attn(v, ow, grids, strides, B, E, H, P)
    y = F.linear(att, sd[a + "output_proj.weight"], sd[a + "output_proj.bias"]) + x
    x1, _ = ref.token_prep(y, grids, B, ln=(sd[p + "norms.0.weight"], sd[p + "norms.0.bias"]))
    h = F.relu(F.linear(x1, sd[p + "ffns.0.layers.0.0.weight"], sd[p + "ffns.0.layers.0.0.bias"]))
    y2 = x1 + F.linear(h, sd[p + "ffns.0.layers.1.weight"], sd[p + "ffns.0.layers.1.bias"])
    got, _ = ref.token_prep(y2, grids, B, ln=(sd[p + "norms.1.weight"], sd[p + "norms.1.bias"]))
    torch.testing.assert_close(got, want, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("fine,coarse", [((8, 6, 4), (4, 3, 2)), ((13, 13, 2), (7, 7, 1)), ((16, 12, 3), (8, 6, 2))])
def test_fpn_step_equals_port_conv_gn_and_interpolate(fine, coarse):
    """gn_stats + gn_upsample_add fed fp64 statistics = port._conv_gn (1x1x1 conv, GroupNorm) + F.interpolate"""
    B, Cin, C, G = 2, 48, 64, 32
    g = torch.Generator().manual_seed(sum(fine))
    sd = {"lat.conv.weight": torch.randn(C, Cin, 1, 1, 1, generator=g, dtype=torch.float64) * Cin ** -0.5,
          "lat.gn.weight": 1 + 0.1 * torch.randn(C, generator=g, dtype=torch.float64),
          "lat.gn.bias": 0.1 * torch.randn(C, generator=g, dtype=torch.float64)}
    feat = torch.randn(B, Cin, *fine, generator=g, dtype=torch.float64) + 0.5
    low = torch.randn(B, C, *coarse, generator=g, dtype=torch.float64)
    want = port._conv_gn(feat, sd, "lat.", G) + F.interpolate(low, size=fine, mode="trilinear", align_corners=False)
    raw = F.conv3d(feat, sd["lat.conv.weight"]).permute(0, 2, 3, 4, 1).contiguous()
    st = ref.gn_stats(raw.view(-1, C), B, G)
    got = ref.gn_upsample_add(raw, st, sd["lat.gn.weight"], sd["lat.gn.bias"], G, low.permute(0, 2, 3, 4, 1))
    torch.testing.assert_close(got, want.permute(0, 2, 3, 4, 1), rtol=1e-10, atol=1e-10)


# ------------------------------------------------------------------------------------------------ sensitivity
def _bites(mutant, want, what):
    r = rel_err(mutant, want)
    assert r > BITE, f"{what}: the planted mistake moves the result by only {r:.2e} (needs > {BITE:.0e})"


@pytest.mark.parametrize("case", [2, 3], ids=["L2-B2-H2", "L4-B2-H4"])
@pytest.mark.parametrize("mistake", ref.MSDA_MISTAKES)
def test_ms_deform_attn_inputs_tell_mistakes_apart(case, mistake):
    grids, strides, E, H, B, lds = ref.MSDA_CASES[case]
    value = ref.value_input(grids, B, E, H, seed=ref.case_seed(case, 1)).double()
    ow = ref.ow_input(grids, B, H, seed=ref.case_seed(case, 2)).double()
    want = ref.ms_deform_attn(value, ow, grids, strides, B, E, H)
    _bites(ref.ms_deform_attn(value, ow, grids, strides, B, E, H, mistake=mistake), want, f"ms_deform_attn {mistake}")


@pytest.mark.parametrize("mistake", ["pos_sample_major", "pos_before_ln", "eps"])
def test_token_prep_inputs_tell_mistakes_apart(mistake):
    """the L = 3, B = 3, C = 192 case of the GPU test"""
    grids, B, C = ref.TOKEN_GRIDS[3], 3, 192
    x, pos = (t.double() for t in ref.token_input(grids, B, C, ref.case_seed(C, len(grids), B)))
    ln = tuple(t.double() for t in ref.affine(C, ref.case_seed(C)))
    want = ref.token_prep(x, grids, B, ln=ln, pos=pos)
    if mistake == "eps":
        _bites(ref.token_prep(x, grids, B, ln=ln, pos=pos, eps=1e-6)[0], want[0], "LayerNorm eps 1e-6")
    else:
        _bites(ref.token_prep(x, grids, B, ln=ln, pos=pos, mistake=mistake)[1], want[1], mistake)


@pytest.mark.parametrize("mistake", list(ref.GN_UP_MISTAKES) + ["neighbour_stats", "eps"])
@pytest.mark.parametrize("case", [0, 4])
def test_gn_upsample_add_inputs_tell_mistakes_apart(case, mistake):
    """a x2 case and a general case of the GPU test, both B = 2"""
    B, (X, Y, Z), (Xc, Yc, Zc), C, groups = ref.GN_UP_CASES[case]
    cur = ref.gn_input(B, X * Y * Z, C, groups, ref.case_seed(case, 1)).double()
    gw, gb = (t.double() for t in ref.affine(C, ref.case_seed(C, groups)))
    coarse = ref.coarse_input(B, Xc, Yc, Zc, C, ref.case_seed(case, 2)).double()
    st = ref.gn_stats(cur, B, groups)
    cur = cur.view(B, X, Y, Z, C)
    want = ref.gn_upsample_add(cur, st, gw, gb, groups, coarse)
    if mistake == "neighbour_stats":
        got = ref.gn_upsample_add(cur, st.roll(1, 0), gw, gb, groups, coarse)
    elif mistake == "eps":
        got = ref.gn_upsample_add(cur, st, gw, gb, groups, coarse, eps=1e-6)
    else:
        got = ref.gn_upsample_add(cur, st, gw, gb, groups, coarse, mistake=mistake)
    _bites(got, want, f"gn_upsample_add {mistake}")


def test_gn_stats_inputs_tell_the_next_sample_apart():
    """the (3, 1250, 192, 6) case of the GPU test, through the GroupNorm its statistics feed"""
    B, rows, C, cpg = ref.GN_STATS_CASES[1]
    groups = C // cpg
    x = ref.gn_input(B, rows, C, groups, ref.case_seed(B, rows, C, cpg)).double()
    w, b = torch.ones(C, dtype=torch.float64), torch.zeros(C, dtype=torch.float64)
    want = ref.group_norm(x, ref.gn_stats(x, B, groups), w, b, rows, groups)
    _bites(ref.group_norm(x, ref.gn_stats(x, B, groups, mistake="next_sample"), w, b, rows, groups), want,
           "rows of sample b + 1 counted in sample b")


def test_ref_points_and_pos_index():
    """the level-major bookkeeping the references share: pos row = start_l + local for every sample, and the reference
    point of a voxel is its centre normalised in its own level"""
    grids, B = [(2, 1, 1), (2, 2, 1)], 2
    assert ref.pos_index(grids, B).tolist() == [0, 1, 0, 1, 2, 3, 4, 5, 2, 3, 4, 5]
    assert ref.ref_points(grids, (8, 4))[:2].tolist() == [[0.5, 0.5, 0.25], [0.5, 0.5, 0.75]]
