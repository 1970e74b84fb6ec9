"""The fp64 reference of tests/test_gpu_encoder_glue.py (tests/encoder_ref.py) against oracle.port and against planted
mistakes.  Composed launch by launch with fp64 torch convolutions and the port's window attention, it equals
port.dualpath_block to fp64 round-off; and on the GPU test's own inputs, each planted mistake moves the result by more
than 10x the GPU gate.  A GPU failure then points at a kernel, and a case that cannot tell a mistake apart fails here."""
import pytest
import torch
import torch.nn.functional as F

import encoder_ref as ref
from oracle import port
from occformer_b200 import synth
from util import rel_err

G = 32                          # the model's GroupNorm groups
BITE = 10 * ref.GATE_S32        # a planted mistake must move the result by more than this (10x the looser gate)


def _f64(sd):
    """the floating-point entries of a state dict in fp64 (the relative position index stays an index)"""
    return {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}


def _rows(t):
    """(B, C, *spatial) -> (B * prod(spatial), C) token rows"""
    return t.movedim(1, -1).reshape(-1, t.shape[1])


def _aspp(xb, sd, p, B, X, Y):
    """BottleNeckASPP on BEV rows xb (B*X*Y, C) from encoder_ref's gn_apply / aspp_gap_branch and fp64 convs, with the
    library's inner-group rule"""
    from occformer_b200.encoder import _BottleNeckASPP
    C = xb.shape[1]
    ch, XY = C // 4, X * Y
    gi = _BottleNeckASPP(C, dict(type="GN", num_groups=G)).inner_groups
    a = p + "aspp."

    def conv(r, w, **kw):
        return _rows(F.conv2d(r.view(B, X, Y, -1).permute(0, 3, 1, 2), w, **kw))

    def norm(t, q, groups, **kw):
        return ref.gn_apply(t, ref.gn_stats(t, B, groups), sd[q + "weight"], sd[q + "bias"], XY, groups, **kw)

    y = norm(conv(xb, sd[p + "input_conv.0.weight"]), p + "input_conv.1.", G)
    branches = [norm(conv(y, sd[a + "aspp1.atrous_conv.weight"]), a + "aspp1.bn.", gi)]
    for i, d in zip((2, 3, 4), (6, 12, 18)):
        branches.append(norm(conv(y, sd[a + f"aspp{i}.atrous_conv.weight"], padding=d, dilation=d), a + f"aspp{i}.bn.", gi))
    branches.append(ref.aspp_gap_branch(y, sd[a + "global_avg_pool.1.weight"].view(ch, ch),
                                        sd[a + "global_avg_pool.2.weight"], sd[a + "global_avg_pool.2.bias"], B, gi))
    y3 = norm(conv(torch.cat(branches, 1), sd[a + "conv1.weight"]), a + "bn1.", gi, residual=y)
    return norm(conv(y3, sd[p + "output_conv.0.weight"]), p + "output_conv.1.", G, residual=xb)


def _block(x, sd, p, stride, shift):
    """port.dualpath_block as the library splits it: conv -> gn_relu_zmean_ln -> window attention on tokn -> proj +
    residual -> layernorm (norm2) -> FFN -> ASPP on the BEV rows -> dualpath_fuse"""
    B = x.shape[0]
    w = sd[p + "input_conv.0.weight"]
    C = w.shape[0]
    y = F.conv3d(x, w, None, stride=stride, padding=1)
    _, _, X, Y, Z = y.shape
    XY, nvox = X * Y, B * X * Y * Z
    y_r = _rows(y)
    st = ref.gn_stats(y_r, B, G)
    be = p + "bev_encoder."
    tok, tokn = ref.gn_relu_zmean_ln(y_r, st, sd[p + "input_conv.1.weight"], sd[p + "input_conv.1.bias"],
                                     sd[be + "norm1.weight"], sd[be + "norm1.bias"], B, XY, Z, G)

    def seqs(t):  # token rows -> the port's image sequences: the B BEV images, then 'b c x y z -> (b z) c x y'
        vox = t[:nvox].view(B, X, Y, Z, C).permute(0, 3, 1, 2, 4).reshape(B * Z, XY, C)
        return torch.cat([t[nvox:].view(B, XY, C), vox])

    att = port.shift_window_msa(seqs(tokn), (X, Y), sd, be + "attn.", C // 32, 3 if shift else 0)
    y1 = seqs(tok) + att
    h = F.gelu(F.linear(ref.layernorm(y1, sd[be + "norm2.weight"], sd[be + "norm2.bias"]),
                        sd[be + "ffn.layers.0.0.weight"], sd[be + "ffn.layers.0.0.bias"]))
    y2 = y1 + F.linear(h, sd[be + "ffn.layers.1.weight"], sd[be + "ffn.layers.1.bias"])
    x_vox = y2[B:].view(B, Z, X, Y, C).permute(0, 2, 3, 1, 4).reshape(nvox, C)
    bev = _aspp(y2[:B].reshape(B * XY, C), sd, p + "aspp.", B, X, Y)
    cw, cb = sd[p + "combine_coeff.weight"].view(C), float(sd[p + "combine_coeff.bias"])
    if stride > 1:
        idr = _rows(F.conv3d(x, sd[p + "downsample.0.weight"], None, stride=stride))
        out = ref.dualpath_fuse(x_vox, bev, cw, cb, idr, B, XY, Z, id_stats=ref.gn_stats(idr, B, G),
                                id_w=sd[p + "downsample.1.weight"], id_b=sd[p + "downsample.1.bias"], groups=G)
    else:
        out = ref.dualpath_fuse(x_vox, bev, cw, cb, _rows(x), B, XY, Z)
    return out, (X, Y, Z)


@pytest.mark.parametrize("B,cin,c,stride,shift,grid", [
    (2, 128, 128, 1, False, (9, 8, 3)),
    (1, 128, 128, 1, True, (15, 10, 4)),
    (2, 128, 256, 2, True, (15, 10, 4)),
    (1, 128, 256, 2, False, (9, 16, 2))])
def test_pieces_compose_to_port_dualpath_block(B, cin, c, stride, shift, grid):
    g = torch.Generator().manual_seed(c + 10 * stride + int(shift))
    sd = _f64(synth.make_block_state(cin, c, stride, g))
    x = torch.randn(B, cin, *grid, generator=g, dtype=torch.float64)
    want = port.dualpath_block(x, sd, "", stride, shift)
    got, (X, Y, Z) = _block(x, sd, "", stride, shift)
    torch.testing.assert_close(got, _rows(want), rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("C", [128, 256, 512])
def test_aspp_pieces_equal_port_bottleneck_aspp(C):
    """including the inner-group rule: C = 128 has ch = 32 <= 32, so ch / 2 = 16 groups; wider C has 32"""
    B, X, Y = 2, 11, 9
    g = torch.Generator().manual_seed(C)
    sd = _f64(synth.make_block_state(C, C, 1, g))
    xb = torch.randn(B, C, X, Y, generator=g, dtype=torch.float64)
    want = port.bottleneck_aspp(xb, sd, "aspp.")
    torch.testing.assert_close(_aspp(_rows(xb), sd, "aspp.", B, X, Y), _rows(want), rtol=1e-10, atol=1e-10)


def test_gn_stats_and_group_norm_equal_torch_group_norm():
    B, rpb, C, groups = 2, 50, 64, 16
    x = ref.gn_input(B, rpb, C, groups, seed=5).double()
    w, b = (t.double() for t in ref.affine(C, 6))
    got = ref.group_norm(x, ref.gn_stats(x, B, groups), w, b, rpb, groups)
    want = F.group_norm(x.view(B, rpb, C).transpose(1, 2), groups, w, b, ref.EPS).transpose(1, 2).reshape(-1, C)
    torch.testing.assert_close(got, want, rtol=1e-10, atol=1e-10)


# ------------------------------------------------------------------------------------------------ sensitivity
def _bites(mutant, want, what):
    r = rel_err(mutant, want)
    assert r > BITE, f"{what}: the planted mistake moves the result by only {r:.2e} (needs > {BITE:.0e})"


def _f64s(*ts):
    return [t.double() for t in ts]


def test_gn_apply_inputs_tell_sample_group_and_eps_mistakes_apart():
    """the (2, 2500, 32, 32) case of the GPU test (cpg 1, the ASPP input conv)"""
    B, rpb, C, groups = 2, 2500, 32, 32
    x, w, b = _f64s(*ref.gn_case(B, rpb, C, groups))
    st = ref.gn_stats(x, B, groups)
    want = ref.gn_apply(x, st, w, b, rpb, groups)
    swapped = st.clone()
    swapped[1] = st[0]
    _bites(ref.gn_apply(x, swapped, w, b, rpb, groups), want, "sample 0's statistics used for sample 1")
    _bites(ref.gn_apply(x, st.roll(-1, 1), w, b, rpb, groups), want, "group g+1's statistics used for group g")
    _bites(ref.gn_apply(x, st, w, b, rpb, groups, eps=1e-6), want, "GroupNorm eps 1e-6")


def test_layernorm_inputs_tell_eps_apart():
    rows, C = 1001, 256
    x = ref.ln_input(rows, C, ref.case_seed(rows, C)).double()
    w, b = _f64s(*ref.affine(C, ref.case_seed(C)))
    _bites(ref.layernorm(x, w, b, eps=1e-6), ref.layernorm(x, w, b), "LayerNorm eps 1e-6")


def test_zmean_inputs_tell_mean_before_relu_apart():
    B, X, Y, Z, C, groups = 2, 7, 5, 8, 128, 32
    XY = X * Y
    y, gw, gb = _f64s(*ref.gn_case(B, XY * Z, C, groups))
    lw, lb = _f64s(*ref.affine(C, ref.case_seed(C, groups, 1)))
    st = ref.gn_stats(y, B, groups)
    tok, _ = ref.gn_relu_zmean_ln(y, st, gw, gb, lw, lb, B, XY, Z, groups)
    before = torch.relu(ref.group_norm(y, st, gw, gb, XY * Z, groups).view(B * XY, Z, C).mean(1))
    _bites(before, tok[B * XY * Z:], "Z-mean taken before the ReLU")
    _bites(ref.gn_relu_zmean_ln(y, st, gw, gb, lw, lb, B, XY, Z, groups, eps=1e-6)[0], tok, "GroupNorm eps 1e-6")


def test_fuse_inputs_tell_the_neighbouring_bev_row_and_sample_apart():
    B, XY, Z, C = 2, 35, 3, 128
    x, bev, cw, idn = _f64s(*ref.fuse_case(B, XY, Z, C))
    want = ref.dualpath_fuse(x, bev, cw, 0.1, idn, B, XY, Z)
    _bites(ref.dualpath_fuse(x, bev.roll(-1, 0), cw, 0.1, idn, B, XY, Z), want, "BEV row of the neighbouring column")
    st = ref.gn_stats(idn, B, 32)
    w, b = _f64s(*ref.affine(C, ref.case_seed(C, 32)))
    want = ref.dualpath_fuse(x, bev, cw, 0.1, idn, B, XY, Z, id_stats=st, id_w=w, id_b=b, groups=32)
    _bites(ref.dualpath_fuse(x, bev, cw, 0.1, idn, B, XY, Z, id_stats=st[:1].expand(B, -1, -1), id_w=w, id_b=b,
                             groups=32), want, "sample 0's identity statistics used for sample 1")


def test_pool_branch_inputs_tell_unbiased_variance_and_global_mean_apart():
    """the (2, 2500, 32, 16) case of the GPU test: cpg 2, where the unbiased variance is twice the biased one"""
    B, rpb, ch, groups = 2, 2500, 32, 16
    x, wconv, gw, gb = _f64s(*ref.gap_case(B, rpb, ch, groups))
    want = ref.aspp_gap_values(ref.pool_means(x, B), wconv, gw, gb, groups)
    _bites(ref.aspp_gap_values(ref.pool_means(x, B), wconv, gw, gb, groups, correction=1), want,
           "unbiased variance in the 1x1 GroupNorm")
    every = x.mean(0, keepdim=True).expand(B, ch)
    _bites(ref.aspp_gap_values(every, wconv, gw, gb, groups), want, "pool mean taken over all samples")
