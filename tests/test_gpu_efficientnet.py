"""CustomEfficientNet on the library's kernels (efficientnet.py _forward_cuda): the depthwise conv, the SE gate and scale,
the Swish epilogue and the generalised stem im2col one launch at a time, single blocks, the whole B7 at the SemanticKITTI
size, SECONDFPN at the KITTI levels, and the chain images -> B7 -> SECONDFPN -> view transformer.  The oracle is
efficientnet.py's torch forward in float64 (pinned to the reference class by tests/test_cpu_efficientnet.py)."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from util import GOLDEN, assert_close, bits, f64, golden, images, parity_log, rel_err, rel_rms, run_trace
from vt_chain import check_pooled, config_view_transformer
from occformer_b200 import BACKBONES, NECKS, ops, synth
from occformer_b200.common import attach_twin, twin_of
from occformer_b200.efficientnet import CustomEfficientNet, adaptive_pad
from occformer_b200.image_encoder import SECONDFPN

pytestmark = pytest.mark.gpu

KERNEL_TOL = 5e-5
OUTS = (2, 3, 4, 5, 6)
FPN = dict(in_channels=[48, 80, 224, 640, 2560], out_channels=[128] * 5, upsample_strides=[0.25, 0.5, 1, 2, 2])
HW = (384, 1280)


def _b7(seed, dev, out_indices=OUTS):
    net = CustomEfficientNet("b7", out_indices=out_indices).eval()
    net.load_state_dict(synth.make_efficientnet_state("b7", seed=seed, out_indices=out_indices), strict=True)
    return net.to(dev)


def _neck(seed, dev):
    net = SECONDFPN(**FPN).eval()
    net.load_state_dict(synth.make_secondfpn_state(seed=seed, out_hw=(6, 20), **FPN), strict=True)
    return net.to(dev)


def _swish(x):
    return x * torch.sigmoid(x)


# ------------------------------------------------------------------ 1. the new kernels, one launch at a time
@pytest.mark.parametrize("k,s,C,H,W", [(3, 1, 288, 48, 160), (3, 2, 192, 96, 320), (5, 1, 1344, 24, 80),
                                       (5, 2, 480, 48, 160), (3, 1, 64, 30, 17), (5, 2, 3840, 12, 40)])
def test_dwconv_swish_against_fp64(cuda, k, s, C, H, W):
    """out and the SE partial sums (their per-image total over the tiles) against F.conv2d(groups=C) + bias + Swish in
    fp64 with mmcv's adaptive padding; odd-chunk widths 288 / 1344 / 480 and a size that is not a multiple of 32.  fp32
    FMAs in a fixed order: 1.3e-7 - 2.6e-7 measured on H100, fp32 rounding"""
    n = 2
    g = torch.Generator().manual_seed(k * 100 + s * 10 + C)
    x = torch.randn(n, C, H, W, generator=g)
    w = torch.randn(C, 1, k, k, generator=g) * (2 / (k * k)) ** 0.5
    b = 0.1 * torch.randn(C, generator=g)
    Ho, Wo = -(-H // s), -(-W // s)
    (pt, pb), (pl, pr) = adaptive_pad(H, k, s), adaptive_pad(W, k, s)
    x_cl = x.permute(0, 2, 3, 1).contiguous().to(cuda)
    wt = w.view(C, k * k).t().contiguous().to(cuda)
    y, part = ops.dwconv_swish(x_cl, wt, b.to(cuda), k, s, pt, pl, Ho, Wo)
    want = _swish(F.conv2d(F.pad(x.double(), [pl, pr, pt, pb]), w.double(), b.double(), stride=s, groups=C))
    want = want.permute(0, 2, 3, 1)
    r = assert_close(y, want, KERNEL_TOL, f"depthwise k{k} s{s} C{C} {H}x{W}")
    rs = assert_close(part.sum(1), want.sum((1, 2)), KERNEL_TOL, f"depthwise SE sums k{k} s{s} C{C}")
    parity_log(f"[efficientnet] depthwise k{k} s{s} C{C} {H}x{W}: rel_max {r:.2e}, SE sums {rs:.2e}")
    # fixed-order partials: a second launch is bit-identical
    y2, part2 = ops.dwconv_swish(x_cl, wt, b.to(cuda), k, s, pt, pl, Ho, Wo)
    assert torch.equal(bits(y2), bits(y)) and torch.equal(bits(part2), bits(part))


@pytest.mark.parametrize("C,S,hw", [(288, 12, 1920), (1344, 56, 480), (64, 16, 122880), (3840, 160, 480)])
def test_se_gate_and_scale_against_fp64(cuda, C, S, hw):
    n = 3
    g = torch.Generator().manual_seed(C + S)
    y = _swish(torch.randn(n, hw, C, generator=g))
    tiles = ops.lib().occ_dw_tiles(1, hw)
    part = torch.zeros(n, tiles, C)
    for t in range(tiles):  # the partial sums occ_dwconv_swish would write for a 1 x hw map
        part[:, t] = y[:, t * 256:(t + 1) * 256].sum(1)
    w1 = torch.randn(S, C, generator=g) * (2 / C) ** 0.5
    b1 = 0.1 * torch.randn(S, generator=g)
    w2 = torch.randn(C, S, generator=g) * (2 / S) ** 0.5
    b2 = 0.1 * torch.randn(C, generator=g)
    d = lambda t: t.contiguous().to(cuda)  # noqa: E731
    gate = ops.se_gate(d(part), hw, d(w1.t()), d(b1), d(w2.t()), d(b2))
    mean = y.double().mean(1)
    want = torch.sigmoid(_swish(mean @ w1.double().t() + b1.double()) @ w2.double().t() + b2.double())
    r = assert_close(gate, want, KERNEL_TOL, f"SE gate C{C} S{S}")
    ys = ops.se_scale(d(y), gate)
    r2 = assert_close(ops.from_split(ys), y.double() * want.unsqueeze(1), KERNEL_TOL, f"SE scale C{C}")
    assert tiles == (hw + 255) // 256
    parity_log(f"[efficientnet] SE gate C{C} S{S}: rel_max {r:.2e}; scale {r2:.2e}")


def test_swish_epilogue_against_fp64(cuda):
    g = torch.Generator().manual_seed(60)
    M, N, K = 1000, 96, 64
    a, w, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * K ** -0.5, torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g)
    y = ops.gemm(ops.to_split(a.to(cuda)), ops.split_weight(w).to(cuda), bias=b.to(cuda), residual=res.to(cuda), act=3)
    want = F.silu(a.double() @ w.double().t() + b.double() + res.double())
    r = assert_close(y, want, KERNEL_TOL, "GEMM Swish epilogue")
    x_s = ops.to_split(a.view(10, 10, 10, 1, K).to(cuda))
    yc = ops.conv(x_s, ops.repack_conv_weight(w.view(N, K, 1, 1).to(cuda))[0], (1, 1, 1), bias=b.to(cuda), act=3)
    assert torch.equal(bits(yc.view(M, N)), bits(ops.gemm(ops.to_split(a.to(cuda)), ops.split_weight(w).to(cuda),
                                                         bias=b.to(cuda), act=3)))
    parity_log(f"[efficientnet] Swish epilogue: rel_max {r:.2e}")


@pytest.mark.parametrize("H,W", [(384, 1280), (37, 50), (8, 9)])
def test_im2col3_bitexact(cuda, H, W):
    """the generalised stem im2col at EfficientNet's 3x3 stride-2 adaptive padding, against F.pad + F.unfold"""
    n = 2
    x = images(n, H, W, seed=61)
    Ho, Wo = -(-H // 2), -(-W // 2)
    (pt, pb), (pl, pr) = adaptive_pad(H, 3, 2), adaptive_pad(W, 3, 2)
    cols = ops.im2col3(x.to(cuda), 3, 2, pt, pl, Ho, Wo, 32)
    u = F.unfold(F.pad(x, [pl, pr, pt, pb]), 3, stride=2)
    L = u.shape[-1]
    assert L == Ho * Wo
    want = torch.cat([u.view(n, 3, 9, L).permute(0, 3, 2, 1).reshape(n * L, 27), torch.zeros(n * L, 5)], dim=1)
    assert torch.equal(bits(cols), bits(ops.split_weight(want)))


# ------------------------------------------------------------------ 2. single blocks
@pytest.mark.parametrize("layer,block,what", [(1, 0, "no expand conv, 64 -> 32"), (2, 0, "stride 2, 32 -> 48 (padded)"),
                                              (2, 1, "residual at 48 (padded to 64)"), (4, 19, "residual at 224, k5")])
def test_block_against_fp64(cuda, layer, block, what):
    net = _b7(62, cuda)
    blocks = [b for l in net.layers[1:6] for b in l]
    idx = sum(len(net.layers[i]) for i in range(1, layer)) + block
    blk = net.layers[layer][block]
    p = net._prepare()["blocks"][idx]
    cin = blk.depthwise_conv.conv.in_channels if not blk.with_expand_conv else blk.expand_conv.conv.in_channels
    h, w = 384 // 2 ** layer, 1280 // 2 ** layer
    if blk.stride == 2:
        h, w = 2 * h, 2 * w
    x = torch.randn(2, cin, h, w, generator=torch.Generator().manual_seed(63))
    cp = (cin + 31) // 32 * 32
    x_cl = F.pad(x.permute(0, 2, 3, 1), (0, cp - cin)).contiguous().to(cuda).view(-1, cp)
    out, _, ho, wo = CustomEfficientNet._block_cuda(p, x_cl, ops.to_split(x_cl), 2, h, w)
    cout = blk.linear_conv.conv.out_channels
    with torch.no_grad():
        want = f64(net).layers[layer][block](x.double()).permute(0, 2, 3, 1)
    got = out.view(2, ho, wo, -1)
    assert bool((got[..., cout:] == 0).all()), "pad channels are not exactly 0"
    r = assert_close(got[..., :cout], want, 1e-3, f"block layers.{layer}.{block}")
    assert blocks[idx] is blk
    parity_log(f"[efficientnet] block layers.{layer}.{block} ({what}): rel_max {r:.2e}")


# ------------------------------------------------------------------ 3. full size
def test_b7_full_size_against_fp64(cuda):
    net = _b7(64, cuda)
    x = images(1, *HW, seed=65)
    outs = net(x.to(cuda))
    ref = f64(net, cuda)
    gates = []
    hooks = [b.se.conv2.register_forward_hook(lambda m, i, o: gates.append(o.flatten().cpu()))
             for l in ref.layers[1:6] for b in l]
    with torch.no_grad():
        want = ref._forward_torch(x.double().to(cuda))
    for h in hooks:
        h.remove()
    gates = torch.cat(gates)
    mid = float(((gates > 0.05) & (gates < 0.95)).double().mean())
    assert len(outs) == 5
    for i, (o, wnt) in enumerate(zip(outs, want)):
        assert o.shape == wnt.shape
        C = o.shape[1]
        assert twin_of(o).shape[-1] == (C + 31) // 32 * 32
        r = assert_close(o, wnt, 1e-3, f"B7 stage {OUTS[i]}")
        pos = float((wnt > 0).double().mean())
        assert 0.05 < pos < 0.95, f"stage {OUTS[i]}: {pos:.1%} positive activations -- a vacuous comparison"
        parity_log(f"[efficientnet] B7 (1, 3, 384, 1280) stage {OUTS[i]}: rel_max {r:.2e}, {pos:.0%} positive")
    parity_log(f"[efficientnet] B7 SE gates in (0.05, 0.95): {mid:.0%} of {gates.numel()}")
    assert mid > 0.5, f"only {mid:.1%} of the SE gates are away from 0 / 1"


def test_secondfpn_kitti_levels_with_attached_twins_against_fp64(cuda):
    """the five KITTI levels with zero-padded S32 twins (48 -> 64, 80 -> 96) handed over by attach_twin, as
    CustomEfficientNet hands them over; a 48-wide level changed in place afterwards cannot be re-split and raises"""
    net = _neck(66, cuda)
    g = torch.Generator().manual_seed(67)
    n = 2
    levels = [torch.randn(n, c, int(24 / s), int(80 / s), generator=g) for c, s in
              zip(FPN["in_channels"], FPN["upsample_strides"])]
    dev = []
    for t in levels:
        C = t.shape[1]
        cp = (C + 31) // 32 * 32
        full = F.pad(t.permute(0, 2, 3, 1), (0, cp - C)).contiguous().to(cuda)
        v = full[..., :C].permute(0, 3, 1, 2)
        dev.append(attach_twin(v, ops.to_split(full)))
    y = net(dev)[0]
    assert y.shape == (n, 640, 24, 80)
    with torch.no_grad():
        want = f64(net)([t.double() for t in levels])[0]
    r = assert_close(y, want, 1e-3, "SECONDFPN KITTI levels")
    parity_log(f"[efficientnet] SECONDFPN at the KITTI levels: rel_max {r:.2e}")
    dev[0].mul_(0.5)
    with pytest.raises(RuntimeError, match="unmodified since"):
        net(dev)


def test_images_to_view_transformer(cuda):
    """images -> B7 -> SECONDFPN -> view transformer built from the unmodified KITTI config, against the same chain in
    float64 (oracle.port lift / pooling), gated as test_gpu_image_encoder.py::test_images_to_view_transformer"""
    cfg = json.load(open(os.path.join(GOLDEN, "image_encoder_cfg_kitti.json")))
    backbone, neck = BACKBONES.build(cfg["img_backbone"]).eval(), NECKS.build(cfg["img_neck"]).eval()
    backbone.load_state_dict(synth.make_efficientnet_state("b7", seed=68, out_indices=OUTS), strict=True)
    neck.load_state_dict(synth.make_secondfpn_state(seed=69, out_hw=(6, 20), **FPN), strict=True)
    B, N = 1, 1
    vt, cams, mlp = config_view_transformer("kitti", 70, B)
    backbone, neck, vt = backbone.to(cuda), neck.to(cuda), vt.to(cuda)
    imgs = images(B * N, *HW, seed=71)

    feat = neck(backbone(imgs.to(cuda)))[0]
    _, C, H, W = feat.shape
    assert (C, H, W) == (640, 24, 80)
    x = feat.view(B, N, C, H, W)
    inp = [x] + [cams[k].to(cuda) for k in ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")]
    bev, prob = vt(inp + [mlp.to(cuda)])

    with torch.no_grad():
        stages = f64(backbone, cuda)._forward_torch(imgs.double().to(cuda))
        out = f64(vt.depth_net)(f64(neck)([s.cpu() for s in stages])[0], mlp.double())
    check_pooled(vt, cams, out, prob, bev, B, N, "[efficientnet] KITTI images -> view transformer", "terms")


def test_golden_on_gpu(cuda):
    """tests/golden/efficientnet_small.npz (the reference class at 'b0') on the kernels"""
    gd = golden("efficientnet_small.npz")
    net = CustomEfficientNet("b0", out_indices=(2, 3)).eval()
    net.load_state_dict({k[2:]: torch.from_numpy(gd[k]) for k in gd.files if k.startswith("w:")}, strict=True)
    outs = net.to(cuda)(torch.from_numpy(gd["x"]).to(cuda))
    for i, o in enumerate(outs):
        r = assert_close(o, torch.from_numpy(gd[f"out{i}"]), 1e-3, f"b0 golden stage {i}")
        parity_log(f"[efficientnet] b0 golden stage {i}: rel_max {r:.2e}")


# ------------------------------------------------------------------ 4. only library kernels, graph-safe
def test_only_library_kernels_and_cuda_graph(cuda):
    res = run_trace("b7", 1200)
    assert res["memsets"] == 0
    # stem im2col + GEMM; 55 blocks x (depthwise + SE gate + SE scale + linear GEMM) + 51 expand GEMMs (layers.1 has
    # none) + 52 splits (after every block followed by an expand conv or by layers.6); layers.6 GEMM + split;
    # SECONDFPN: 2 x (space_to_depth + conv) + conv + 2 x (GEMM + depth_to_space)
    assert res["counted"] == res["kernels"] == res["expected"] == 2 + 55 * 4 + 51 + 52 + 2 + 9
    assert res["graph_equals_eager"], "CUDA-graph replay differs from the eager forward"


# ------------------------------------------------------------------ 5. shape contract, bf16 mode
def test_shape_contract(cuda):
    net = CustomEfficientNet("b0", out_indices=(2, 3)).eval().to(cuda)
    with pytest.raises(RuntimeError, match="multiples of 32"):
        net(images(1, 100, 128).to(cuda))
    assert net.cpu()(images(1, 100, 128))[1].shape == (1, 40, 13, 16)  # the CPU forward still runs
    net = net.to(cuda).train()
    with pytest.raises(RuntimeError, match="eval mode"):
        net(images(1, 64, 64).to(cuda))


def test_bf16_mode(cuda):
    net, neck = _b7(72, cuda), _neck(73, cuda)
    x = images(1, *HW, seed=74)
    with ops.precision("bf16"):
        y = neck(list(net(x.to(cuda))))[0]
    with torch.no_grad():
        want = f64(neck)([s.cpu() for s in f64(net, cuda)._forward_torch(x.double().to(cuda))])[0]
    # single-pass bf16 operands (~3e-3 per contraction) through 112 GEMMs and the FPN, a mode without a reference twin:
    # bounded by its max and rms error (9.7e-3 / 3.9e-3 measured on H100)
    r, q = rel_err(y, want), rel_rms(y, want)
    parity_log(f"[efficientnet] bf16 mode: rel_max {r:.2e}, rel_rms {q:.2e}")
    assert r <= 3e-2 and q <= 1.5e-2, f"EfficientNet bf16: rel_max {r:.2e}, rel_rms {q:.2e}"
