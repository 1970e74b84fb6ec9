"""The image encoder on the library's kernels (image_encoder.py _forward_cuda): the stem im2col, the stem max-pool and
SECONDFPN's pixel reshuffles one launch at a time, the 2-D stride-2 conv, Bottlenecks, the whole ResNet-50 and SECONDFPN,
the chain images -> ResNet -> SECONDFPN -> view transformer, and DepthNet on the encoder's channels_last map.  The
oracle is image_encoder.py's torch forward on the host in float64 (pinned to torchvision's resnet50 and to the reference
SECONDFPN by tests/test_cpu_image_encoder.py)."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from util import GOLDEN, assert_close, bits, f64, images, parity_log, rel_err, rel_rms, run_trace
from vt_chain import check_pooled, config_view_transformer
from occformer_b200 import BACKBONES, NECKS, ops, synth
from occformer_b200.common import attach_twin, twin_of
from occformer_b200.depthnet import DepthNet
from occformer_b200.image_encoder import SECONDFPN, ResNet

pytestmark = pytest.mark.gpu

KERNEL_TOL = 5e-5
SENTINEL = -1234.5
FPN = dict(in_channels=[256, 512, 1024, 2048], out_channels=[128, 128, 128, 128], upsample_strides=[0.25, 0.5, 1, 2])
HW = (256, 704)


def _backbone(seed, dev):
    net = ResNet(50).eval()
    net.load_state_dict(synth.make_resnet_state(seed), strict=True)
    return net.to(dev)


def _neck(seed, dev, cfg=FPN):
    net = SECONDFPN(**cfg).eval()
    net.load_state_dict(synth.make_secondfpn_state(seed=seed, **cfg), strict=True)
    return net.to(dev)


# ------------------------------------------------------------------ 1. the new kernels, one launch at a time
@pytest.mark.parametrize("H,W", [(256, 704), (37, 50), (8, 9)])
def test_stem_im2col_bitexact(cuda, H, W):
    """against F.unfold reordered to (ky, kx, c) columns, padded to 160 with zeros and split by split_weight: the image
    borders (zero padding) and the zero pad columns included"""
    n = 2
    x = images(n, H, W, seed=1)
    cols = ops.stem_im2col(x.to(cuda))
    u = F.unfold(x, 7, padding=3, stride=2)  # (n, c*49 + ky*7 + kx, L)
    L = u.shape[-1]
    want = u.view(n, 3, 49, L).permute(0, 3, 2, 1).reshape(n * L, 147)
    want = torch.cat([want, torch.zeros(n * L, 13)], dim=1)
    assert cols.shape == (n * ((H - 1) // 2 + 1) * ((W - 1) // 2 + 1), 160) == want.shape
    assert torch.equal(bits(cols), bits(ops.split_weight(want)))


@pytest.mark.parametrize("H,W,C", [(128, 352, 64), (15, 22, 96), (1, 3, 32)])
def test_maxpool_bitexact(cuda, H, W, C):
    """against F.max_pool2d(3, 2, 1): an odd size, and all-negative borders so that a zero padding would show"""
    n = 2
    x = torch.randn(n, C, H, W, generator=torch.Generator().manual_seed(2))
    x[:, :, 0], x[:, :, -1], x[:, :, :, 0], x[:, :, :, -1] = (-x[:, :, 0].abs() - 1, -x[:, :, -1].abs() - 1,
                                                              -x[:, :, :, 0].abs() - 1, -x[:, :, :, -1].abs() - 1)
    got = ops.maxpool3x3s2(x.permute(0, 2, 3, 1).contiguous().to(cuda))
    want = F.max_pool2d(x, 3, 2, 1).permute(0, 2, 3, 1).contiguous()
    assert got.shape == want.shape
    assert torch.equal(bits(got).view(-1, C), bits(ops.split_weight(want.view(-1, C))))
    if H > 2:
        assert bool((want[:, 0] < 0).any())  # a border window whose maximum is negative


@pytest.mark.parametrize("f", [2, 4])
def test_space_to_depth_bitexact(cuda, f):
    n, H, W, C = 2, 8 * f, 12 * f, 64
    x = ops.to_split(torch.randn(n, H, W, C, generator=torch.Generator().manual_seed(3)).to(cuda))
    got = ops.space_to_depth(x, f)
    want = x.cpu().view(n, H // f, f, W // f, f, C).permute(0, 1, 3, 2, 4, 5).reshape(n, H // f, W // f, f * f * C)
    assert torch.equal(bits(got), bits(want))


@pytest.mark.parametrize("f,C,ldo,off", [(2, 128, 512, 384), (2, 64, 200, 8), (4, 32, 96, 32)])
def test_depth_to_space_bitexact(cuda, f, C, ldo, off):
    n, h, w = 2, 5, 7
    y = torch.randn(n * h * w, f * f * C, generator=torch.Generator().manual_seed(4)).to(cuda)
    out = torch.full((n * h * w * f * f, ldo), SENTINEL, device=cuda)
    ops.depth_to_space_into(y, n, h, w, f, out, off)
    want = y.cpu().view(n, h, w, f, f, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, C)
    assert torch.equal(bits(out[:, off:off + C]), bits(want))
    outside = torch.cat([out[:, :off], out[:, off + C:]], dim=1)
    assert bool((bits(outside) == bits(torch.tensor(SENTINEL))).all()), "columns outside the slice changed"


# ------------------------------------------------------------------ 2. the 2-D stride-2 conv (Z = KZ = 1)
@pytest.mark.parametrize("k,H,W,Cin,Cout", [(3, 32, 88, 128, 128), (1, 32, 88, 256, 512), (3, 15, 22, 64, 64),
                                            (1, 15, 22, 64, 96)])
def test_conv2d_stride2_against_fp64(cuda, k, H, W, Cin, Cout):
    n = 3
    g = torch.Generator().manual_seed(5)
    x = torch.randn(n, Cin, H, W, generator=g)
    w = torch.randn(Cout, Cin, k, k, generator=g) * (k * k * Cin) ** -0.5
    b = 0.1 * torch.randn(Cout, generator=g)
    x_s = ops.to_split(x.permute(0, 2, 3, 1).contiguous().to(cuda)).unsqueeze(3)
    w2, ks = ops.repack_conv_weight(w.to(cuda))
    y = ops.conv(x_s, w2, ks, stride=2, bias=b.to(cuda))
    want = F.conv2d(x.double(), w.double(), b.double(), stride=2, padding=k // 2).permute(0, 2, 3, 1)
    assert y.shape == (n, (H - 1) // 2 + 1, (W - 1) // 2 + 1, 1, Cout)
    r = assert_close(y[:, :, :, 0], want, KERNEL_TOL, f"2-D stride-2 conv k={k} {H}x{W} {Cin}->{Cout}")
    parity_log(f"[image encoder] 2-D stride-2 conv k={k} {H}x{W}: rel_max {r:.2e}")


# ------------------------------------------------------------------ 3. Bottlenecks, whole ResNet, SECONDFPN
@pytest.mark.parametrize("layer,block", [("layer2", 0), ("layer2", 1)])
def test_bottleneck_against_fp64(cuda, layer, block):
    """layer2.0 (stride 2, downsample) and layer2.1 (identity shortcut) on a non-negative 256 / 512-channel map"""
    net = _backbone(6, cuda)
    blk = getattr(net, layer)[block]
    idx = 3 + block  # layer1 has 3 blocks
    cin = blk.conv1.in_channels
    x = torch.randn(4, cin, 32, 88, generator=torch.Generator().manual_seed(7)).abs()
    x_cl = x.permute(0, 2, 3, 1).contiguous().to(cuda).unsqueeze(3)
    out, out_s = ResNet._bottleneck_cuda(net._prepare()["blocks"][idx], x_cl, ops.to_split(x_cl))
    ref = f64(net)
    with torch.no_grad():
        want = getattr(ref, layer)[block](x.double()).permute(0, 2, 3, 1)
    r = assert_close(out[:, :, :, 0], want, 1e-3, f"Bottleneck {layer}.{block}")
    assert torch.equal(bits(out_s), bits(ops.to_split(out)))
    parity_log(f"[image encoder] Bottleneck {layer}.{block}: rel_max {r:.2e}")


def test_resnet50_against_fp64(cuda):
    net = _backbone(8, cuda)
    x = images(6, *HW, seed=9)
    outs = net(x.to(cuda))
    with torch.no_grad():
        want = f64(net)(x.double())
    assert len(outs) == 4
    for i, (o, w) in enumerate(zip(outs, want)):
        assert o.shape == w.shape and o.is_contiguous(memory_format=torch.channels_last)
        assert torch.equal(bits(twin_of(o)), bits(ops.to_split(o.permute(0, 2, 3, 1).contiguous())))
        r = assert_close(o, w, 1e-3, f"ResNet-50 stage {i}")
        pos = float((w > 0).double().mean())
        assert 0.05 < pos < 0.95, f"stage {i}: {pos:.1%} positive activations -- a vacuous comparison"
        parity_log(f"[image encoder] ResNet-50 (6, 3, 256, 704) stage {i}: rel_max {r:.2e}, {pos:.0%} positive")


@pytest.mark.parametrize("twin", [True, False, "modified"])
def test_secondfpn_against_fp64(cuda, twin):
    """at R50 shapes: levels with their S32 twin (as the ResNet hands them over), plain NCHW levels, and levels with
    twins of which one was scaled in place after the hand-over (its twin is stale: SECONDFPN must split the level)"""
    net = _neck(10, cuda)
    g = torch.Generator().manual_seed(11)
    n = 6
    levels = [torch.randn(n, c, 64 // 2 ** i, 176 // 2 ** i, generator=g).abs() for i, c in enumerate(FPN["in_channels"])]
    dev_levels = []
    for t in levels:
        d = t.to(cuda)
        if twin:
            d = d.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
            attach_twin(d, ops.to_split(d.permute(0, 2, 3, 1).contiguous()))
        dev_levels.append(d)
    if twin == "modified":
        dev_levels[1].mul_(0.5)
        levels[1] = levels[1] * 0.5
    out = net(dev_levels)
    assert isinstance(out, list) and len(out) == 1
    y = out[0]
    assert y.shape == (n, 512, 16, 44) and y.is_contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        want = f64(net)([t.double() for t in levels])[0]
    r = assert_close(y, want, 1e-3, f"SECONDFPN R50 twin={twin}")
    parity_log(f"[image encoder] SECONDFPN R50 (twin={twin if isinstance(twin, str) else int(twin)}): rel_max {r:.2e}")


def test_secondfpn_other_strides(cuda):
    """use_conv_for_no_stride and a stride-4 deconv (depth_to_space with f = 4)"""
    for cfg in (dict(in_channels=[64, 32], out_channels=[32, 64], upsample_strides=[1, 4]),
                dict(in_channels=[64], out_channels=[96], upsample_strides=[1], use_conv_for_no_stride=True)):
        net = SECONDFPN(**cfg).eval()
        net.load_state_dict(synth.make_secondfpn_state(seed=12, **cfg), strict=True)
        net = net.to(cuda)
        g = torch.Generator().manual_seed(13)
        levels = [torch.randn(2, c, int(8 / s), int(12 / s), generator=g) for c, s in
                  zip(cfg["in_channels"], cfg["upsample_strides"])]
        y = net([t.to(cuda) for t in levels])[0]
        with torch.no_grad():
            want = f64(net)([t.double() for t in levels])[0]
        assert_close(y, want, 1e-3, f"SECONDFPN {cfg}")


# ------------------------------------------------------------------ 4. connected: images -> view transformer
def test_images_to_view_transformer(cuda):
    """images -> ResNet -> SECONDFPN -> the reference glue's x.view(B, N, C, H, W) -> the view transformer built from the
    unmodified nuScenes R50 config, against the same chain on the host (torch modules in float64, oracle.port lift /
    voxel pooling) as test_gpu_depthnet.py::test_view_transformer_from_config"""
    cfg = json.load(open(os.path.join(GOLDEN, "image_encoder_cfg_nusc.json")))
    backbone, neck = BACKBONES.build(cfg["img_backbone"]).eval(), NECKS.build(cfg["img_neck"]).eval()
    backbone.load_state_dict(synth.make_resnet_state(14), strict=True)
    neck.load_state_dict(synth.make_secondfpn_state(seed=15, **FPN), strict=True)
    B, N = 1, 6
    vt, cams, mlp = config_view_transformer("nusc_r50", 16, B)
    backbone, neck, vt = backbone.to(cuda), neck.to(cuda), vt.to(cuda)
    imgs = images(B * N, *HW, seed=17)

    feat = neck(backbone(imgs.to(cuda)))[0]
    _, C, H, W = feat.shape
    x = feat.view(B, N, C, H, W)  # occupancyformer.py:22-35
    inp = [x] + [cams[k].to(cuda) for k in ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")]
    bev, prob = vt(inp + [mlp.to(cuda)])

    with torch.no_grad():
        out = f64(vt.depth_net)(f64(neck)(list(f64(backbone)(imgs.double())))[0], mlp.double())
    # every voxel within 1e-2 of the magnitude of its terms: 2.1e-3 measured on H100
    check_pooled(vt, cams, out, prob, bev, B, N, "[image encoder] images -> view transformer", "terms")


def test_depthnet_on_channels_last_map_is_bitwise_nchw(cuda):
    cin, mid, ctx, D, cam = 512, 512, 128, 112, 27
    net = DepthNet(cin, mid, ctx, D, cam_channels=cam).eval()
    net.load_state_dict(synth.make_depthnet_state(cin, mid, ctx, D, cam, seed=18), strict=True)
    net = net.to(cuda)
    g = torch.Generator().manual_seed(19)
    x = torch.randn(6, cin, 16, 44, generator=g).to(cuda)
    mlp = torch.randn(1, 6, cam, generator=g).to(cuda)
    x_cl = x.contiguous(memory_format=torch.channels_last)
    assert not x_cl.is_contiguous()
    assert torch.equal(bits(net(x_cl, mlp)), bits(net(x, mlp)))


# ------------------------------------------------------------------ 5. only library kernels, graph-safe
def test_only_library_kernels_and_cuda_graph(cuda):
    res = run_trace("r50", 900)
    # stem im2col + GEMM + max-pool, 16 Bottlenecks x (3 convs + split) + 4 downsamples, SECONDFPN: 2 space_to_depth +
    # 3 convs + GEMM + depth_to_space
    assert res["counted"] == res["kernels"] + res["memsets"] == 3 + 16 * 4 + 4 + 7
    assert res["graph_equals_eager"], "CUDA-graph replay differs from the eager forward"


# ------------------------------------------------------------------ 6. shape contract, bf16 mode
def test_shape_contract(cuda):
    net = _backbone(20, cuda)
    x = images(1, 100, 128, seed=21)
    with pytest.raises(RuntimeError, match="multiples of 32"):
        net(x.to(cuda))
    y = net.cpu()(x)  # the CPU forward still runs
    assert y[3].shape == (1, 2048, 4, 4)
    net = net.to(cuda).train()
    with pytest.raises(RuntimeError, match="eval mode"):
        net(images(1, 64, 64).to(cuda))
    neck = _neck(22, cuda)
    with pytest.raises(RuntimeError, match="one output size"):
        neck([torch.rand(1, c, 16, 16, device=cuda) for c in FPN["in_channels"]])
    narrow = SECONDFPN([16], [32], [1]).eval()
    t = torch.rand(1, 16, 4, 4)
    with pytest.raises(RuntimeError, match="multiples of 32"):
        narrow.to(cuda)([t.to(cuda)])
    assert narrow.cpu()([t])[0].shape == (1, 32, 4, 4)  # the CPU forward still runs
    neck = neck.to(cuda).train()
    with pytest.raises(RuntimeError, match="eval mode"):
        neck([torch.rand(1, c, 16 // 2 ** i, 16 // 2 ** i, device=cuda) for i, c in enumerate(FPN["in_channels"])])


def test_bf16_mode(cuda):
    backbone, neck = _backbone(23, cuda), _neck(24, cuda)
    x = images(6, *HW, seed=25)
    with ops.precision("bf16"):
        y = neck(list(backbone(x.to(cuda))))[0]
    with torch.no_grad():
        want = f64(neck)(list(f64(backbone)(x.double())))[0]
    # single-pass bf16 operands (~3e-3 per contraction) through 53 stacked convs and the FPN, a mode without a reference
    # twin: bounded by its max and rms error (5.5e-2 / 3.5e-2 measured on H100)
    r, q = rel_err(y, want), rel_rms(y, want)
    parity_log(f"[image encoder] bf16 mode: rel_max {r:.2e}, rel_rms {q:.2e}")
    assert r <= 1e-1 and q <= 5e-2, f"image encoder bf16: rel_max {r:.2e}, rel_rms {q:.2e}"
