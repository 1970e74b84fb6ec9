"""ResNetDCN and its DCNv2 layer on the CPU (float64): the ModulatedDeformConv2dPack sampling rules pinned by identities
and by hand-computed bilinear samples (mmcv's own op is not available here), caffe-style R101 against torchvision's
resnet101 with the stage strides moved to conv1, ResNetDCN(50) against ResNet(50), the R101 config's keys, the folded
parameters of the CUDA path, the unsupported options and the local-only registration."""
import importlib.util
import json
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from util import GOLDEN, assert_close, rel_err
import occformer_b200
from occformer_b200 import BACKBONES, HEADS, NECKS, registry, synth
from occformer_b200.depthnet import deform_columns
from occformer_b200.image_encoder import ModulatedDeformConv2dPack, ResNet, ResNetDCN

DCN = dict(type="DCNv2", deform_groups=1, fallback_on_stride=False)
R101 = dict(style="caffe", dcn=DCN, stage_with_dcn=(False, False, True, True))


def _cfg():
    return json.load(open(os.path.join(GOLDEN, "image_encoder_cfg_nusc_r101.json")))


def _layer(C, off_bias, mask_logit, weight=None):
    """a float64 DCNv2 layer whose conv_offset is the constant off_bias (27,) and whose weight is the identity on the
    centre tap unless given"""
    m = ModulatedDeformConv2dPack(C, C).double()
    with torch.no_grad():
        m.conv_offset.weight.zero_()
        m.conv_offset.bias.copy_(torch.as_tensor(off_bias, dtype=torch.float64))
        m.conv_offset.bias[18:] = torch.as_tensor(mask_logit, dtype=torch.float64)
        if weight is None:
            m.weight.zero_()
            m.weight[:, :, 1, 1] = torch.eye(C, dtype=torch.float64)
        else:
            m.weight.copy_(weight)
    return m


# ------------------------------------------------------------------ the DCNv2 layer
def test_dcnv2_zero_offsets_is_mask_weighted_sum_of_taps():
    """offsets 0: sum over the kernel points k of sigmoid(m_k) * (tap k of the plain 3x3 conv)"""
    g = torch.Generator().manual_seed(1)
    C, O = 8, 6
    x = torch.randn(2, C, 7, 9, generator=g).double()
    w = torch.randn(O, C, 3, 3, generator=g).double()
    logits = torch.randn(9, generator=g).double()
    m = ModulatedDeformConv2dPack(C, O).double()
    with torch.no_grad():
        m.conv_offset.weight.zero_()
        m.conv_offset.bias.zero_()
        m.conv_offset.bias[18:] = logits
        m.weight.copy_(w)
        got = m(x)
    want = 0
    for k in range(9):
        wk = torch.zeros_like(w)
        wk[:, :, k // 3, k % 3] = w[:, :, k // 3, k % 3]
        want = want + torch.sigmoid(logits[k]) * F.conv2d(x, wk, padding=1)
    assert_close(got, want, 1e-12, "DCNv2 with zero offsets")


@pytest.mark.parametrize("dy,dx", [(2, -1), (-3, 0), (0, 4)])
def test_dcnv2_integer_offsets_shift_the_map(dy, dx):
    """the centre point offset by integers (dy, dx), mask logit 0, identity weight: 0.5 * x[y + dy, x + dx], zero where
    that lies outside the map"""
    C, H, W = 3, 6, 7
    x = torch.randn(1, C, H, W, generator=torch.Generator().manual_seed(2)).double()
    off = torch.zeros(27)
    off[8], off[9] = dy, dx
    with torch.no_grad():
        got = _layer(C, off, 0.0)(x)
    want = torch.zeros_like(x)
    ys, xs = slice(max(-dy, 0), min(H - dy, H)), slice(max(-dx, 0), min(W - dx, W))
    want[:, :, ys, xs] = 0.5 * x[:, :, max(dy, 0):min(H + dy, H), max(dx, 0):min(W + dx, W)]
    assert_close(got, want, 1e-12, f"DCNv2 with integer offsets ({dy}, {dx})")  # grid_sample's normalisation: 1e-17


def _mmcv_sample(img, h, w):
    """mmcv-full 1.4.0 modulated_deformable_im2col_gpu_kernel for one sample of a (H, W) map, written out as it is:
    zero unless h > -1 && w > -1 && h < H && w < W, then dmcn_im2col_bilinear with each corner outside the map zero."""
    H, W = img.shape
    if not (h > -1 and w > -1 and h < H and w < W):
        return 0.0
    h_low, w_low = math.floor(h), math.floor(w)
    h_high, w_high = h_low + 1, w_low + 1
    lh, lw = h - h_low, w - w_low
    hh, hw = 1 - lh, 1 - lw
    v1 = float(img[h_low, w_low]) if h_low >= 0 and w_low >= 0 else 0.0
    v2 = float(img[h_low, w_high]) if h_low >= 0 and w_high <= W - 1 else 0.0
    v3 = float(img[h_high, w_low]) if h_high <= H - 1 and w_low >= 0 else 0.0
    v4 = float(img[h_high, w_high]) if h_high <= H - 1 and w_high <= W - 1 else 0.0
    return hh * hw * v1 + hh * lw * v2 + lh * hw * v3 + lh * lw * v4


OFFSETS = [(0.25, 0.5), (-0.75, 0.4), (-1.0, 0.0), (-1.5, 0.2), (0.3, -0.6), (-0.5, -0.5), (2.5, 3.25), (1.0, -1.0),
           (3.6, 4.7), (-4.2, 1.1)]


def test_dcnv2_hand_computed_bilinear_samples():
    """every point k of a 4x5 map at ten constant offsets against _mmcv_sample; the cases cover h <= -1 and h >= H
    (no contribution), a row or column of corners outside the map (two corners), a row and a column (three corners), and
    interior samples"""
    H, W = 4, 5
    img = torch.arange(1, H * W + 1, dtype=torch.float64).view(1, 1, H, W) * 0.1 + 1.0
    kinds = set()
    for dy, dx in OFFSETS:
        logits = torch.linspace(-2, 2, 9).double()
        off = torch.zeros(27, dtype=torch.float64)
        off[0:18:2], off[1:18:2] = dy, dx
        col = deform_columns(img, off.view(1, 27, 1, 1).expand(1, 27, H, W))[0, 0]  # (9, H, W)
        with torch.no_grad():
            for k in range(9):
                wk = torch.zeros(1, 1, 3, 3, dtype=torch.float64)
                wk[0, 0, k // 3, k % 3] = 1.0
                got = _layer(1, off, logits, wk)(img)[0, 0]
                for y in range(H):
                    for x in range(W):
                        h, w = y - 1 + k // 3 + dy, x - 1 + k % 3 + dx
                        want = _mmcv_sample(img[0, 0], h, w)
                        assert abs(float(col[k, y, x]) - want) <= 1e-12, (dy, dx, k, y, x)
                        assert abs(float(got[y, x]) - want * float(torch.sigmoid(logits[k]))) <= 1e-12
                        if not (h > -1 and w > -1 and h < H and w < W):
                            kinds.add("h<=-1" if h <= -1 else "h>=H" if h >= H else "w out")
                        else:
                            hl, wl = math.floor(h), math.floor(w)
                            out_rows = (hl < 0) + (hl + 1 > H - 1)
                            out_cols = (wl < 0) + (wl + 1 > W - 1)
                            n_out = sum(not (0 <= a < H and 0 <= b < W) for a in (hl, hl + 1) for b in (wl, wl + 1))
                            if (h != hl and out_rows) or (w != wl and out_cols) or n_out:
                                kinds.add(f"{n_out} corners out")
                            else:
                                kinds.add("inside")
    assert {"h<=-1", "h>=H", "2 corners out", "3 corners out", "inside"} <= kinds, kinds


def test_dcn_layer_keys_and_unsupported_options():
    m = ModulatedDeformConv2dPack(64, 32)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {
        "weight": (32, 64, 3, 3), "conv_offset.weight": (27, 64, 3, 3), "conv_offset.bias": (27,)}
    for kw in (dict(stride=2), dict(deform_groups=2), dict(bias=True), dict(dilation=2)):
        with pytest.raises(NotImplementedError):
            ModulatedDeformConv2dPack(64, 32, **kw)


# ------------------------------------------------------------------ the backbone
def test_caffe_r101_without_dcn_equals_torchvision_with_strides_on_conv1():
    tv = pytest.importorskip("torchvision")
    sd = synth.make_resnet_dcn_state(3, style="caffe", calib_shape=(1, 3, 64, 96))
    ref = tv.models.resnet101()
    assert set(ref.state_dict()) - {"fc.weight", "fc.bias"} == set(sd)
    for i in range(2, 5):
        blk = getattr(ref, f"layer{i}")[0]
        blk.conv1.stride, blk.conv2.stride = blk.conv2.stride, (1, 1)
    ref.load_state_dict(sd, strict=False)
    ref = ref.double().eval()
    net = ResNetDCN(101, style="caffe").eval()
    net.load_state_dict(sd, strict=True)
    x = torch.randn(2, 3, 64, 96, generator=torch.Generator().manual_seed(4)).double()
    with torch.no_grad():
        got = net.double()(x)
        y = ref.maxpool(ref.relu(ref.bn1(ref.conv1(x))))
        for i in range(4):
            y = getattr(ref, f"layer{i + 1}")(y)
            assert_close(got[i], y, 1e-6, f"caffe ResNet-101 stage {i} vs torchvision with conv1 strides")


def test_resnet_dcn_50_is_resnet_50_bit_for_bit():
    sd = synth.make_resnet_state(5)
    a, b = ResNet(50).eval(), ResNetDCN(50).eval()
    a.load_state_dict(sd, strict=True)
    b.load_state_dict(sd, strict=True)
    x = torch.randn(1, 3, 64, 96, generator=torch.Generator().manual_seed(6))
    with torch.no_grad():
        for u, v in zip(a(x), b(x)):
            assert torch.equal(u, v)
    for fa, fb in zip(a._folded()["blocks"], b._folded()["blocks"]):
        assert fa[0] == fb[0] and fb[5:] == (False, None)
        for u, v in zip(fa[1:5], fb[1:5]):
            assert (u is None and v is None) or all(torch.equal(p, q) for p, q in zip(u, v))


def test_r101_config_keys_and_strict_load():
    tv = pytest.importorskip("torchvision")
    cfg = _cfg()["img_backbone"]
    assert cfg["type"] == "ResNet" and cfg["depth"] == 101 and cfg["style"] == "caffe"
    net = BACKBONES.build(dict(cfg, type=ResNetDCN))
    assert type(net) is ResNetDCN and net.out_indices == (0, 1, 2, 3)
    keys = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    tv_keys = {k: tuple(v.shape) for k, v in tv.models.resnet101().state_dict().items() if not k.startswith("fc.")}
    extra = {}
    for i, (blocks, planes) in enumerate(zip((3, 4, 23, 3), (64, 128, 256, 512))):
        if i >= 2:
            for j in range(blocks):
                extra[f"layer{i + 1}.{j}.conv2.conv_offset.weight"] = (27, planes, 3, 3)
                extra[f"layer{i + 1}.{j}.conv2.conv_offset.bias"] = (27,)
    assert keys == {**tv_keys, **extra}
    assert len(extra) == 2 * 26
    assert net.layer3[0].conv1.stride == (2, 2) and isinstance(net.layer3[0].conv2, ModulatedDeformConv2dPack)
    assert net.layer2[0].conv1.stride == (2, 2) and net.layer2[0].conv2.stride == (1, 1)
    net.load_state_dict(synth.make_resnet_dcn_state(7, calib_shape=(1, 3, 64, 96), **R101), strict=True)


def test_r101_model_builds_through_the_registries():
    """the whole R101 model dict: the image encoder with ResNetDCN opted in as `type`, and the hot-path sections of the
    unmodified config (tests/golden/model_cfg_nusc_r101.json) as they are"""
    enc = _cfg()
    backbone = BACKBONES.build(dict(enc["img_backbone"], type=ResNetDCN))
    neck = NECKS.build(enc["img_neck"])
    cfg = json.load(open(os.path.join(GOLDEN, "model_cfg_nusc_r101.json")))
    vt = NECKS.build(cfg["img_view_transformer"])
    bev = BACKBONES.build(cfg["img_bev_encoder_backbone"])
    bev_neck = NECKS.build(cfg["img_bev_encoder_neck"])
    head = HEADS.build(cfg["pts_bbox_head"])
    assert type(backbone) is ResNetDCN and type(neck).__name__ == "SECONDFPN"
    assert vt.data_config["input_size"] == [896, 1600] and vt.D == 112 and vt.numC_input == 512
    assert vt.grid_size() == (128, 128, 16)
    assert len(bev.layers) == 4 and bev_neck.num_encoder_levels == 3 and head.num_classes == 17
    assert BACKBONES.get("ResNetDCN") is ResNetDCN and occformer_b200.ResNetDCN is ResNetDCN


@pytest.mark.parametrize("kw,name", [
    (dict(dcn=dict(type="DCN", deform_groups=1, fallback_on_stride=False)), "dcn"),
    (dict(dcn=dict(type="DCNv2", deform_groups=4, fallback_on_stride=False)), "dcn"),
    (dict(dcn=dict(type="DCNv2", deform_groups=1, fallback_on_stride=True)), "dcn"),
    (dict(style="pytorch"), "stage_with_dcn"), (dict(stage_with_dcn=(False, True, True)), "stage_with_dcn"),
    (dict(depth=152), "depth"), (dict(style="other"), "style"), (dict(deep_stem=True), "deep_stem"),
    (dict(avg_down=True), "avg_down"), (dict(plugins=[dict(cfg=dict(type="ContextBlock"))]), "plugins"),
    (dict(strides=(1, 2, 2, 1)), "strides"), (dict(dilations=(1, 1, 1, 2)), "dilations"),
    (dict(norm_cfg=dict(type="GN", num_groups=32)), "norm_cfg")])
def test_unsupported_options_raise(kw, name):
    with pytest.raises(NotImplementedError, match=name):
        ResNetDCN(**{"depth": 101, **R101, **kw})


def test_supported_options():
    ResNetDCN(101, style="pytorch", dcn=DCN, stage_with_dcn=(True, False, False, False))  # stride-1 stage: fine
    ResNetDCN(50, style="caffe", dcn=DCN, stage_with_dcn=(False, True, True, True), frozen_stages=1, norm_eval=True,
              with_cp=True, norm_cfg=dict(type="BN2d", requires_grad=False))
    assert not ResNetDCN(101, stage_with_dcn=(False, False, True, True)).stage_dcn[2]  # mmdet: no dcn, no DCN stage


def test_folded_parameters_reproduce_forward():
    net = ResNetDCN(101, **R101).eval()
    net.load_state_dict(synth.make_resnet_dcn_state(8, calib_shape=(1, 3, 64, 96), **R101), strict=True)
    x = torch.randn(1, 3, 64, 96, generator=torch.Generator().manual_seed(9)).double()
    Fp = net._folded()
    with torch.no_grad():
        want = net.double()._forward_torch(x)
        w, b = (t.double() for t in Fp["stem"])
        y = F.max_pool2d(torch.relu(F.conv2d(x, w, b, stride=2, padding=3)), 3, 2, 1)
        outs, i = [], 0
        for blocks in (3, 4, 23, 3):
            for _ in range(blocks):
                s, c1, c2, c3, ds, caffe, off = Fp["blocks"][i]
                i += 1
                assert caffe
                t = torch.relu(F.conv2d(y, c1[0].double(), c1[1].double(), stride=s))
                if off is None:
                    t = torch.relu(F.conv2d(t, c2[0].double(), c2[1].double(), padding=1))
                else:
                    o = F.conv2d(t, off[0].double(), off[1].double(), padding=1)
                    assert o.shape[1] == 32 and float(o[:, 27:].abs().max()) == 0.0
                    col = deform_columns(t, o) * torch.sigmoid(o[:, 18:27]).unsqueeze(1)
                    C = t.shape[1]
                    t = torch.einsum("bckhw,ock->bohw", col, c2[0].double().view(C, C, 9)) + c2[1].double().view(1, -1, 1, 1)
                    t = torch.relu(t)
                ident = y if ds is None else F.conv2d(y, ds[0].double(), ds[1].double(), stride=s)
                y = torch.relu(F.conv2d(t, c3[0].double(), c3[1].double()) + ident)
            outs.append(y)
    for si, (a, b) in enumerate(zip(outs, want)):
        assert rel_err(a, b) <= 1e-5, f"folded ResNetDCN stage {si}: rel_max {rel_err(a, b):.2e}"


def test_cpu_forward_is_the_torch_forward():
    net = ResNetDCN(50, **R101).eval()
    x = torch.randn(1, 3, 64, 64, generator=torch.Generator().manual_seed(10))
    with torch.no_grad():
        assert torch.equal(net(x)[3], net._forward_torch(x)[3])


def test_name_stays_out_of_upstream_registries(monkeypatch):
    fake = registry.Registry("fake upstream")
    monkeypatch.setattr(registry.BACKBONES, "upstreams", [fake])
    monkeypatch.setattr(registry.BACKBONES.local, "_module_dict", dict(registry.BACKBONES.local._module_dict))
    path = os.path.join(os.path.dirname(registry.__file__), "image_encoder.py")
    spec = importlib.util.spec_from_file_location("occformer_b200._image_encoder_probe_dcn", path)
    mod = importlib.util.module_from_spec(spec)
    monkeypatch.setitem(sys.modules, spec.name, mod)
    spec.loader.exec_module(mod)
    assert fake.get("ResNetDCN") is None and registry.BACKBONES.get("ResNetDCN") is mod.ResNetDCN
