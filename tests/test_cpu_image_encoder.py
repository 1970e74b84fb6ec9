"""The image encoder's torch forwards (the oracle of its GPU tests) and its construction surface, on the CPU:
ResNet against torchvision's resnet50, SECONDFPN against the reference class (tests/golden/secondfpn_small.npz), the
folded parameters of the CUDA path applied with plain torch ops, the R50 config dicts through the local registries, and
the names kept out of the upstream registries."""
import importlib.util
import json
import os
import sys
import types

import pytest
import torch
import torch.nn.functional as F

from util import GOLDEN, assert_close, golden, rel_err
from occformer_b200 import BACKBONES, NECKS, registry, synth
from occformer_b200.image_encoder import SECONDFPN, ResNet

FPN_CASE = dict(in_channels=[32, 64, 64, 96], out_channels=[32, 32, 64, 32], upsample_strides=[0.25, 0.5, 1, 2])


def _resnet(seed=0, **kw):
    net = ResNet(depth=50, **kw).eval()
    net.load_state_dict(synth.make_resnet_state(seed, **kw), strict=True)
    return net


# ------------------------------------------------------------------ ResNet = torchvision resnet50 (same keys, same arithmetic)
@pytest.mark.parametrize("out_indices", [(0, 1, 2, 3), (3,), (1, 2)])
def test_resnet_equals_torchvision(out_indices):
    tv = pytest.importorskip("torchvision")
    sd = synth.make_resnet_state(1)
    ref = tv.models.resnet50()
    assert set(ref.state_dict()) - {"fc.weight", "fc.bias"} == set(sd)
    ref.load_state_dict(sd, strict=False)
    ref = ref.double().eval()
    net = ResNet(50, out_indices=out_indices).eval()
    net.load_state_dict(sd, strict=True)
    x = torch.randn(2, 3, 64, 96, generator=torch.Generator().manual_seed(2)).double()
    with torch.no_grad():
        got = net.double()(x)
        y = ref.maxpool(ref.relu(ref.bn1(ref.conv1(x))))
        want = []
        for i in range(4):
            y = getattr(ref, f"layer{i + 1}")(y)
            if i in out_indices:
                want.append(y)
    assert isinstance(got, tuple) and len(got) == len(want)
    for i, (a, b) in zip(out_indices, zip(got, want)):
        assert_close(a, b, 1e-6, f"ResNet stage {i} vs torchvision resnet50")


def test_resnet_keys_and_kwargs():
    cfg = json.load(open(os.path.join(GOLDEN, "image_encoder_cfg_nusc.json")))["img_backbone"]
    net = BACKBONES.build(cfg)  # pretrained / frozen_stages / norm_eval / requires_grad: accepted, nothing is read
    assert type(net) is ResNet and net.out_indices == (0, 1, 2, 3)
    keys = set(net.state_dict())
    assert {"conv1.weight", "bn1.running_var", "layer1.0.downsample.0.weight", "layer1.0.downsample.1.bias",
            "layer4.2.conv3.weight", "layer4.2.bn3.weight"} <= keys
    assert not any(k.startswith("fc.") for k in keys)
    assert net.bn1.eps == 1e-5 and net.layer2[0].conv2.stride == (2, 2) and net.layer2[0].conv1.stride == (1, 1)
    ResNet(50, frozen_stages=2, norm_eval=True, with_cp=True, zero_init_residual=False, pretrained="/nonexistent.pth",
           init_cfg=dict(type="Pretrained", checkpoint="/nonexistent.pth"))


@pytest.mark.parametrize("kw,name", [(dict(dcn=dict(type="DCNv2")), "dcn"),
                                     (dict(stage_with_dcn=(False, True, True, True)), "stage_with_dcn"),
                                     (dict(deep_stem=True), "deep_stem"), (dict(avg_down=True), "avg_down"),
                                     (dict(plugins=[dict(cfg=dict(type="ContextBlock"))]), "plugins"),
                                     (dict(depth=101), "depth"), (dict(style="caffe"), "style")])
def test_resnet_unsupported_options_raise(kw, name):
    kw = {"depth": 50, **kw}
    with pytest.raises(NotImplementedError, match=name):
        ResNet(**kw)


# ------------------------------------------------------------------ SECONDFPN = the reference class
def test_secondfpn_matches_reference_golden():
    z = golden("secondfpn_small.npz")
    net = SECONDFPN(**FPN_CASE).eval()
    net.load_state_dict({k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w:")}, strict=True)
    levels = [torch.from_numpy(z[f"level{i}"]) for i in range(4)]
    with torch.no_grad():
        out = net(levels)
    assert isinstance(out, list) and len(out) == 1
    assert_close(out[0], torch.from_numpy(z["out"]), 1e-6, "SECONDFPN vs reference class")


def test_secondfpn_defaults():
    cfg = json.load(open(os.path.join(GOLDEN, "image_encoder_cfg_nusc.json")))["img_neck"]
    net = NECKS.build(cfg)
    assert type(net) is SECONDFPN
    for blk, s in zip(net.deblocks, (4, 2, 1, 2)):
        assert blk[0].bias is None and blk[1].eps == 1e-3 and blk[0].stride == (s, s)
    assert [type(b[0]).__name__ for b in net.deblocks] == ["Conv2d", "Conv2d", "ConvTranspose2d", "ConvTranspose2d"]
    assert tuple(net.deblocks[3][0].weight.shape) == (2048, 128, 2, 2)


# ------------------------------------------------------------------ folded parameters (the CUDA path's source)
def test_resnet_folded_parameters_reproduce_forward():
    net = _resnet(3)
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(4))
    Fp = net._folded()
    with torch.no_grad():
        want = net.double()._forward_torch(x.double())
        w, b = (t.double() for t in Fp["stem"])
        y = F.max_pool2d(torch.relu(F.conv2d(x.double(), w, b, stride=2, padding=3)), 3, 2, 1)
        outs, i = [], 0
        for si, blocks in enumerate((3, 4, 6, 3)):
            for _ in range(blocks):
                s, c1, c2, c3, ds = Fp["blocks"][i]
                i += 1
                t = torch.relu(F.conv2d(y, c1[0].double(), c1[1].double()))
                t = torch.relu(F.conv2d(t, c2[0].double(), c2[1].double(), stride=s, padding=1))
                ident = y if ds is None else F.conv2d(y, ds[0].double(), ds[1].double(), stride=s)
                y = torch.relu(F.conv2d(t, c3[0].double(), c3[1].double()) + ident)
            outs.append(y)
    # each folded weight is rounded to fp32 (relative 6e-8); through up to 53 stacked convs that adds up to a few 1e-6
    # of the tensor's maximum (3.4e-6 at layer3 here): the bound is 1e-5, two orders below the 1e-3 parity gate
    for si, (a, b) in enumerate(zip(outs, want)):
        assert rel_err(a, b) <= 1e-5, f"folded ResNet stage {si}: rel_max {rel_err(a, b):.2e}"


def test_secondfpn_folded_parameters_reproduce_forward():
    cases = [FPN_CASE, dict(in_channels=[64, 32], out_channels=[32, 64], upsample_strides=[1, 4]),
             dict(in_channels=[32], out_channels=[64], upsample_strides=[1], use_conv_for_no_stride=True)]
    for c in cases:
        net = SECONDFPN(**c).eval()
        net.load_state_dict(synth.make_secondfpn_state(seed=5, **c), strict=True)
        g = torch.Generator().manual_seed(6)
        levels = [torch.randn(2, ch, int(4 / s), int(8 / s), generator=g) for ch, s in
                  zip(c["in_channels"], c["upsample_strides"])]
        with torch.no_grad():
            want = net.double()._forward_torch([t.double() for t in levels])[0]
        ups = []
        for t, (kind, f, w, b) in zip(levels, net._folded()):
            op = F.conv2d if kind == "conv" else F.conv_transpose2d
            ups.append(torch.relu(op(t.double(), w.double(), b.double(), stride=f)))
        assert_close(torch.cat(ups, 1), want, 1e-6, f"folded SECONDFPN {c}")


def test_cpu_forward_is_the_torch_forward():
    net = _resnet(0, out_indices=(1,))
    x = torch.randn(1, 3, 32, 64, generator=torch.Generator().manual_seed(7))
    with torch.no_grad():
        a, b = net(x), net._forward_torch(x)
    assert torch.equal(a[0], b[0])


def test_prepare_cache_dropped_by_load_state_dict():
    net = SECONDFPN(**FPN_CASE).eval()
    net.load_state_dict(synth.make_secondfpn_state(seed=8, **FPN_CASE))
    net._prep = object()
    net.load_state_dict(synth.make_secondfpn_state(seed=9, **FPN_CASE))
    assert net._prep is None
    net._prep = object()
    net.double()
    assert net._prep is None


# ------------------------------------------------------------------ registries: local only
def test_image_encoder_names_stay_out_of_upstream_registries(monkeypatch):
    """ResNet and SECONDFPN are general mmdet / mmdet3d names: re-running image_encoder.py's registrations with an
    upstream registry present must leave that registry alone, while a module registered the default way reaches it."""
    fake = registry.Registry("fake upstream")
    for mirror in (registry.BACKBONES, registry.NECKS):
        monkeypatch.setattr(mirror, "upstreams", [fake])
        monkeypatch.setattr(mirror.local, "_module_dict", dict(mirror.local._module_dict))
    path = os.path.join(os.path.dirname(registry.__file__), "image_encoder.py")
    spec = importlib.util.spec_from_file_location("occformer_b200._image_encoder_probe", path)
    mod = importlib.util.module_from_spec(spec)
    monkeypatch.setitem(sys.modules, spec.name, mod)
    spec.loader.exec_module(mod)
    assert fake.get("ResNet") is None and fake.get("SECONDFPN") is None
    assert registry.BACKBONES.get("ResNet") is mod.ResNet and registry.NECKS.get("SECONDFPN") is mod.SECONDFPN
    other = types.new_class("SomeBackbone", (torch.nn.Module,))
    registry.BACKBONES.register_module(module=other)
    assert fake.get("SomeBackbone") is other
