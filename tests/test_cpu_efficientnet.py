"""CustomEfficientNet's torch forward (efficientnet.py _forward_torch, the CPU path and the GPU tests' oracle) against the
reference class, its keys against the reference's at the SemanticKITTI config, and its construction rules."""
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

from util import GOLDEN, golden, rel_err
from occformer_b200 import BACKBONES, NECKS
from occformer_b200.efficientnet import CustomEfficientNet, adaptive_pad, make_divisible, scaled_layers


def test_forward_torch_equals_reference_golden():
    """tests/golden/efficientnet_small.npz: the reference class at 'b0', out_indices (2, 3) -- k3 / k5 depthwise convs at
    stride 1 and 2, SE, residuals, no-expand blocks, odd widths 24 / 40"""
    g = golden("efficientnet_small.npz")
    net = CustomEfficientNet("b0", out_indices=(2, 3)).eval()
    net.load_state_dict({k[2:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("w:")}, strict=True)
    with torch.no_grad():
        outs = net(torch.from_numpy(g["x"]))
    assert len(outs) == 2
    for i, o in enumerate(outs):
        want = torch.from_numpy(g[f"out{i}"])
        assert o.shape == want.shape
        assert rel_err(o, want) <= 1e-5, f"stage {i}: {rel_err(o, want):.2e}"


def test_kitti_config_keys_and_shapes():
    cfg = json.load(open(os.path.join(GOLDEN, "image_encoder_cfg_kitti.json")))
    net = BACKBONES.build(cfg["img_backbone"])
    assert isinstance(net, CustomEfficientNet)
    got = {k: list(v.shape) for k, v in net.state_dict().items()}
    assert got == cfg["img_backbone_state_shapes"]
    for k in ("layers.2.0.expand_conv.conv.weight", "layers.4.3.depthwise_conv.bn.running_var",
              "layers.5.0.se.conv1.conv.bias", "layers.6.bn.weight"):
        assert k in got
    assert [len(net.layers[i]) for i in range(1, 6)] == [4, 7, 7, 20, 17]
    neck = NECKS.build(cfg["img_neck"])
    assert neck.in_channels == [48, 80, 224, 640, 2560]


def test_unbuilt_layers_follow_out_indices():
    """the reference builds no layer after max(out_indices), and layers.6 only when it is an output"""
    assert len(CustomEfficientNet("b7", out_indices=(2, 3)).layers) == 4
    assert len(CustomEfficientNet("b7", out_indices=(5,)).layers) == 6
    assert len(CustomEfficientNet("b7", out_indices=(6,)).layers) == 7


def test_unsupported_kwargs():
    with pytest.raises(NotImplementedError, match="arch"):
        CustomEfficientNet("es")
    with pytest.raises(NotImplementedError, match="conv_cfg"):
        CustomEfficientNet("b0", conv_cfg=dict(type="Conv2d"))
    with pytest.raises(NotImplementedError, match="norm_cfg"):
        CustomEfficientNet("b0", norm_cfg=dict(type="GN", num_groups=8))
    with pytest.raises(NotImplementedError, match="act_cfg"):
        CustomEfficientNet("b0", act_cfg=dict(type="ReLU"))
    # the training-only kwargs are accepted
    CustomEfficientNet("b1", drop_path_rate=0.2, with_cp=True, frozen_stages=2, norm_eval=True, init_cfg=dict(type="x"))


@pytest.mark.parametrize("size", [7, 8, 31, 32, 33, 96, 97])
@pytest.mark.parametrize("k,s", [(3, 1), (3, 2), (5, 1), (5, 2), (1, 1)])
def test_adaptive_pad_is_mmcv_rule(size, k, s):
    """against the rule written out (mmcv Conv2dAdaptivePadding.forward) and the output size of F.conv2d after it"""
    out = math.ceil(size / s)
    pad = max((out - 1) * s + (k - 1) + 1 - size, 0)
    assert adaptive_pad(size, k, s) == (pad // 2, pad - pad // 2)
    x = torch.zeros(1, 1, size, size)
    before, after = adaptive_pad(size, k, s)
    y = F.conv2d(F.pad(x, [before, after, before, after]), torch.zeros(1, 1, k, k), stride=s)
    assert y.shape[-1] == out


def test_model_scaling_b7():
    """B7: the stage widths and block counts of the SemanticKITTI backbone"""
    layers = scaled_layers(2.0, 3.1)
    assert [len(l) for l in layers] == [1, 4, 7, 7, 20, 17, 1]
    assert [make_divisible(b[1], 8) for b in (layers[2][-1], layers[3][-1], layers[4][-1], layers[5][-1])] == \
        [48, 80, 224, 640]
    assert layers[-1][0][1] == 2560
