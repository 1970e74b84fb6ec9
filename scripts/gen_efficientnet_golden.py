"""TEST INFRASTRUCTURE ONLY -- the EfficientNet fixtures, generated from the reference tree (needs it on disk):

    python scripts/gen_efficientnet_golden.py

tests/golden/efficientnet_small.npz      the reference CustomEfficientNet (P/occformer/backbones/efficientnet.py, imported
                                         verbatim under oracle/shim.py plus the mmcv / mmdet pieces below) at arch 'b0',
                                         out_indices (2, 3), on seeded (2, 3, 64, 96) images: the images, the state_dict
                                         and the outputs
tests/golden/image_encoder_cfg_kitti.json   the img_backbone / img_neck dicts of the unmodified SemanticKITTI config, and
                                         the key -> shape list of the reference CustomEfficientNet built from that dict

The mmcv 1.4.0 / mmdet 2.14.0 pieces the reference file imports are restated here from their published sources and put
on the shim's modules at run time: Conv2dAdaptivePadding (mmcv/cnn/bricks/conv2d_adaptive_padding.py), Swish
(mmcv/cnn/bricks/swish.py), DropPath (identity in eval), make_divisible and SELayer (mmdet/models/utils).
"""
import importlib.util
import json
import math
import os
import sys

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from occformer_b200 import synth  # noqa: E402
from oracle import shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SMALL = dict(arch="b0", out_indices=(2, 3), shape=(2, 3, 64, 96), wseed=51, xseed=53)


class Conv2dAdaptivePadding(nn.Conv2d):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True):
        super().__init__(in_channels, out_channels, kernel_size, stride, 0, dilation, groups, bias)

    def forward(self, x):
        img_h, img_w = x.size()[-2:]
        kernel_h, kernel_w = self.weight.size()[-2:]
        stride_h, stride_w = self.stride
        output_h = math.ceil(img_h / stride_h)
        output_w = math.ceil(img_w / stride_w)
        pad_h = max((output_h - 1) * self.stride[0] + (kernel_h - 1) * self.dilation[0] + 1 - img_h, 0)
        pad_w = max((output_w - 1) * self.stride[1] + (kernel_w - 1) * self.dilation[1] + 1 - img_w, 0)
        if pad_h > 0 or pad_w > 0:
            x = F.pad(x, [pad_w // 2, pad_w - pad_w // 2, pad_h // 2, pad_h - pad_h // 2])
        return F.conv2d(x, self.weight, self.bias, self.stride, self.padding, self.dilation, self.groups)


class Swish(nn.Module):
    def __init__(self, inplace=False):
        super().__init__()

    def forward(self, x):
        return x * torch.sigmoid(x)


class DropPath(nn.Module):
    def __init__(self, drop_prob=0.1):
        super().__init__()

    def forward(self, x):
        return x


def make_divisible(value, divisor, min_value=None, min_ratio=0.9):
    if min_value is None:
        min_value = divisor
    new_value = max(min_value, int(value + divisor / 2) // divisor * divisor)
    if new_value < min_ratio * value:
        new_value += divisor
    return new_value


class SELayer(shim.BaseModule):
    def __init__(self, channels, ratio=16, conv_cfg=None, act_cfg=(dict(type="ReLU"), dict(type="Sigmoid")),
                 init_cfg=None):
        super().__init__(init_cfg)
        self.global_avgpool = nn.AdaptiveAvgPool2d(1)
        self.conv1 = shim.ConvModule(channels, int(channels / ratio), 1, stride=1, conv_cfg=conv_cfg, act_cfg=act_cfg[0])
        self.conv2 = shim.ConvModule(int(channels / ratio), channels, 1, stride=1, conv_cfg=conv_cfg, act_cfg=act_cfg[1])

    def forward(self, x):
        out = self.global_avgpool(x)
        out = self.conv1(out)
        out = self.conv2(out)
        return x * out


def reference_efficientnet():
    """the reference CustomEfficientNet class, its file imported verbatim under the extended shim"""
    shim.install()
    shim.CONV_LAYERS["Conv2dAdaptivePadding"] = Conv2dAdaptivePadding
    shim.ACT_LAYERS["Swish"] = Swish
    shim.ACT_LAYERS["Sigmoid"] = lambda inplace=None: nn.Sigmoid()  # mmcv's Sigmoid takes no inplace
    sys.modules["mmcv.cnn.bricks"].ConvModule = shim.ConvModule
    sys.modules["mmcv.cnn.bricks"].DropPath = DropPath
    sys.modules["mmdet.models.utils"].SELayer = SELayer
    sys.modules["mmdet.models.utils"].make_divisible = make_divisible
    path = os.path.join(shim.PLUGIN, "occformer", "backbones", "efficientnet.py")
    spec = importlib.util.spec_from_file_location("reference_efficientnet", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.CustomEfficientNet


def gen_small(ref_cls):
    c = SMALL
    ref = ref_cls(arch=c["arch"], out_indices=c["out_indices"])
    ref.eval()  # the reference train() returns None
    sd = synth.make_efficientnet_state(c["arch"], seed=c["wseed"], out_indices=c["out_indices"])
    ref.load_state_dict(sd, strict=True)
    x = torch.randn(*c["shape"], generator=torch.Generator().manual_seed(c["xseed"]))
    with torch.no_grad():
        outs = ref(x.clone())
    np.savez_compressed(os.path.join(OUT, "efficientnet_small.npz"), x=x.numpy(),
                        **{f"out{i}": o.numpy() for i, o in enumerate(outs)}, **{"w:" + k: v.numpy() for k, v in sd.items()})
    print("efficientnet_small", [tuple(o.shape) for o in outs], len(sd), "keys")


def gen_cfg(ref_cls):
    rel = "projects/configs/occformer_kitti/occformer_kitti.py"
    ns = {}
    exec(compile(open(os.path.join(shim.REFERENCE_ROOT, rel)).read(), rel, "exec"), ns)
    keep = {k: ns["model"][k] for k in ("img_backbone", "img_neck")}
    args = {k: v for k, v in keep["img_backbone"].items() if k != "type"}
    ref = ref_cls(**args)
    keep["img_backbone_state_shapes"] = {k: list(v.shape) for k, v in ref.state_dict().items()}
    cfg = json.loads(json.dumps({k: keep[k] for k in ("img_backbone", "img_neck")}, default=list))
    text = json.dumps(cfg, indent=1)[:-2] + ',\n "img_backbone_state_shapes": {\n' + ",\n".join(
        f"  {json.dumps(k)}: {json.dumps(v)}" for k, v in keep["img_backbone_state_shapes"].items()) + "\n }\n}\n"
    with open(os.path.join(OUT, "image_encoder_cfg_kitti.json"), "w") as f:  # one key per line
        f.write(text)
    print("image_encoder_cfg_kitti", {k: keep[k] for k in ("img_backbone", "img_neck")},
          len(keep["img_backbone_state_shapes"]), "keys")


def main():
    assert shim.reference_available(), "needs the reference tree"
    cls = reference_efficientnet()
    gen_small(cls)
    gen_cfg(cls)


if __name__ == "__main__":
    main()
