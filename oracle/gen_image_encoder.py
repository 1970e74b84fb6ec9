"""TEST INFRASTRUCTURE ONLY -- the image encoder's fixtures, generated from the reference tree (needs it on disk):

    python -m oracle.gen_image_encoder

tests/golden/secondfpn_small.npz   mmdet3d's SECONDFPN class (mmdetection3d/mmdet3d/models/necks/second_fpn.py, imported
                                   verbatim under oracle/shim.py) on small seeded levels: the levels, the state_dict and
                                   the reference output
tests/golden/image_encoder_cfg_nusc.json   the img_backbone / img_neck dicts of the unmodified nuScenes R50 config

mmdet's ResNet is not part of the reference tree; tests/test_cpu_image_encoder.py pins image_encoder.ResNet to
torchvision's resnet50 instead (same arithmetic, same keys).
"""
import importlib.util
import json
import os
import sys

import numpy as np
import torch
import torch.nn as nn

from occformer_b200 import synth

from . import shim

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
SECONDFPN_CASE = dict(in_channels=[32, 64, 64, 96], out_channels=[32, 32, 64, 32], upsample_strides=[0.25, 0.5, 1, 2],
                      n=2, out_hw=(4, 6), wseed=41, xseed=43)


def build_upsample_layer(cfg, *args, **kwargs):
    """mmcv.cnn.build_upsample_layer for the 'deconv' type SECONDFPN uses (mmcv/cnn/bricks/upsample.py): the cfg's other
    keys are nn.ConvTranspose2d kwargs"""
    cfg_ = dict(cfg)
    kind = cfg_.pop("type")
    if kind != "deconv":
        raise NotImplementedError(kind)
    return nn.ConvTranspose2d(*args, **kwargs, **cfg_)


def reference_secondfpn():
    """the reference SECONDFPN class, its file imported verbatim (the shim's mmcv.cnn extended by build_upsample_layer)"""
    shim.install()
    sys.modules["mmcv.cnn"].build_upsample_layer = build_upsample_layer
    path = os.path.join(shim.REFERENCE_ROOT, "mmdetection3d", "mmdet3d", "models", "necks", "second_fpn.py")
    spec = importlib.util.spec_from_file_location("reference_second_fpn", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.SECONDFPN


def gen_secondfpn():
    c = SECONDFPN_CASE
    ref = reference_secondfpn()(in_channels=c["in_channels"], out_channels=c["out_channels"],
                                upsample_strides=c["upsample_strides"]).eval()
    sd = synth.make_secondfpn_state(c["in_channels"], c["out_channels"], c["upsample_strides"], seed=c["wseed"])
    ref.load_state_dict(sd, strict=True)
    g = torch.Generator().manual_seed(c["xseed"])
    H, W = c["out_hw"]
    levels = [torch.randn(c["n"], ch, int(H / s), int(W / s), generator=g).abs()
              for ch, s in zip(c["in_channels"], c["upsample_strides"])]
    with torch.no_grad():
        out = ref([t.clone() for t in levels])
    assert len(out) == 1
    np.savez(os.path.join(OUT, "secondfpn_small.npz"), out=out[0].numpy(),
             **{f"level{i}": t.numpy() for i, t in enumerate(levels)}, **{"w:" + k: v.numpy() for k, v in sd.items()})
    print("secondfpn_small", tuple(out[0].shape), len(sd), "keys")


def gen_cfg():
    rel = "projects/configs/occformer_nusc/occformer_nusc_r50_256x704.py"
    ns = {}
    exec(compile(open(os.path.join(shim.REFERENCE_ROOT, rel)).read(), rel, "exec"), ns)
    keep = {k: ns["model"][k] for k in ("img_backbone", "img_neck")}
    with open(os.path.join(OUT, "image_encoder_cfg_nusc.json"), "w") as f:
        json.dump(keep, f, indent=1, default=lambda o: list(o))
    print("image_encoder_cfg_nusc", keep)


def main():
    assert shim.reference_available(), "needs the reference tree"
    os.makedirs(OUT, exist_ok=True)
    gen_secondfpn()
    gen_cfg()


if __name__ == "__main__":
    main()
