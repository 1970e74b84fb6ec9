"""TEST INFRASTRUCTURE ONLY -- the nuScenes R101 fixtures, read from the reference tree (needs it on disk):

    python scripts/gen_resnet_dcn_golden.py

tests/golden/image_encoder_cfg_nusc_r101.json   the img_backbone / img_neck dicts of the unmodified
                                                occformer_nusc_r101_896x1600.py config
tests/golden/model_cfg_nusc_r101.json           its img_view_transformer / img_bev_encoder_backbone /
                                                img_bev_encoder_neck / pts_bbox_head dicts (the view transformer at 896x1600)

Both are written as oracle/gen_image_encoder.py and oracle/gen_golden.py write the R50 ones; the existing fixtures are
not touched.  mmdet's ResNet and mmcv's ModulatedDeformConv2dPack are not part of the reference tree:
tests/test_cpu_resnet_dcn.py pins image_encoder.ResNetDCN to torchvision's resnet101 and the DCNv2 layer to its
sampling identities instead.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
CONFIG = "projects/configs/occformer_nusc/occformer_nusc_r101_896x1600.py"


def main():
    assert shim.reference_available(), "needs the reference tree"
    ns = {}
    exec(compile(open(os.path.join(shim.REFERENCE_ROOT, CONFIG)).read(), CONFIG, "exec"), ns)
    m = ns["model"]
    for name, keys in (("image_encoder_cfg_nusc_r101", ("img_backbone", "img_neck")),
                       ("model_cfg_nusc_r101", ("img_view_transformer", "img_bev_encoder_backbone",
                                                "img_bev_encoder_neck", "pts_bbox_head"))):
        keep = {k: m[k] for k in keys}
        with open(os.path.join(OUT, name + ".json"), "w") as f:
            json.dump(keep, f, indent=1, default=lambda o: list(o))
        print(name, list(keep))


if __name__ == "__main__":
    main()
