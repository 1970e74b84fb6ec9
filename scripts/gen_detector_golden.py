"""TEST INFRASTRUCTURE ONLY -- the whole-model fixtures, read from the reference tree (needs it on disk):

    python scripts/gen_detector_golden.py

tests/golden/detector_cfg_<name>.json   the ``model`` dict of an unmodified reference config, verbatim (``type``,
                                        ``img_backbone``, ``img_neck``, ``train_cfg``, ``test_cfg`` and the rest), the
                                        input of DETECTORS.build

    nusc_r50        occformer_nusc_r50_256x704.py
    nusc_r101       occformer_nusc_r101_896x1600.py (occformer_nusc_r101_896x1600_trainval.py has the same ``model``)
    nusc_panoptic   occformer_nusc_panoptic_r50_256x704.py
    kitti           occformer_kitti.py

Written as scripts/gen_resnet_dcn_golden.py writes the R101 fixtures; the existing fixtures are not touched.
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import shim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
CONFIGS = {"nusc_r50": "projects/configs/occformer_nusc/occformer_nusc_r50_256x704.py",
           "nusc_r101": "projects/configs/occformer_nusc/occformer_nusc_r101_896x1600.py",
           "nusc_panoptic": "projects/configs/occformer_nusc/occformer_nusc_panoptic_r50_256x704.py",
           "kitti": "projects/configs/occformer_kitti/occformer_kitti.py"}
SAME_MODEL = {"nusc_r101": "projects/configs/occformer_nusc/occformer_nusc_r101_896x1600_trainval.py"}


def model_dict(rel):
    """the ``model`` of a config file (pure-python assignments; ``_base_`` inheritance only adds dataset / runtime keys)"""
    ns = {}
    exec(compile(open(os.path.join(shim.REFERENCE_ROOT, rel)).read(), rel, "exec"), ns)
    return ns["model"]


def main():
    assert shim.reference_available(), "needs the reference tree"
    for name, rel in CONFIGS.items():
        m = model_dict(rel)
        if name in SAME_MODEL:
            assert model_dict(SAME_MODEL[name]) == m, f"{SAME_MODEL[name]} has another model dict than {rel}"
        with open(os.path.join(OUT, f"detector_cfg_{name}.json"), "w") as f:
            json.dump(m, f, indent=1, default=lambda o: list(o))
        print(f"detector_cfg_{name}", list(m))


if __name__ == "__main__":
    main()
