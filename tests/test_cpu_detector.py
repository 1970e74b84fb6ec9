"""The OccupancyFormer detector on the host: the unmodified configs' ``model`` dicts (tests/golden/detector_cfg_*.json,
written verbatim by scripts/gen_detector_golden.py) build through DETECTORS, the submodules are the ones the configs name,
the state_dict is the reference checkpoint's key set in its order, and what the detector does not build is refused."""
import json
import os

import numpy as np
import pytest
import torch

import occformer_b200
from occformer_b200 import DETECTORS, BACKBONES, HEADS, NECKS, OccupancyFormer, synth
from occformer_b200.efficientnet import CustomEfficientNet
from occformer_b200.head import Mask2FormerNuscOccHead, Mask2FormerNuscPanopticOccHead, Mask2FormerOccHead
from occformer_b200.image_encoder import SECONDFPN, ModulatedDeformConv2dPack, ResNet, ResNetDCN
from util import GOLDEN

NAMES = ["nusc_r50", "nusc_r101", "nusc_panoptic", "kitti"]
ORDER = ["pts_bbox_head", "img_backbone", "img_neck", "img_view_transformer", "img_bev_encoder_backbone",
         "img_bev_encoder_neck"]
REGISTRY = {"pts_bbox_head": HEADS, "img_backbone": BACKBONES, "img_neck": NECKS, "img_view_transformer": NECKS,
            "img_bev_encoder_backbone": BACKBONES, "img_bev_encoder_neck": NECKS}


def _cfg(name):
    return json.load(open(os.path.join(GOLDEN, f"detector_cfg_{name}.json")))


_built = {}


def _model(name):
    if name not in _built:
        _built[name] = DETECTORS.build(_cfg(name)).eval()
    return _built[name]


@pytest.mark.parametrize("name", NAMES)
def test_config_builds_unedited(name):
    cfg = _cfg(name)
    assert cfg["type"] == "OccupancyFormer" and DETECTORS.get("OccupancyFormer") is OccupancyFormer
    m = _model(name)
    assert [n for n, _ in m.named_children()] == ORDER
    want = {"nusc_r50": (ResNet, Mask2FormerNuscOccHead), "nusc_r101": (ResNetDCN, Mask2FormerNuscOccHead),
            "nusc_panoptic": (ResNet, Mask2FormerNuscPanopticOccHead), "kitti": (CustomEfficientNet, Mask2FormerOccHead)}
    assert type(m.img_backbone) is want[name][0] and type(m.pts_bbox_head) is want[name][1]
    assert type(m.img_neck) is SECONDFPN
    if name == "nusc_r101":
        for i, stage in enumerate([m.img_backbone.layer1, m.img_backbone.layer2, m.img_backbone.layer3,
                                   m.img_backbone.layer4]):
            dcn = [isinstance(b.conv2, ModulatedDeformConv2dPack) for b in stage]
            assert all(dcn) if i >= 2 else not any(dcn), f"layer{i + 1}: DCN {dcn}"
    if name == "kitti":
        assert len(m.img_neck.deblocks) == 5
    # MVXTwoStageDetector hands the head train_cfg['pts'] / test_cfg['pts']
    assert m.pts_bbox_head.test_cfg == cfg["test_cfg"]["pts"] and m.pts_bbox_head.train_cfg == cfg["train_cfg"]["pts"]
    assert m.with_img_neck and m.with_img_backbone and m.with_pts_bbox


@pytest.mark.parametrize("name", NAMES)
def test_state_dict_is_the_prefixed_union_of_the_submodules(name):
    """keys and shapes in registration order = each submodule built alone from its section (the reference contracts the
    module tests pin), prefixed; the detector adds no parameter or buffer of its own"""
    cfg, m = _cfg(name), _model(name)
    want = []
    for sub in ORDER:
        section = dict(cfg[sub])
        if sub == "pts_bbox_head":
            section.update(train_cfg=cfg["train_cfg"]["pts"], test_cfg=cfg["test_cfg"]["pts"])
        if section["type"] == "ResNet":
            section["type"] = ResNetDCN if section.get("dcn") else ResNet
        alone = REGISTRY[sub].build(section)
        want += [(f"{sub}.{k}", tuple(v.shape)) for k, v in alone.state_dict().items()]
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == want
    assert not list(m.named_parameters(recurse=False)) and not list(m.named_buffers(recurse=False))
    if name != "kitti":  # the reference DepthNet's keys of the nuScenes configs
        dn = json.load(open(os.path.join(GOLDEN, "depthnet_keys_nusc.json")))
        got = {k[len("img_view_transformer.depth_net."):]: list(v.shape) for k, v in m.state_dict().items()
               if k.startswith("img_view_transformer.depth_net.")}
        assert got == dn


@pytest.mark.parametrize("name", ["nusc_r50", "kitti"])
def test_strict_load(name):
    cfg = _cfg(name)
    m = DETECTORS.build(cfg)
    sd = synth.make_detector_state(cfg, seed=1)
    assert list(sd) == list(m.state_dict())
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.pts_bbox_head.query_feat.weight, sd["pts_bbox_head.query_feat.weight"])
    missing = dict(sd)
    missing.pop("img_neck.deblocks.0.1.weight")
    with pytest.raises(RuntimeError, match="Missing key"):
        m.load_state_dict(missing, strict=True)
    with pytest.raises(RuntimeError, match="Unexpected key"):
        m.load_state_dict(dict(sd, **{"img_backbone.fc.weight": torch.zeros(1)}), strict=True)


@pytest.mark.parametrize("kwarg", ["pts_voxel_layer", "pts_voxel_encoder", "pts_middle_encoder", "pts_backbone",
                                   "pts_fusion_layer", "pts_neck", "img_rpn_head", "img_roi_head"])
def test_lidar_branches_are_refused(kwarg):
    cfg = dict(_cfg("nusc_r50"), **{kwarg: dict(type="Anything")})
    with pytest.raises(NotImplementedError, match=kwarg):
        DETECTORS.build(cfg)


def test_training_and_unknown_types_are_refused():
    m = _model("nusc_r50")
    with pytest.raises(NotImplementedError, match="inference-only"):
        m(return_loss=True, img_metas=[{}], img_inputs=[])
    with pytest.raises(NotImplementedError, match="inference-only"):
        m.forward_train(img_metas=[{}], img_inputs=[])
    cfg = _cfg("nusc_r50")
    with pytest.raises(KeyError, match="NoSuchBackbone"):
        DETECTORS.build(dict(cfg, img_backbone=dict(cfg["img_backbone"], type="NoSuchBackbone")))
    with pytest.raises(ValueError, match="pretrained"):
        DETECTORS.build(dict(cfg, pretrained="ckpts/x.pth"))
    with pytest.raises(TypeError):
        DETECTORS.build(dict(cfg, no_such_kwarg=1))


def test_type_given_as_a_class_and_local_only_names():
    cfg = _cfg("nusc_r50")
    m = DETECTORS.build(dict(cfg, type=OccupancyFormer, img_backbone=dict(cfg["img_backbone"], type=ResNetDCN)))
    assert type(m.img_backbone) is ResNetDCN
    # outside a detector the general mmdet names keep their local-only registration
    assert BACKBONES.get("ResNet") is ResNet and NECKS.get("SECONDFPN") is SECONDFPN
    assert occformer_b200.DETECTORS.get("OccupancyFormer") is OccupancyFormer


def test_evaluation_semantic_is_fast_hist_crop():
    """simple_evaluation_semantic from labels (any of 0..16) and from point scores = the reference's
    fast_hist_crop(pred, gt[:, 3], np.arange(16)), restated in numpy, as a numpy int64 array"""
    def fast_hist_crop(output, target, unique_label):
        n = np.max(unique_label) + 2
        k = (target >= 0) & (target < n)
        hist = np.bincount(n * target[k].astype(int) + output[k], minlength=n ** 2)[:n ** 2].reshape(n, n)
        return hist[unique_label + 1, :][:, unique_label + 1]

    g = torch.Generator().manual_seed(0)
    scores = torch.randn(500, 17, generator=g)
    pts = torch.cat([torch.randn(500, 3, generator=g), torch.randint(0, 17, (500, 1), generator=g).float()], dim=1)
    pred = torch.argmax(scores[:, 1:], dim=1) + 1
    want = fast_hist_crop(pred.numpy(), pts[:, 3].numpy().astype(int), np.arange(16))
    m = _model("nusc_r50")
    for p in (pred, scores):
        got = m.simple_evaluation_semantic(p, pts, None)
        assert type(got) is np.ndarray and got.dtype == np.int64 and got.shape == (16, 16)
        assert np.array_equal(got, want)
    # labels as the reference's caller may pass them, 0 (cropped away by fast_hist_crop) included
    labels = torch.randint(0, 17, (500,), generator=g)
    assert int((labels == 0).sum()) > 0
    got = m.simple_evaluation_semantic(labels, pts, None)
    assert got.dtype == np.int64 and np.array_equal(got, fast_hist_crop(labels.numpy(), pts[:, 3].numpy().astype(int),
                                                                        np.arange(16)))
    vol = torch.randn(2, 17, 4, 4, 2, generator=g)
    assert torch.equal(m.post_process_semantic([vol * 0, vol]), vol.argmax(1))
