"""The whole OccFormer model: camera images -> image encoder -> view transformer -> occupancy encoder -> pixel decoder ->
head, behind the reference's detector surface.

    DETECTORS 'OccupancyFormer'   P/occformer/detectors/occupancyformer.py:14-254
    (the parts of its bases that inference uses)   P/occformer/detectors/bevdepth.py:15-60,
                                  mmdetection3d/mmdet3d/models/detectors/mvx_two_stage.py:23-105, base.py:47-61

The constructor takes a reference config's ``model`` dict as it stands (``type`` popped by the registry) and builds every
submodule through this package's registries, in the reference's registration order, so ``state_dict()`` lists the keys
of a checkpoint the reference saves and ``load_state_dict(torch.load('occformer_*.pth')['state_dict'])`` loads it with
``strict=True``.  The detector owns no parameters or buffers of its own; the arithmetic is the submodules'.

Inside the detector the general mmdet names of the image encoder resolve to this package's classes: ``type='ResNet'``
builds ``ResNetDCN`` when the dict has a ``dcn`` (the R101 config) and ``ResNet`` otherwise, ``type='SECONDFPN'``
builds ``SECONDFPN``.  A ``type`` given as a class is used as is.

Inference only: ``forward(return_loss=True)`` and ``forward_train`` raise NotImplementedError, and the submodules refuse
to run in training mode.  The forward has no host synchronisation (it can be captured in a CUDA graph) except
``evaluation_semantic``, which is handed back as a numpy array when LiDAR points are given, as the reference's test loop
expects (occformer/apis/test.py:156,203).
"""
import numpy as np
import torch
import torch.nn as nn

from . import dist_eval, image_prep, targets
from .head import Mask2FormerNuscOccHead, Mask2FormerNuscPanopticOccHead, Mask2FormerOccHead
from .image_encoder import SECONDFPN, ResNet, ResNetDCN
from .registry import BACKBONES, DETECTORS, HEADS, NECKS

# fast_hist_crop(pred, gt, np.arange(16)) (occupancyformer.py:246-254): the 16 nuScenes lidarseg classes 1..16
LIDARSEG_CLASSES = 17


def _build(registry, cfg, default_args=None):
    cfg = dict(cfg)
    if cfg.get("type") == "ResNet":
        cfg["type"] = ResNetDCN if cfg.get("dcn") else ResNet
    elif cfg.get("type") == "SECONDFPN":
        cfg["type"] = SECONDFPN
    return registry.build(cfg, default_args)


def _voxel_files(img_metas):
    """every sample's metas carry the SemanticKITTI voxel files of pipelines.LoadSemKittiVoxelFiles"""
    return bool(img_metas) and all("semkitti_voxels" in m for m in img_metas)


def _pts(cfg):
    if not cfg:
        return None
    return cfg.get("pts") if isinstance(cfg, dict) else getattr(cfg, "pts", None)


@DETECTORS.register_module()
class OccupancyFormer(nn.Module):
    def __init__(self, img_view_transformer, img_bev_encoder_backbone, img_bev_encoder_neck, pts_voxel_layer=None,
                 pts_voxel_encoder=None, pts_middle_encoder=None, pts_fusion_layer=None, img_backbone=None,
                 pts_backbone=None, img_neck=None, pts_neck=None, pts_bbox_head=None, img_roi_head=None,
                 img_rpn_head=None, train_cfg=None, test_cfg=None, pretrained=None, init_cfg=None,
                 occ_targets_from_points=False):
        """occ_targets_from_points (not a reference kwarg): simple_test called without gt_occ builds 'target_voxels' from
        points_occ on the GPU (occupancy_targets), for a pipeline whose loader skips the host-side ground truth
        (occformer_b200.pipelines, INTEGRATION.md)."""
        super().__init__()
        self.occ_targets_from_points = bool(occ_targets_from_points)
        lidar = dict(pts_voxel_layer=pts_voxel_layer, pts_voxel_encoder=pts_voxel_encoder,
                     pts_middle_encoder=pts_middle_encoder, pts_backbone=pts_backbone, pts_fusion_layer=pts_fusion_layer,
                     pts_neck=pts_neck, img_rpn_head=img_rpn_head, img_roi_head=img_roi_head)
        for kwarg, value in lidar.items():
            if value is not None:
                raise NotImplementedError(f"occformer_b200.OccupancyFormer: {kwarg} is not built (no OccFormer config "
                                          "sets it; the detector is camera-only)")
        if pretrained is not None and not isinstance(pretrained, dict):
            raise ValueError(f"pretrained should be a dict, got {type(pretrained)}")
        # MVXTwoStageDetector.__init__ (mvx_two_stage.py:57-67), then BEVDet.__init__ (bevdepth.py:19-34)
        if pts_bbox_head:
            self.pts_bbox_head = _build(HEADS, dict(pts_bbox_head, train_cfg=_pts(train_cfg), test_cfg=_pts(test_cfg)))
        if img_backbone:
            self.img_backbone = _build(BACKBONES, img_backbone)
        if img_neck is not None:
            self.img_neck = _build(NECKS, img_neck)
        self.train_cfg, self.test_cfg = train_cfg, test_cfg
        self.pretrained, self.init_cfg = pretrained, init_cfg
        self.img_view_transformer = _build(NECKS, img_view_transformer) if img_view_transformer is not None else None
        self.img_bev_encoder_backbone = (_build(BACKBONES, img_bev_encoder_backbone)
                                         if img_bev_encoder_backbone is not None else nn.Identity())
        self.img_bev_encoder_neck = (_build(NECKS, img_bev_encoder_neck)
                                     if img_bev_encoder_neck is not None else nn.Identity())

    @property
    def with_img_neck(self):
        return getattr(self, "img_neck", None) is not None

    @property
    def with_img_backbone(self):
        return getattr(self, "img_backbone", None) is not None

    @property
    def with_pts_bbox(self):
        return getattr(self, "pts_bbox_head", None) is not None

    # ------------------------------------------------------------------ occupancyformer.py:22-97
    def image_encoder(self, img):
        """(B, N, 3, H, W) normalised images -> (B, N, C, h, w) features"""
        B, N, C, imH, imW = img.shape
        x = self.img_backbone(img.view(B * N, C, imH, imW))
        if self.with_img_neck:
            x = self.img_neck(x)
            if type(x) in [list, tuple]:
                x = x[0]
        _, output_dim, output_H, output_W = x.shape
        return x.view(B, N, output_dim, output_H, output_W)

    def bev_encoder(self, x):
        x = self.img_bev_encoder_backbone(x)
        return self.img_bev_encoder_neck(x)

    def extract_img_feat(self, img, img_metas):
        """img = [imgs, rots, trans, intrins, post_rots, post_trans, bda, ...] -> (voxel_feats list, depth, img_feats).
        The reference clones the image features for a head that ignores them; they are handed on as they are.
        imgs may also be the uint8 (B, N, H, W, 3) BGR frames of occformer_b200.pipelines' LoadMultiViewImageFrames_*
        transforms: they are resized, cropped and normalised on the GPU first (image_prep.prepare_images), from the
        'img_aug' of each sample's metas.  An empty uint8 (B, N, 0) imgs is LoadMultiViewJpegBytes_OccFormer's
        placeholder: the JPEG files in each 'img_aug' are decoded on the GPU first (image_prep.decode_jpeg); so is
        LoadMultiViewPngBytes_SemanticKitti's (B, 1, 0) one, whose 'img_aug' carries PNG files (image_prep.decode_png)."""
        imgs = image_prep.input_frames(
            img[0], img_metas,
            "OccupancyFormer: the empty image placeholder needs each sample's 'img_aug' meta with its 'jpeg' files, "
            "which LoadMultiViewJpegBytes_OccFormer produces, or its 'png' files, which "
            "LoadMultiViewPngBytes_SemanticKitti produces; add 'img_aug' to Collect3D's meta_keys")
        if (imgs.dtype if torch.is_tensor(imgs) else imgs[0].dtype) == torch.uint8:
            if img_metas is None or any("img_aug" not in m for m in img_metas):
                raise ValueError("OccupancyFormer: uint8 camera frames need each sample's 'img_aug' meta, which the "
                                 "LoadMultiViewImageFrames_OccFormer / LoadMultiViewImageFrames_SemanticKitti transforms "
                                 "produce; add 'img_aug' to Collect3D's meta_keys")
            imgs = image_prep.prepare_images(imgs, [m["img_aug"] for m in img_metas])
        x = self.image_encoder(imgs)
        img_feats = x
        rots, trans, intrins, post_rots, post_trans, bda = img[1:7]
        mlp_input = self.img_view_transformer.get_mlp_input(rots, trans, intrins, post_rots, post_trans, bda)
        x, depth = self.img_view_transformer([x, rots, trans, intrins, post_rots, post_trans, bda, mlp_input])
        x = self.bev_encoder(x)
        if type(x) is not list:
            x = [x]
        return x, depth, img_feats

    def extract_feat(self, points, img, img_metas):
        voxel_feats, depth, img_feats = self.extract_img_feat(img, img_metas)
        return voxel_feats, img_feats, depth

    # ------------------------------------------------------------------ inference entry points
    def forward(self, return_loss=True, **kwargs):
        """Base3DDetector.forward (base.py:47-61)"""
        if return_loss:
            return self.forward_train(**kwargs)
        return self.forward_test(**kwargs)

    def forward_train(self, *args, **kwargs):
        raise NotImplementedError("occformer_b200.OccupancyFormer is inference-only: forward_train, the losses and "
                                  "get_depth_loss are not built (call model(return_loss=False, ...))")

    def forward_test(self, img_metas=None, img_inputs=None, **kwargs):
        return self.simple_test(img_metas, img_inputs, **kwargs)

    @torch.no_grad()
    def simple_test(self, img_metas, img=None, rescale=False, points_occ=None, gt_occ=None, points_uv=None):
        """occupancyformer.py:209-237 -> the head's dict with 'output_voxels' (B, K, *occ_size) and 'target_voxels' = gt_occ;
        with LiDAR points also 'output_points' (int64 labels), 'target_points' and 'evaluation_semantic'.  Without gt_occ,
        the SemanticKITTI head builds 'target_voxels' from the voxel files of LoadSemKittiVoxelFiles when every sample's
        metas carry 'semkitti_voxels' (occupancy_targets).

        The panoptic head's dict is returned as the head makes it, plus 'target_voxels' and 'target_points': its
        'output_voxels' is [(semantic, panoptic)] and its 'output_points' are labels already, which the reference detector
        cannot take (INTEGRATION.md)."""
        if gt_occ is None and points_occ is not None and self.occ_targets_from_points:
            gt_occ = self.occupancy_targets(points_occ, img_metas)
        elif gt_occ is None and _voxel_files(img_metas) and isinstance(self.pts_bbox_head, Mask2FormerOccHead):
            gt_occ = self.occupancy_targets(points_occ, img_metas)
        voxel_feats, img_feats, depth = self.extract_feat(points=None, img=img, img_metas=img_metas)
        output = self.pts_bbox_head.simple_test(voxel_feats=voxel_feats, points=points_occ, img_metas=img_metas,
                                                img_feats=img_feats, points_uv=points_uv)
        if isinstance(self.pts_bbox_head, Mask2FormerNuscPanopticOccHead):
            output["target_voxels"] = gt_occ
            output["target_points"] = torch.cat(points_occ, dim=0) if points_occ is not None else None
            return output
        if output["output_points"] is not None and points_occ is not None:
            scores = output["output_points"]
            target_points = torch.cat(points_occ, dim=0)
            output["output_points"] = torch.argmax(scores[:, 1:], dim=1) + 1
            output["evaluation_semantic"] = self.simple_evaluation_semantic(scores, target_points, img_metas)
            output["target_points"] = target_points
        # The reference resizes output_voxels trilinearly to img_metas[0]['occ_size'] when their sizes differ; the head
        # already interpolates to that size (head.simple_test), so the resize could never fire and is not built.
        output["output_voxels"] = output["output_voxels"][0]
        output["target_voxels"] = gt_occ
        return output

    def occupancy_targets(self, points_occ, img_metas, unoccupied_id=17):
        """The gt_occ the reference's nuScenes loader builds for these points (occformer_b200.targets), on their device:
        points_occ = list of per-sample (n_i, 4) CUDA tensors [x, y, z, label | panoptic id], occ_size and pc_range from
        img_metas[0] -> int64 (B, X, Y, Z): semantic labels for Mask2FormerNuscOccHead, panoptic ids for
        Mask2FormerNuscPanopticOccHead.  Reads one invalid-point count back to the host (ValueError if nonzero).
        Mask2FormerOccHead (SemanticKITTI): points_occ is unused; every sample's img_metas carry the 'semkitti_voxels' of
        LoadSemKittiVoxelFiles -> int64 (B, 256, 256, 32) from those files (targets.semantic_kitti_occupancy); those of
        the training transform LoadSemKittiVoxelFilesAug also carry its 'augment', which gives the augmented volume of
        LoadSemKittiAnnotation(is_train=True) (semantic_kitti_occupancy(..., augment=))."""
        head = self.pts_bbox_head
        if isinstance(head, Mask2FormerNuscPanopticOccHead):
            build = targets.panoptic_occupancy
        elif isinstance(head, Mask2FormerNuscOccHead):
            build = targets.lidarseg_occupancy
        elif isinstance(head, Mask2FormerOccHead) and _voxel_files(img_metas):
            vox = [m["semkitti_voxels"] for m in img_metas]
            if any(v["learning_map"] != vox[0]["learning_map"] for v in vox[1:]):
                raise ValueError("occupancy_targets: every sample of a batch needs the same learning map")
            aug = {"augment" in v for v in vox}
            if len(aug) != 1:
                raise ValueError("occupancy_targets: a batch mixes the voxel files of LoadSemKittiVoxelFiles and of "
                                 "LoadSemKittiVoxelFilesAug")
            kw = dict(augment=[v["augment"] for v in vox]) if aug == {True} else {}
            return targets.semantic_kitti_occupancy([v["label"] for v in vox], [v["invalid"] for v in vox],
                                                    vox[0]["learning_map"], names=[v["files"] for v in vox], **kw)
        else:
            raise NotImplementedError(f"occupancy_targets: {type(head).__name__} scores against preprocessed voxel labels "
                                      "(SemanticKITTI), not a LiDAR point scan; pass gt_occ, or the voxel files of "
                                      "LoadSemKittiVoxelFiles ('semkitti_voxels' in every sample's metas)")
        # the reference's datasets store both fields as numpy arrays (nuscenes_lss_dataset.py:86-87), configs as lists
        occ_size, pc_range = (np.asarray(img_metas[0][k]) for k in ("occ_size", "pc_range"))
        same = (np.array_equal(np.asarray(m["occ_size"]), occ_size) and np.array_equal(np.asarray(m["pc_range"]), pc_range)
                for m in img_metas[1:])
        if not all(same):
            raise ValueError("occupancy_targets: every sample of a batch needs the same occ_size and pc_range")
        return build(list(points_occ), [int(v) for v in occ_size], [float(v) for v in pc_range], unoccupied_id)

    def post_process_semantic(self, pred_occ):
        """occupancyformer.py:239-244: class of the largest softmax probability, (B, K, ...) -> (B, ...).  An evaluation
        helper outside the forward; simple_test's 'output_labels' is the same argmax, made by the head's kernel."""
        if type(pred_occ) == list:
            pred_occ = pred_occ[-1]
        score, clses = torch.max(torch.softmax(pred_occ, dim=1), dim=1)
        return clses

    def simple_evaluation_semantic(self, pred, gt, img_metas):
        """occupancyformer.py:246-254: fast_hist_crop(pred, gt[:, 3], arange(16)) -> numpy int64 (16, 16).

        pred: the head's (n, 17) point scores, whose prediction is 1 + argmax(scores[:, 1:]) (what simple_test passes):
        counted on the tensors' device by dist_eval.lidarseg_hist, hist[label - 1, pred - 1] over the points labelled
        1..16; the numpy conversion is the one host synchronisation of simple_test.  Or (n,) predicted labels, as the
        reference passes them: counted on the host exactly as the reference's fast_hist_crop (metric_util.py:8-23)
        counts any integer labels, including the ones it crops away."""
        if pred.dim() == 2:
            return dist_eval.lidarseg_hist(pred, gt[:, 3], LIDARSEG_CLASSES).cpu().numpy()
        n = LIDARSEG_CLASSES
        pred = pred.cpu().numpy().astype(np.int64)
        label = gt[:, 3].cpu().numpy().astype(np.int64)
        k = (label >= 0) & (label < n)
        hist = np.bincount(n * label[k] + pred[k], minlength=n ** 2)[:n ** 2].reshape(n, n)
        return hist[1:, 1:]
