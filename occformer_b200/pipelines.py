"""Loader transforms that leave the occupancy ground truth (occformer_b200.targets), the camera images' resize, crop and
normalisation (occformer_b200.image_prep, the LoadMultiViewImageFrames_* transforms) or also the JPEG decoding
(LoadMultiViewJpegBytes_OccFormer) to the GPU.  In training pipelines, the LoadMultiViewImageFramesAug_* transforms
also leave the flip and rotation, and LoadLidarDepthPoints the depth maps of CreateDepthFromLiDAR, to the GPU
(image_prep.camera_inputs), and the byte transforms' training twins (LoadMultiViewJpegBytesAug_OccFormer,
LoadMultiViewPngBytesAug_SemanticKitti) also the decode.  LoadSemKittiVoxelFiles, at the end of this file, hands
SemanticKITTI's voxel files to the GPU in place of the preprocessed labels, and LoadSemKittiVoxelFilesAug does so in
training pipelines with LoadSemKittiAnnotation's augmentation.

    LoadNuscOccupancyPoints          = LoadNuscOccupancyAnnotations          P/datasets/pipelines/loading_nusc_occ.py:13-120
    LoadNuscPanopticOccupancyPoints  = LoadNuscPanopticOccupancyAnnotations  P/datasets/pipelines/loading_nusc_panoptic_occ.py:32-145

Same kwargs, same ``points_occ`` and ``img_inputs`` (with the augmentation matrix ``bda_rot``), same numpy RNG draws in
training mode, but no ``gt_occ``: the float64 voxelisation, the lexsort and the per-voxel counter loop are skipped, and
``OccupancyFormer(occ_targets_from_points=True)`` builds the volume from ``points_occ`` on the device (INTEGRATION.md).
Registered under these new names, so a config opts in by swapping the transform's ``type``.
"""
import os

import numpy as np
import torch

from . import jpeg, png
from .registry import PIPELINES


def bda_matrix(rotate_deg, flip_dx, flip_dy, flip_dz):
    """The 3x3 float32 augmentation matrix flip @ rot of the reference's voxel_transform (loading_nusc_occ.py:140-177),
    in its float32 torch arithmetic: rot = BEV rotation by rotate_deg, flip = diag(+-1) per flipped axis."""
    a = torch.tensor(rotate_deg / 180 * np.pi)
    s, c = torch.sin(a), torch.cos(a)
    rot = torch.Tensor([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    flip = torch.eye(4)
    for axis, on in enumerate((flip_dx, flip_dy, flip_dz)):
        if on:
            f = torch.eye(4)
            f[axis, axis] = -1
            flip = flip @ f
    return (flip @ rot)[:3, :3]


class _OccupancyPoints:
    """the shared part of both transforms"""

    def __init__(self, data_root="data/nuscenes", is_train=False, is_test_submit=False, grid_size=None,
                 point_cloud_range=None, bda_aug_conf=None, unoccupied_id=17, cls_metas="nuscenes.yaml"):
        if is_test_submit:
            raise ValueError(f"{type(self).__name__}: is_test_submit=True builds no ground truth; keep the reference "
                             "transform for the test-submission pipeline")
        import yaml
        with open(cls_metas, "r") as f:
            self.learning_map = yaml.safe_load(f)["learning_map"]
        self.data_root, self.is_train, self.is_test_submit = data_root, is_train, is_test_submit
        self.cls_metas, self.bda_aug_conf, self.unoccupied_id = cls_metas, bda_aug_conf, unoccupied_id
        self.grid_size = np.array(grid_size)
        self.point_cloud_range = np.array(point_cloud_range)

    def sample_3d_augmentation(self):
        """five numpy draws in the reference's order (rotation, scale, three flips); only the flips and the rotation
        enter the matrix"""
        conf = self.bda_aug_conf
        rotate = np.random.uniform(*conf["rot_lim"])
        scale = np.random.uniform(*conf["scale_lim"])
        flip_dx = np.random.uniform() < conf["flip_dx_ratio"]
        flip_dy = np.random.uniform() < conf["flip_dy_ratio"]
        flip_dz = np.random.uniform() < conf.get("flip_dz_ratio", 0.0)
        return rotate, scale, flip_dx, flip_dy, flip_dz

    def _labels(self, results):
        raise NotImplementedError

    def __call__(self, results):
        labels = self._labels(results)
        points = np.fromfile(results["pts_filename"], dtype=np.float32, count=-1).reshape(-1, 5)[..., :3]
        lidarseg = np.concatenate([points, labels], axis=-1)
        if self.is_train:
            rotate, _, flip_dx, flip_dy, flip_dz = self.sample_3d_augmentation()
            bda_rot = bda_matrix(rotate, flip_dx, flip_dy, flip_dz)
        else:
            bda_rot = torch.eye(3).float()
        lidarseg[:, :3] = points @ bda_rot.t().numpy()
        results["points_occ"] = torch.from_numpy(lidarseg).float()
        imgs, rots, trans, intrins, post_rots, post_trans, gt_depths, sensor2sensors = results["img_inputs"]
        results["img_inputs"] = (imgs, rots, trans, intrins, post_rots, post_trans, bda_rot, gt_depths, sensor2sensors)
        return results


@PIPELINES.register_module()
class LoadNuscOccupancyPoints(_OccupancyPoints):
    """LoadNuscOccupancyAnnotations without gt_occ: column 3 of points_occ is the lidarseg label after the learning map."""

    def _labels(self, results):
        raw = np.fromfile(os.path.join(self.data_root, results["lidarseg"]), dtype=np.uint8).reshape([-1, 1])
        lut, known = np.zeros(256, np.int64), np.zeros(256, bool)
        for k, v in self.learning_map.items():
            if 0 <= int(k) < 256:
                lut[int(k)], known[int(k)] = v, True
        if not known[raw].all():
            raise KeyError(int(raw[~known[raw]][0]))  # as the reference's dict lookup
        return lut[raw]


@PIPELINES.register_module()
class LoadNuscPanopticOccupancyPoints(_OccupancyPoints):
    """LoadNuscPanopticOccupancyAnnotations without gt_occ: column 3 of points_occ is the mapped panoptic id
    (mapped label * 1000 + instance)."""

    def _labels(self, results):
        path = results["lidarseg"].replace("lidarseg", "panoptic").replace(".bin", ".npz")
        pan = np.load(os.path.join(self.data_root, path))["data"]
        sem = pan // 1e3
        # The reference's in-place remap (loading_nusc_panoptic_occ.py:98-104): the raw labels are visited in ascending
        # order, and a point already remapped to a label visited later is remapped again (2 -> 7, then raw 7 -> 0).
        for label in np.unique(sem):
            hit = sem == label
            mapped = self.learning_map[int(label)]
            sem[hit] = mapped
            pan[hit] = mapped * 1e3 + (pan[hit] - label * 1e3)
        return pan.reshape(-1, 1)


# ---------------------------------------------------------------------------------------------- camera images
class _ImageFrames:
    """the shared part of the image transforms: sample_augmentation (loading_nusc_imgs.py:72-96) in test mode, or with
    the training-mode draws when the class sets ``training``, the post-homography in the reference's float32 torch
    arithmetic (:34-53), and the frame decode.  A transform serves one mode and refuses the other."""

    training = False

    def __init__(self, data_config, is_train=False, img_norm_cfg=None):
        if is_train and not self.training:
            raise ValueError(f"{type(self).__name__}: is_train=True is not supported by this test-mode transform; "
                             "training pipelines take LoadMultiViewImageFramesAug_OccFormer / "
                             "LoadMultiViewImageFramesAug_SemanticKitti (with LoadLidarDepthPoints in place of "
                             "CreateDepthFromLiDAR), or keep the reference transform")
        if self.training and not is_train:
            raise ValueError(f"{type(self).__name__}: is_train=False: this is the training-mode transform; test "
                             "pipelines take LoadMultiViewImageFrames_OccFormer / LoadMultiViewImageFrames_SemanticKitti")
        from .image_prep import norm_config
        self.is_train, self.data_config, self.img_norm_cfg = is_train, data_config, img_norm_cfg
        self.norm = norm_config(img_norm_cfg)

    def sample_augmentation(self, H, W):
        fH, fW = self.data_config["input_size"]
        resize = float(fW) / float(W)
        resize += self.data_config.get("resize_test", 0.0)
        resize_dims = (int(W * resize), int(H * resize))
        newW, newH = resize_dims
        crop_h = int((1 - np.mean(self.data_config["crop_h"])) * newH) - fH
        crop_w = int(max(0, newW - fW) / 2)
        return resize, resize_dims, (crop_w, crop_h, crop_w + fW, crop_h + fH)

    def train_augmentation(self, H, W):
        """training-mode sample_augmentation: five numpy draws in the reference's order (resize, crop_h, crop_w, flip,
        rotate; no flip draw when data_config['flip'] is falsy) -> (resize, resize_dims, crop, flip, rotate)"""
        cfg = self.data_config
        fH, fW = cfg["input_size"]
        resize = float(fW) / float(W)
        resize += np.random.uniform(*cfg["resize"])
        resize_dims = (int(W * resize), int(H * resize))
        newW, newH = resize_dims
        crop_h = int((1 - np.random.uniform(*cfg["crop_h"])) * newH) - fH
        crop_w = int(np.random.uniform(0, max(0, newW - fW)))
        flip = cfg["flip"] and np.random.choice([0, 1])
        rotate = np.random.uniform(*cfg["rot"])
        return resize, resize_dims, (crop_w, crop_h, crop_w + fW, crop_h + fH), flip, rotate

    def choose_cams(self):
        """the camera names of a sample: in training mode Ncams of them drawn without replacement when Ncams is fewer"""
        cams = self.data_config["cams"]
        if self.training and self.data_config["Ncams"] < len(cams):
            return np.random.choice(cams, self.data_config["Ncams"], replace=False)
        return cams

    @staticmethod
    def post_homography(resize, crop, flip=False, rotate=0):
        """(post_rot (3, 3), post_tran (3,)) of img_transform"""
        post_rot2 = torch.eye(2) * resize
        post_tran2 = torch.zeros(2) - torch.Tensor(crop[:2])
        if flip:
            A = torch.Tensor([[-1, 0], [0, 1]])
            b = torch.Tensor([crop[2] - crop[0], 0])
            post_rot2 = A.matmul(post_rot2)
            post_tran2 = A.matmul(post_tran2) + b
        h = rotate / 180 * np.pi
        A = torch.Tensor([[np.cos(h), np.sin(h)], [-np.sin(h), np.cos(h)]])
        b = torch.Tensor([crop[2] - crop[0], crop[3] - crop[1]]) / 2
        b = A.matmul(-b) + b
        post_rot2 = A.matmul(post_rot2)
        post_tran2 = A.matmul(post_tran2) + b
        post_rot, post_tran = torch.eye(3), torch.zeros(3)
        post_rot[:2, :2] = post_rot2
        post_tran[:2] = post_tran2
        return post_rot, post_tran

    @staticmethod
    def decode(path):
        """cv2.imread(path, IMREAD_UNCHANGED): the pixels of mmcv.imread(path, 'unchanged') with its cv2 backend"""
        import cv2
        img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        if img is None:
            raise FileNotFoundError(path)
        if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3:
            raise ValueError(f"{path}: a 3-channel uint8 frame is needed, got {img.dtype} {img.shape}")
        return img

    def load(self, path):
        """one camera's file -> (its payload, (H, W)): the decoded frame"""
        img = self.decode(path)
        return img, img.shape[:2]

    def image_input(self, payloads):
        """img_inputs[0] of a sample from its cameras' payloads: the uint8 (N, H, W, 3) frames"""
        return torch.stack([torch.from_numpy(p) for p in payloads])

    def file_meta(self, payloads, paths):
        """what results['img_aug'] carries besides the augmentation: nothing"""
        return {}

    def camera_size(self, H, W):
        """one camera of an H x W frame -> (resize_dims, crop, flip, rotate, post_rot, post_tran)"""
        if self.training:
            resize, resize_dims, crop, flip, rotate = self.train_augmentation(H, W)
        else:
            (resize, resize_dims, crop), flip, rotate = self.sample_augmentation(H, W), False, 0
        return (resize_dims, crop, flip, rotate) + self.post_homography(resize, crop, flip, rotate)

    def img_aug(self, dims, crops, flips=(), rotates=()):
        aug = dict(resize_dims=[list(d) for d in dims], crop=[list(c) for c in crops],
                   input_size=list(self.data_config["input_size"]), **self.norm)
        if self.training:
            aug.update(flip=[bool(f) for f in flips], rotate=[float(r) for r in rotates])
        return aug


@PIPELINES.register_module()
class LoadMultiViewImageFrames_OccFormer(_ImageFrames):
    """LoadMultiViewImageFromFiles_OccFormer (loading_nusc_imgs.py:10-179) in test mode, leaving the resize, crop and
    normalisation to the GPU (image_prep.prepare_images, called by OccupancyFormer.extract_img_feat).  img_inputs[0] is
    the decoded uint8 (N, H, W, 3) BGR frames; img_inputs[1:] are the reference's; results['img_aug'] describes each
    camera's resize and crop and the normalisation, and must be collected into the img_metas (Collect3D meta_keys).
    results['canvas'] (the cropped uint8 images, read only by a commented-out visualisation) is not produced."""

    def __call__(self, results):
        cam_names = self.choose_cams()
        results["cam_names"] = cam_names
        payloads, paths, sizes, rots, trans, intrins, post_rots, post_trans, sensor2sensors, dims, crops, flips, \
            rotates = ([] for _ in range(13))
        for cam_name in cam_names:
            cam_data = results["curr"]["cams"][cam_name]
            payload, (H, W) = self.load(cam_data["data_path"])
            intrin = torch.Tensor(cam_data["cam_intrinsic"])
            sensor2lidar = torch.tensor(results["lidar2cam_dic"][cam_name]).inverse().float()
            resize_dims, crop, flip, rotate, post_rot, post_tran = self.camera_size(H, W)
            payloads.append(payload)
            paths.append(cam_data["data_path"])
            sizes.append((H, W))
            intrins.append(intrin)
            rots.append(sensor2lidar[:3, :3])
            trans.append(sensor2lidar[:3, 3])
            post_rots.append(post_rot)
            post_trans.append(post_tran)
            sensor2sensors.append(sensor2lidar)
            dims.append(resize_dims)
            crops.append(crop)
            flips.append(flip)
            rotates.append(rotate)
        if len(set(sizes)) != 1:
            raise ValueError(f"{type(self).__name__}: the cameras of a sample need one frame size")
        gt_depths = [torch.zeros(1) for _ in cam_names]
        results["img_inputs"] = (self.image_input(payloads),) + tuple(
            torch.stack(x) for x in (rots, trans, intrins, post_rots, post_trans, gt_depths, sensor2sensors))
        results["img_aug"] = dict(self.img_aug(dims, crops, flips, rotates), **self.file_meta(payloads, paths))
        return results


@PIPELINES.register_module()
class LoadMultiViewImageFrames_SemanticKitti(_ImageFrames):
    """LoadMultiViewImageFromFiles_SemanticKitti (loading_kitti_imgs.py:12-146) in test mode, leaving the resize, crop
    and normalisation to the GPU: img_inputs[0] is the decoded uint8 (1, H, W, 3) BGR frame, img_inputs[1:] are the
    reference's, results['raw_img'] is kept and results['img_aug'] added; results['canvas'] is not produced."""

    keep_raw_img = True  # results['raw_img'] = the decoded frame

    def __call__(self, results):
        img_filenames = results["img_filename"]
        assert len(img_filenames) == 1
        payload, (H, W) = self.load(img_filenames[0])
        if self.keep_raw_img:
            results["raw_img"] = payload
        resize_dims, crop, flip, rotate, post_rot, post_tran = self.camera_size(H, W)
        intrin = torch.Tensor(results["cam_intrinsic"][0])
        lidar2cam = torch.Tensor(results["lidar2cam"][0])
        cam2lidar = lidar2cam.inverse()
        res = [cam2lidar[:3, :3], cam2lidar[:3, 3], intrin, post_rot, post_tran, torch.zeros(1), cam2lidar]
        results["img_inputs"] = (self.image_input([payload]),) + tuple(x[None] for x in res)
        results["img_aug"] = dict(self.img_aug([resize_dims], [crop], [flip], [rotate]),
                                  **self.file_meta([payload], [img_filenames[0]]))
        return results


@PIPELINES.register_module()
class LoadMultiViewImageFramesAug_OccFormer(LoadMultiViewImageFrames_OccFormer):
    """LoadMultiViewImageFromFiles_OccFormer (loading_nusc_imgs.py:10-179) in training mode (is_train=True is required),
    leaving the resize, crop, flip, rotation and normalisation to the GPU (image_prep.camera_inputs).  The same numpy
    draws in the same order as the reference (choose_cams when Ncams < len(cams), then per camera resize, crop_h,
    crop_w, flip when data_config['flip'], rotate) and the same img_inputs[1:]; img_inputs[0] is the decoded uint8
    (N, H, W, 3) BGR frames and results['img_aug'] also carries each camera's 'flip' and 'rotate'."""

    training = True


@PIPELINES.register_module()
class LoadMultiViewImageFramesAug_SemanticKitti(LoadMultiViewImageFrames_SemanticKitti):
    """LoadMultiViewImageFromFiles_SemanticKitti (loading_kitti_imgs.py:12-146) in training mode (is_train=True is
    required), leaving the resize, crop, flip, rotation and normalisation to the GPU: the reference's draws and
    img_inputs[1:], the decoded uint8 (1, H, W, 3) BGR frame in img_inputs[0], and 'flip' / 'rotate' in
    results['img_aug']."""

    training = True


@PIPELINES.register_module()
class LoadLidarDepthPoints:
    """CreateDepthFromLiDAR (P/datasets/pipelines/lidar2depth.py:8-87) leaving the projection to the GPU: reads the same
    scan (nuScenes: pts_filename as (-1, 5) float32 rows; KITTI: the velodyne .bin of the camera frame under data_root,
    as (-1, 4) rows), keeps x, y, z, and computes rots.inverse() of img_inputs[1] here, in CPU fp32 torch as the
    reference does (a device inverse would give other bits).  Both go into results['img_aug'] ('lidar_points',
    'lidar_inv_rots'); img_inputs keeps its 8-tuple layout with the gt_depths placeholder, which
    image_prep.camera_inputs fills on the GPU.  Makes no random draws."""

    def __init__(self, data_root=None, dataset="kitti"):
        if dataset not in ("kitti", "nusc"):
            raise ValueError(f"LoadLidarDepthPoints: dataset must be 'kitti' or 'nusc', got {dataset!r}")
        self.data_root, self.dataset = data_root, dataset

    def scan_path(self, results):
        if self.dataset == "nusc":
            return results["pts_filename"]
        seq_id, _, filename = results["img_filename"][0].split("/")[-3:]
        return os.path.join(self.data_root, "data_velodyne/velodyne/sequences", seq_id, "velodyne",
                            filename.replace(".png", ".bin"))

    def __call__(self, results):
        cols = 4 if self.dataset == "kitti" else 5
        pts = np.fromfile(self.scan_path(results), dtype=np.float32).reshape(-1, cols)[:, :3]
        inv_rots = results["img_inputs"][1].inverse()
        results["img_aug"] = dict(results["img_aug"], lidar_points=torch.from_numpy(np.ascontiguousarray(pts)),
                                  lidar_inv_rots=inv_rots)
        return results


class _FileBytes:
    """the byte transforms' part (mixed into a frame transform): a camera's payload is its file's bytes and (H, W) comes
    from the file's header (frame_size, whose error names the file in a ValueError); img_inputs[0] is an empty
    uint8 (N, 0) placeholder and results['img_aug'] also carries the files (kind) and their paths (kind + '_files').
    The class sets kind, frame_size and error."""

    def load(self, path):
        with open(path, "rb") as f:
            data = f.read()
        try:
            return data, self.frame_size(data)
        except self.error as e:
            raise ValueError(f"{path}: {e}") from None

    def image_input(self, payloads):
        return torch.zeros((len(payloads), 0), dtype=torch.uint8)

    def file_meta(self, payloads, paths):
        return {self.kind: list(payloads), self.kind + "_files": list(paths)}


@PIPELINES.register_module()
class LoadMultiViewJpegBytes_OccFormer(_FileBytes, LoadMultiViewImageFrames_OccFormer):
    """LoadMultiViewImageFrames_OccFormer without the decode: each camera file's bytes are read and the frame size comes
    from its SOF header (jpeg.frame_size), so img_aug and img_inputs[1:] are the frame transform's.  results['img_aug']
    also carries 'jpeg' (the N files' bytes, in camera order) and 'jpeg_files' (their paths); img_inputs[0] is an empty
    uint8 (N, 0) placeholder, which collates to (B, N, 0), a shape no other transform produces.  OccupancyFormer then
    decodes the files on the GPU (image_prep.decode_jpeg) and prepares the images from the frames.  Files the device
    decoder does not take (progressive, grayscale, ...) raise ValueError here, in the loader."""

    kind, frame_size, error = "jpeg", staticmethod(jpeg.frame_size), jpeg.JpegError


@PIPELINES.register_module()
class LoadMultiViewPngBytes_SemanticKitti(_FileBytes, LoadMultiViewImageFrames_SemanticKitti):
    """LoadMultiViewImageFrames_SemanticKitti without the decode: the frame file's bytes are read and the frame size
    comes from its IHDR chunk (png.frame_size), so img_aug and img_inputs[1:] are the frame transform's.
    results['img_aug'] also carries 'png' (the file's bytes, in a list of one) and 'png_files' (its path); img_inputs[0]
    is an empty uint8 (1, 0) placeholder, which collates to (B, 1, 0).  OccupancyFormer then decodes the file on the GPU
    (image_prep.decode_png) and prepares the image from the frame.  Files the device decoder does not take (16-bit,
    grayscale, alpha, palette, tRNS, interlaced, animated, ...) raise ValueError here, in the loader.
    results['raw_img'] needs the decoded frame on the host and is not produced: only the visualisation dump of the
    test loop (pred_save) reads it, and that keeps the frame transform.  Test pipelines only: is_train=True is refused,
    as the frame transform refuses it."""

    kind, frame_size, error = "png", staticmethod(png.frame_size), png.PngError
    keep_raw_img = False


@PIPELINES.register_module()
class LoadMultiViewJpegBytesAug_OccFormer(LoadMultiViewJpegBytes_OccFormer):
    """LoadMultiViewImageFramesAug_OccFormer without the decode (is_train=True is required): the reference's training
    draws (choose_cams when Ncams < len(cams), then per camera resize, crop_h, crop_w, flip when data_config['flip'],
    rotate) with the frame size from each file's SOF header, the same img_inputs[1:] and img_aug ('flip' / 'rotate'
    included), plus the files as LoadMultiViewJpegBytes_OccFormer adds them.  image_prep.camera_inputs decodes them on
    the GPU first."""

    training = True


@PIPELINES.register_module()
class LoadMultiViewPngBytesAug_SemanticKitti(LoadMultiViewPngBytes_SemanticKitti):
    """LoadMultiViewImageFramesAug_SemanticKitti without the decode (is_train=True is required): the reference's
    training draws with the frame size from the IHDR chunk, the same img_inputs[1:] and img_aug ('flip' / 'rotate'
    included), plus the file as LoadMultiViewPngBytes_SemanticKitti adds it; no raw_img.  image_prep.camera_inputs
    decodes it on the GPU first."""

    training = True


# ---------------------------------------------------------------------------------------------- SemanticKITTI labels
@PIPELINES.register_module()
class LoadSemKittiVoxelFiles:
    """The SemanticKITTI ground truth from the dataset's own voxel files instead of the preprocessed '<frame>_1_1.npy'
    (tools/kitti_process/semantic_kitti_preprocess.py): reads dataset/sequences/{sequence}/voxels/{frame_id}.label and
    .invalid under data_root, and the learning map from the dataset yaml at data_info_path (the file the preprocessing
    step takes).  results['semkitti_voxels'] = dict(label=, invalid= (the files' bytes), files= (their paths),
    learning_map=); results['gt_occ'] = None, so a following LoadSemKittiAnnotation takes its test-mode path and the
    npy the dataset may have loaded is dropped.  OccupancyFormer.simple_test then builds 'target_voxels' on the GPU
    (targets.semantic_kitti_occupancy); 'semkitti_voxels' must be collected into the img_metas (Collect3D meta_keys).
    Files of the wrong size raise ValueError here, in the loader.  Test pipelines only: before a training-mode
    LoadSemKittiAnnotation the None would silently skip its augmentation and its gt_occ, so is_train=True (the
    annotation transform's flag, repeated here) is refused."""

    def __init__(self, data_root="data/SemanticKITTI", data_info_path="projects/configs/_base_/semantickitti.yaml",
                 is_train=False):
        if is_train:
            raise ValueError("LoadSemKittiVoxelFiles: is_train=True is not supported: the transform hands no gt_occ to "
                             "LoadSemKittiAnnotation, whose training path needs it for the augmentation; keep the "
                             "preprocessed labels for training pipelines")
        self.learning_map = _learning_map(data_info_path)
        self.data_root, self.data_info_path = data_root, data_info_path

    def __call__(self, results):
        results["semkitti_voxels"] = _voxel_files(self.data_root, results, self.learning_map)
        results["gt_occ"] = None
        return results


def _learning_map(data_info_path):
    import yaml
    with open(data_info_path, "r") as f:
        return yaml.safe_load(f)["learning_map"]


def _voxel_files(data_root, results, learning_map):
    """dataset/sequences/{sequence}/voxels/{frame_id}.label and .invalid under data_root -> the 'semkitti_voxels' dict
    (label=, invalid= (the files' bytes), files= (their paths), learning_map=); ValueError for a wrong size"""
    from .targets import SEMKITTI_INVALID_BYTES, SEMKITTI_LABEL_BYTES
    base = os.path.join(data_root, "dataset", "sequences", results["sequence"], "voxels", results["frame_id"])
    files, data = [base + ".label", base + ".invalid"], []
    for path, size in zip(files, (SEMKITTI_LABEL_BYTES, SEMKITTI_INVALID_BYTES)):
        with open(path, "rb") as f:
            data.append(f.read())
        if len(data[-1]) != size:
            raise ValueError(f"{path}: a SemanticKITTI voxel file of {size} bytes is needed, got {len(data[-1])}")
    return dict(label=data[0], invalid=data[1], files=files, learning_map=learning_map)


def semkitti_bda_matrix(rotate_deg, flip_dx, flip_dy, flip_dz, point_cloud_range):
    """the 4x4 float32 bda_mat of the reference's SemanticKITTI voxel_transform (loading_kitti_occ.py:55-95), in its
    torch arithmetic and product order: ((denorm @ flip) @ rot) @ norm, about the centre of point_cloud_range (taken
    through torch.tensor, as LoadSemKittiAnnotation.__init__ takes it)"""
    pcr = torch.tensor(point_cloud_range)
    center = (pcr[:3] + pcr[3:]) / 2
    norm, denorm = torch.eye(4), torch.eye(4)
    norm[:3, -1] = -center
    denorm[:3, -1] = center
    a = torch.tensor(rotate_deg / 180 * np.pi)
    s, c = torch.sin(a), torch.cos(a)
    rot = torch.Tensor([[c, -s, 0, 0], [s, c, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    flip = torch.eye(4)
    for axis, on in enumerate((flip_dx, flip_dy, flip_dz)):
        if on:
            f = torch.eye(4)
            f[axis, axis] = -1
            flip = flip @ f
    return denorm @ flip @ rot @ norm


@PIPELINES.register_module()
class LoadSemKittiVoxelFilesAug:
    """LoadSemKittiAnnotation(is_train=True) (P/datasets/pipelines/loading_kitti_occ.py:8-53) from the dataset's own voxel
    files, leaving the volume and its augmentation to the GPU; it takes LoadSemKittiAnnotation's place in a training
    pipeline.  The same kwargs (bda_aug_conf, is_train, point_cloud_range) plus LoadSemKittiVoxelFiles' data_root and
    data_info_path.  It makes the reference's five numpy draws in its order (rotate, scale, flip_dx, flip_dy, flip_dz;
    only the rotation and the flips are used), inserts the reference's 4x4 bda_mat (semkitti_bda_matrix) into
    img_inputs as the reference does (the 9-tuple), and puts the files, the learning map and
    augment=dict(rotate=, flip_dx=, flip_dy=, flip_dz=) into results['semkitti_voxels']; results['gt_occ'] = None.  The
    training step then builds gt_occ on the GPU (targets.semantic_kitti_occupancy(..., augment=), through
    OccupancyFormer.occupancy_targets); 'semkitti_voxels' must be collected into the img_metas.  Files of the wrong size
    raise ValueError here.  Training pipelines only: is_train=False is refused (test pipelines take
    LoadSemKittiVoxelFiles before LoadSemKittiAnnotation)."""

    def __init__(self, bda_aug_conf, is_train=True, point_cloud_range=(0, -25.6, -2, 51.2, 25.6, 4.4),
                 data_root="data/SemanticKITTI", data_info_path="projects/configs/_base_/semantickitti.yaml"):
        if not is_train:
            raise ValueError("LoadSemKittiVoxelFilesAug: is_train=False: this is the training-mode transform; test "
                             "pipelines take LoadSemKittiVoxelFiles before LoadSemKittiAnnotation")
        self.bda_aug_conf, self.is_train = bda_aug_conf, is_train
        self.point_cloud_range = list(point_cloud_range)
        self.learning_map = _learning_map(data_info_path)
        self.data_root, self.data_info_path = data_root, data_info_path

    def sample_bda_augmentation(self):
        """the reference's five draws in its order -> (rotate, scale, flip_dx, flip_dy, flip_dz)"""
        conf = self.bda_aug_conf
        rotate = np.random.uniform(*conf["rot_lim"])
        scale = np.random.uniform(*conf["scale_lim"])
        flip_dx = np.random.uniform() < conf["flip_dx_ratio"]
        flip_dy = np.random.uniform() < conf["flip_dy_ratio"]
        flip_dz = np.random.uniform() < conf["flip_dz_ratio"]
        return rotate, scale, flip_dx, flip_dy, flip_dz

    def __call__(self, results):
        vox = _voxel_files(self.data_root, results, self.learning_map)
        rotate, _, flip_dx, flip_dy, flip_dz = self.sample_bda_augmentation()
        bda_mat = semkitti_bda_matrix(rotate, flip_dx, flip_dy, flip_dz, self.point_cloud_range)
        vox["augment"] = dict(rotate=float(rotate), flip_dx=bool(flip_dx), flip_dy=bool(flip_dy), flip_dz=bool(flip_dz))
        results["semkitti_voxels"] = vox
        results["gt_occ"] = None
        imgs, rots, trans, intrins, post_rots, post_trans, gt_depths, sensor2sensors = results["img_inputs"]
        results["img_inputs"] = (imgs, rots, trans, intrins, post_rots, post_trans, bda_mat, gt_depths, sensor2sensors)
        return results
