"""Loader transforms that leave the occupancy ground truth to the GPU (occformer_b200.targets).

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
