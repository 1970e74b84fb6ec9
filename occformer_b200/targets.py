"""Occupancy ground truth of nuScenes on the GPU, built from the labelled LiDAR points the test loop already hands to the
model (``points_occ``), bit for bit the ``gt_occ`` of the reference's loaders:

    lidarseg_occupancy   LoadNuscOccupancyAnnotations          P/datasets/pipelines/loading_nusc_occ.py:95-138
    panoptic_occupancy   LoadNuscPanopticOccupancyAnnotations  P/datasets/pipelines/loading_nusc_panoptic_occ.py:120-166

``points_occ`` holds the float32 xyz after the batch augmentation (exact in the float64 array the loader voxelises) and
the mapped label (semantic) or id (panoptic) in column 3, an integer below 2^24 and so exact in float32.  The kernel
(occ_lidarseg_occupancy, csrc/occ_targets.cu) voxelises in float64 as numpy does and takes each voxel's majority id with
no sort.  Out-of-contract points (a label that is negative, not an integer or at or above 256 / 65536, a non-finite
coordinate, more than 65535 points of one id in one voxel) raise ValueError; there is no CPU fallback.
"""
import torch

from . import ops

SEMANTIC_IGNORE = 255
PANOPTIC_IGNORE = 65535


def _occupancy(points, occ_size, point_cloud_range, panoptic, empty_id, ignore):
    single = torch.is_tensor(points)
    pts = [points] if single else list(points)
    if not pts:
        raise ValueError("occupancy targets of an empty batch")
    for p in pts:
        if not torch.is_tensor(p) or p.dim() != 2 or p.shape[1] < 4:
            raise ValueError("points: (n, >= 4) tensors of rows [x, y, z, label, ...]")
        if p.shape[1] != pts[0].shape[1]:
            raise ValueError("points: every sample needs the same number of columns")
    if len(occ_size) != 3 or len(point_cloud_range) != 6:
        raise ValueError("occ_size is (X, Y, Z) and point_cloud_range (x_min, y_min, z_min, x_max, y_max, z_max)")
    if not all(p.is_cuda for p in pts):
        raise RuntimeError("occformer_b200.targets: points must be CUDA tensors (no CPU fallback exists)")
    flat = (pts[0] if len(pts) == 1 else torch.cat(pts, dim=0)).float().contiguous()
    vol, invalid = ops.lidarseg_occupancy(flat, [p.shape[0] for p in pts], point_cloud_range, occ_size, panoptic,
                                          empty_id, ignore)
    bad = int(invalid.item())  # the one host synchronisation
    if bad:
        raise ValueError(f"{bad} LiDAR points or voxel votes are outside the ground truth's contract (label not an "
                         f"integer in [0, {65536 if panoptic else 256}), non-finite coordinate, or more than 65535 "
                         "points of one id in one voxel)")
    return vol[0] if single else vol


def lidarseg_occupancy(points, occ_size, point_cloud_range, unoccupied_id=17):
    """Semantic occupancy ground truth: points = list of per-sample (n_i, >= 4) CUDA tensors [x, y, z, label, ...] (labels
    after the learning map, 0..255) or one such tensor -> int64 (B, X, Y, Z) (or (X, Y, Z)): each occupied voxel's
    majority label with noise 0 -> 255 and unoccupied_id -> 0, empty voxels 0."""
    return _occupancy(points, occ_size, point_cloud_range, 0, int(unoccupied_id), SEMANTIC_IGNORE)


def panoptic_occupancy(points, occ_size, point_cloud_range, unoccupied_id=17):
    """Panoptic occupancy ground truth: column 3 holds the mapped panoptic id (label * 1000 + instance, < 65536) ->
    int64 (B, X, Y, Z) (or (X, Y, Z)): each occupied voxel's majority id without id 0 (which still decides the voxel the
    reference writes last, as its loader does), 0 -> 65535, unoccupied_id * 1000 -> 0, empty voxels 0."""
    return _occupancy(points, occ_size, point_cloud_range, 1, int(unoccupied_id * 1e3), PANOPTIC_IGNORE)
