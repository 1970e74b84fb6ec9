"""Occupancy ground truth of nuScenes on the GPU, built from the labelled LiDAR points the test loop already hands to the
model (``points_occ``), bit for bit the ``gt_occ`` of the reference's loaders:

    lidarseg_occupancy   LoadNuscOccupancyAnnotations          P/datasets/pipelines/loading_nusc_occ.py:95-138
    panoptic_occupancy   LoadNuscPanopticOccupancyAnnotations  P/datasets/pipelines/loading_nusc_panoptic_occ.py:120-166

``points_occ`` holds the float32 xyz after the batch augmentation (exact in the float64 array the loader voxelises) and
the mapped label (semantic) or id (panoptic) in column 3, an integer below 2^24 and so exact in float32.  The kernel
(occ_lidarseg_occupancy, csrc/occ_targets.cu) voxelises in float64 as numpy does and takes each voxel's majority id with
no sort.  Out-of-contract points (a label that is negative, not an integer or at or above 256 / 65536, a non-finite
coordinate, more than 65535 points of one id in one voxel) raise ValueError; there is no CPU fallback.

SemanticKITTI's ground truth comes from the dataset's own voxel files instead of the offline preprocessing step:

    semantic_kitti_occupancy   semantic_kitti_preprocess.main (_1_1)  P/tools/kitti_process/semantic_kitti_preprocess.py:117-142
                               + LoadSemKittiAnnotation's .long()     P/datasets/pipelines/loading_kitti_occ.py:34-53

The 4 MB .label and 256 KB .invalid files of a frame cross PCIe instead of the 16 MB int64 volume, and the kernel
(occ_semkitti_labels, csrc/semkitti_labels.cu) remaps and masks them in one pass.  In training pipelines
(semantic_kitti_occupancy(..., augment=)) one launch of another kernel also applies LoadSemKittiAnnotation's
augmentation:

    + voxel_transform's slice rotation and flips   P/datasets/pipelines/loading_kitti_occ.py:55-117,
                                                    loading_nusc_occ.py:206-225 (occ_semkitti_labels_aug)
"""
import numpy as np
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


# ---------------------------------------------------------------------------------------------- SemanticKITTI
SEMKITTI_SHAPE = (256, 256, 32)
SEMKITTI_LABEL_BYTES = 2 * 256 * 256 * 32   # .label: one uint16 per voxel
SEMKITTI_INVALID_BYTES = 256 * 256 * 32 // 8  # .invalid: one bit per voxel


def semkitti_remap_lut(learning_map):
    """io_data.get_remap_lut (P/tools/kitti_process/io_data.py:173-193) from the dataset yaml's learning_map -> int32
    numpy table of max key + 100 entries: learning_map[k], 255 for keys the map lacks or maps to 0, 0 for key 0."""
    keys = [int(k) for k in learning_map]
    if not keys or min(keys) < 0 or max(keys) + 100 > 65536:
        raise ValueError("semkitti_remap_lut: learning_map keys must be labels in [0, 65436)")
    lut = np.zeros(max(keys) + 100, dtype=np.int32)
    lut[keys] = [int(v) for v in learning_map.values()]
    lut[lut == 0] = 255
    lut[0] = 0
    return lut


def _bytes(x, size, what, name):
    m = memoryview(x).cast("B")
    if m.nbytes != size:
        raise ValueError(f"semantic_kitti_occupancy: {name}: a {what} file holds {size} bytes, got {m.nbytes}")
    return m


def semkitti_augment_rows(augment):
    """per-sample augmentation dicts (rotate in degrees, flip_dx, flip_dy, flip_dz) -> int32 numpy (B, 10) rows of
    occ_semkitti_labels_aug: the three flips, the rotate flag (not np.isclose(rotate, 0), as voxel_transform decides)
    and the 16.16 coefficients of Image.rotate(rotate) of a 256 x 256 slice (image_prep.rotate_coeffs)"""
    from .image_prep import rotate_coeffs
    rows = []
    for a in augment:
        angle = float(a["rotate"])
        rot = not np.isclose(angle, 0)
        coeffs = rotate_coeffs(angle, SEMKITTI_SHAPE[1], SEMKITTI_SHAPE[0]) if rot else (1 << 16, 0, 0, 0, 1 << 16, 0)
        rows.append([int(bool(a["flip_dx"])), int(bool(a["flip_dy"])), int(bool(a["flip_dz"])), int(rot), *coeffs])
    return np.asarray(rows, dtype=np.int32).reshape(-1, 10)


def semantic_kitti_occupancy(labels, invalids, learning_map, names=None, augment=None):
    """SemanticKITTI occupancy ground truth from the voxel files: labels / invalids = the bytes (bytes-like) of one
    sample's voxels/*.label and voxels/*.invalid, or lists of B of each; learning_map = the dataset yaml's -> int64 CUDA
    (256, 256, 32) (or (B, 256, 256, 32)) on the current device, equal to the reference's
    torch.tensor(np.load('<frame>_1_1.npy')).long(): remap_lut[label], then 255 where the invalid bit is set.  The files
    travel in one pinned host buffer and one host-to-device copy (ops._stage).  A file of the wrong size, or a label
    at or past the LUT (the reference's IndexError; one count read back), raises ValueError naming the file (names: B
    (.label name, .invalid name) pairs for the messages; default: the sample index).

    augment: None, or one dict per sample with 'rotate' (degrees), 'flip_dx', 'flip_dy', 'flip_dz', as
    pipelines.LoadSemKittiVoxelFilesAug draws them -> the volume LoadSemKittiAnnotation(is_train=True) returns from the
    same files: each z slice rotated as Pillow's Image.rotate(rotate, NEAREST, fillcolor=255) when not
    np.isclose(rotate, 0), then the flips (occ_semkitti_labels_aug, one launch).  The learning map's values must then
    lie in [0, 255], the reference's uint8 cast."""
    single = not isinstance(labels, (list, tuple))
    labels = [labels] if single else list(labels)
    invalids = [invalids] if single else list(invalids)
    B = len(labels)
    if B == 0 or len(invalids) != B:
        raise ValueError("semantic_kitti_occupancy: needs one .label and one .invalid file per sample")
    names = [tuple(n) for n in names] if names is not None else [(f"sample {b}",) * 2 for b in range(B)]
    if len(names) != B or any(len(n) != 2 for n in names):
        raise ValueError("semantic_kitti_occupancy: names are B (.label name, .invalid name) pairs")
    lab = [_bytes(x, SEMKITTI_LABEL_BYTES, ".label", n[0]) for x, n in zip(labels, names)]
    inv = [_bytes(x, SEMKITTI_INVALID_BYTES, ".invalid", n[1]) for x, n in zip(invalids, names)]
    lut = semkitti_remap_lut(learning_map)
    if augment is not None:
        augment = list(augment)
        if len(augment) != B:
            raise ValueError(f"semantic_kitti_occupancy: augment needs one dict per sample, got {len(augment)} for {B}")
        if lut.min() < 0 or lut.max() > 255:
            raise ValueError("semantic_kitti_occupancy: with augment, the learning map's values must lie in [0, 255] "
                             "(voxel_transform casts the volume to uint8)")
        aug = semkitti_augment_rows(augment)
    if not torch.cuda.is_available():
        raise RuntimeError("occformer_b200.targets: semantic_kitti_occupancy needs a CUDA device (no CPU fallback exists)")
    dev = torch.device("cuda", torch.cuda.current_device())
    lut_d = ops._device_table(dev, ("semkitti_lut", lut.tobytes()), lambda: lut)
    # one copy: the labels, then the invalid bits, then the augmentation rows
    data, _ = ops._stage(lab + inv + ([] if augment is None else [aug.reshape(-1).view(np.uint8)]))
    split = B * SEMKITTI_LABEL_BYTES
    aug_at = split + B * SEMKITTI_INVALID_BYTES
    nvox = SEMKITTI_LABEL_BYTES // 2
    if augment is None:
        vol, bad = ops.semkitti_labels(data[:split], data[split:], B, nvox, lut_d)
    else:
        vol, bad = ops.semkitti_labels_aug(data[:split], data[split:aug_at], B, data[aug_at:].view(torch.int32), lut_d)
    bad = bad.cpu()  # the one host synchronisation
    if bool(bad.any()):
        b = int(bad.nonzero()[0, 0])
        raise ValueError(f"semantic_kitti_occupancy: {names[b][0]}: {int(bad[b])} voxel labels are at or past the remap "
                         f"table's {lut.size} entries (the learning map's largest key + 100)")
    vol = vol.view(B, *SEMKITTI_SHAPE)
    return vol[0] if single else vol
