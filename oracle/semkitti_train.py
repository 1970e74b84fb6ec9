"""TEST INFRASTRUCTURE ONLY (oracle) -- SemanticKITTI's training-mode ground truth (P/ = projects/mmdet3d_plugin/):

    LoadSemKittiAnnotation(is_train=True), voxel_transform   P/datasets/pipelines/loading_kitti_occ.py:8-117
    custom_rotate_3d                                         P/datasets/pipelines/loading_nusc_occ.py:206-225

A numpy restatement of the augmented volume: the preprocessed volume of oracle/semkitti_labels.py, cast to uint8, each
z slice rotated by Pillow's Image.rotate(angle, NEAREST, fillcolor=255) when not np.isclose(angle, 0) (the fixed-point
restatement of oracle/train_inputs.py, with 255 instead of black outside the slice), then the z, y and x reversals.
For the build container that has the reference checkout, the fixture generator runs the reference's transform verbatim
under oracle/shim.py on the preprocessed volumes of seeded synthetic voxel files:

    python -m oracle.semkitti_train gen        # tests/golden/semkitti_train_labels.npz

Only the first half is imported by tests/; it needs no reference checkout.
"""
import hashlib
import os
import sys

import numpy as np

from . import semkitti_labels as sk
from . import train_inputs as ti

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                      "semkitti_train_labels.npz")
KITTI_RANGE = [0, -25.6, -2, 51.2, 25.6, 4.4]
CONFIG_CONF = dict(rot_lim=(0, 0), scale_lim=(0.95, 1.05), flip_dx_ratio=0.5, flip_dy_ratio=0.5, flip_dz_ratio=0.5)


# =============================================================================
# restatement
# =============================================================================
def rotate_slices(vol, angle, fill=255):
    """Image.fromarray(vol[..., z]).rotate(angle, resample=NEAREST, fillcolor=fill) of every z slice of a uint8 (X, Y, Z)
    volume: oracle.train_inputs.rotate gathers all slices at once (they share one gather), and the pixels it takes
    from outside the slice (where a rotated all-ones image is 0) become fill"""
    out = ti.rotate(vol, angle)
    outside = ti.rotate(np.ones(vol.shape[:2] + (1,), np.uint8), angle)[..., 0] == 0
    out[outside] = fill
    return out


def augment(vol, rotate, flip_dx, flip_dy, flip_dz):
    """voxel_transform's volume: int64 (X, Y, Z) preprocessed volume -> int64 (X, Y, Z)"""
    v = vol.astype(np.uint8)
    if not np.isclose(rotate, 0):
        v = rotate_slices(v, rotate)
    if flip_dz:
        v = v[:, :, ::-1]
    if flip_dy:
        v = v[:, ::-1]
    if flip_dx:
        v = v[::-1]
    return np.ascontiguousarray(v).astype(np.int64)


def volume(label_bytes, invalid_bytes, learning_map, aug):
    """one frame's files and augmentation dict (rotate, flip_dx, flip_dy, flip_dz) -> LoadSemKittiAnnotation's
    training-mode gt_occ as an int64 array"""
    return augment(sk.occupancy(label_bytes, invalid_bytes, learning_map), aug["rotate"], aug["flip_dx"],
                   aug["flip_dy"], aug["flip_dz"])


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.int64).tobytes()).hexdigest()


# =============================================================================
# the fixture's cases
# =============================================================================
def conf(rot, fx=0.0, fy=0.0, fz=0.0):
    """a bda_aug_conf whose draws are fixed: uniform(a, a) is a, uniform() < 0 never and < 1 always holds"""
    return dict(rot_lim=(rot, rot), scale_lim=(0.95, 1.05), flip_dx_ratio=fx, flip_dy_ratio=fy, flip_dz_ratio=fz)


# name -> (bda_aug_conf, samples, synthetic frame mode)
CASES = {
    "none": (conf(0.0), 1, "mixed"),
    "flip_dx": (conf(0.0, fx=1.0), 1, "mixed"),
    "flip_dy": (conf(0.0, fy=1.0), 1, "mixed"),
    "flip_dz": (conf(0.0, fz=1.0), 1, "structured"),
    "flip_all": (conf(0.0, 1.0, 1.0, 1.0), 1, "mixed"),
    "rot90": (conf(90.0), 1, "mixed"),
    "rot180": (conf(180.0, fz=1.0), 1, "mixed"),
    "rot270": (conf(270.0, fx=1.0), 1, "mixed"),
    "rot17_3": (conf(17.3, fy=1.0), 1, "mixed"),
    "rot_neg": (conf(-33.7, 1.0, 0.0, 1.0), 1, "structured"),
    "rot_tiny": (conf(1e-9, fx=1.0), 1, "mixed"),
    "random": (dict(CONFIG_CONF, rot_lim=(-180.0, 180.0)), 3, "mixed"),
    "config": (CONFIG_CONF, 4, "mixed"),
}
CASE_SEED = {name: 7000 + 97 * i for i, name in enumerate(CASES)}


def frames(name, learning_map):
    """the case's synthetic (label bytes, invalid bytes) per sample"""
    _, n, mode = CASES[name]
    return [sk.synthetic_voxels(learning_map, CASE_SEED[name] + s, mode) for s in range(n)]


def img_inputs():
    """a stand-in for the image loader's 8-tuple (imgs, rots, trans, intrins, post_rots, post_trans, gt_depths,
    sensor2sensors): distinct tensors, to follow their positions"""
    import torch
    return tuple(torch.full((1,), float(k)) for k in range(8))


def run_case(name, make_transform, learning_map, results_of):
    """every sample of a case through one transform from the case's seed -> (results, numpy RNG state after the case)"""
    np.random.seed(CASE_SEED[name])
    t = make_transform(CASES[name][0])
    out = []
    for s, f in enumerate(frames(name, learning_map)):
        out.append(t(results_of(s, f)))
    return out, np.random.get_state()


# =============================================================================
# reference side (build container only)
# =============================================================================
def _reference_transform():
    from . import occ_targets, shim
    occ_targets._reference_transforms()  # the datasets namespace and the PIPELINES registry
    return shim.load("projects.mmdet3d_plugin.datasets.pipelines.loading_kitti_occ").LoadSemKittiAnnotation


def gen():
    """tests/golden/semkitti_train_labels.npz: the learning map; per case and sample the reference's draws (rotate,
    scale, three flips), bda_mat's float32 bits and the SHA-256 of the int64 gt_occ; the numpy RNG state after each
    case"""
    import PIL
    import torch
    torch.set_num_threads(1)
    cls = _reference_transform()
    yaml_path = sk.reference_yaml()
    lm = sk._learning_map(yaml_path)
    out = dict(learning_map=np.array(sorted(lm.items()), dtype=np.int64), cases=np.array(list(CASES)),
               pil_version=np.array(PIL.__version__), torch_version=np.array(torch.__version__))
    for name in CASES:
        fr = frames(name, lm)
        pre = sk.reference_occupancy(fr, yaml_path)  # the preprocessing script's _1_1 volumes, as int64

        def results_of(s, f):
            return dict(gt_occ=pre[s].astype(np.float32), img_inputs=img_inputs())  # np.load of the float32 .npy

        res, state = run_case(name, lambda c: cls(bda_aug_conf=c, is_train=True, point_cloud_range=KITTI_RANGE), lm,
                              results_of)
        np.random.seed(CASE_SEED[name])  # the draws alone, by the reference's own method
        t = cls(bda_aug_conf=CASES[name][0], is_train=True, point_cloud_range=KITTI_RANGE)
        draws = [t.sample_bda_augmentation() for _ in fr]
        state_d = np.random.get_state()
        assert state_d[2] == state[2] and np.array_equal(state_d[1], state[1])
        for s, (r, d) in enumerate(zip(res, draws)):
            gt = r["gt_occ"].numpy()
            assert r["gt_occ"].dtype == torch.int64 and gt.shape == sk.SHAPE
            out[f"{name}_{s}_draws"] = np.array([float(d[0]), float(d[1]), float(d[2]), float(d[3]), float(d[4])])
            out[f"{name}_{s}_rotate_type"] = np.array(type(d[0]).__name__)
            out[f"{name}_{s}_bda"] = r["img_inputs"][6].numpy().view(np.int32)
            out[f"{name}_{s}_sha"] = np.array(sha(gt))
            out[f"{name}_{s}_n255"] = np.array(int((gt == 255).sum()))
            mine = volume(*fr[s], lm, dict(rotate=d[0], flip_dx=d[2], flip_dy=d[3], flip_dz=d[4]))
            assert np.array_equal(mine, gt), f"{name} sample {s}: the restatement differs from the reference"
        out[f"{name}_rng_pos"] = np.array(state[2])
        out[f"{name}_rng_sha"] = np.array(hashlib.sha256(state[1].tobytes()).hexdigest())
        print(f"{name}: {len(res)} samples, draws {[tuple(np.round(np.asarray(d, float), 3)) for d in draws]}")
    np.savez_compressed(GOLDEN, **out)
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    from . import shim
    assert shim.reference_available(), "needs the reference checkout"
    {"gen": gen}[sys.argv[1] if len(sys.argv) > 1 else "gen"]()
