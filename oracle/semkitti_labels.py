"""TEST INFRASTRUCTURE ONLY (oracle) -- SemanticKITTI's occupancy ground truth from the voxel files, as the reference's
offline preprocessing writes it (P/tools/kitti_process/semantic_kitti_preprocess.py:117-142, with io_data's readers
and get_remap_lut, P/tools/kitti_process/io_data.py) and LoadSemKittiAnnotation turns it into int64
(P/datasets/pipelines/loading_kitti_occ.py:34-53; P/ = projects/mmdet3d_plugin/).

A numpy restatement (np.unpackbits for the invalid mask, the LUT built from the learning map), synthetic voxel files for
the tests and the benchmark, and, for the build container that has the reference checkout, the fixture generator and
the check of this restatement against the reference's preprocessing script itself (its main() run on synthetic files):

    python -m oracle.semkitti_labels gen        # tests/golden/semkitti_labels.npz
    python -m oracle.semkitti_labels validate   # this restatement == the reference script

Only the first half is imported by tests/; it needs no reference checkout.
"""
import os
import sys
import tempfile
import types

import numpy as np

SHAPE = (256, 256, 32)
NVOX = 256 * 256 * 32
GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                      "semkitti_labels.npz")


# =============================================================================
# restatement
# =============================================================================
def remap_lut(learning_map):
    """max key + 100 int32 entries: the map's value, 255 where it is 0 or missing, 0 for key 0"""
    lut = np.full(max(int(k) for k in learning_map) + 100, 255, dtype=np.int32)
    for k, v in learning_map.items():
        if int(v) != 0:
            lut[int(k)] = int(v)
    lut[0] = 0
    return lut


def occupancy(label_bytes, invalid_bytes, learning_map):
    """one frame's .label and .invalid bytes -> int64 (256, 256, 32), torch.tensor(np.load(_1_1.npy)).long() as an
    array; IndexError for a label past the LUT, as the reference"""
    label = np.frombuffer(label_bytes, dtype="<u2").astype(np.int64)
    invalid = np.unpackbits(np.frombuffer(invalid_bytes, dtype=np.uint8))  # most significant bit first
    lut = remap_lut(learning_map)
    if label.size and label.max() >= lut.size:
        raise IndexError(f"label {int(label.max())} is past the remap table's {lut.size} entries")
    out = lut[label].astype(np.int64)
    out[invalid == 1] = 255
    return out.reshape(SHAPE)


# =============================================================================
# synthetic voxel files
# =============================================================================
def synthetic_voxels(learning_map, seed, mode="mixed"):
    """(label bytes, invalid bytes) of one synthetic frame.  mixed: every learning-map key, unknown keys below the LUT
    size (up to max key + 99) and mostly-empty space, a few invalid bits; 'no_invalid' / 'all_invalid': the same labels
    with no / every invalid bit set; 'sparse': mixed in the first 1/32 of the volume, empty and valid after it;
    'structured': runs of keys, the kind of content that compresses"""
    rng = np.random.default_rng(seed)
    keys = np.array(sorted(int(k) for k in learning_map), dtype=np.int64)
    top = int(keys.max()) + 100
    if mode == "structured":
        i = np.arange(NVOX)
        label = np.where((i // 4096) % 3 == 0, 0, keys[(i // 1024) % keys.size])
        label[(i % 65536) == 7] = top - 1
        invalid = np.where((np.arange(NVOX // 8) // 512) % 5 == 0, 0x5A, 0).astype(np.uint8)
        return label.astype("<u2").tobytes(), invalid.tobytes()
    draw = rng.random(NVOX)
    label = np.where(draw < 0.6, 0, keys[rng.integers(0, keys.size, NVOX)])
    label = np.where(draw > 0.95, rng.integers(0, top, NVOX), label)
    label[:keys.size] = keys
    label[keys.size:keys.size + 100] = np.arange(top - 100, top)
    invalid = np.where(rng.random(NVOX // 8) < 0.2, rng.integers(0, 256, NVOX // 8), 0).astype(np.uint8)
    if mode == "sparse":
        label[NVOX // 32:] = 0
        invalid[NVOX // 256:] = 0
    elif mode == "no_invalid":
        invalid[:] = 0
    elif mode == "all_invalid":
        invalid[:] = 0xFF
    return label.astype("<u2").tobytes(), invalid.tobytes()


# =============================================================================
# reference (build container only)
# =============================================================================
def _reference_modules():
    """the reference's preprocessing script and io_data, imported verbatim (imageio, which io_data imports for RGB
    frames the preprocessing never reads, is stubbed when absent)"""
    from . import shim
    tools = os.path.join(shim.PLUGIN, "tools", "kitti_process")
    if "imageio" not in sys.modules:
        try:
            import imageio  # noqa: F401
        except ImportError:
            sys.modules["imageio"] = types.ModuleType("imageio")
    sys.path.insert(0, tools)
    try:
        import io_data
        import semantic_kitti_preprocess
    finally:
        sys.path.remove(tools)
    return io_data, semantic_kitti_preprocess


def reference_yaml():
    from . import shim
    return os.path.join(shim.REFERENCE_ROOT, "projects", "configs", "_base_", "semantickitti.yaml")


def reference_occupancy(frames, yaml_path):
    """frames: [(label bytes, invalid bytes)] -> the reference script's _1_1.npy of each as int64 (its main() run over
    a temporary dataset/sequences/08/voxels tree, then LoadSemKittiAnnotation's torch.tensor(...).long())"""
    import torch
    _, pre = _reference_modules()
    out = []
    with tempfile.TemporaryDirectory() as root:
        vox = os.path.join(root, "kitti", "dataset", "sequences", "08", "voxels")
        os.makedirs(vox)
        for i, (lab, inv) in enumerate(frames):
            for ext, data in ((".label", lab), (".invalid", inv)):
                with open(os.path.join(vox, f"{i:06d}{ext}"), "wb") as f:
                    f.write(data)
        cfg = types.SimpleNamespace(kitti_root=os.path.join(root, "kitti"), kitti_preprocess_root=os.path.join(root, "pre"),
                                    data_info_path=yaml_path)
        pre.main(cfg)
        for i in range(len(frames)):
            npy = np.load(os.path.join(root, "pre", "labels", "08", f"{i:06d}_1_1.npy"))
            out.append(torch.tensor(npy).long().numpy())
    return out


def _learning_map(yaml_path):
    import yaml
    with open(yaml_path) as f:
        return yaml.safe_load(f)["learning_map"]


MODES = ("structured", "sparse")


def gen():
    """tests/golden/semkitti_labels.npz: the dataset yaml's learning map, the reference's get_remap_lut, and per case
    the voxel files and the reference's volume (as uint8: every value is below 256)"""
    io_data, _ = _reference_modules()
    yaml_path = reference_yaml()
    lm = _learning_map(yaml_path)
    out = {"learning_map": np.array(sorted(lm.items()), dtype=np.int64),
           "remap_lut": io_data.get_remap_lut(yaml_path).astype(np.int32), "modes": np.array(MODES)}
    frames = [synthetic_voxels(lm, 11 + i, mode) for i, mode in enumerate(MODES)]
    for mode, (lab, inv), ref in zip(MODES, frames, reference_occupancy(frames, yaml_path)):
        assert ref.min() >= 0 and ref.max() < 256
        out[f"{mode}_label"] = np.frombuffer(lab, np.uint8)
        out[f"{mode}_invalid"] = np.frombuffer(inv, np.uint8)
        out[f"{mode}_gt"] = ref.astype(np.uint8)
    np.savez_compressed(GOLDEN, **out)
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")


def validate():
    """this restatement against the reference script on every synthetic mode and against get_remap_lut; exit status 1
    on any difference"""
    io_data, _ = _reference_modules()
    yaml_path = reference_yaml()
    lm = _learning_map(yaml_path)
    bad = int(not np.array_equal(remap_lut(lm), io_data.get_remap_lut(yaml_path)))
    print(f"{'OK ' if not bad else 'BAD'} remap LUT")
    modes = ("mixed", "no_invalid", "all_invalid", "sparse", "structured")
    frames = [synthetic_voxels(lm, 21 + i, mode) for i, mode in enumerate(modes)]
    for mode, f, ref in zip(modes, frames, reference_occupancy(frames, yaml_path)):
        n_bad = int((occupancy(*f, lm) != ref).sum())
        bad += n_bad
        print(f"{'OK ' if n_bad == 0 else 'BAD'} {mode}: {n_bad} differing voxels, {int((ref == 255).sum())} at 255")
    if bad:
        sys.exit(1)
    print("SemanticKITTI label restatement == reference preprocessing on all cases")


if __name__ == "__main__":
    from . import shim
    assert shim.reference_available(), "needs the reference checkout"
    {"gen": gen, "validate": validate}[sys.argv[1] if len(sys.argv) > 1 else "validate"]()
