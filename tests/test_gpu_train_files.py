"""Training pipelines from the dataset's own files on the H100, bit for bit: SemanticKITTI's augmented gt_occ
(targets.semantic_kitti_occupancy(..., augment=), occ_semkitti_labels_aug in csrc/semkitti_labels.cu) against the
reference's LoadSemKittiAnnotation(is_train=True) (SHA-256 in tests/golden/semkitti_train_labels.npz, voxel files
regenerated from their seeds) and the numpy restatement (oracle/semkitti_train.py); and image_prep.camera_inputs from
the training byte transforms' JPEG / PNG files against camera_inputs from the cv2-decoded frames of the same files."""
import os

import numpy as np
import pytest
import torch

from util import GOLDEN, graph_replay, misaligned, rejected, same_bits
from oracle import semkitti_labels as sk
from oracle import semkitti_train as st
from oracle import train_inputs as ti
from occformer_b200 import image_prep, ops, targets

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(GOLDEN, "semkitti_train_labels.npz")))


@pytest.fixture(scope="module")
def lm(gold):
    return {int(k): int(v) for k, v in gold["learning_map"]}


def _aug(draws):
    rotate, _, fx, fy, fz = draws
    return dict(rotate=float(rotate), flip_dx=bool(fx), flip_dy=bool(fy), flip_dz=bool(fz))


@pytest.mark.parametrize("name", list(st.CASES))
def test_volume_equals_the_fixture(cuda, gold, lm, name):
    fr = st.frames(name, lm)
    augs = [_aug(gold[f"{name}_{s}_draws"]) for s in range(len(fr))]
    n0 = ops.LAUNCH_COUNT[0]
    out = targets.semantic_kitti_occupancy([f[0] for f in fr], [f[1] for f in fr], lm, augment=augs)
    assert ops.LAUNCH_COUNT[0] - n0 == 1
    assert out.shape == (len(fr), 256, 256, 32) and out.dtype == torch.int64 and out.device == cuda
    for s, (f, a) in enumerate(zip(fr, augs)):
        got = out[s].cpu().numpy()
        assert st.sha(got) == str(gold[f"{name}_{s}_sha"]), (name, s)
        assert np.array_equal(got, st.volume(*f, lm, a)), (name, s)


def test_batch1_and_batch4_mixed(cuda, gold, lm):
    """one sample (the (256, 256, 32) form), and four samples of four augmentations in one call"""
    picks = [("rot17_3", 0), ("flip_all", 0), ("rot90", 0), ("random", 1)]
    fr = [st.frames(n, lm)[s] for n, s in picks]
    augs = [_aug(gold[f"{n}_{s}_draws"]) for n, s in picks]
    out = targets.semantic_kitti_occupancy([f[0] for f in fr], [f[1] for f in fr], lm, augment=augs).cpu().numpy()
    for b, (n, s) in enumerate(picks):
        assert st.sha(out[b]) == str(gold[f"{n}_{s}_sha"]), (n, s)
    one = targets.semantic_kitti_occupancy(fr[0][0], fr[0][1], lm, augment=augs[:1])
    assert one.shape == (256, 256, 32) and st.sha(one.cpu().numpy()) == str(gold["rot17_3_0_sha"])


def test_augment_none_is_todays_call(cuda, lm):
    fr = [sk.synthetic_voxels(lm, 60 + i, m) for i, m in enumerate(("mixed", "structured"))]
    n0 = ops.LAUNCH_COUNT[0]
    a = targets.semantic_kitti_occupancy([f[0] for f in fr], [f[1] for f in fr], lm)
    assert ops.LAUNCH_COUNT[0] - n0 == 1
    b = targets.semantic_kitti_occupancy([f[0] for f in fr], [f[1] for f in fr], lm, augment=None)
    assert torch.equal(a, b)
    lut = torch.from_numpy(targets.semkitti_remap_lut(lm)).to(cuda)
    label = torch.from_numpy(np.frombuffer(b"".join(f[0] for f in fr), np.uint8).copy()).to(cuda)
    invalid = torch.from_numpy(np.frombuffer(b"".join(f[1] for f in fr), np.uint8).copy()).to(cuda)
    vol, _ = ops.semkitti_labels(label, invalid, 2, sk.NVOX, lut)
    assert torch.equal(a.view(2, -1), vol)
    # the identity augmentation through the new entry gives the same volume
    ident = [dict(rotate=0.0, flip_dx=False, flip_dy=False, flip_dz=False)] * 2
    assert torch.equal(targets.semantic_kitti_occupancy([f[0] for f in fr], [f[1] for f in fr], lm, augment=ident), a)


def _device_inputs(cuda, lm, frames, augs):
    lut = torch.from_numpy(targets.semkitti_remap_lut(lm)).to(cuda)
    label = torch.from_numpy(np.frombuffer(b"".join(f[0] for f in frames), np.uint8).copy()).to(cuda)
    invalid = torch.from_numpy(np.frombuffer(b"".join(f[1] for f in frames), np.uint8).copy()).to(cuda)
    aug = torch.from_numpy(targets.semkitti_augment_rows(augs)).to(cuda)
    return label, invalid, aug, lut


def test_one_launch_and_graph_replay(cuda, gold, lm):
    picks = [("rot_neg", 0), ("flip_dz", 0), ("rot270", 0), ("config", 2)]
    fr = [st.frames(n, lm)[s] for n, s in picks]
    augs = [_aug(gold[f"{n}_{s}_draws"]) for n, s in picks]
    label, invalid, aug, lut = _device_inputs(cuda, lm, fr, augs)
    counts = set()
    for B in (1, 4):
        n0 = ops.LAUNCH_COUNT[0]
        ops.semkitti_labels_aug(label[:B * targets.SEMKITTI_LABEL_BYTES], invalid[:B * targets.SEMKITTI_INVALID_BYTES],
                                B, aug[:B], lut)
        counts.add(ops.LAUNCH_COUNT[0] - n0)
    assert counts == {1}
    eager, _ = ops.semkitti_labels_aug(label, invalid, 4, aug, lut)
    outs = []
    graph_replay(lambda: outs.extend(ops.semkitti_labels_aug(label, invalid, 4, aug, lut)), outs)
    vol, bad = outs
    assert int(bad.abs().sum()) == 0
    same_bits(vol, eager, "volume after graph replay")
    for b, (n, s) in enumerate(picks):
        assert st.sha(vol[b].cpu().numpy()) == str(gold[f"{n}_{s}_sha"]), (n, s)


@pytest.mark.parametrize("rotate", [0.0, 45.0])
def test_label_past_the_lut_raises(cuda, lm, rotate):
    """every voxel of the source volume is checked, also the corners a 45 degree rotation never reads"""
    lab, inv = sk.synthetic_voxels(lm, 6, "no_invalid")
    bad = np.frombuffer(lab, np.uint16).copy()
    bad[[0, sk.NVOX - 1]] = 359  # columns (0, 0) and (255, 255)
    aug = dict(rotate=rotate, flip_dx=True, flip_dy=False, flip_dz=True)
    with pytest.raises(ValueError, match=r"b\.label: 2 voxel labels are at or past the remap table's 359 entries"):
        targets.semantic_kitti_occupancy([lab, bad.tobytes()], [inv, inv], lm, augment=[aug, aug],
                                         names=[("a.label", "a.invalid"), ("b.label", "b.invalid")])
    ok = np.frombuffer(lab, np.uint16).copy()
    ok[[0, sk.NVOX - 1]] = 358  # the last in-table value is an unknown key: 255, no error
    out = targets.semantic_kitti_occupancy(ok.tobytes(), inv, lm, augment=[aug]).cpu().numpy()
    assert np.array_equal(out, st.volume(ok.tobytes(), inv, lm, aug))


def test_misaligned_inputs_are_refused(cuda, lm):
    aug0 = [dict(rotate=0.0, flip_dx=False, flip_dy=False, flip_dz=False)]
    label, invalid, aug, lut = _device_inputs(cuda, lm, [sk.synthetic_voxels(lm, 7, "sparse")], aug0)
    out = torch.zeros((1, 256, 256, 32), dtype=torch.int64, device=cuda)
    bad = torch.zeros(1, dtype=torch.int32, device=cuda)
    big = torch.zeros(label.numel() + 16, dtype=torch.uint8, device=cuda)
    rejected("occ_semkitti_labels_aug", misaligned(big), invalid, 1, aug, lut, lut.numel(), bad, out,
             buffers=(out, bad))
    inv2 = torch.zeros(invalid.numel() + 4, dtype=torch.uint8, device=cuda)
    rejected("occ_semkitti_labels_aug", label, inv2[1:], 1, aug, lut, lut.numel(), bad, out, buffers=(out, bad))
    rejected("occ_semkitti_labels_aug", label, invalid, 0, aug, lut, lut.numel(), bad, out, buffers=(out, bad))
    rejected("occ_semkitti_labels_aug", label, invalid, 1, aug, lut, 0, bad, out, buffers=(out, bad))


# ---------------------------------------------------------------------------------------------- camera files
def _collate(results, cuda):
    """the collate of img_inputs: a stacked tensor, or the list of per-sample frames of different sizes"""
    first = [r["img_inputs"][0] for r in results]
    same = len({tuple(f.shape) for f in first}) == 1
    imgs = torch.stack(first).to(cuda) if same else [f.to(cuda) for f in first]
    rest = tuple(torch.stack([r["img_inputs"][k] for r in results]).to(cuda) for k in range(1, 8))
    return (imgs,) + rest


@pytest.mark.parametrize("name", ["r50", "kitti", "small"])
def test_camera_inputs_from_files_equal_from_frames(cuda, name, tmp_path):
    """nuScenes from JPEG files, SemanticKITTI from PNG files (three frame sizes), training mode with flips and
    rotations: the same img_inputs as from the cv2-decoded frames of the same files"""
    pytest.importorskip("cv2")
    from test_cpu_train_files import camera_pipelines
    frames, _ = camera_pipelines(name, str(tmp_path), False)
    files, _ = camera_pipelines(name, str(tmp_path), True)
    assert any(any(r["img_aug"]["flip"]) for r in frames) or not ti.CASES[name][7]
    a = image_prep.camera_inputs(_collate(frames, cuda), [dict(img_aug=r["img_aug"]) for r in frames])
    fi = _collate(files, cuda)
    assert fi[0].shape[-1] == 0
    b = image_prep.camera_inputs(fi, [dict(img_aug=r["img_aug"]) for r in files])
    assert len(a) == len(b) == 8
    same_bits(b[0], a[0], f"{name}: images from files")
    same_bits(b[6], a[6], f"{name}: depth maps")
    for k in (1, 2, 3, 4, 5, 7):
        assert torch.equal(a[k], b[k])
