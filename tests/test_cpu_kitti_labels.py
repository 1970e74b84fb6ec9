"""SemanticKITTI ground truth from the voxel files, host side: the numpy restatement (oracle/semkitti_labels.py) and the
package's remap LUT against the reference's preprocessing and get_remap_lut (tests/golden/semkitti_labels.npz, written
by ``python -m oracle.semkitti_labels gen``), the loader transform, the detector's dispatch, and the C ABI entry bound
from the header."""
import os

import numpy as np
import pytest
import torch

from util import GOLDEN, FakeLibrary
from oracle import semkitti_labels as sk

KITTI_RANGE = [0, -25.6, -2, 51.2, 25.6, 4.4]


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(GOLDEN, "semkitti_labels.npz")))


def _map(gold):
    return {int(k): int(v) for k, v in gold["learning_map"]}


def _write(root, lm, label, invalid, sequence="08", frame_id="000123"):
    vox = os.path.join(root, "dataset", "sequences", sequence, "voxels")
    os.makedirs(vox, exist_ok=True)
    for ext, data in ((".label", label), (".invalid", invalid)):
        with open(os.path.join(vox, frame_id + ext), "wb") as f:
            f.write(bytes(data))
    yaml_path = os.path.join(root, "semantickitti.yaml")
    with open(yaml_path, "w") as f:
        f.write("labels:\n  0: unlabeled\nlearning_map:\n" + "".join(f"  {k}: {v}\n" for k, v in sorted(lm.items())))
    return yaml_path, os.path.join(vox, frame_id)


def test_fixture_covers_the_cases(gold):
    assert os.path.getsize(os.path.join(GOLDEN, "semkitti_labels.npz")) < 256 << 10
    assert list(gold["modes"]) == list(sk.MODES)
    lm = _map(gold)
    assert len(lm) == 34 and max(lm) == 259 and gold["remap_lut"].size == 359
    for mode in sk.MODES:
        assert gold[f"{mode}_label"].size == 2 * sk.NVOX and gold[f"{mode}_invalid"].size == sk.NVOX // 8
        gt = gold[f"{mode}_gt"]
        assert (gt == 255).any() and (gt == 0).any() and set(np.unique(gt)) - {0, 255}


def test_remap_lut_equals_reference(gold):
    from occformer_b200 import targets
    lut = targets.semkitti_remap_lut(_map(gold))
    assert lut.dtype == np.int32 and np.array_equal(lut, gold["remap_lut"])
    assert np.array_equal(sk.remap_lut(_map(gold)), gold["remap_lut"])
    # the rules: key 0 stays 0, keys mapped to 0 and keys the map lacks become 255
    assert lut[0] == 0 and lut[1] == 255 and lut[52] == 255 and lut[2] == 255 and lut[10] == 1 and lut[358] == 255
    with pytest.raises(ValueError, match="keys"):
        targets.semkitti_remap_lut({-1: 3, 0: 0})


@pytest.mark.parametrize("mode", sk.MODES)
def test_restatement_matches_reference(gold, mode):
    got = sk.occupancy(gold[f"{mode}_label"].tobytes(), gold[f"{mode}_invalid"].tobytes(), _map(gold))
    assert got.dtype == np.int64 and got.shape == (256, 256, 32)
    assert np.array_equal(got, gold[f"{mode}_gt"].astype(np.int64))


def test_restatement_label_past_the_lut_raises(gold):
    label, invalid = sk.synthetic_voxels(_map(gold), 3, "no_invalid")
    lab = np.frombuffer(label, np.uint16).copy()
    lab[12345] = 359
    with pytest.raises(IndexError):
        sk.occupancy(lab.tobytes(), invalid, _map(gold))
    lab[12345] = 358  # the last entry: an unknown key, 255
    assert sk.occupancy(lab.tobytes(), invalid, _map(gold)).reshape(-1)[12345] == 255


def test_transform_reads_the_voxel_files(gold, tmp_path):
    from occformer_b200 import PIPELINES
    from occformer_b200.pipelines import LoadSemKittiVoxelFiles
    lm = _map(gold)
    label, invalid = gold["sparse_label"].tobytes(), gold["sparse_invalid"].tobytes()
    yaml_path, base = _write(str(tmp_path), lm, label, invalid)
    t = PIPELINES.build(dict(type="LoadSemKittiVoxelFiles", data_root=str(tmp_path), data_info_path=yaml_path))
    assert isinstance(t, LoadSemKittiVoxelFiles)
    npy = np.zeros((256, 256, 32), np.float32)  # what the dataset loads when the preprocessed labels exist
    out = t(dict(sequence="08", frame_id="000123", gt_occ=npy, img_inputs=()))
    assert out["gt_occ"] is None
    vox = out["semkitti_voxels"]
    assert vox["label"] == label and vox["invalid"] == invalid
    assert vox["files"] == [base + ".label", base + ".invalid"] and vox["learning_map"] == lm
    # the reference's test-mode annotation path then runs as it does for the test-submission split
    assert t(dict(sequence="08", frame_id="000123", gt_occ=None))["gt_occ"] is None


@pytest.mark.parametrize("which", [".label", ".invalid"])
def test_transform_refuses_wrong_file_sizes(gold, tmp_path, which):
    from occformer_b200.pipelines import LoadSemKittiVoxelFiles
    label, invalid = gold["sparse_label"].tobytes(), gold["sparse_invalid"].tobytes()
    if which == ".label":
        label = label[:-2]
    else:
        invalid = invalid + b"\0"
    yaml_path, base = _write(str(tmp_path), _map(gold), label, invalid)
    t = LoadSemKittiVoxelFiles(data_root=str(tmp_path), data_info_path=yaml_path)
    with pytest.raises(ValueError, match=base + which):
        t(dict(sequence="08", frame_id="000123", gt_occ=None))


def test_transform_refuses_training_mode(gold, tmp_path):
    from occformer_b200 import PIPELINES
    yaml_path, _ = _write(str(tmp_path), _map(gold), b"", b"")
    with pytest.raises(ValueError, match="is_train=True"):
        PIPELINES.build(dict(type="LoadSemKittiVoxelFiles", data_root=str(tmp_path), data_info_path=yaml_path,
                             is_train=True))


def test_header_entry_bound():
    from occformer_b200 import _lib
    params = _lib.parameters()
    assert params["occ_semkitti_labels"] == [("label", "unsigned char"), ("invalid", "unsigned char"), ("B", None),
                                             ("nvox", None), ("lut", "int"), ("lut_size", None), ("bad", "int"),
                                             ("out", "long long"), ("stream", None)]


def test_wrong_sizes_and_cpu_raise_before_the_device(gold, monkeypatch):
    from occformer_b200 import ops, targets
    fake = FakeLibrary()
    monkeypatch.setattr(ops, "lib", lambda: fake)
    lm = _map(gold)
    label, invalid = gold["sparse_label"].tobytes(), gold["sparse_invalid"].tobytes()
    names = [("frame_a.label", "frame_a.invalid")]
    with pytest.raises(ValueError, match=r"frame_a\.label: a \.label file holds 4194304 bytes, got 4194302"):
        targets.semantic_kitti_occupancy([label[:-2]], [invalid], lm, names=names)
    with pytest.raises(ValueError, match=r"frame_a\.invalid: a \.invalid file holds 262144 bytes, got 262143"):
        targets.semantic_kitti_occupancy([label], [invalid[:-1]], lm, names=names)
    with pytest.raises(ValueError, match=r"sample 1: a \.invalid file"):
        targets.semantic_kitti_occupancy([label, label], [invalid, invalid[:-1]], lm)
    with pytest.raises(ValueError, match="pairs"):
        targets.semantic_kitti_occupancy([label], [invalid], lm, names=["frame_a.label"])
    with pytest.raises(ValueError, match="one .label and one .invalid"):
        targets.semantic_kitti_occupancy([label], [], lm)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        targets.semantic_kitti_occupancy(label, invalid, lm)
    with pytest.raises(RuntimeError, match=r"occ_semkitti_labels\(label\) must be a CUDA tensor"):
        ops.semkitti_labels(torch.zeros(16, dtype=torch.uint8), torch.zeros(1, dtype=torch.uint8), 1, 8,
                            torch.zeros(4, dtype=torch.int32))
    assert fake.calls == []


def _kitti_model():
    from occformer_b200 import Mask2FormerOccHead, OccupancyFormer
    from occformer_b200.head import head_cfg
    model = OccupancyFormer(None, None, None)
    model.pts_bbox_head = Mask2FormerOccHead(**head_cfg(96, 12, 20, 3, 3, KITTI_RANGE, ffn=192))
    return model


def test_detector_targets_from_the_voxel_files(gold, monkeypatch):
    """batch 2: one call with both samples' files, named by their paths; without the metas the KITTI head still
    asks for gt_occ; differing learning maps raise"""
    from occformer_b200 import targets
    model = _kitti_model()
    calls = []
    monkeypatch.setattr(targets, "semantic_kitti_occupancy", lambda *a, **k: calls.append((a, k)) or "volume")
    lm = _map(gold)
    metas = [dict(occ_size=[256, 256, 32], pc_range=KITTI_RANGE,
                  semkitti_voxels=dict(label=f"L{b}", invalid=f"I{b}", files=[f"f{b}.label", f"f{b}.invalid"],
                                       learning_map=lm)) for b in range(2)]
    assert model.occupancy_targets(None, metas) == "volume"
    ((labels, invalids, learning_map), kw), = calls
    assert labels == ["L0", "L1"] and invalids == ["I0", "I1"] and learning_map is lm
    assert kw == dict(names=[["f0.label", "f0.invalid"], ["f1.label", "f1.invalid"]])
    with pytest.raises(NotImplementedError, match="pass gt_occ"):
        model.occupancy_targets(None, [dict(occ_size=[256, 256, 32], pc_range=KITTI_RANGE)])
    with pytest.raises(NotImplementedError, match="pass gt_occ"):
        model.occupancy_targets(None, metas[:1] + [dict(occ_size=[256, 256, 32], pc_range=KITTI_RANGE)])
    metas[1]["semkitti_voxels"] = dict(metas[1]["semkitti_voxels"], learning_map={**lm, 1: 1})
    with pytest.raises(ValueError, match="same learning map"):
        model.occupancy_targets(None, metas)
