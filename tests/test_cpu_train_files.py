"""Training pipelines from the dataset's own files, host side: the numpy restatement of LoadSemKittiAnnotation's
training-mode volume (oracle/semkitti_train.py) against the reference's (tests/golden/semkitti_train_labels.npz,
written by ``python -m oracle.semkitti_train gen``) and against the installed Pillow; LoadSemKittiVoxelFilesAug's draws,
bda_mat and img_inputs; the byte transforms' training twins against the frame transforms; the refusals; and the C ABI
entry bound from the header."""
import hashlib
import os

import numpy as np
import pytest
import torch

from util import GOLDEN, FakeLibrary
from oracle import semkitti_labels as sk
from oracle import semkitti_train as st
from oracle import train_inputs as ti

FIXTURE = os.path.join(GOLDEN, "semkitti_train_labels.npz")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(FIXTURE))


def _map(gold):
    return {int(k): int(v) for k, v in gold["learning_map"]}


def _aug(draws):
    rotate, _, fx, fy, fz = draws
    return dict(rotate=float(rotate), flip_dx=bool(fx), flip_dy=bool(fy), flip_dz=bool(fz))


def _rng_matches(gold, name, state):
    assert int(gold[f"{name}_rng_pos"]) == state[2]
    assert str(gold[f"{name}_rng_sha"]) == hashlib.sha256(state[1].tobytes()).hexdigest()


def test_fixture_covers_the_cases(gold):
    assert os.path.getsize(FIXTURE) < 64 << 10
    assert list(gold["cases"]) == list(st.CASES)
    d = {name: gold[f"{name}_0_draws"] for name in st.CASES}
    assert d["none"][[0, 2, 3, 4]].tolist() == [0, 0, 0, 0] and d["flip_all"][2:].tolist() == [1, 1, 1]
    for name, k in (("flip_dx", 2), ("flip_dy", 3), ("flip_dz", 4)):
        assert d[name][2:].tolist() == [float(j == k) for j in (2, 3, 4)]
    assert [d[n][0] for n in ("rot90", "rot180", "rot270", "rot17_3", "rot_neg", "rot_tiny")] == [
        90.0, 180.0, 270.0, 17.3, -33.7, 1e-9]
    # the arbitrary angles leave voxels outside the slice at 255; the tiny one is not rotated at all
    assert int(gold["rot17_3_0_n255"]) > int(gold["none_0_n255"])
    lab, inv = st.frames("rot_tiny", _map(gold))[0]
    unrotated = st.volume(lab, inv, _map(gold), dict(rotate=0.0, flip_dx=True, flip_dy=False, flip_dz=False))
    assert st.sha(unrotated) == str(gold["rot_tiny_0_sha"])
    assert str(gold["rot17_3_0_rotate_type"]) == "float"


@pytest.mark.parametrize("name", list(st.CASES))
def test_restatement_equals_the_fixture(gold, name):
    lm = _map(gold)
    for s, (lab, inv) in enumerate(st.frames(name, lm)):
        got = st.volume(lab, inv, lm, _aug(gold[f"{name}_{s}_draws"]))
        assert got.dtype == np.int64 and got.shape == sk.SHAPE
        assert st.sha(got) == str(gold[f"{name}_{s}_sha"]), (name, s)


@pytest.mark.parametrize("angle", [17.3, -33.7, 90.0, 180.0, 270.0, -90.0, 45.0, 359.99, 0.004, 360.0])
def test_slice_rotation_equals_pillow(angle):
    from PIL import Image
    rng = np.random.default_rng(int(abs(angle) * 100))
    vol = rng.integers(0, 21, (256, 256, 4)).astype(np.uint8)
    got = st.rotate_slices(vol, angle)
    for z in range(vol.shape[2]):
        ref = np.array(Image.fromarray(vol[..., z]).rotate(angle, resample=Image.Resampling.NEAREST, fillcolor=255))
        assert np.array_equal(got[..., z], ref), (angle, z)


def _write(root, lm, frames):
    """the samples' voxel files as dataset/sequences/08/voxels/{frame_id} under root and the yaml -> (yaml path, results
    per sample)"""
    vox = os.path.join(root, "dataset", "sequences", "08", "voxels")
    os.makedirs(vox, exist_ok=True)
    results = []
    for s, (lab, inv) in enumerate(frames):
        for ext, data in ((".label", lab), (".invalid", inv)):
            with open(os.path.join(vox, f"{s:06d}{ext}"), "wb") as f:
                f.write(data)
        results.append(dict(sequence="08", frame_id=f"{s:06d}", gt_occ=np.zeros(1), img_inputs=st.img_inputs()))
    yaml_path = os.path.join(root, "semantickitti.yaml")
    with open(yaml_path, "w") as f:
        f.write("learning_map:\n" + "".join(f"  {k}: {v}\n" for k, v in sorted(lm.items())))
    return yaml_path, results


@pytest.mark.parametrize("name", list(st.CASES))
def test_voxel_files_aug_equals_the_fixture(gold, name, tmp_path):
    """the reference's draws in its order, its bda_mat bits, the 9-tuple and the RNG state after the case"""
    from occformer_b200 import PIPELINES
    from occformer_b200.pipelines import LoadSemKittiVoxelFilesAug
    lm = _map(gold)
    yaml_path, results = _write(str(tmp_path), lm, st.frames(name, lm))

    def make(conf):
        return PIPELINES.build(dict(type="LoadSemKittiVoxelFilesAug", bda_aug_conf=conf, is_train=True,
                                    point_cloud_range=st.KITTI_RANGE, data_root=str(tmp_path),
                                    data_info_path=yaml_path))

    res, state = st.run_case(name, make, lm, lambda s, f: dict(results[s]))
    _rng_matches(gold, name, state)
    for s, r in enumerate(res):
        assert isinstance(make(st.CONFIG_CONF), LoadSemKittiVoxelFilesAug)
        assert r["gt_occ"] is None
        vox = r["semkitti_voxels"]
        assert vox["augment"] == _aug(gold[f"{name}_{s}_draws"])
        assert vox["learning_map"] == lm and vox["files"][0].endswith(f"08/voxels/{s:06d}.label")
        lab, inv = st.frames(name, lm)[s]
        assert vox["label"] == lab and vox["invalid"] == inv
        imgs = r["img_inputs"]
        assert len(imgs) == 9 and [float(imgs[k]) for k in (0, 1, 2, 3, 4, 5, 7, 8)] == [0, 1, 2, 3, 4, 5, 6, 7]
        bda = imgs[6]
        assert bda.dtype == torch.float32 and bda.shape == (4, 4)
        assert np.array_equal(bda.numpy().view(np.int32), gold[f"{name}_{s}_bda"]), (name, s)


def test_voxel_files_aug_defaults(gold, tmp_path):
    """the reference's default point_cloud_range"""
    from occformer_b200.pipelines import LoadSemKittiVoxelFilesAug, semkitti_bda_matrix
    yaml_path, _ = _write(str(tmp_path), _map(gold), [])
    t = LoadSemKittiVoxelFilesAug(bda_aug_conf=st.CONFIG_CONF, data_info_path=yaml_path)
    assert t.point_cloud_range == st.KITTI_RANGE and t.is_train
    g = gold["rot17_3_0_bda"]
    assert np.array_equal(semkitti_bda_matrix(17.3, False, True, False, t.point_cloud_range).numpy().view(np.int32), g)


def _camera_results(name, s, root, jpeg):
    """sample s of a train_inputs case written under root (camera files as JPEG when jpeg, else PNG) -> results"""
    import cv2
    r = ti.write_results(root, name, s, ti.case_frames(name, s), ti.scan(name, s))
    if jpeg:
        for cam in r["curr"]["cams"].values():
            path = cam["data_path"][:-4] + ".jpg"
            cv2.imwrite(path, cv2.imread(cam["data_path"], cv2.IMREAD_UNCHANGED), [cv2.IMWRITE_JPEG_QUALITY, 93])
            cam["data_path"] = path
    return r


def camera_pipelines(name, root, bytes_transform):
    """every sample of a train_inputs case through the training frame transform or its byte twin, then
    LoadLidarDepthPoints, from the case's seed -> (results, numpy RNG state after the case)"""
    from occformer_b200 import PIPELINES
    kind = ti.CASES[name][0]
    frames_t = "LoadMultiViewImageFramesAug_" + ("SemanticKitti" if kind == "kitti" else "OccFormer")
    bytes_t = "LoadMultiViewPngBytesAug_SemanticKitti" if kind == "kitti" else "LoadMultiViewJpegBytesAug_OccFormer"
    loaders = [PIPELINES.build(dict(type=bytes_t if bytes_transform else frames_t, **ti.transform_kwargs(name))),
               PIPELINES.build(dict(type="LoadLidarDepthPoints", data_root=root, dataset=kind))]
    np.random.seed(ti.CASE_SEED[name])
    out = []
    for s in range(ti.CASES[name][1]):
        r = _camera_results(name, s, root, kind != "kitti")
        for t in loaders:
            r = t(r)
        out.append(r)
    return out, np.random.get_state()


@pytest.mark.parametrize("name", list(ti.CASES))
def test_byte_transforms_draw_as_the_frame_transforms(name, tmp_path):
    pytest.importorskip("cv2")
    a, sa = camera_pipelines(name, str(tmp_path), False)
    b, sb = camera_pipelines(name, str(tmp_path), True)
    assert sa[2] == sb[2] and np.array_equal(sa[1], sb[1])
    kind = ti.CASES[name][0]
    key = "png" if kind == "kitti" else "jpeg"
    for ra, rb in zip(a, b):
        ia, ib = ra["img_inputs"], rb["img_inputs"]
        assert len(ib) == 8 and ib[0].dtype == torch.uint8 and tuple(ib[0].shape) == (ia[0].shape[0], 0)
        for k in range(1, 8):
            assert ia[k].dtype == ib[k].dtype and torch.equal(ia[k], ib[k]), (name, k)
        aug = dict(rb["img_aug"])
        files = aug.pop(key)
        paths = aug.pop(key + "_files")
        assert len(files) == len(paths) == ia[0].shape[0]
        for f, p in zip(files, paths):
            with open(p, "rb") as fh:
                assert fh.read() == f
        for k in ("lidar_points", "lidar_inv_rots"):
            assert np.array_equal(aug.pop(k).numpy(), ra["img_aug"][k].numpy(), equal_nan=True)  # the scans hold NaN
        assert aug == {k: v for k, v in ra["img_aug"].items() if k not in ("lidar_points", "lidar_inv_rots")}
        assert "flip" in aug and "rotate" in aug
        if kind != "kitti":
            assert list(ra["cam_names"]) == list(rb["cam_names"])
        else:
            assert "raw_img" not in rb


def test_refusals(gold, tmp_path):
    from occformer_b200 import PIPELINES
    yaml_path, _ = _write(str(tmp_path), _map(gold), [])
    with pytest.raises(ValueError, match="LoadSemKittiVoxelFilesAug: is_train=False"):
        PIPELINES.build(dict(type="LoadSemKittiVoxelFilesAug", bda_aug_conf=st.CONFIG_CONF, is_train=False,
                             data_info_path=yaml_path))
    with pytest.raises(ValueError, match="is_train=True"):
        PIPELINES.build(dict(type="LoadSemKittiVoxelFiles", data_info_path=yaml_path, is_train=True))
    for t in ("LoadMultiViewJpegBytesAug_OccFormer", "LoadMultiViewPngBytesAug_SemanticKitti"):
        with pytest.raises(ValueError, match="is_train=False"):
            PIPELINES.build(dict(type=t, **ti.transform_kwargs("kitti", is_train=False)))
    for t in ("LoadMultiViewJpegBytes_OccFormer", "LoadMultiViewPngBytes_SemanticKitti"):
        with pytest.raises(ValueError, match="is_train=True"):
            PIPELINES.build(dict(type=t, **ti.transform_kwargs("kitti")))


def test_voxel_files_aug_refuses_wrong_file_sizes(gold, tmp_path):
    from occformer_b200.pipelines import LoadSemKittiVoxelFilesAug
    lab, inv = st.frames("none", _map(gold))[0]
    yaml_path, results = _write(str(tmp_path), _map(gold), [(lab[:-2], inv)])
    t = LoadSemKittiVoxelFilesAug(bda_aug_conf=st.CONFIG_CONF, data_root=str(tmp_path), data_info_path=yaml_path)
    with pytest.raises(ValueError, match=r"000000\.label"):
        t(results[0])


def test_header_entry_bound():
    from occformer_b200 import _lib
    assert _lib.parameters()["occ_semkitti_labels_aug"] == [
        ("label", "unsigned char"), ("invalid", "unsigned char"), ("B", None), ("aug", "int"), ("lut", "int"),
        ("lut_size", None), ("bad", "int"), ("out", "long long"), ("stream", None)]


def test_augment_rows():
    from occformer_b200 import image_prep, targets
    rows = targets.semkitti_augment_rows([dict(rotate=0.0, flip_dx=True, flip_dy=False, flip_dz=True),
                                          dict(rotate=1e-9, flip_dx=False, flip_dy=True, flip_dz=False),
                                          dict(rotate=-33.7, flip_dx=False, flip_dy=False, flip_dz=False),
                                          dict(rotate=90.0, flip_dx=False, flip_dy=False, flip_dz=False)])
    one = 1 << 16
    assert rows.dtype == np.int32 and rows.shape == (4, 10)
    assert rows[0].tolist() == [1, 0, 1, 0, one, 0, 0, 0, one, 0]
    assert rows[1].tolist() == [0, 1, 0, 0, one, 0, 0, 0, one, 0]   # np.isclose(1e-9, 0): no rotation
    assert rows[2, :4].tolist() == [0, 0, 0, 1] and tuple(rows[2, 4:]) == image_prep.rotate_coeffs(-33.7, 256, 256)
    assert tuple(rows[3, 4:]) == (0, -one, 255 << 16, one, 0, 0)     # Pillow's transpose


def test_wrong_sizes_and_cpu_raise_before_the_device(gold, monkeypatch):
    from occformer_b200 import image_prep, ops, targets
    fake = FakeLibrary()
    monkeypatch.setattr(ops, "lib", lambda: fake)
    lm = _map(gold)
    lab, inv = st.frames("none", lm)[0]
    aug = dict(rotate=0.0, flip_dx=False, flip_dy=False, flip_dz=False)
    with pytest.raises(ValueError, match="one dict per sample"):
        targets.semantic_kitti_occupancy([lab], [inv], lm, augment=[aug, aug])
    with pytest.raises(ValueError, match=r"\[0, 255\]"):
        targets.semantic_kitti_occupancy([lab], [inv], {**lm, 10: 300}, augment=[aug])
    with pytest.raises(ValueError, match=r"frame_a\.label: a \.label file"):
        targets.semantic_kitti_occupancy([lab[:-2]], [inv], lm, names=[("frame_a.label", "frame_a.invalid")],
                                         augment=[aug])
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        targets.semantic_kitti_occupancy(lab, inv, lm, augment=[aug])
    lut = torch.zeros(359, dtype=torch.int32)
    with pytest.raises(RuntimeError, match=r"occ_semkitti_labels_aug\(label\) must be a CUDA tensor"):
        ops.semkitti_labels_aug(torch.zeros(sk.NVOX * 2, dtype=torch.uint8), torch.zeros(sk.NVOX // 8, dtype=torch.uint8),
                                1, torch.zeros(10, dtype=torch.int32), lut)
    with pytest.raises(RuntimeError, match="B = 2 needs"):
        ops.semkitti_labels_aug(torch.zeros(sk.NVOX * 2, dtype=torch.uint8), torch.zeros(sk.NVOX // 8, dtype=torch.uint8),
                                2, torch.zeros(20, dtype=torch.int32), lut)
    with pytest.raises(ValueError, match="placeholder"):
        image_prep.camera_inputs((torch.zeros(1, 1, 0, dtype=torch.uint8),), [dict(img_aug={})])
    assert fake.calls == []


def test_detector_targets_take_the_augmentation(gold, monkeypatch):
    """the training transform's 'augment' reaches semantic_kitti_occupancy; the test transform's metas call it as
    before; a batch mixing both raises"""
    from test_cpu_kitti_labels import KITTI_RANGE, _kitti_model
    from occformer_b200 import targets
    model = _kitti_model()
    calls = []
    monkeypatch.setattr(targets, "semantic_kitti_occupancy", lambda *a, **k: calls.append((a, k)) or "volume")
    lm = _map(gold)
    augs = [dict(rotate=17.3, flip_dx=True, flip_dy=False, flip_dz=False),
            dict(rotate=0.0, flip_dx=False, flip_dy=False, flip_dz=True)]
    metas = [dict(occ_size=[256, 256, 32], pc_range=KITTI_RANGE,
                  semkitti_voxels=dict(label=f"L{b}", invalid=f"I{b}", files=[f"f{b}.label", f"f{b}.invalid"],
                                       learning_map=lm, augment=augs[b])) for b in range(2)]
    assert model.occupancy_targets(None, metas) == "volume"
    ((labels, invalids, learning_map), kw), = calls
    assert labels == ["L0", "L1"] and learning_map is lm
    assert kw == dict(names=[["f0.label", "f0.invalid"], ["f1.label", "f1.invalid"]], augment=augs)
    plain = dict(metas[1], semkitti_voxels={k: v for k, v in metas[1]["semkitti_voxels"].items() if k != "augment"})
    with pytest.raises(ValueError, match="mixes"):
        model.occupancy_targets(None, [metas[0], plain])
