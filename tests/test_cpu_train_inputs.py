"""The training pipelines' camera inputs on the host: the numpy restatement (oracle/train_inputs.py) against Pillow and
against the reference transforms' fixture (tests/golden/train_inputs.npz), the package's rotation coefficients against
it, and the new loader transforms (LoadMultiViewImageFramesAug_*, LoadLidarDepthPoints) against the fixture: the same
draws in the same order, the same img_inputs bits and the same scan."""
import hashlib
import os

import numpy as np
import pytest
import torch

from util import GOLDEN
from oracle import image_prep as ip
from oracle import train_inputs as ti
from occformer_b200 import image_prep

FIXTURE = os.path.join(GOLDEN, "train_inputs.npz")


def _sweep():
    """(frame H, W, resize (W', H'), crop box, flip, angle): the configs' geometries, crops past every edge (KITTI's
    negative crop_h where the resized frame is shorter than the crop, nuScenes' narrower resized frame), square and
    non-square crops at the angles where Pillow copies or transposes, and seeded angles in +-5.4 and the full circle"""
    geo = [(900, 1600, (704, 396), (0, 140, 704, 396)), (900, 1600, (1717, 965), (13, 69, 1613, 965)),
           (376, 1241, (1241, 376), (-19, -8, 1261, 376)), (370, 1226, (1200, 362), (0, -22, 1280, 362)),
           (90, 160, (66, 37), (-3, -11, 69, 37)), (50, 50, (50, 50), (0, 0, 50, 50)), (40, 70, (70, 40), (9, 0, 49, 40)),
           (37, 53, (53, 37), (0, 0, 53, 37))]
    out = []
    rng = np.random.default_rng(11)
    for i, g in enumerate(geo):
        angles = [0.0, 180.0, 90.0, -90.0, 270.0, 360.0, -180.0] if i >= 5 else [0.0]
        angles += [float(a) for a in rng.uniform(-5.4, 5.4, 2)] + [float(rng.uniform(-180.0, 180.0))]
        for j, a in enumerate(angles):
            out.append(g + (bool((i + j) % 2), a))
    return out


SWEEP = _sweep()


@pytest.mark.parametrize("i", range(len(SWEEP)))
def test_restatement_equals_pillow(i):
    Image = pytest.importorskip("PIL.Image")
    H, W, size, box, flip, angle = SWEEP[i]
    f = ip.frame(700 + i, H, W)
    img = Image.fromarray(f).resize(size).crop(box)
    if flip:
        img = img.transpose(method=Image.FLIP_LEFT_RIGHT)
    ref = np.asarray(img.rotate(angle))
    assert np.array_equal(ti.augment_uint8(f, size, box, flip, angle), ref)


def _gather(img, flip, a):
    """the device's read of a (mirrored) crop through the package's coefficients"""
    h, w = img.shape[:2]
    y, x = np.arange(h)[:, None], np.arange(w)[None, :]
    xs, ys = (a[2] + y * a[1] + x * a[0]) >> 16, (a[5] + y * a[4] + x * a[3]) >> 16
    ok = (xs >= 0) & (xs < w) & (ys >= 0) & (ys < h)
    xs = np.where(flip, w - 1 - xs, xs)
    out = img[np.clip(ys, 0, h - 1), np.clip(xs, 0, w - 1)]
    out[~ok] = 0
    return out


@pytest.mark.parametrize("i", range(len(SWEEP)))
def test_package_coefficients_equal_the_restatement(i):
    H, W, size, box, flip, angle = SWEEP[i]
    crop = ip.crop(ip.resize(ip.frame(700 + i, H, W), size), box)
    a = image_prep.rotate_coeffs(angle, crop.shape[1], crop.shape[0])
    assert all(isinstance(v, int) and -(1 << 31) <= v < (1 << 31) for v in a)
    ref = ti.rotate(crop[:, ::-1] if flip else crop, angle)
    assert np.array_equal(_gather(crop, flip, a), ref)


def test_rotate_coeffs_refuses_what_pillow_interpolates_in_float():
    with pytest.raises(ValueError, match="fixed-point"):
        image_prep.rotate_coeffs(45.0, 30000, 30000)


def test_fixture_records_versions():
    g = np.load(FIXTURE)
    assert str(g["pil_version"]) and str(g["torch_version"])
    assert os.path.getsize(FIXTURE) < 1 << 20


def _rng_matches(g, name, state):
    assert int(g[f"{name}_rng_pos"]) == state[2]
    assert str(g[f"{name}_rng_sha"]) == hashlib.sha256(state[1].tobytes()).hexdigest()


@pytest.mark.parametrize("name", list(ti.CASES))
def test_restatement_equals_the_fixture(name):
    """the oracle's draws, images and depth maps against the reference's, from the fixture's seed"""
    g = np.load(FIXTURE)
    kind, B, ncam, Ncams, shapes, size, norm = ti.CASES[name][:7]
    draws, state = ti.oracle_case(name)
    _rng_matches(g, name, state)
    for s, (cams, dr) in enumerate(draws):
        assert cams == g[f"{name}_{s}_cams"].tolist()
        frames = ti.case_frames(name, s)
        pts = ti.scan(name, s)
        rots, trans, intrins, post_rots, post_trans = (g[f"{name}_{s}_in{k}"] for k in range(1, 6))
        inv = torch.from_numpy(rots).inverse().numpy()
        for j, (c, (_, dims, box, flip, rot)) in enumerate(zip(cams, dr)):
            img = ti.augment(frames[c], dims, box, flip, rot, norm or ip.NORM_R50)
            assert ti.sha(img) == str(g[f"{name}_{s}_img_sha"][j]), (name, s, j)
            d = ti.depth_map(pts, inv[j], trans[j], intrins[j], post_rots[j], post_trans[j], *size)
            assert ti.sha(d) == str(g[f"{name}_{s}_depth_sha"][j]), (name, s, j)
            assert int((d > 0).sum()) == int(g[f"{name}_{s}_depth_valid"][j]) > 0


@pytest.mark.parametrize("name", list(ti.CASES))
def test_new_transforms_equal_the_fixture(name, tmp_path):
    pytest.importorskip("cv2")
    from occformer_b200.pipelines import (LoadLidarDepthPoints, LoadMultiViewImageFramesAug_OccFormer,
                                          LoadMultiViewImageFramesAug_SemanticKitti)
    g = np.load(FIXTURE)
    kind = ti.CASES[name][0]
    cls = LoadMultiViewImageFramesAug_SemanticKitti if kind == "kitti" else LoadMultiViewImageFramesAug_OccFormer
    loaders = [cls(**ti.transform_kwargs(name)), LoadLidarDepthPoints(data_root=str(tmp_path), dataset=kind)]
    res, state = ti.run_case(name, loaders, str(tmp_path))
    _rng_matches(g, name, state)
    draws, _ = ti.oracle_case(name)
    for s, (r, (cams, dr)) in enumerate(zip(res, draws)):
        imgs, aug = r["img_inputs"], r["img_aug"]
        assert len(imgs) == 8 and imgs[0].dtype == torch.uint8
        frames = ti.case_frames(name, s)
        assert np.array_equal(imgs[0].numpy(), np.stack([frames[c] for c in cams]))
        for k in range(1, 6):
            ref = g[f"{name}_{s}_in{k}"]
            assert imgs[k].dtype == torch.float32 and np.array_equal(imgs[k].numpy(), ref), (name, s, k)
        assert torch.equal(imgs[6], torch.zeros(len(cams), 1))
        assert aug["resize_dims"] == [list(d[1]) for d in dr] and aug["crop"] == [list(d[2]) for d in dr]
        assert aug["flip"] == [d[3] for d in dr] and aug["rotate"] == [d[4] for d in dr]
        assert np.array_equal(aug["lidar_points"].numpy(), ti.scan(name, s), equal_nan=True)
        assert torch.equal(aug["lidar_inv_rots"], imgs[1].inverse())
        if kind != "kitti":
            assert [ip.NUSC_CAMS.index(c) for c in r["cam_names"]] == cams


def test_flip_draw_is_skipped_without_flip():
    """data_config['flip'] False: four draws per camera, not five"""
    assert ti.CASES["small"][7] is False
    _, state = ti.oracle_case("small")
    np.random.seed(ti.CASE_SEED["small"])
    np.random.choice(5, 3, replace=False)
    np.random.uniform(size=4 * 3)
    np.random.choice(5, 3, replace=False)
    np.random.uniform(size=4 * 3)
    assert np.random.get_state()[2] == state[2] and np.array_equal(np.random.get_state()[1], state[1])


def test_refusals():
    from occformer_b200.pipelines import (LoadLidarDepthPoints, LoadMultiViewImageFrames_OccFormer,
                                          LoadMultiViewImageFramesAug_OccFormer,
                                          LoadMultiViewImageFramesAug_SemanticKitti)
    for cls in (LoadMultiViewImageFramesAug_OccFormer, LoadMultiViewImageFramesAug_SemanticKitti):
        with pytest.raises(ValueError, match="is_train=False.*LoadMultiViewImageFrames_"):
            cls(**ti.transform_kwargs("kitti", is_train=False))
        cls(**ti.transform_kwargs("kitti"))
    with pytest.raises(ValueError, match="LoadMultiViewImageFramesAug_OccFormer"):
        LoadMultiViewImageFrames_OccFormer(**ti.transform_kwargs("r50"))
    with pytest.raises(ValueError, match="dataset"):
        LoadLidarDepthPoints(dataset="waymo")


def test_camera_inputs_checks_its_metas():
    with pytest.raises(ValueError, match="img_aug metas"):
        image_prep.lidar_depth_maps([np.zeros((4, 3), np.float32)], [None] * 8, [])
    aug = dict(resize_dims=[[72, 48]], crop=[[0, 0, 72, 48]], input_size=[48, 72], flip=[False], rotate=[0.0],
               **image_prep.norm_config(None))
    with pytest.raises(ValueError, match="mixes"):
        image_prep.prepare_images([torch.zeros(1, 48, 72, 3, dtype=torch.uint8)] * 2,
                                  [aug, {k: v for k, v in aug.items() if k not in ("flip", "rotate")}])
