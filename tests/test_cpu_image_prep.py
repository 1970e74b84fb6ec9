"""The image side of the test loaders on the host: the numpy restatement (oracle/image_prep.py) against Pillow and
OpenCV bit for bit, the package's coefficient and normalisation tables against it, and the new loader transforms
(occformer_b200.pipelines) against the reference transforms' fixture (tests/golden/image_prep.npz)."""
import os

import numpy as np
import pytest
import torch

from util import GOLDEN
from oracle import image_prep as ip
from occformer_b200 import image_prep

FIXTURE = os.path.join(GOLDEN, "image_prep.npz")


def _sweep():
    """(source H, W, resize (W', H'), crop box) of the configs and a seeded sweep, every axis downscaled by at most 32
    (the kernel's bound; test_gpu_image_prep checks that a larger one is refused)"""
    geo = [(900, 1600, (704, 396), (0, 140, 704, 396)), (900, 1600, (1600, 900), (0, 4, 1600, 900)),
           (376, 1241, (1279, 387), (0, 3, 1280, 387)), (370, 1226, (1280, 386), (0, 2, 1280, 386))]
    geo += [(300, 400, (20, 15), (0, 0, 20, 15)),            # 1/20 downscale
            (40, 30, (90, 120), (5, 7, 60, 100)),            # x3 upscale
            (57, 83, (83, 57), (-3, -4, 80, 50)),            # identity, crop partly outside
            (64, 300, (13, 64), (0, 0, 13, 64)),             # one axis only: 13 columns from 300
            (200, 50, (50, 77), (10, 10, 40, 60)),           # the other axis only
            (20, 31, (1, 1), (0, 0, 1, 1)), (33, 47, (19, 11), (0, 0, 1, 1)),  # 1 x 1 outputs
            (50, 60, (30, 25), (40, 30, 52, 41))]            # crop wholly outside
    rng = np.random.default_rng(7)
    for _ in range(8):
        H, W = (int(v) for v in rng.integers(8, 400, 2))
        rW, rH = int(rng.integers(-(-W // 32), 600)), int(rng.integers(-(-H // 32), 600))
        x0, y0 = (int(v) for v in rng.integers(-20, 40, 2))
        geo.append((H, W, (rW, rH), (x0, y0, x0 + int(rng.integers(1, 300)), y0 + int(rng.integers(1, 200)))))
    return geo


SWEEP = _sweep()


@pytest.mark.parametrize("i", range(len(SWEEP)))
def test_resample_equals_pillow(i):
    Image = pytest.importorskip("PIL.Image")
    H, W, size, box = SWEEP[i]
    f = ip.frame(500 + i, H, W)
    ref = np.asarray(Image.fromarray(f).resize(size).crop(box))
    assert np.array_equal(ip.crop(ip.resize(f, size), box), ref)


@pytest.mark.parametrize("in_size,out_size", [(1600, 704), (900, 396), (1241, 1279), (376, 387), (1600, 1600),
                                              (300, 13), (40, 120), (6000, 200), (1, 1), (5, 1)])
def test_package_tables_equal_the_restatement(in_size, out_size):
    t = image_prep.resample_table(in_size, out_size)
    first, count, kk = ip.coeffs(in_size, out_size)
    n = out_size
    assert t.dtype == np.int32 and t.size == n * (2 + kk.shape[1])
    assert np.array_equal(t[:2 * n:2], first) and np.array_equal(t[1:2 * n:2], count)
    assert np.array_equal(t[2 * n:].reshape(-1, n).T, kk)


@pytest.mark.parametrize("cfg", [ip.NORM_R50, ip.NORM_R101, None], ids=["r50_kitti", "r101_caffe", "default"])
def test_normalisation_table_equals_opencv(cfg):
    cv2 = pytest.importorskip("cv2")
    norm = image_prep.norm_config(cfg)
    mean, std = np.array(norm["mean"], np.float32), np.array(norm["std"], np.float32)
    # every value in every channel, through mmcv 1.4.0 imnormalize_'s cv2 call sequence
    img = np.stack([np.arange(256, dtype=np.uint8)] * 3, axis=-1)[None].astype(np.float32)
    img[0, :, 1] = img[0, ::-1, 1]  # the channels differ, so a swapped channel would show
    src = img.copy()
    if norm["to_rgb"]:
        cv2.cvtColor(img, cv2.COLOR_BGR2RGB, img)
    cv2.subtract(img, np.float64(mean.reshape(1, -1)), img)
    cv2.multiply(img, 1 / np.float64(std.reshape(1, -1)), img)
    t = image_prep.normalize_table(norm["mean"], norm["std"], norm["to_rgb"])
    assert np.array_equal(t, ip.norm_table(norm["mean"], norm["std"], norm["to_rgb"]))
    v = src[0].astype(np.int64)
    mine = np.stack([t[c][v[:, 2 - c if norm["to_rgb"] else c]] for c in range(3)], axis=-1)
    assert np.array_equal(mine.view(np.int32), img[0].view(np.int32))


def test_fixture_records_versions_and_small_case():
    g = np.load(FIXTURE)
    assert str(g["pil_version"]) and str(g["cv2_version"])
    assert os.path.getsize(FIXTURE) < 1 << 20
    name = "small"
    _, shapes, size, norm = ip.CASES[name]
    for c, f in enumerate(ip.case_frames(name)[0]):
        dims, box = g[f"{name}_0_resize_dims"][c], g[f"{name}_0_crop"][c]
        mine = ip.prepare(f, tuple(dims), tuple(box), norm or ip.NORM_R50)
        assert np.array_equal(mine.view(np.int32), g[f"{name}_0_img"][c].view(np.int32))
        assert ip.sha(mine) == str(g[f"{name}_sha"][c])


@pytest.mark.parametrize("name", list(ip.CASES))
def test_new_transforms_equal_the_fixture(name, tmp_path):
    pytest.importorskip("cv2")
    from occformer_b200.pipelines import LoadMultiViewImageFrames_OccFormer, LoadMultiViewImageFrames_SemanticKitti
    g = np.load(FIXTURE)
    res = ip.run_case(name, LoadMultiViewImageFrames_OccFormer, LoadMultiViewImageFrames_SemanticKitti, str(tmp_path))
    kind, shapes, size, norm = ip.CASES[name]
    for s, (r, frames) in enumerate(zip(res, ip.case_frames(name))):
        imgs = r["img_inputs"]
        assert len(imgs) == 8 and imgs[0].dtype == torch.uint8
        assert np.array_equal(imgs[0].numpy(), np.stack(frames))
        for k in range(1, 8):
            ref = g[f"{name}_{s}_in{k}"]
            assert imgs[k].dtype == torch.float32 and np.array_equal(imgs[k].numpy(), ref), (name, s, k)
        aug = r["img_aug"]
        assert aug["resize_dims"] == g[f"{name}_{s}_resize_dims"].tolist()
        assert aug["crop"] == g[f"{name}_{s}_crop"].tolist()
        assert aug["input_size"] == list(size)
        assert {k: aug[k] for k in ("mean", "std", "to_rgb")} == image_prep.norm_config(norm)
        assert "canvas" not in r
        if kind == "kitti":
            assert np.array_equal(r["raw_img"], frames[0])
        else:
            assert list(r["cam_names"]) == ip.NUSC_CAMS[:len(frames)]


def test_refusals(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from occformer_b200.pipelines import LoadMultiViewImageFrames_OccFormer, LoadMultiViewImageFrames_SemanticKitti
    for cls in (LoadMultiViewImageFrames_OccFormer, LoadMultiViewImageFrames_SemanticKitti):
        with pytest.raises(ValueError, match="is_train=True"):
            cls(**ip.transform_kwargs("kitti", is_train=True))
    gray = os.path.join(str(tmp_path), "gray.png")
    cv2.imwrite(gray, np.zeros((20, 30), np.uint8))
    rgba = os.path.join(str(tmp_path), "rgba.png")
    cv2.imwrite(rgba, np.zeros((20, 30, 4), np.uint8))
    deep = os.path.join(str(tmp_path), "deep.png")
    cv2.imwrite(deep, np.zeros((20, 30, 3), np.uint16))
    t = LoadMultiViewImageFrames_SemanticKitti(**ip.transform_kwargs("kitti"))
    for path in (gray, rgba, deep):
        with pytest.raises(ValueError, match="3-channel uint8"):
            t(dict(img_filename=[path], cam_intrinsic=[np.eye(3).tolist()], lidar2cam=[np.eye(4).tolist()]))


def test_uint8_frames_need_img_aug():
    from occformer_b200.detector import OccupancyFormer
    frames = torch.zeros(1, 6, 9, 16, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match="LoadMultiViewImageFrames_OccFormer"):
        OccupancyFormer.extract_img_feat(None, [frames], [dict(pc_range=[0] * 6)])
