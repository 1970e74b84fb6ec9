"""TEST INFRASTRUCTURE ONLY (oracle) -- the image side of the test loaders (LoadMultiViewImageFromFiles_OccFormer,
P/datasets/pipelines/loading_nusc_imgs.py:34-62,181-195; LoadMultiViewImageFromFiles_SemanticKitti,
P/datasets/pipelines/loading_kitti_imgs.py:35-65; P/ = projects/mmdet3d_plugin/).

A numpy restatement of Pillow's Image.resize (BICUBIC, resample.c: precompute_coeffs, normalize_coeffs_8bpc, the
horizontal then vertical 8-bit passes over the rows the vertical pass reads), Image.crop (0 outside the image) and
mmcv's imnormalize as a 3 x 256 table; deterministic synthetic frames; and, for the build container that has the
reference checkout, the fixture generator and the check of this restatement against the reference transforms, run
verbatim on PNG-written frames (PNG is lossless, so the decode is exact):

    python -m oracle.image_prep gen        # tests/golden/image_prep.npz
    python -m oracle.image_prep validate   # this restatement == the reference transforms

mmcv is not installed there, so two mmcv 1.4.0 functions are restated under oracle/shim.py's fake mmcv and are the one
part not run from the real package: mmcv.imread (its cv2 backend: cv2.imdecode(bytes, IMREAD_UNCHANGED)) and
mmcv.image.photometric.imnormalize (imnormalize_'s cv2 calls: float32 copy, float64 mean and 1 / std, cvtColor BGR2RGB,
subtract, multiply).  Pillow's C source is not at hand either: these rules are restated from its published resample.c
and checked against the installed Pillow by tests/test_cpu_image_prep.py.

The fixture records the Pillow and OpenCV versions that wrote it (Pillow 12.2.0, OpenCV 4.13).  The reference
environment pins Pillow 9.4.0 and opencv-python 4.7.0.72; Pillow's resample code is believed unchanged between these
versions, but that is unverified.

Only the first half is imported by tests/; it needs no reference checkout.
"""
import hashlib
import math
import os
import sys
import tempfile
import types

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "image_prep.npz")
NORM_R50 = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)
NORM_R101 = dict(mean=[103.530, 116.280, 123.675], std=[1.0, 1.0, 1.0], to_rgb=False)
NUSC_CAMS = ["CAM_FRONT_LEFT", "CAM_FRONT", "CAM_FRONT_RIGHT", "CAM_BACK_LEFT", "CAM_BACK", "CAM_BACK_RIGHT"]


# =============================================================================
# restatement
# =============================================================================
def bicubic(x):
    """resample.c bicubic_filter, a = -0.5 (scalar, float64)"""
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def coeffs(in_size, out_size):
    """precompute_coeffs(in_size, 0, in_size, out_size, bicubic) + normalize_coeffs_8bpc -> (first (n,), count (n,),
    int64 weights (n, ksize))"""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    first = np.zeros(out_size, np.int64)
    count = np.zeros(out_size, np.int64)
    kk = np.zeros((out_size, ksize), np.int64)
    for xx in range(out_size):
        center = 0.0 + (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = [bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        kk[xx, :xmax] = [int(-0.5 + w * (1 << 22)) if w < 0 else int(0.5 + w * (1 << 22)) for w in k]
        first[xx], count[xx] = xmin, xmax
    return first, count, kk


def _pass(img, first, kk, axis):
    """one 8-bit pass along axis (0: rows, 1: columns) of an (H, W, 3) uint8 image -> uint8"""
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    acc = np.full((len(first),) + src.shape[1:], 1 << 21, np.int64)
    for k in range(kk.shape[1]):
        idx = np.minimum(first + k, src.shape[0] - 1)  # taps past the count have weight 0
        acc += kk[:, k][:, None, None] * src[idx]
    return np.moveaxis(np.clip(acc >> 22, 0, 255).astype(np.uint8), 0, axis)


def resize(img, size):
    """Image.fromarray(img).resize(size) for an (H, W, 3) uint8 array, size = (W', H')"""
    H, W = img.shape[:2]
    rW, rH = size
    if (rW, rH) == (W, H):
        return img.copy()
    hf, _, hk = coeffs(W, rW)
    vf, vc, vk = coeffs(H, rH)
    y0, y1 = vf[0], vf[-1] + vc[-1]  # ybox_first, ybox_last
    out = img
    if rW != W:
        out = _pass(img[y0:y1], hf, hk, 1)
        vf = vf - y0
    if rH != H:
        out = _pass(out, vf, vk, 0)
    return out


def crop(img, box):
    """Image.crop(box): pixels outside img are 0"""
    x0, y0, x1, y1 = (int(v) for v in box)
    H, W = img.shape[:2]
    out = np.zeros((y1 - y0, x1 - x0) + img.shape[2:], img.dtype)
    sy0, sy1, sx0, sx1 = max(y0, 0), min(y1, H), max(x0, 0), min(x1, W)
    if sy0 < sy1 and sx0 < sx1:
        out[sy0 - y0:sy1 - y0, sx0 - x0:sx1 - x0] = img[sy0:sy1, sx0:sx1]
    return out


def norm_table(mean, std, to_rgb):
    """mmcv imnormalize_ of each uint8 value (cv2.subtract of the float64 mean into float32, cv2.multiply by the float64
    1 / std into float32) -> float32 (3, 256), row c = output channel c (with to_rgb: source channel 2 - c)"""
    m = np.asarray(mean, np.float32).astype(np.float64)
    s = 1 / np.asarray(std, np.float32).astype(np.float64)
    v = np.arange(256, dtype=np.float64)
    return np.stack([((v - m[c]).astype(np.float32).astype(np.float64) * s[c]).astype(np.float32) for c in range(3)])


def prepare(frame, resize_dims, box, norm):
    """one camera: uint8 (H, W, 3) BGR frame -> float32 (3, fH, fW), the reference transform's normalised image"""
    img = crop(resize(frame, resize_dims), box)
    t = norm_table(norm["mean"], norm["std"], norm["to_rgb"])
    return np.stack([t[c][img[..., 2 - c if norm["to_rgb"] else c]] for c in range(3)])


def test_augmentation(H, W, input_size, crop_h=(0.0, 0.0), resize_test=0.0):
    """sample_augmentation in test mode (loading_nusc_imgs.py:84-95) -> (resize, resize_dims, crop)"""
    fH, fW = input_size
    resize = float(fW) / float(W) + resize_test
    resize_dims = (int(W * resize), int(H * resize))
    newW, newH = resize_dims
    crop_y = int((1 - np.mean(crop_h)) * newH) - fH
    crop_x = int(max(0, newW - fW) / 2)
    return resize, resize_dims, (crop_x, crop_y, crop_x + fW, crop_y + fH)


# =============================================================================
# synthetic frames
# =============================================================================
def _mix(h):
    h = h ^ (h >> np.uint32(16))
    h = h * np.uint32(0x7FEB352D)
    h = h ^ (h >> np.uint32(15))
    h = h * np.uint32(0x846CA68B)
    return h ^ (h >> np.uint32(16))


def frame(image, H, W):
    """uint8 (H, W, 3) frame `image` from an integer hash of (image, y, x, c): 8 x 8 cells, each black, white, noise or
    a ramp, so that cell edges jump 0 <-> 255 and drive the bicubic past both clips"""
    y = np.arange(H, dtype=np.uint32)[:, None, None]
    x = np.arange(W, dtype=np.uint32)[None, :, None]
    c = np.arange(3, dtype=np.uint32)[None, None, :]
    seed = np.uint32((image * 0x9E3779B1) & 0xFFFFFFFF)
    cell = _mix(seed ^ _mix((y >> np.uint32(3)) * np.uint32(0x10001) + (x >> np.uint32(3)) * np.uint32(0x3F1)))
    noise = _mix(seed ^ (y * np.uint32(0x1F123BB5) + x * np.uint32(0x5F356495) + c * np.uint32(0x2C1B3C6D)))
    kind = (cell >> np.uint32(7)) & np.uint32(3)
    ramp = (x * np.uint32(7) + y * np.uint32(3) + c * np.uint32(50)) & np.uint32(255)
    v = np.where(kind == 0, 0, np.where(kind == 1, 255, np.where(kind == 2, noise >> np.uint32(24), ramp)))
    return v.astype(np.uint8)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


# =============================================================================
# the fixture's cases
# =============================================================================
def data_config(input_size, cams=NUSC_CAMS):
    return dict(cams=list(cams), Ncams=len(cams), input_size=tuple(input_size), crop_h=(0.0, 0.0), resize_test=0.0,
                resize=(-0.06, 0.11), rot=(-5.4, 5.4), flip=True)


# name -> (kind, per-sample list of per-camera (H, W), input_size, norm); image index = running count over the case
CASES = {
    "r50": ("nusc", [[(900, 1600)] * 6] * 4, (256, 704), NORM_R50),
    "r101": ("nusc", [[(900, 1600)] * 2], (896, 1600), NORM_R101),
    "kitti": ("kitti", [[(376, 1241)], [(375, 1242)], [(370, 1226)]], (384, 1280), NORM_R50),
    "small": ("nusc", [[(90, 160), (90, 160)]], (48, 72), None),  # stored in full; its crop starts above the image
}
CASE_SEED = {"r50": 0, "r101": 1000, "kitti": 2000, "small": 3000}


def case_frames(name):
    """-> list (samples) of lists (cameras) of uint8 frames"""
    _, shapes, _, _ = CASES[name]
    out, i = [], CASE_SEED[name]
    for cams in shapes:
        s = []
        for H, W in cams:
            s.append(frame(i, H, W))
            i += 1
        out.append(s)
    return out


def calib(i):
    """deterministic intrinsics (3, 3) and lidar2cam (4, 4) of camera i"""
    a = 0.3 + 0.7 * i
    rot = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
    l2c = np.eye(4)
    l2c[:3, :3] = rot
    l2c[:3, 3] = [0.5 * i, -0.2, 1.5]
    K = np.array([[1260.0 + i, 0, 800.0 - i], [0, 1260.0 + i, 450.0 + i], [0, 0, 1]])
    return K, l2c


def write_results(root, name, s, frames):
    """write sample s's frames as PNG under root -> the results dict its loader reads"""
    import cv2
    kind = CASES[name][0]
    paths = []
    for c, f in enumerate(frames):
        p = os.path.join(root, f"{name}_{s}_{c}.png")
        cv2.imwrite(p, f)
        paths.append(p)
    if kind == "kitti":
        K, l2c = calib(s)
        return dict(img_filename=[paths[0]], cam_intrinsic=[K.tolist()], lidar2cam=[l2c.tolist()])
    cams = NUSC_CAMS[:len(frames)]
    cal = [calib(c) for c in range(len(frames))]
    return dict(curr=dict(cams={cam: dict(data_path=p, cam_intrinsic=cal[c][0].tolist())
                                for c, (cam, p) in enumerate(zip(cams, paths))}),
                lidar2cam_dic={cam: cal[c][1].tolist() for c, cam in enumerate(cams)})


def transform_kwargs(name, is_train=False):
    kind, shapes, size, norm = CASES[name]
    return dict(data_config=data_config(size, NUSC_CAMS[:len(shapes[0])]), is_train=is_train, img_norm_cfg=norm)


def run_case(name, nusc_cls, kitti_cls, root):
    """every sample of a case through a loader class pair (the reference's or this package's) -> list of results"""
    out = []
    for s, frames in enumerate(case_frames(name)):
        cls = kitti_cls if CASES[name][0] == "kitti" else nusc_cls
        out.append(cls(**transform_kwargs(name))(write_results(root, name, s, frames)))
    return out


# =============================================================================
# reference side (build container only)
# =============================================================================
def _install_mmcv_image():
    """mmcv 1.4.0's imread (cv2 backend) and imnormalize, restated on the shim's fake mmcv"""
    import cv2
    from . import shim
    shim.install()

    def imread(path, flag="color"):
        assert flag == "unchanged"
        with open(path, "rb") as f:
            buf = np.frombuffer(f.read(), np.uint8)
        return cv2.imdecode(buf, cv2.IMREAD_UNCHANGED)

    def imnormalize(img, mean, std, to_rgb=True):
        img = img.copy().astype(np.float32)
        assert img.dtype != np.uint8
        mean = np.float64(mean.reshape(1, -1))
        stdinv = 1 / np.float64(std.reshape(1, -1))
        if to_rgb:
            cv2.cvtColor(img, cv2.COLOR_BGR2RGB, img)
        cv2.subtract(img, mean, img)
        cv2.multiply(img, stdinv, img)
        return img

    sys.modules["mmcv"].imread = imread
    image = types.ModuleType("mmcv.image")
    photometric = types.ModuleType("mmcv.image.photometric")
    photometric.imnormalize = imnormalize
    image.photometric = photometric
    sys.modules["mmcv.image"], sys.modules["mmcv.image.photometric"] = image, photometric
    sys.modules["mmcv"].image = image


def _reference_transforms():
    from . import occ_targets
    occ_targets._reference_transforms()  # the datasets namespace and the PIPELINES registry
    _install_mmcv_image()
    from . import shim
    nusc = shim.load("projects.mmdet3d_plugin.datasets.pipelines.loading_nusc_imgs")
    kitti = shim.load("projects.mmdet3d_plugin.datasets.pipelines.loading_kitti_imgs")
    return nusc.LoadMultiViewImageFromFiles_OccFormer, kitti.LoadMultiViewImageFromFiles_SemanticKitti


def gen():
    """tests/golden/image_prep.npz: per case img_inputs[1:] and the img_aug the new transforms produce (as the reference's
    sample_augmentation gives it), the SHA-256 of every image's float32 bytes; the small case's images in full"""
    import cv2
    import PIL
    nusc_cls, kitti_cls = _reference_transforms()
    out = dict(pil_version=np.array(PIL.__version__), cv2_version=np.array(cv2.__version__))
    with tempfile.TemporaryDirectory() as root:
        for name, (kind, shapes, size, norm) in CASES.items():
            res = run_case(name, nusc_cls, kitti_cls, root)
            shas = []
            for s, r in enumerate(res):
                imgs = r["img_inputs"][0].numpy()
                shas += [sha(im) for im in imgs]
                for k in range(1, 8):
                    out[f"{name}_{s}_in{k}"] = r["img_inputs"][k].numpy()
                aug = [test_augmentation(H, W, size) for H, W in shapes[s]]
                out[f"{name}_{s}_resize_dims"] = np.array([a[1] for a in aug], np.int64)
                out[f"{name}_{s}_crop"] = np.array([a[2] for a in aug], np.int64)
                if name == "small":
                    out[f"{name}_{s}_img"] = imgs
            out[f"{name}_sha"] = np.array(shas)
            print(f"{name}: {len(shas)} images")
    np.savez_compressed(GOLDEN, **out)
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")


def validate():
    """this restatement against the reference transforms on every case, image by image; exit status 1 on a difference"""
    nusc_cls, kitti_cls = _reference_transforms()
    bad = 0
    with tempfile.TemporaryDirectory() as root:
        for name, (kind, shapes, size, norm) in CASES.items():
            res = run_case(name, nusc_cls, kitti_cls, root)
            n_img = n_bad = 0
            for s, (r, frames) in enumerate(zip(res, case_frames(name))):
                for c, f in enumerate(frames):
                    _, dims, box = test_augmentation(*f.shape[:2], size)
                    mine = prepare(f, dims, box, norm or NORM_R50)
                    ref = r["img_inputs"][0][c].numpy()
                    n_bad += int(not np.array_equal(mine.view(np.int32), ref.view(np.int32)))
                    n_img += 1
            bad += n_bad
            print(f"{'OK ' if n_bad == 0 else 'BAD'} {name}: {n_bad} of {n_img} images differ")
    if bad:
        sys.exit(1)
    print("image restatement == reference transforms on all cases")


if __name__ == "__main__":
    from . import shim
    assert shim.reference_available(), "needs the reference checkout"
    {"gen": gen, "validate": validate}[sys.argv[1] if len(sys.argv) > 1 else "validate"]()
