"""TEST INFRASTRUCTURE ONLY (oracle) -- the camera inputs of the training pipelines (P/ = projects/mmdet3d_plugin/):

    LoadMultiViewImageFromFiles_OccFormer(is_train=True)      P/datasets/pipelines/loading_nusc_imgs.py:34-96
    LoadMultiViewImageFromFiles_SemanticKitti(is_train=True)  P/datasets/pipelines/loading_kitti_imgs.py:35-95
    CreateDepthFromLiDAR                                      P/datasets/pipelines/lidar2depth.py:15-82

A numpy restatement of the training-mode image transform (resize and crop as oracle/image_prep.py, then
FLIP_LEFT_RIGHT, then Pillow's Image.rotate with its defaults, then the normalisation table) and of the depth map
(fp32 projection, one operation at a time, then np.minimum.at); deterministic synthetic scans and camera files; and,
for the build container that has the reference checkout, the fixture generator, which runs the reference transforms
verbatim under oracle/shim.py with torch.set_num_threads(1), as a DataLoader worker runs them:

    python -m oracle.train_inputs gen        # tests/golden/train_inputs.npz

Pillow's rotation, restated from its published Image.py and Geometry.c: Image.rotate(angle) copies at angle % 360 == 0,
transposes at 180 (and at 90 / 270 when the image is square), and otherwise gathers the nearest pixel through the
matrix [round(cos a, 15), round(sin a, 15), ., round(-sin a, 15), round(cos a, 15), .], a = -radians(angle), about
(w / 2, h / 2), in 16.16 fixed point (affine_fixed): a2 = FIX(m2 + m1 / 2 + m0 / 2), a5 = FIX(m5 + m4 / 2 + m3 / 2),
FIX(v) = floor(v * 65536 + 0.5), source ((a2 + y a1 + x a0) >> 16, (a5 + y a4 + x a3) >> 16), black outside.
tests/test_cpu_train_inputs.py checks it against the installed Pillow.

Only the first half is imported by tests/; it needs no reference checkout.
"""
import hashlib
import math
import os
import sys
import tempfile

import numpy as np

from . import image_prep as ip

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                      "train_inputs.npz")


# =============================================================================
# restatement
# =============================================================================
def rotate(img, angle):
    """Image.fromarray(img).rotate(angle) of an (h, w, 3) uint8 array"""
    h, w = img.shape[:2]
    angle = angle % 360.0
    if angle == 0:
        return img.copy()
    if angle == 180:
        return img[::-1, ::-1].copy()
    if angle in (90, 270) and w == h:
        return np.rot90(img, 1 if angle == 90 else -1).copy()  # counter-clockwise for a positive angle
    a = -math.radians(angle)
    m0, m1, m3, m4 = round(math.cos(a), 15), round(math.sin(a), 15), round(-math.sin(a), 15), round(math.cos(a), 15)
    m2 = m0 * (-w / 2.0) + m1 * (-h / 2.0) + 0.0 + w / 2.0
    m5 = m3 * (-w / 2.0) + m4 * (-h / 2.0) + 0.0 + h / 2.0
    fix = lambda v: math.floor(v * 65536.0 + 0.5)  # noqa: E731
    a0, a1, a3, a4 = fix(m0), fix(m1), fix(m3), fix(m4)
    a2, a5 = fix(m2 + m1 * 0.5 + m0 * 0.5), fix(m5 + m4 * 0.5 + m3 * 0.5)
    y = np.arange(h, dtype=np.int64)[:, None]
    x = np.arange(w, dtype=np.int64)[None, :]
    xs = (a2 + y * a1 + x * a0) >> 16
    ys = (a5 + y * a4 + x * a3) >> 16
    inside = (xs >= 0) & (xs < w) & (ys >= 0) & (ys < h)
    out = img[np.clip(ys, 0, h - 1), np.clip(xs, 0, w - 1)]
    out[~inside] = 0
    return out


def augment_uint8(frame, resize_dims, box, flip, angle):
    """img_transform_core: resize, crop, FLIP_LEFT_RIGHT when flip, rotate -> uint8 (fH, fW, 3)"""
    img = ip.crop(ip.resize(frame, resize_dims), box)
    if flip:
        img = img[:, ::-1].copy()
    return rotate(img, angle)


def augment(frame, resize_dims, box, flip, angle, norm):
    """one camera of a training loader: uint8 (H, W, 3) BGR frame -> float32 (3, fH, fW), the normalised image"""
    img = augment_uint8(frame, resize_dims, box, flip, angle)
    t = ip.norm_table(norm["mean"], norm["std"], norm["to_rgb"])
    return np.stack([t[c][img[..., 2 - c if norm["to_rgb"] else c]] for c in range(3)])


def _dot(m, v):
    """rows of m (..., k) times v (P, k) in float32, summed left to right without fused multiply-add -> (P,)"""
    acc = m[0] * v[:, 0]
    for k in range(1, v.shape[1]):
        acc = acc + m[k] * v[:, k]
    return acc


def depth_map(points, inv_rot, tran, intrin, post_rot, post_tran, fH, fW):
    """CreateDepthFromLiDAR for one camera: float32 points (P, 3), the camera's float32 rots.inverse(), trans, 3 x 3 or
    4 x 4 intrinsics, post_rot, post_tran -> float32 (fH, fW), the nearest valid point's depth per pixel, else 0"""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        return _depth_map(points, inv_rot, tran, intrin, post_rot, post_tran, fH, fW)


def _depth_map(points, inv_rot, tran, intrin, post_rot, post_tran, fH, fW):
    f = np.float32
    q = points.astype(f) - tran.astype(f)[None, :]
    c = np.stack([_dot(inv_rot[i].astype(f), q) for i in range(3)], axis=1)
    if intrin.shape[-1] == 4:
        c = np.concatenate([c, np.ones((len(c), 1), f)], axis=1)
    x, y, d = (_dot(intrin[i].astype(f), c) for i in range(3))
    u, v = x / d, y / d
    uv = np.stack([u, v], axis=1)
    pu = _dot(post_rot[0, :2].astype(f), uv) + f(post_tran[0])
    pv = _dot(post_rot[1, :2].astype(f), uv) + f(post_tran[1])
    ok = (pu >= 0) & (pv >= 0) & (pu <= fW - 1) & (pv <= fH - 1) & (d > 0)
    idx = (np.rint(pv[ok]).astype(np.int64), np.rint(pu[ok]).astype(np.int64))
    out = np.full((fH, fW), np.inf, f)
    np.minimum.at(out, idx, d[ok])
    hit = np.zeros((fH, fW), bool)
    hit[idx] = True
    out[~hit] = 0
    return out


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float32).tobytes()).hexdigest()


# =============================================================================
# synthetic inputs and the fixture's cases
# =============================================================================
KITTI_SIZES = [(376, 1241), (375, 1242), (370, 1226)]

# name -> (kind, samples, cameras per sample (listed), Ncams, frame (H, W) per sample, input_size, norm, flip, rot,
#          scan points per sample)
CASES = {
    "r50": ("nusc", 1, 6, 6, [(900, 1600)], (256, 704), ip.NORM_R50, True, (-5.4, 5.4), 34720),
    "r101": ("nusc", 1, 2, 2, [(900, 1600)], (896, 1600), ip.NORM_R101, True, (-5.4, 5.4), 34720),
    "kitti": ("kitti", 3, 1, 1, KITTI_SIZES, (384, 1280), ip.NORM_R50, True, (-5.4, 5.4), 120000),
    "small": ("nusc", 2, 5, 3, [(90, 160), (60, 100)], (48, 72), None, False, (-180.0, 180.0), 3000),
}
CASE_SEED = {"r50": 0, "r101": 1000, "kitti": 2000, "small": 3000}


def data_config(name):
    kind, _, ncam, Ncams, _, size, _, flip, rot, _ = CASES[name]
    return dict(cams=list(ip.NUSC_CAMS[:ncam]), Ncams=Ncams, input_size=tuple(size), src_size=(900, 1600),
                resize=(-0.06, 0.11), rot=tuple(rot), flip=flip, crop_h=(0.0, 0.0), resize_test=0.0)


def transform_kwargs(name, is_train=True):
    return dict(data_config=data_config(name), is_train=is_train, img_norm_cfg=CASES[name][6])


def calib(name, i):
    """camera i's float64 intrinsics (3 x 3, or KITTI's 4 x 4 projection with a translation column) and lidar2cam"""
    K, l2c = ip.calib(i)
    if CASES[name][0] == "kitti":
        K4 = np.eye(4)
        K4[:3, :3] = K
        K4[:3, 3] = [44.86, 0.2163, 0.002745]
        K = K4
    return K, l2c


def scan(name, s):
    """sample s's float32 (P, 3) scan: points in front of each camera over its frame and a margin around it (collisions
    come from the crop's downscale), exact duplicates, points behind the cameras, and NaN / inf rows"""
    kind, _, ncam, _, shapes, _, _, _, _, n = CASES[name]
    H, W = shapes[s % len(shapes)]
    rng = np.random.default_rng(CASE_SEED[name] + 17 * s)
    parts = []
    for c in range(ncam):
        K, l2c = calib(name, c)
        m = n // ncam
        u = rng.uniform(-0.1 * W, 1.1 * W, m)
        v = rng.uniform(-0.1 * H, 1.1 * H, m)
        z = rng.uniform(-3.0, 60.0, m)
        cam = np.stack([(u - K[0, 2]) * z / K[0, 0], (v - K[1, 2]) * z / K[1, 1], z, np.ones(m)], axis=1)
        parts.append((np.linalg.inv(l2c) @ cam.T).T[:, :3])
    pts = np.concatenate(parts).astype(np.float32)
    k = len(pts) // 50
    pts[-k:] = pts[:k]                                  # exact duplicates: equal depths on one pixel
    pts[-2 * k:-k] = pts[k:2 * k] * np.float32(1.001)   # near copies: distinct depths on a pixel or its neighbour
    pts[5] = [np.nan, 1.0, 2.0]
    pts[6] = [np.inf, 1.0, 2.0]
    pts[7] = [1.0, -np.inf, 2.0]
    return pts


def write_results(root, name, s, frames, pts):
    """write sample s's frames as PNG and its scan as the dataset's .bin under root -> the results dict of its loaders"""
    import cv2
    kind, _, ncam = CASES[name][:3]
    if kind == "kitti":
        seq = f"{s:02d}"
        d = os.path.join(root, "sequences", seq, "image_2")
        os.makedirs(d, exist_ok=True)
        path = os.path.join(d, f"{100 + s:06d}.png")
        cv2.imwrite(path, frames[0])
        vd = os.path.join(root, "data_velodyne", "velodyne", "sequences", seq, "velodyne")
        os.makedirs(vd, exist_ok=True)
        ref = np.concatenate([pts, np.full((len(pts), 1), 0.5, np.float32)], axis=1)
        ref.tofile(os.path.join(vd, f"{100 + s:06d}.bin"))
        K, l2c = calib(name, s)
        return dict(img_filename=[path], cam_intrinsic=[K.tolist()], lidar2cam=[l2c.tolist()])
    paths = []
    for c, f in enumerate(frames):
        p = os.path.join(root, f"{name}_{s}_{c}.png")
        cv2.imwrite(p, f)
        paths.append(p)
    pts_file = os.path.join(root, f"{name}_{s}_lidar.bin")
    np.concatenate([pts, np.zeros((len(pts), 2), np.float32)], axis=1).tofile(pts_file)
    cams = ip.NUSC_CAMS[:ncam]
    cal = [calib(name, c) for c in range(ncam)]
    return dict(curr=dict(cams={cam: dict(data_path=p, cam_intrinsic=cal[c][0].tolist())
                                for c, (cam, p) in enumerate(zip(cams, paths))}),
                lidar2cam_dic={cam: cal[c][1].tolist() for c, cam in enumerate(cams)}, pts_filename=pts_file)


def case_frames(name, s):
    kind, _, ncam, _, shapes = CASES[name][:5]
    H, W = shapes[s % len(shapes)]
    return [ip.frame(CASE_SEED[name] + 10 * s + c, H, W) for c in range(ncam)]


def draws(name, H, W):
    """one camera's training-mode sample_augmentation from the global numpy RNG, in the reference's order ->
    (resize, resize_dims, crop, flip, rotate)"""
    cfg = data_config(name)
    fH, fW = cfg["input_size"]
    resize = float(fW) / float(W) + np.random.uniform(*cfg["resize"])
    dims = (int(W * resize), int(H * resize))
    crop_h = int((1 - np.random.uniform(*cfg["crop_h"])) * dims[1]) - fH
    crop_w = int(np.random.uniform(0, max(0, dims[0] - fW)))
    flip = bool(cfg["flip"] and np.random.choice([0, 1]))
    rotate = float(np.random.uniform(*cfg["rot"]))
    return resize, dims, (crop_w, crop_h, crop_w + fW, crop_h + fH), flip, rotate


def run_case(name, loaders, root):
    """every sample of a case through loaders (a list of transforms, the reference's or this package's) from the case's
    seed -> (list of results, numpy RNG state after the case)"""
    np.random.seed(CASE_SEED[name])
    out = []
    for s in range(CASES[name][1]):
        r = write_results(root, name, s, case_frames(name, s), scan(name, s))
        for t in loaders:
            r = t(r)
        out.append(r)
    return out, np.random.get_state()


def oracle_case(name):
    """the restatement's draws for every sample of a case -> per sample, (camera indices, per camera draws)"""
    kind, B, ncam, Ncams = CASES[name][:4]
    np.random.seed(CASE_SEED[name])
    out = []
    for s in range(B):
        cams = list(range(ncam))
        if Ncams < ncam:
            names = np.random.choice(ip.NUSC_CAMS[:ncam], Ncams, replace=False)
            cams = [ip.NUSC_CAMS.index(c) for c in names]
        H, W = CASES[name][4][s % len(CASES[name][4])]
        out.append((cams, [draws(name, H, W) for _ in cams]))
    return out, np.random.get_state()


# =============================================================================
# reference side (build container only)
# =============================================================================
def _reference_transforms():
    nusc_cls, kitti_cls = ip._reference_transforms()
    from . import shim
    depth = shim.load("projects.mmdet3d_plugin.datasets.pipelines.lidar2depth")
    return nusc_cls, kitti_cls, depth.CreateDepthFromLiDAR


def gen():
    """tests/golden/train_inputs.npz: per case and sample the camera names, img_inputs[1:6] (post_rot / post_tran
    bits), the SHA-256 of every image's and depth map's float32 bytes, and the numpy RNG state after the case"""
    import PIL
    import torch
    torch.set_num_threads(1)
    nusc_cls, kitti_cls, depth_cls = _reference_transforms()
    out = dict(pil_version=np.array(PIL.__version__), torch_version=np.array(torch.__version__))
    with tempfile.TemporaryDirectory() as root:
        for name, case in CASES.items():
            kind = case[0]
            cls = kitti_cls if kind == "kitti" else nusc_cls
            loaders = [cls(**transform_kwargs(name)), depth_cls(data_root=root, dataset=kind)]
            res, state = run_case(name, loaders, root)
            draws_, state_o = oracle_case(name)
            assert state_o[2] == state[2] and np.array_equal(state_o[1], state[1]), "the draw order differs"
            for s, (r, (cams, dr)) in enumerate(zip(res, draws_)):
                imgs = r["img_inputs"]
                out[f"{name}_{s}_cams"] = np.array(cams, np.int64)
                for k in range(1, 6):
                    out[f"{name}_{s}_in{k}"] = imgs[k].numpy()
                out[f"{name}_{s}_img_sha"] = np.array([sha(im) for im in imgs[0].numpy()])
                out[f"{name}_{s}_depth_sha"] = np.array([sha(d) for d in imgs[6].numpy()])
                out[f"{name}_{s}_depth_valid"] = (imgs[6].numpy() > 0).sum(axis=(1, 2))
            out[f"{name}_rng_pos"] = np.array(state[2])
            out[f"{name}_rng_sha"] = np.array(hashlib.sha256(state[1].tobytes()).hexdigest())
            print(f"{name}: {len(res)} samples")
    np.savez_compressed(GOLDEN, **out)
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    from . import shim
    assert shim.reference_available(), "needs the reference checkout"
    {"gen": gen}[sys.argv[1] if len(sys.argv) > 1 else "gen"]()
