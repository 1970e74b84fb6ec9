"""The training pipelines' camera inputs on the H100 (occformer_b200.image_prep: prepare_images with flip / rotate,
lidar_depth_maps, camera_inputs; csrc/image_prep.cu, csrc/lidar_depth.cu), bit for bit: against the reference
transforms' SHA-256 in tests/golden/train_inputs.npz (frames and scans regenerated from their seeds) and against the
numpy restatement (oracle/train_inputs.py, itself checked against Pillow and the reference); planted depth-map corners,
launch counts, graph replay and argument errors."""
import ctypes
import os

import numpy as np
import pytest
import torch

from util import GOLDEN, graph_replay, launches, rejected, same_bits, sentinel
from oracle import image_prep as ip
from oracle import train_inputs as ti
from occformer_b200 import image_prep, ops

pytestmark = pytest.mark.gpu


def _golden():
    return np.load(os.path.join(GOLDEN, "train_inputs.npz"))


def _case(name):
    """per sample of a fixture case: (uint8 frames of the chosen cameras, img_aug as the new transforms give it)"""
    draws, _ = ti.oracle_case(name)
    norm = image_prep.norm_config(ti.CASES[name][6])
    out = []
    for s, (cams, dr) in enumerate(draws):
        frames = ti.case_frames(name, s)
        aug = dict(resize_dims=[list(d[1]) for d in dr], crop=[list(d[2]) for d in dr],
                   input_size=list(ti.CASES[name][5]), flip=[d[3] for d in dr], rotate=[d[4] for d in dr], **norm)
        out.append((np.stack([frames[c] for c in cams]), aug))
    return out


def _frames(cuda, samples):
    f = [torch.from_numpy(s).to(cuda) for s in samples]
    return torch.stack(f) if len({tuple(x.shape) for x in f}) == 1 else f


@pytest.mark.parametrize("name", list(ti.CASES))
def test_images_equal_the_fixture(cuda, name):
    g = _golden()
    case = _case(name)
    n0 = ops.LAUNCH_COUNT[0]
    out = image_prep.prepare_images(_frames(cuda, [c[0] for c in case]), [c[1] for c in case])
    assert ops.LAUNCH_COUNT[0] - n0 == 2
    for s, (frames, aug) in enumerate(case):
        assert [ti.sha(im) for im in out[s].cpu().numpy()] == [str(h) for h in g[f"{name}_{s}_img_sha"]]
    if name in ("small", "kitti"):
        norm = ti.CASES[name][6] or ip.NORM_R50
        for s, (frames, aug) in enumerate(case):
            for c, f in enumerate(frames):
                ref = ti.augment(f, aug["resize_dims"][c], aug["crop"][c], aug["flip"][c], aug["rotate"][c], norm)
                same_bits(out[s, c], torch.from_numpy(ref).to(cuda), f"{name} sample {s} camera {c}")


def test_256_mixed_images_equal_the_restatement(cuda):
    """32 samples x 8 cameras in one call: frame sizes per sample, resizes, crops past every edge, flips, and angles
    where Pillow copies, transposes (the crop is square) or gathers"""
    rng = np.random.default_rng(5)
    size = (40, 40)
    special = [0.0, 180.0, 90.0, 270.0, -90.0, 360.0]
    samples, augs = [], []
    for s in range(32):
        H, W = int(rng.integers(20, 120)), int(rng.integers(20, 160))
        frames, dims, crops, flips, rots = [], [], [], [], []
        for c in range(8):
            frames.append(ip.frame(3000 + 8 * s + c, H, W))
            rW, rH = int(rng.integers(max(1, -(-W // 32)), 90)), int(rng.integers(max(1, -(-H // 32)), 90))
            x0, y0 = int(rng.integers(-20, max(rW - 20, -19))), int(rng.integers(-25, max(rH - 15, -24)))
            dims.append([rW, rH])
            crops.append([x0, y0, x0 + size[1], y0 + size[0]])
            flips.append(bool(rng.integers(0, 2)))
            k = 8 * s + c
            rots.append(special[k % 6] if k % 4 == 0 else float(rng.uniform(-5.4, 5.4) if k % 4 == 1
                                                                else rng.uniform(-360.0, 360.0)))
        samples.append(np.stack(frames))
        augs.append(dict(resize_dims=dims, crop=crops, input_size=list(size), flip=flips, rotate=rots,
                         **image_prep.norm_config(ip.NORM_R101)))
    out = image_prep.prepare_images(_frames(cuda, samples), augs)
    ref = np.stack([np.stack([ti.augment(f, a["resize_dims"][c], a["crop"][c], a["flip"][c], a["rotate"][c],
                                         ip.NORM_R101) for c, f in enumerate(fr)]) for fr, a in zip(samples, augs)])
    same_bits(out, torch.from_numpy(ref).to(cuda), "256 mixed images")


def test_test_mode_through_the_new_entry_equals_the_old(cuda):
    samples = ip.case_frames("r50")[:2]
    frames = torch.from_numpy(np.stack([np.stack(s) for s in samples])).to(cuda)
    _, _, size, norm = ip.CASES["r50"]
    aug = [ip.test_augmentation(900, 1600, size) for _ in range(6)]
    test = dict(resize_dims=[list(a[1]) for a in aug], crop=[list(a[2]) for a in aug], input_size=list(size),
                **image_prep.norm_config(norm))
    train = dict(test, flip=[False] * 6, rotate=[0.0] * 6)
    same_bits(image_prep.prepare_images(frames, [train] * 2), image_prep.prepare_images(frames, [test] * 2),
              "test-mode img_aug through occ_prepare_images_aug")


# ---------------------------------------------------------------------------------------------- depth maps
def _golden_inputs(name, s, cuda):
    g = _golden()
    rots, trans, intrins, post_rots, post_trans = (torch.from_numpy(g[f"{name}_{s}_in{k}"]) for k in range(1, 6))
    img_inputs = [None, rots[None].to(cuda), trans[None].to(cuda), intrins[None].to(cuda), post_rots[None].to(cuda),
                  post_trans[None].to(cuda)]
    return img_inputs, dict(lidar_inv_rots=rots.inverse(), input_size=list(ti.CASES[name][5]))


def _oracle_depths(pts, img_inputs, aug):
    inv = torch.as_tensor(aug["lidar_inv_rots"]).numpy()
    trans, intrins, post_rots, post_trans = (t[0].cpu().numpy() for t in img_inputs[2:6])
    return np.stack([ti.depth_map(pts, inv[j], trans[j], intrins[j], post_rots[j], post_trans[j], *aug["input_size"])
                     for j in range(len(inv))])


@pytest.mark.parametrize("name", list(ti.CASES))
def test_depth_maps_equal_the_fixture(cuda, name):
    g = _golden()
    for s in range(ti.CASES[name][1]):
        img_inputs, aug = _golden_inputs(name, s, cuda)
        pts = ti.scan(name, s)
        n0 = ops.LAUNCH_COUNT[0]
        out = image_prep.lidar_depth_maps([pts], img_inputs, [aug])
        assert ops.LAUNCH_COUNT[0] - n0 == 3
        assert [ti.sha(d) for d in out[0].cpu().numpy()] == [str(h) for h in g[f"{name}_{s}_depth_sha"]], (name, s)
        same_bits(out[0], torch.from_numpy(_oracle_depths(pts, img_inputs, aug)).to(cuda), f"{name} sample {s}")


def _planted(W, H):
    """points for an identity camera (u = x / z, v = y / z): collisions with distinct and equal depths, the last column
    and row, rounding ties, d <= 0, NaN and inf"""
    f = np.float32
    p = [[(W - 1) * 2.0, (H - 1) * 2.0, 2.0],               # exactly (W - 1, H - 1)
         [(W - 1) * 4.0 + 0.1, 0.0, 4.0],                    # just past the last column
         [2.5, 3.5, 1.0], [4.5, 0.5, 1.0], [1.5, 6.5, 1.0],  # ties: round half to even
         [10.0, 10.0, 5.0], [20.0, 20.0, 10.0], [30.0, 30.0, 15.0], [10.0, 10.0, 5.0],  # one pixel, equal and distinct
         [9.0, 9.0, 3.0], [9.0, 9.0, 3.0],                   # one pixel, equal depths only
         [1.0, 1.0, 0.0], [1.0, 1.0, -1.0], [-1.0, -1.0, -1.0],  # d <= 0
         [np.nan, 1.0, 1.0], [1.0, np.inf, 1.0], [1.0, 1.0, np.inf], [np.inf, np.inf, np.inf], [0.0, 0.0, np.nan],
         [-0.2, -0.2, 1.0], [-0.6, 0.0, 1.0]]                # rounds to 0 from below the edge: invalid
    return np.array(p, f)


def test_planted_depths(cuda):
    """B = 4 samples x 6 cameras, different scan sizes (one empty, one with no valid point), identity and golden
    cameras, 3 x 3 intrinsics; and KITTI's 4 x 4"""
    H, W = 48, 72
    B, N = 4, 6
    eye = torch.eye(3).expand(B, N, 3, 3).clone()
    img_inputs = [None, eye, torch.zeros(B, N, 3), eye.clone(), eye.clone(), torch.zeros(B, N, 3)]
    rng = np.random.default_rng(3)
    for b in range(B):
        for n in range(1, N):
            img_inputs[3][b, n] = torch.tensor([[40.0 + n, 0, 36], [0, 40.0 + b, 24], [0, 0, 1]])
            img_inputs[4][b, n, :2, :2] = torch.tensor([[0.9, 0.05], [-0.05, 0.9]]) * (1 + 0.1 * n)
            img_inputs[5][b, n, :2] = torch.tensor([-3.0 * n, 2.0])
            img_inputs[2][b, n] = torch.tensor([0.1 * n, -0.2, 0.3])
    rand = (rng.standard_normal((3000, 3)) * [3, 2, 5] + [0, 0, 4]).astype(np.float32)
    scans = [_planted(W, H), np.zeros((0, 3), np.float32),
             np.array([[1.0, 1.0, -2.0], [np.nan, 0, 1], [1e6, 1e6, 1.0]], np.float32),
             np.concatenate([_planted(W, H), rand])]
    aug = [dict(lidar_inv_rots=eye[b], input_size=[H, W]) for b in range(B)]
    dev_inputs = [None] + [t.to(cuda) for t in img_inputs[1:]]
    out = image_prep.lidar_depth_maps(scans, dev_inputs, aug)
    assert out.shape == (B, N, H, W)
    for b in range(B):
        ref = _oracle_depths(scans[b], [None] + [t[b:b + 1] for t in img_inputs[1:]], aug[b])
        same_bits(out[b], torch.from_numpy(ref).to(cuda), f"sample {b}")
    d = out[0, 0].cpu()  # the identity camera: the planted points alone
    assert d[H - 1, W - 1] == 2.0 and d[4, 2] == 1.0 and d[0, 4] == 1.0 and d[6, 2] == 1.0
    assert d[2, 2] == 5.0 and d[3, 3] == 3.0 and int((d > 0).sum()) == 6
    assert bool((out[1] == 0).all()) and bool((out[2] == 0).all())
    # KITTI: one camera, 4 x 4 intrinsics with a translation column
    img_inputs, k_aug = _golden_inputs("kitti", 0, cuda)
    pts = np.concatenate([ti.scan("kitti", 0)[:5000], _planted(1280, 384)])
    same_bits(image_prep.lidar_depth_maps([pts], img_inputs, [k_aug])[0],
              torch.from_numpy(_oracle_depths(pts, img_inputs, k_aug)).to(cuda), "KITTI planted")


# ---------------------------------------------------------------------------------------------- the whole call
def _pipeline(name, tmp_path):
    from occformer_b200.pipelines import (LoadLidarDepthPoints, LoadMultiViewImageFramesAug_OccFormer,
                                          LoadMultiViewImageFramesAug_SemanticKitti)
    kind = ti.CASES[name][0]
    cls = LoadMultiViewImageFramesAug_SemanticKitti if kind == "kitti" else LoadMultiViewImageFramesAug_OccFormer
    res, _ = ti.run_case(name, [cls(**ti.transform_kwargs(name)), LoadLidarDepthPoints(str(tmp_path), kind)],
                         str(tmp_path))
    return res


@pytest.mark.parametrize("name", ["r50", "kitti"])
def test_camera_inputs_equal_the_reference_tuple(cuda, name, tmp_path):
    pytest.importorskip("cv2")
    g = _golden()
    for s, r in enumerate(_pipeline(name, tmp_path)):
        img_inputs = tuple(t[None].to(cuda) for t in r["img_inputs"])
        metas = [dict(img_aug=r["img_aug"])]
        out = image_prep.camera_inputs(img_inputs, metas)
        assert len(out) == 8
        assert [ti.sha(im) for im in out[0][0].cpu().numpy()] == [str(h) for h in g[f"{name}_{s}_img_sha"]]
        assert [ti.sha(d) for d in out[6][0].cpu().numpy()] == [str(h) for h in g[f"{name}_{s}_depth_sha"]]
        for k in (1, 2, 3, 4, 5, 7):
            assert out[k] is img_inputs[k]
        # after an occupancy annotation transform: bda_rot at 6, gt_depths at 7
        bda = torch.eye(3, device=cuda)[None]
        nine = img_inputs[:6] + (bda,) + img_inputs[6:]
        out9 = image_prep.camera_inputs(nine, metas)
        assert len(out9) == 9 and out9[6] is bda and out9[8] is nine[8]
        same_bits(out9[7], out[6], "gt_depths of the 9-tuple")


def test_graph_replay_equals_eager(cuda, tmp_path):
    pytest.importorskip("cv2")
    r = _pipeline("small", tmp_path)
    frames = [x["img_inputs"][0].to(cuda) for x in r]  # two frame sizes: the list form
    img_inputs = (frames,) + tuple(torch.stack([x["img_inputs"][k] for x in r]).to(cuda) for k in range(1, 8))
    metas = [dict(img_aug=dict(x["img_aug"], lidar_points=x["img_aug"]["lidar_points"].to(cuda),
                               lidar_inv_rots=x["img_aug"]["lidar_inv_rots"].to(cuda))) for x in r]
    eager = image_prep.camera_inputs(img_inputs, metas)
    outs = []
    graph_replay(lambda: outs.extend(image_prep.camera_inputs(img_inputs, metas)[i] for i in (0, 6)), outs)
    same_bits(outs[0], eager[0], "images after graph replay")
    same_bits(outs[1], eager[6], "depth maps after graph replay")


# ---------------------------------------------------------------------------------------------- the C ABI
def _depth_args(cuda, B=2, N=3, H=20, W=30):
    pts = torch.from_numpy(_planted(W, H)).to(cuda)
    n = pts.shape[0]
    eye = torch.eye(3, device=cuda).expand(B, N, 3, 3).contiguous()
    out = sentinel(B * N * H, W, cuda)
    offsets = (ctypes.c_longlong * (B + 1))(*[n * b // B for b in range(B + 1)])
    return [pts, offsets, B, N, eye, torch.zeros(B, N, 3, device=cuda), eye.clone(), 3, eye.clone(),
            torch.zeros(B, N, 3, device=cuda), H, W, out], out


def test_lidar_depth_argument_errors(cuda):
    args, out = _depth_args(cuda)
    assert launches("occ_lidar_depth", *args) == 3

    def bad(i, value):
        a, o = _depth_args(cuda)
        a[i] = value
        rejected("occ_lidar_depth", *a, buffers=[o], rc=-1)

    bad(1, (ctypes.c_longlong * 3)(1, 5, 10))       # offsets[0] != 0
    bad(1, (ctypes.c_longlong * 3)(0, 10, 5))       # decreasing
    bad(2, 0)                                       # B = 0
    bad(2, 257)                                     # B above the bound
    bad(3, 0)                                       # N = 0
    bad(7, 5)                                       # intrinsics neither 3 x 3 nor 4 x 4
    bad(10, 0)                                      # fH = 0
    bad(11, -1)                                     # fW < 0
    bad(0, None)                                    # no points but offsets[B] > 0


def _aug_args(cuda, flip=0, coeffs=(65536, 0, 0, 0, 65536, 0)):
    geoms = [(90, 160, 70, 39, 0, 14), (90, 160, 70, 39, -3, 2)]
    frames = torch.from_numpy(np.stack([ip.frame(40 + m, 90, 160) for m in range(2)])).reshape(-1).to(cuda)
    tables = []
    for H, W, rW, rH, _, _ in geoms:
        tables += [ops._prep_table(cuda, W, rW).data_ptr(), ops._prep_table(cuda, H, rH).data_ptr()]
    geom = (ctypes.c_int * 12)(*[v for g in geoms for v in g])
    nbytes = ops.lib().occ_prepare_images_workspace_bytes(geom, 2, 25, 70)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=cuda)
    norm = torch.from_numpy(image_prep.normalize_table(**image_prep.norm_config(None))).to(cuda)
    out = sentinel(2 * 3 * 25, 70, cuda)
    aug = (ctypes.c_int * 14)(*([flip, *coeffs] * 2))
    return [frames, frames.numel(), (ctypes.c_longlong * 2)(0, 90 * 160 * 3), geom, aug, 2, 25, 70,
            (ctypes.c_longlong * 4)(*tables), norm, 1, ws, ws.numel(), out], out


def test_prepare_images_aug_argument_errors(cuda):
    args, out = _aug_args(cuda, 1, image_prep.rotate_coeffs(3.0, 70, 25))
    assert launches("occ_prepare_images_aug", *args) == 2
    for a, o in (_aug_args(cuda, flip=2), _aug_args(cuda, coeffs=(65536, 0, (1 << 31) - 65536 * 30, 0, 65536, 0)),
                 _aug_args(cuda, coeffs=(0, -65536, -(1 << 31) + 65536 * 10, 65536, 0, 0))):
        rejected("occ_prepare_images_aug", *a, buffers=[o], rc=-1)
    a, o = _aug_args(cuda)
    a[4] = None
    rejected("occ_prepare_images_aug", *a, buffers=[o], rc=-1)
    a, o = _aug_args(cuda)
    a[12] = 0                                        # workspace too short
    rejected("occ_prepare_images_aug", *a, buffers=[o], rc=-1)
