"""Camera images on the GPU from the decoded frames: the resize, crop and normalisation of the reference's test loaders
(LoadMultiViewImageFromFiles_OccFormer, P/datasets/pipelines/loading_nusc_imgs.py:34-62,181-195;
LoadMultiViewImageFromFiles_SemanticKitti, loading_kitti_imgs.py:35-65), bit for bit (csrc/image_prep.cu).

The loader transforms of occformer_b200.pipelines hand the model uint8 BGR frames and, per sample, an ``img_aug`` meta:

    {"resize_dims": [[rW, rH], ...], "crop": [[x0, y0, x1, y1], ...],   # one per camera, as sample_augmentation gives
     "input_size": [fH, fW], "mean": [3 floats], "std": [3 floats], "to_rgb": bool}   # mmlabNormalize's config

decode_jpeg decodes the camera files themselves on the device (csrc/jpeg_decode.cu), bit for bit as cv2.imdecode,
into the frames prepare_images takes; the loader then ships the JPEG bytes instead of the decoded frames
(pipelines.LoadMultiViewJpegBytes_OccFormer).  decode_png does the same for SemanticKITTI's PNG frames
(csrc/png_decode.cu, pipelines.LoadMultiViewPngBytes_SemanticKitti).

Training pipelines add per camera 'flip' and 'rotate' to img_aug (pipelines.LoadMultiViewImageFramesAug_*), which
prepare_images then applies as Pillow's FLIP_LEFT_RIGHT and Image.rotate (rotate_coeffs); LoadLidarDepthPoints adds
the LiDAR scan, from which lidar_depth_maps builds CreateDepthFromLiDAR's depth maps; camera_inputs does both for a
training step.

The host part here is table building: Pillow's bicubic coefficients per (source size, resized size) of an axis and the
normalisation as a 3 x 256 table, both in float64 numpy, one operation at a time as x86-64 builds of Pillow and OpenCV
compute them (no fused multiply-add).  ops.prepare_images caches them on the device.
"""
import math

import numpy as np
import torch

from . import jpeg, ops, png

PRECISION_BITS = 22  # Pillow's resample.c: 32 - 8 - 2
DEFAULT_NORM = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)  # mmlabNormalize's


def _bicubic(x):
    """Pillow's bicubic_filter, a = -0.5, in its operation order"""
    x = np.abs(x)
    a = -0.5
    near = ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    far = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def resample_table(in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for one axis of Image.resize (box (0, in_size)) -> int32
    [2 * out_size] (first tap, tap count per output index) ++ [ksize * out_size] weights tap-major, 22 fractional bits"""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    center = (np.arange(out_size) + 0.5) * scale
    first = np.maximum(np.trunc(center - support + 0.5).astype(np.int64), 0)
    last = np.minimum(np.trunc(center + support + 0.5).astype(np.int64), in_size)
    count = last - first
    ss = 1.0 / filterscale
    taps = np.arange(ksize)
    w = _bicubic(((taps[None, :] + first[:, None]) - center[:, None] + 0.5) * ss)
    w = np.where(taps[None, :] < count[:, None], w, 0.0)
    ww = np.zeros(out_size)
    for k in range(ksize):  # the C loop's order, not numpy's pairwise sum
        ww = ww + w[:, k]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    fixed = w * (1 << PRECISION_BITS)
    fixed = np.trunc(np.where(w < 0, -0.5 + fixed, 0.5 + fixed)).astype(np.int32)
    bounds = np.stack([first, count], axis=1).astype(np.int32)
    return np.concatenate([bounds.reshape(-1), fixed.T.reshape(-1)])


def normalize_table(mean, std, to_rgb):
    """mmcv's imnormalize of every uint8 value -> float32 (3, 256) in output channel order: cv2.subtract of the float64
    mean, rounded to float32, then cv2.multiply by the float64 1 / std, rounded to float32.  to_rgb (cvtColor BGR2RGB
    first) leaves the table as it is: output channel c then reads source channel 2 - c (the kernel's swap_rb)."""
    mean = np.asarray(mean, dtype=np.float32).astype(np.float64)
    stdinv = 1 / np.asarray(std, dtype=np.float32).astype(np.float64)
    v = np.arange(256, dtype=np.float64)
    rows = [((v - mean[c]).astype(np.float32).astype(np.float64) * stdinv[c]).astype(np.float32) for c in range(3)]
    return np.stack(rows)


def norm_config(img_norm_cfg):
    """mmlabNormalize's reading of img_norm_cfg (None: its defaults) -> dict(mean, std, to_rgb) of plain Python values"""
    cfg = DEFAULT_NORM if img_norm_cfg is None else img_norm_cfg
    return dict(mean=[float(v) for v in cfg["mean"]], std=[float(v) for v in cfg["std"]], to_rgb=bool(cfg["to_rgb"]))


def prepare_images(frames, img_aug):
    """frames: uint8 CUDA (B, N, H, W, 3) BGR, or a list of B per-sample (N, H_i, W_i, 3) tensors; img_aug: B metas (the
    module docstring) -> float32 (B, N, 3, fH, fW), the reference loaders' img_inputs[0] stacked by the collate.
    All samples must share input_size and the normalisation config."""
    if torch.is_tensor(frames):
        if frames.dim() != 5:
            raise ValueError(f"prepare_images: frames must be (B, N, H, W, 3), got {tuple(frames.shape)}")
        samples = list(frames.unbind(0))
    else:
        samples = list(frames)
    if len(samples) != len(img_aug) or not samples:
        raise ValueError(f"prepare_images: {len(samples)} samples of frames but {len(img_aug)} img_aug metas")
    train = [("flip" in a) or ("rotate" in a) for a in img_aug]
    if any(train) and not all(train):
        raise ValueError("prepare_images: a batch mixes training-mode img_aug (flip / rotate) and test-mode img_aug")
    for s in samples:
        if s.dtype != torch.uint8 or s.dim() != 4 or s.shape[-1] != 3:
            raise ValueError(f"prepare_images: every sample must be uint8 (N, H, W, 3), got {s.dtype} "
                             f"{tuple(s.shape)}")
        if not s.is_cuda:
            raise RuntimeError("prepare_images: frames must be CUDA tensors (no CPU fallback exists)")
    a0 = img_aug[0]
    size = [int(v) for v in a0["input_size"]]
    norm = norm_config(a0)
    N = samples[0].shape[0]
    for s, a in zip(samples, img_aug):
        if [int(v) for v in a["input_size"]] != size or norm_config(a) != norm:
            raise ValueError("prepare_images: every sample of a batch needs the same input_size and normalisation")
        if s.shape[0] != N or len(a["resize_dims"]) != N or len(a["crop"]) != N:
            raise ValueError("prepare_images: every sample needs the same number of cameras, one resize and crop each")
        for (rW, rH), (x0, y0, x1, y1) in zip(a["resize_dims"], a["crop"]):
            if (int(x1) - int(x0), int(y1) - int(y0)) != (size[1], size[0]):
                raise ValueError(f"prepare_images: crop {(x0, y0, x1, y1)} is not input_size {tuple(size)}")
    if torch.is_tensor(frames) and frames.is_contiguous():
        flat = frames.reshape(-1)
    else:
        flat = torch.cat([s.contiguous().reshape(-1) for s in samples])
    offsets, geoms, aug, off = [], [], [], 0
    for s, a in zip(samples, img_aug):
        H, W = int(s.shape[1]), int(s.shape[2])
        for c, ((rW, rH), crop) in enumerate(zip(a["resize_dims"], a["crop"])):
            offsets.append(off)
            geoms.append((H, W, int(rW), int(rH), int(crop[0]), int(crop[1])))
            off += H * W * 3
            if train[0]:
                flip = bool(a.get("flip", [False] * N)[c])
                aug.append((int(flip),) + rotate_coeffs(a.get("rotate", [0.0] * N)[c], size[1], size[0]))
    out = ops.prepare_images(flat, offsets, geoms, size, norm["mean"], norm["std"], norm["to_rgb"],
                             aug if train[0] else None)
    return out.view(len(samples), N, 3, *size)


def rotate_coeffs(angle, w, h):
    """Pillow's Image.rotate(angle) (NEAREST, no expand, black fill) of a w x h image as the six 16.16 fixed-point
    coefficients (a0, .., a5) of its affine_fixed gather: output (x, y) reads ((a2 + y a1 + x a0) >> 16,
    (a5 + y a4 + x a3) >> 16), 0 outside.  Pillow copies at angle 0 and transposes at 180, and at 90 / 270 for a square
    image: those take the coefficients of the same permutation.  Otherwise the matrix is Image.rotate's float64 one
    about (w / 2, h / 2), and FIX(v) = floor(v * 65536 + 0.5) as in Pillow's Geometry.c."""
    angle = angle % 360.0
    one = 1 << 16
    if angle == 0:
        return (one, 0, 0, 0, one, 0)
    if angle == 180:
        return (-one, 0, (w - 1) << 16, 0, -one, (h - 1) << 16)
    if angle == 90 and w == h:   # Transpose.ROTATE_90: out (x, y) = in (w - 1 - y, x)
        return (0, -one, (w - 1) << 16, one, 0, 0)
    if angle == 270 and w == h:  # Transpose.ROTATE_270: out (x, y) = in (y, h - 1 - x)
        return (0, one, 0, -one, 0, (h - 1) << 16)
    a = -math.radians(angle)
    m = [round(math.cos(a), 15), round(math.sin(a), 15), 0.0, round(-math.sin(a), 15), round(math.cos(a), 15), 0.0]
    cx, cy = w / 2.0, h / 2.0
    m[2] = m[0] * -cx + m[1] * -cy + m[2] + cx
    m[5] = m[3] * -cx + m[4] * -cy + m[5] + cy
    # Pillow takes the fixed-point path while the far corner maps inside +-32768 (check_fixed); past that it would
    # interpolate in float64, which this gather does not restate
    if not (abs(w * m[0] + h * m[1] + m[2]) < 32768.0 and abs(w * m[3] + h * m[4] + m[5]) < 32768.0):
        raise ValueError(f"rotate_coeffs: a {w} x {h} image is past Pillow's fixed-point rotation")

    def fix(v):
        return math.floor(v * 65536.0 + 0.5)
    return (fix(m[0]), fix(m[1]), fix(m[2] + m[1] * 0.5 + m[0] * 0.5), fix(m[3]), fix(m[4]),
            fix(m[5] + m[4] * 0.5 + m[3] * 0.5))


def lidar_depth_maps(points, img_inputs, img_aug):
    """CreateDepthFromLiDAR's gt_depths on the GPU (csrc/lidar_depth.cu), bit for bit as a loader worker computes them:
    points, B scans of float32 (P_b, 3) (host or CUDA); img_inputs, the collated tuple (trans, intrins, post_rots,
    post_trans at [2:6], CUDA); img_aug, B metas with 'lidar_inv_rots' (pipelines.LoadLidarDepthPoints) and
    'input_size' -> float32 (B, N, fH, fW).  The scans travel in one pinned host buffer and one host-to-device copy."""
    if len(points) != len(img_aug) or not img_aug:
        raise ValueError(f"lidar_depth_maps: {len(points)} scans but {len(img_aug)} img_aug metas")
    trans, intrins, post_rots, post_trans = img_inputs[2:6]
    dev = trans.device
    B, N = trans.shape[:2]
    size = [int(v) for v in img_aug[0]["input_size"]]
    if any([int(v) for v in a["input_size"]] != size for a in img_aug):
        raise ValueError("lidar_depth_maps: every sample of a batch needs the same input_size")
    pts = [torch.as_tensor(p, dtype=torch.float32).reshape(-1, 3) for p in points]
    offsets = np.cumsum([0] + [len(p) for p in pts]).tolist()
    if all(p.is_cuda for p in pts):
        flat = torch.cat(pts).contiguous()
    else:
        flat, _ = ops._stage([p.cpu().contiguous().numpy().view(np.uint8).reshape(-1) for p in pts])
        flat = flat.view(torch.float32).view(-1, 3)
    inv_rots = torch.stack([torch.as_tensor(a["lidar_inv_rots"], dtype=torch.float32) for a in img_aug]).to(dev)
    return ops.lidar_depth(flat, offsets, inv_rots.contiguous(), trans.float().contiguous(),
                           intrins.float().contiguous(), post_rots.float().contiguous(),
                           post_trans.float().contiguous(), size)


def is_file_placeholder(imgs):
    """the empty uint8 (B, N, 0) img_inputs[0] of the byte transforms (pipelines.LoadMultiView*Bytes*)"""
    return torch.is_tensor(imgs) and imgs.dtype == torch.uint8 and imgs.dim() == 3 and imgs.shape[-1] == 0


def decode_files(img_aug):
    """the frames of the files the byte transforms put into img_aug: 'png' files in every meta (decode_png), else
    'jpeg' files in every meta (decode_jpeg), named by 'png_files' / 'jpeg_files' -> decoded frames; None when the metas
    carry neither"""
    kind = next((k for k in ("png", "jpeg") if img_aug and all(k in a for a in img_aug)), None)
    if kind is None:
        return None
    names = [a.get(kind + "_files") for a in img_aug]
    decode = decode_png if kind == "png" else decode_jpeg
    return decode([a[kind] for a in img_aug], None if None in names else names)


def input_frames(imgs, img_metas, missing):
    """img_inputs[0] -> the camera frames: the byte transforms' placeholder (is_file_placeholder) decoded from the files
    in the 'img_aug' of img_metas (decode_files), anything else as it is; missing: the message of the ValueError raised
    when the placeholder comes without files"""
    if not is_file_placeholder(imgs):
        return imgs
    frames = decode_files([m.get("img_aug", {}) for m in img_metas or []])
    if frames is None:
        raise ValueError(missing)
    return frames


def camera_inputs(img_inputs, img_metas):
    """The reference training pipeline's collated img_inputs on the GPU, from those of LoadMultiViewImageFramesAug_* (or
    LoadMultiViewJpegBytesAug_OccFormer / LoadMultiViewPngBytesAug_SemanticKitti) + LoadLidarDepthPoints: img_inputs[0]
    the uint8 frames (prepare_images), or the byte transforms' empty placeholder, whose files are decoded first
    (input_frames); the gt_depths placeholder (the slot before sensor2sensors: 6 of the loaders' 8-tuple, 7 once an
    occupancy annotation transform has added bda_rot) replaced by lidar_depth_maps; every other element passed through.
    img_metas: B dicts carrying 'img_aug'."""
    img_aug = [m["img_aug"] for m in img_metas]
    frames = input_frames(img_inputs[0], img_metas, "camera_inputs: the empty image placeholder needs each sample's "
                          "'img_aug' meta with its 'jpeg' or 'png' files, which the byte transforms produce")
    imgs = prepare_images(frames, img_aug)
    depths = lidar_depth_maps([a["lidar_points"] for a in img_aug], img_inputs, img_aug)
    k = len(img_inputs) - 2
    return (imgs,) + tuple(img_inputs[1:k]) + (depths,) + tuple(img_inputs[k + 1:])


def _decode(what, files, names, parse, error, payload, decode, complaint, status_bits):
    """the front end of decode_jpeg / decode_png (what): files B samples of N files, each parsed on the host by parse
    (its error, an exception class, re-raised as ValueError naming the file) into a header; payload(file as a uint8
    memoryview, header) -> the file's bytes to stage; decode(headers, payloads) -> (flat frames, int32 (M, 2) status)
    of ops.decode_*.  One status read-back then raises ValueError naming the first file whose status is not 0 with
    complaint and the names of its status_bits ((bit, name) pairs) -> the frames as _frames gives them"""
    samples = [list(s) for s in files]
    if not samples or any(not s for s in samples):
        raise ValueError(f"{what}: needs at least one sample of at least one file")
    label = [[names[b][n] if names is not None else f"sample {b} camera {n}" for n in range(len(s))]
             for b, s in enumerate(samples)]
    headers, payloads = [], []
    for s, lab in zip(samples, label):
        for f, name in zip(s, lab):
            try:
                h = parse(f)
            except error as e:
                raise ValueError(f"{what}: {name}: {e}") from None
            headers.append(h)
            payloads += payload(memoryview(f).cast("B"), h)
    first = np.cumsum([0] + [len(s) for s in samples])  # each sample's first image, then M
    for b0, b1 in zip(first[:-1], first[1:]):
        sizes = {(h.height, h.width) for h in headers[b0:b1]}
        if len(sizes) != 1:
            raise ValueError(f"{what}: the cameras of a sample need one frame size, got {sorted(sizes)}")
    out, status = decode(headers, payloads)
    bad = status[:, 0].cpu()
    if bool(bad.any()):
        m = int(bad.nonzero()[0, 0])
        b = int(np.searchsorted(first[1:], m, side="right"))
        raise ValueError(f"{what}: {label[b][m - first[b]]}: {complaint} (status {int(bad[m])}: "
                         + ", ".join(w for bit, w in status_bits if int(bad[m]) & bit) + ")")
    return _frames(out, samples, headers)


def _frames(out, samples, headers):
    """the decoders' flat frames -> (B, N, H, W, 3) when every sample shares N and the frame size, else the list of B
    per-sample (N, H_i, W_i, 3) views"""
    shapes = [(len(s), headers[b0].height, headers[b0].width)
              for s, b0 in zip(samples, np.cumsum([0] + [len(s) for s in samples])[:-1])]
    if len(set(shapes)) == 1 and len({len(s) for s in samples}) == 1:
        return out.view(len(samples), *shapes[0], 3)
    res, o = [], 0
    for N, H, W in shapes:
        res.append(out[o:o + N * H * W * 3].view(N, H, W, 3))
        o += N * H * W * 3
    return res


JPEG_STATUS = ((1, "unexpected marker"), (2, "bad restart markers"), (4, "invalid Huffman code or run"),
               (8, "data ends early"))


def decode_jpeg(files, names=None, seq_bits=ops.JPEG_SEQ_BITS, sync_rounds=ops.JPEG_SYNC_ROUNDS):
    """files: B samples, each a list of N JPEG files (bytes-like) -> uint8 CUDA (B, N, H, W, 3) B, G, R frames when all
    share one size, else a list of B per-sample (N, H_i, W_i, 3) tensors: the two forms prepare_images takes, equal to
    cv2.imdecode(buf, IMREAD_UNCHANGED) of each file.  The files travel in one pinned host buffer and one host-to-device
    copy, and decode in one occ_decode_jpeg call; one status read-back then raises ValueError naming a file whose
    entropy-coded data is corrupt (libjpeg would warn and fill in grey).  names: the same nesting of file names for the
    messages (default: sample and camera indices).  seq_bits / sync_rounds tune the parallel Huffman decode and do not
    change the result."""
    def decode(headers, payloads):
        data, offsets = ops._stage(payloads)
        return ops.decode_jpeg(data, offsets, headers, seq_bits, sync_rounds)
    return _decode("decode_jpeg", files, names, jpeg.parse, jpeg.JpegError, lambda f, h: [f], decode,
                   "corrupt entropy-coded data", JPEG_STATUS)


PNG_STATUS = ((1, "invalid deflate data"), (2, "data ends early or too little image data"),
              (4, "incorrect Adler-32 check"), (8, "bad filter type"))


def decode_png(files, names=None):
    """files: B samples, each a list of N 8-bit RGB PNG files (bytes-like) -> uint8 CUDA (B, N, H, W, 3) B, G, R frames
    when all share one size, else a list of B per-sample (N, H_i, W_i, 3) tensors: the two forms prepare_images takes,
    equal to cv2.imdecode(buf, IMREAD_UNCHANGED) of each file.  png.parse walks the chunks on the host (refused kinds
    raise ValueError naming the file); the zlib streams and the IDAT chunk starts travel in one pinned host buffer and
    one host-to-device copy, and decode in one occ_decode_png call; one status read-back then raises ValueError naming
    a file cv2 would not decode.  names: the same nesting of file names for the messages (default: sample and camera
    indices)."""
    def decode(headers, payloads):
        starts = [s for h in headers for s in np.cumsum([0] + [n for _, n in h.idat])[:-1].tolist()]
        streams = sum((h.stream_len for h in headers), 0)
        pad = -streams % 4
        data, _ = ops._stage(payloads + [bytes(pad), np.asarray(starts, np.int32).tobytes()])
        stream_off = np.cumsum([0] + [h.stream_len for h in headers])[:-1].tolist()
        idat = data[streams + pad:].view(torch.int32)
        return ops.decode_png(data[:max(streams, 1)], stream_off, headers, idat)
    return _decode("decode_png", files, names, png.parse, png.PngError, lambda f, h: [f[o:o + n] for o, n in h.idat],
                   decode, "cv2 would not decode it", PNG_STATUS)
