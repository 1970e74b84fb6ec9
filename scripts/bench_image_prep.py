"""What the image side of the test loaders costs: the resize, crop and normalisation on the GPU
(occformer_b200.image_prep.prepare_images, occ_prepare_images) next to the reference's steps 2-4 on the host (Pillow
resize + crop, mmcv's imnormalize by its cv2 calls, a float32 CHW tensor), from decoded frames.

    python scripts/bench_image_prep.py [--iters 30]

Per config (nuScenes R50: 6 cameras 900x1600 -> 256x704; R101: 6 x 900x1600 -> 896x1600; SemanticKITTI: 1 x 376x1241
-> 384x1280) and batch 1 and 4:
  device   the call captured once into a CUDA graph and replayed between CUDA events, L2 flushed before each, median
  bound    the bytes the call must move (source rows the resize reads + the float32 output) over 3.35 TB/s
  host     one core, per sample: the reference's steps 2-4 (Pillow + cv2), and the new transform's non-decode work
  upload   host-to-device bytes and time from pinned memory of the uint8 frames and of the float32 images
Prints the card name, power limit and max SM clock with the numbers.  Needs a GPU; there is no CPU fallback.
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from occformer_b200 import image_prep  # noqa: E402
from occformer_b200.pipelines import _ImageFrames  # noqa: E402
from oracle import image_prep as ip  # noqa: E402
from gpu_bench import card, graphed  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM data sheet
CONFIGS = {"nusc_r50": ([(900, 1600)] * 6, (256, 704), ip.NORM_R50),
           "nusc_r101": ([(900, 1600)] * 6, (896, 1600), ip.NORM_R101),
           "kitti": ([(376, 1241)], (384, 1280), ip.NORM_R50)}


def aug(shapes, size, norm):
    a = [ip.test_augmentation(H, W, size) for H, W in shapes]
    return dict(resize_dims=[list(x[1]) for x in a], crop=[list(x[2]) for x in a], input_size=list(size),
                **image_prep.norm_config(norm))


def bytes_needed(shapes, size):
    """source rows the vertical taps of the cropped rows read (whole rows) + the float32 output, per sample"""
    total = 0
    for H, W in shapes:
        _, (rW, rH), (x0, y0, x1, y1) = ip.test_augmentation(H, W, size)
        first, count, _ = ip.coeffs(H, rH)
        r0, r1 = max(y0, 0), min(y1, rH) - 1
        rows = first[r1] + count[r1] - first[r0] if r0 <= r1 else 0
        total += rows * W * 3 + 3 * size[0] * size[1] * 4
    return total


def host_reference(frame, a, c, norm):
    """steps 2-4 of the reference for one decoded frame: Pillow resize + crop, imnormalize's cv2 calls, CHW tensor"""
    import cv2
    from PIL import Image
    img = np.array(Image.fromarray(frame).resize(tuple(a["resize_dims"][c])).crop(tuple(a["crop"][c])))
    img = img.astype(np.float32)
    mean = np.float64(np.array(norm["mean"], np.float32).reshape(1, -1))
    stdinv = 1 / np.float64(np.array(norm["std"], np.float32).reshape(1, -1))
    if norm["to_rgb"]:
        cv2.cvtColor(img, cv2.COLOR_BGR2RGB, img)
    cv2.subtract(img, mean, img)
    cv2.multiply(img, stdinv, img)
    return torch.tensor(img).float().permute(2, 0, 1).contiguous()


def timed(run, iters, flush):
    ms = []
    for i in range(iters):
        flush.fill_(float(i))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return ms[len(ms) // 2], ms[0], ms[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_image_prep: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.set_num_threads(1)
    try:
        import cv2
        cv2.setNumThreads(1)
    except ImportError:
        cv2 = None
    print(f"card: {card()}")
    print(f"host: {os.cpu_count()} cores, timed on one thread")
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)  # 256 MB > L2
    for name, (shapes, size, norm) in CONFIGS.items():
        frames = [ip.frame(100 + c, H, W) for c, (H, W) in enumerate(shapes)]
        a = aug(shapes, size, norm)
        need = bytes_needed(shapes, size)
        for B in (1, 4):
            host = torch.from_numpy(np.stack([np.stack(frames)] * B)).pin_memory()
            x = host.to(dev)
            g, out = graphed(lambda: image_prep.prepare_images(x, [a] * B))
            g.replay()
            torch.cuda.synchronize()
            ref = torch.from_numpy(np.stack([ip.prepare(f, a["resize_dims"][c], a["crop"][c], norm)
                                             for c, f in enumerate(frames)]))
            assert all(torch.equal(out[b].cpu().view(torch.int32), ref.view(torch.int32)) for b in range(B)), \
                "device images differ from the restatement"
            med, lo, hi = timed(g.replay, args.iters, flush)
            bound_ms = need * B / HBM_BPS * 1e3
            print(f"  {name} batch {B}: device {med:.4f} ms (graph replay, median of {args.iters}; {lo:.4f} .. "
                  f"{hi:.4f}); moves >= {need * B / 1e6:.1f} MB -> {need * B / med / 1e6:.0f} GB/s, "
                  f"bound {bound_ms:.4f} ms at 3.35 TB/s ({bound_ms / med:.0%} of it)")
            host_f = torch.empty(out.shape, dtype=torch.float32).pin_memory()
            for what, src in (("uint8 frames", host), ("float32 images", host_f)):
                dst = torch.empty(src.shape, dtype=src.dtype, device=dev)
                up = timed(lambda: dst.copy_(src, non_blocking=True), 10, flush)[0]
                print(f"    upload {what}: {src.numel() * src.element_size() / 1e6:.1f} MB in {up:.3f} ms "
                      f"(pinned, median of 10)")
        if cv2 is None:
            print("  host reference: not run (cv2 not importable)")
            continue
        ts = []
        for _ in range(2):
            t = time.perf_counter()
            for c, f in enumerate(frames):
                host_reference(f, a, c, norm)
            ts.append((time.perf_counter() - t) * 1e3)
        tr = _ImageFrames(dict(input_size=size, crop_h=(0.0, 0.0), resize_test=0.0), img_norm_cfg=norm)
        tn = []
        for _ in range(5):
            t = time.perf_counter()
            for f in frames:
                tr.camera_size(*f.shape[:2])
            torch.from_numpy(np.stack(frames))
            tn.append((time.perf_counter() - t) * 1e3)
        print(f"  {name} host per sample, one thread: reference steps 2-4 (Pillow + cv2) {min(ts):.1f} ms; "
              f"new transform's non-decode work {min(tn):.2f} ms")


if __name__ == "__main__":
    main()
