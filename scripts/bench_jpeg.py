"""What decoding the camera files costs: the JPEG decode on the GPU (occformer_b200.image_prep.decode_jpeg,
occ_decode_jpeg) next to cv2.imdecode on the host, which the reference's loader runs on every camera file.

    python scripts/bench_jpeg.py [--iters 30] [--profile]

Per config (nuScenes R50: 6 cameras 900x1600 -> 256x704; R101: 6 x 900x1600 -> 896x1600) and batch 1 and 4, on
synthetic frames (oracle.image_prep.frame, cv2.imencode quality 95, 4:2:0, no restart markers):
  decode   occ_decode_jpeg captured once into a CUDA graph and replayed between CUDA events, L2 flushed, median
  +prep    the same for decode_jpeg's kernels followed by prepare_images
  upload   host-to-device bytes and time from pinned memory of the files and of the decoded uint8 frames
  host     cv2.imdecode per frame on one host core
  files    the sizes of the synthetic files, which set the Huffman work
--profile adds the device time of every kernel of one batch-4 call (torch.profiler), to show where the time goes.
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
from occformer_b200 import image_prep, jpeg, ops  # noqa: E402
from oracle import image_prep as ip  # noqa: E402
from oracle import jpeg as oj  # noqa: E402
from gpu_bench import card, graphed  # noqa: E402

CONFIGS = {"nusc_r50": ((256, 704), ip.NORM_R50), "nusc_r101": ((896, 1600), ip.NORM_R101)}
N, H, W = 6, 900, 1600


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
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--tune", action="store_true", help="batch-4 decode time over subsequence lengths and rounds")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg: needs a CUDA device")
    import cv2
    cv2.setNumThreads(1)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.set_num_threads(1)
    print(f"card: {card()}")
    print(f"host: {os.cpu_count()} cores, timed on one thread")
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)  # 256 MB > L2
    files = [oj.encode(ip.frame(300 + c, H, W), 95, "420") for c in range(N)]
    sizes = [len(f) for f in files]
    print(f"files: {N} synthetic {W}x{H} frames, quality 95, 4:2:0: {min(sizes) / 1e6:.3f} .. {max(sizes) / 1e6:.3f} MB, "
          f"{sum(sizes) / 1e6:.2f} MB per sample against {N * H * W * 3 / 1e6:.1f} MB decoded")
    refs = [oj.cv2_decode(f) for f in files]
    ts = []
    for _ in range(3):
        t = time.perf_counter()
        for f in files:
            oj.cv2_decode(f)
        ts.append((time.perf_counter() - t) * 1e3 / N)
    print(f"host cv2.imdecode, one thread: {min(ts):.2f} ms per frame, {min(ts) * N:.1f} ms per sample")
    for B in (1, 4):
        batch = [files] * B
        headers = [jpeg.parse(f) for s in batch for f in s]
        offsets = np.cumsum([0] + [len(f) for s in batch for f in s]).tolist()
        host = torch.from_numpy(np.frombuffer(b"".join(f for s in batch for f in s), np.uint8).copy()).pin_memory()
        data = host.to(dev)
        t0 = time.perf_counter()
        for s in batch:
            for f in s:
                jpeg.parse(f)
        parse_us = (time.perf_counter() - t0) * 1e6 / (B * N)
        g, (out, status) = graphed(lambda: ops.decode_jpeg(data, offsets[:-1], headers))
        g.replay()
        torch.cuda.synchronize()
        assert int(status[:, 0].abs().sum()) == 0
        got = out.view(B * N, H, W, 3).cpu().numpy()
        assert all(np.array_equal(got[i], refs[i % N]) for i in range(B * N)), "device frames differ from cv2"
        med, lo, hi = timed(g.replay, args.iters, flush)
        print(f"  batch {B} ({B * N} frames): decode {med:.3f} ms (graph replay, median of {args.iters}; {lo:.3f} .. "
              f"{hi:.3f}); fix-up re-decoded {int(status[:, 1].sum())} subsequences; host header parse "
              f"{parse_us:.0f} us per file")
        for name, (size, norm) in CONFIGS.items():
            a = [ip.test_augmentation(H, W, size) for _ in range(N)]
            aug = dict(resize_dims=[list(x[1]) for x in a], crop=[list(x[2]) for x in a], input_size=list(size),
                       **image_prep.norm_config(norm))

            def both():
                o, _ = ops.decode_jpeg(data, offsets[:-1], headers)
                return image_prep.prepare_images(o.view(B, N, H, W, 3), [aug] * B)
            g2, _ = graphed(both)
            m2 = timed(g2.replay, args.iters, flush)[0]
            print(f"    {name}: decode + prepare_images {m2:.3f} ms (graph replay, median of {args.iters})")
        frames = torch.empty((B, N, H, W, 3), dtype=torch.uint8).pin_memory()
        for what, src in (("JPEG files", host), ("decoded frames", frames)):
            dst = torch.empty(src.shape, dtype=src.dtype, device=dev)
            up = timed(lambda: dst.copy_(src, non_blocking=True), 10, flush)[0]
            print(f"    upload {what}: {src.numel() / 1e6:.2f} MB in {up:.3f} ms (pinned, median of 10)")
        if args.tune and B == 4:
            for S in (1024, 2048, 4096, 8192, 16384):
                for R in (1, 2, 3, 4, 6):
                    gt, (o, st) = graphed(lambda: ops.decode_jpeg(data, offsets[:-1], headers, S, R))
                    gt.replay()
                    torch.cuda.synchronize()
                    assert torch.equal(o, out)
                    print(f"    tune S {S} R {R}: decode {timed(gt.replay, 5, flush)[0]:.3f} ms, fix-up re-decoded "
                          f"{int(st[:, 1].sum())} subsequences")
        if args.profile and B == 4:
            from torch.profiler import ProfilerActivity, profile
            ops.decode_jpeg(data, offsets[:-1], headers)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ops.decode_jpeg(data, offsets[:-1], headers)
                torch.cuda.synchronize()
            per = {}
            for e in prof.events():
                if str(e.device_type).endswith("CUDA"):
                    k = e.name.split("(")[0].replace("void ", "").replace("occ::", "")
                    per[k] = per.get(k, 0.0) + (e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total) / 1e3
            print("    kernels of one batch-4 call (torch.profiler, ms): "
                  + ", ".join(f"{k} {v:.3f}" for k, v in sorted(per.items(), key=lambda kv: -kv[1])))


if __name__ == "__main__":
    main()
