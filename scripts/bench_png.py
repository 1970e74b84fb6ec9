"""What decoding the SemanticKITTI camera files costs: the PNG decode on the GPU (occformer_b200.image_prep.decode_png,
occ_decode_png) next to cv2.imdecode on the host, which the reference's loader runs on every frame.

    python scripts/bench_png.py [--iters 30] [--profile]

At the KITTI odometry frame size 1241x376, batch 1 and 4, on seeded photo-like frames (oracle.png.content) written by
cv2.imencode at its default level:
  decode   occ_decode_png captured once into a CUDA graph and replayed between CUDA events, L2 flushed, median
  upload   host-to-device bytes and time from pinned memory of the files and of the decoded uint8 frames
  host     cv2.imdecode per frame on one host core; png.parse (chunk walk + CRCs) per file
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
from occformer_b200 import image_prep, ops, png  # noqa: E402
from oracle import png as op  # noqa: E402
from gpu_bench import card, graphed  # noqa: E402

H, W = 376, 1241


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
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_png: needs a CUDA device")
    import cv2
    cv2.setNumThreads(1)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.set_num_threads(1)
    print(f"card: {card()}")
    print(f"host: {os.cpu_count()} cores, timed on one thread")
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)  # 256 MB > L2
    srcs = [op.content(H, W, 900 + k) for k in range(4)]
    files = [cv2.imencode(".png", s)[1].tobytes() for s in srcs]
    sizes = [len(f) for f in files]
    print(f"files: {len(files)} synthetic {W}x{H} frames, cv2.imencode default level: {min(sizes) / 1e3:.0f} .. "
          f"{max(sizes) / 1e3:.0f} KB against {H * W * 3 / 1e6:.2f} MB decoded")
    ts = []
    for _ in range(3):
        t = time.perf_counter()
        for f in files:
            op.cv2_decode(f)
        ts.append((time.perf_counter() - t) * 1e3 / len(files))
    print(f"host cv2.imdecode, one thread: {min(ts):.2f} ms per frame")
    t = time.perf_counter()
    for _ in range(5):
        for f in files:
            png.parse(f)
    print(f"host png.parse (chunk walk and CRCs): {(time.perf_counter() - t) * 1e3 / (5 * len(files)):.3f} ms per file")
    for B in (1, 4):
        batch = files[:B]
        headers = [png.parse(f) for f in batch]
        streams = [b"".join(f[o:o + n] for o, n in h.idat) for f, h in zip(batch, headers)]
        offsets = np.cumsum([0] + [len(s) for s in streams]).tolist()
        host = torch.from_numpy(np.frombuffer(b"".join(streams), np.uint8).copy()).pin_memory()
        data = host.to(dev)
        starts = sum((np.cumsum([0] + [n for _, n in h.idat])[:-1].tolist() for h in headers), [])
        idat = torch.tensor(starts, dtype=torch.int32, device=dev)
        g, (out, status) = graphed(lambda: ops.decode_png(data, offsets[:-1], headers, idat))
        g.replay()
        torch.cuda.synchronize()
        assert int(status[:, 0].abs().sum()) == 0
        got = out.view(B, H, W, 3).cpu().numpy()
        assert all(np.array_equal(got[i], srcs[i]) for i in range(B)), "device frames differ from the source"
        med, lo, hi = timed(g.replay, args.iters, flush)
        print(f"  batch {B}: decode {med:.3f} ms (graph replay, median of {args.iters}; {lo:.3f} .. {hi:.3f}); "
              f"blocks decoded serially while linking: {int(status[:, 1].sum())}")
        frames = torch.empty((B, H, W, 3), dtype=torch.uint8).pin_memory()
        for what, src in (("PNG streams", host), ("decoded frames", frames)):
            dst = torch.empty(src.shape, dtype=src.dtype, device=dev)
            up = timed(lambda: dst.copy_(src, non_blocking=True), 10, flush)[0]
            print(f"    upload {what}: {src.numel() / 1e6:.2f} MB in {up:.3f} ms (pinned, median of 10)")
        t = time.perf_counter()
        for _ in range(5):
            image_prep.decode_png([[f] for f in batch])
        torch.cuda.synchronize()
        print(f"    whole eager decode_png call (parse, staging, copy, decode, status read-back): "
              f"{(time.perf_counter() - t) * 1e3 / 5:.2f} ms")
        if args.profile and B == 4:
            from torch.profiler import ProfilerActivity, profile
            ops.decode_png(data, offsets[:-1], headers, idat)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ops.decode_png(data, offsets[:-1], headers, idat)
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
