"""What panoptic evaluation (PanopticEval.addBatch, occ_panoptic_eval) costs on the GPU, next to the plain-torch
restatement of the reference's per-class np.unique algorithm (oracle/panoptic_eval.py) on the host.

    python scripts/bench_panoptic_eval.py [--iters 20]

Inputs: one 256x256x32 voxel scan (~5000 thing instances, 20 % ignored) and one 34 720-point LiDAR scan, int64 on the
device.  Device time per addBatch with CUDA events, L2 flushed before every call; host time of the restatement on the
same inputs already in host memory (the device-to-host copy is not counted).  Prints the card name, power limit and max
SM clock and the host's core count with the numbers.  Needs a GPU; there is no CPU fallback.
"""
import argparse
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from occformer_b200.dist_eval import PanopticEval  # noqa: E402
from oracle import panoptic_eval as pe  # noqa: E402
from gpu_bench import card  # noqa: E402


def device_ms(scan, iters, flush):
    ev = PanopticEval(17, ignore=[0], min_points=15)
    for _ in range(3):
        ev.addBatch(*scan)
    torch.cuda.synchronize()
    ms = []
    for i in range(iters):
        flush.fill_(float(i))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ev.addBatch(*scan)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return ms[len(ms) // 2], ms[0], ms[-1]


def host_ms(scan, reps):
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        pe.panoptic_counts(*scan, 17, [0], 15)
        ts.append((time.perf_counter() - t) * 1e3)
    return min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_panoptic_eval: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    print(f"host: {os.cpu_count()} cores, torch {torch.get_num_threads()} threads")
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)  # 256 MB > L2
    for name, scan in (("voxels 256x256x32", pe.voxel_scan(1)), ("LiDAR 34720 points", pe.point_scan(10))):
        med, lo, hi = device_ms([t.to(dev).reshape(-1) for t in scan], args.iters, flush)
        h = host_ms([t.reshape(-1) for t in scan], 3)
        print(f"  {name}: addBatch on the device {med:.3f} ms (median of {args.iters}; {lo:.3f} .. {hi:.3f}), "
              f"restatement on the host {h:.1f} ms")


if __name__ == "__main__":
    main()
