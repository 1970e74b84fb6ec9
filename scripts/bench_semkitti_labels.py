"""What SemanticKITTI's ground truth costs when it is built from the voxel files on the GPU
(targets.semantic_kitti_occupancy, occ_semkitti_labels), next to what the reference's test loop does per sample with the
preprocessed labels: np.load of the float32 '<frame>_1_1.npy', torch.tensor(...).long() (LoadSemKittiAnnotation), then
the collate's copy of the 16 MB int64 volume to the device.

    python scripts/bench_semkitti_labels.py [--iters 30]

Inputs: synthetic 256x256x32 frames (oracle.semkitti_labels.synthetic_voxels, 'mixed'), batch 1 and 4.  Device time:
the one kernel captured into a CUDA graph and replayed between CUDA events, L2 flushed before every run, median.  Call
time: the whole eager semantic_kitti_occupancy (pinned staging, one host-to-device copy of the 4.25 MB files per
sample, the kernel and the one status read-back), host clock around a device synchronise, median.  Host time of the
reference's np.load + torch.tensor(...).long() per sample (the npy in the page cache), and host-to-device time of the
16 MB int64 volume from pageable memory (as the collate hands it over) against the files from pinned memory.  Prints
the card name, power limit and max SM clock and the host's core count with the numbers.  Needs a GPU.
"""
import argparse
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from occformer_b200 import ops, targets  # noqa: E402
from oracle import semkitti_labels as sk  # noqa: E402
from gpu_bench import card, graphed  # noqa: E402

# the learning_map of the dataset yaml (semantickitti.yaml), as the fixture stores it
GOLDEN = os.path.join(ROOT, "tests", "golden", "semkitti_labels.npz")


def _median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2], xs[0], xs[-1]


def _events(run, iters, flush):
    ms = []
    for i in range(iters):
        flush.fill_(float(i))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return _median(ms)


def _host(run, iters, flush=None):
    ms = []
    for i in range(iters):
        if flush is not None:
            flush.fill_(float(i))
        torch.cuda.synchronize()
        t = time.perf_counter()
        run()
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t) * 1e3)
    return _median(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_semkitti_labels: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    print(f"host: {os.cpu_count()} cores")
    lm = {int(k): int(v) for k, v in np.load(GOLDEN)["learning_map"]}
    frames = [sk.synthetic_voxels(lm, 70 + b, "mixed") for b in range(4)]
    refs = [sk.occupancy(lab, inv, lm) for lab, inv in frames]
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)  # 256 MB > L2
    lut = torch.from_numpy(targets.semkitti_remap_lut(lm)).to(dev)
    file_mb = (targets.SEMKITTI_LABEL_BYTES + targets.SEMKITTI_INVALID_BYTES) / 2 ** 20
    vol_mb = sk.NVOX * 8 / 2 ** 20
    for B in (1, 4):
        label = torch.from_numpy(np.frombuffer(b"".join(f[0] for f in frames[:B]), np.uint8).copy()).to(dev)
        invalid = torch.from_numpy(np.frombuffer(b"".join(f[1] for f in frames[:B]), np.uint8).copy()).to(dev)
        g, (vol, bad) = graphed(lambda: ops.semkitti_labels(label, invalid, B, sk.NVOX, lut))
        g.replay()
        torch.cuda.synchronize()
        assert int(bad.sum()) == 0
        assert np.array_equal(vol.view(B, *sk.SHAPE).cpu().numpy(), np.stack(refs[:B])), "differs from restatement"
        med, lo, hi = _events(g.replay, args.iters, flush)
        moved = B * (file_mb + vol_mb) * 2 ** 20
        print(f"  batch {B}: device {med:.4f} ms per batch (graph replay, median of {args.iters}; {lo:.4f} .. {hi:.4f}), "
              f"{moved / (med * 1e-3) / 1e9:.0f} GB/s of files read + int64 volume written")
        call = lambda: targets.semantic_kitti_occupancy([f[0] for f in frames[:B]], [f[1] for f in frames[:B]], lm)
        for _ in range(3):
            call()
        cmed, clo, chi = _host(call, args.iters, flush)
        print(f"  batch {B}: eager call {cmed:.3f} ms per batch ({clo:.3f} .. {chi:.3f}): staging, one host-to-device "
              f"copy of {B * file_mb:.2f} MB, the kernel and one read-back")
    with tempfile.TemporaryDirectory() as tmp:
        npy = os.path.join(tmp, "000000_1_1.npy")
        np.save(npy, refs[0].astype(np.float32))  # what the preprocessing writes
        load = lambda: torch.tensor(np.load(npy)).long()
        load()
        hmed, hlo, hhi = _host(load, args.iters)
        print(f"  reference per sample: np.load + torch.tensor(...).long() {hmed:.3f} ms on one host core "
              f"({hlo:.3f} .. {hhi:.3f}), {os.path.getsize(npy) / 2 ** 20:.1f} MB npy read from the page cache")
    volume = torch.from_numpy(refs[0])
    files = torch.from_numpy(np.frombuffer(frames[0][0] + frames[0][1], np.uint8).copy()).pin_memory()
    for what, src, mb in (("int64 volume, pageable", volume, vol_mb), ("voxel files, pinned", files, file_mb)):
        src.to(dev)
        tmed, tlo, thi = _host(lambda: src.to(dev, non_blocking=True), args.iters)
        print(f"  host-to-device per sample, {what}: {mb:.2f} MB in {tmed:.3f} ms ({tlo:.3f} .. {thi:.3f})")


if __name__ == "__main__":
    main()
