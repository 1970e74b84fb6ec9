"""What SemanticKITTI's training-mode ground truth costs when it is built from the voxel files on the GPU
(targets.semantic_kitti_occupancy(..., augment=), occ_semkitti_labels_aug), next to what the reference's training
loader does per sample on one host core: np.load of the float32 '<frame>_1_1.npy', torch.tensor(...), then
voxel_transform (.numpy().astype(np.uint8), a Pillow NEAREST rotation of each of the 32 slices when the angle is
nonzero, the flips, .copy()) and .long().

    python scripts/bench_semkitti_train_labels.py [--iters 30]

Inputs: synthetic 256x256x32 frames (oracle.semkitti_labels.synthetic_voxels, 'mixed'), batch 1 and 4, two
augmentations: flips only (flip_dx, flip_dz) and rotated (17.3 degrees and flip_dy).  Device time: the one kernel
captured into a CUDA graph and replayed between CUDA events, L2 flushed before every run, median.  Call time: the whole
eager semantic_kitti_occupancy (pinned staging, one host-to-device copy of the files and the augmentation rows, the
kernel and the one status read-back), host clock around a device synchronise, median.  The reference's host steps are
restated here with the same library calls, under torch.set_num_threads(1) as in a DataLoader worker.  Prints the card
name, power limit and max SM clock and the host's core count with the numbers.  Needs a GPU.
"""
import argparse
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from occformer_b200 import ops, targets  # noqa: E402
from oracle import semkitti_labels as sk  # noqa: E402
from oracle import semkitti_train as st  # noqa: E402
from gpu_bench import card, graphed  # noqa: E402
from bench_semkitti_labels import _events, _host  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "semkitti_train_labels.npz")
AUGS = {"flips": dict(rotate=0.0, flip_dx=True, flip_dy=False, flip_dz=True),
        "rotated": dict(rotate=17.3, flip_dx=False, flip_dy=True, flip_dz=False)}


def reference_host(npy, aug):
    """the reference loader's per-sample host steps, with its library calls: np.load, torch.tensor, the uint8 cast,
    Image.rotate of each z slice (when not np.isclose(angle, 0)), the flips, .copy() and .long()"""
    from PIL import Image
    v = torch.tensor(np.load(npy)).numpy().astype(np.uint8)
    if not np.isclose(aug["rotate"], 0):
        v = np.stack([np.array(Image.fromarray(v[..., z]).rotate(aug["rotate"], resample=Image.Resampling.NEAREST,
                                                                 fillcolor=255)) for z in range(v.shape[-1])], axis=-1)
    if aug["flip_dz"]:
        v = v[:, :, ::-1]
    if aug["flip_dy"]:
        v = v[:, ::-1]
    if aug["flip_dx"]:
        v = v[::-1]
    return torch.from_numpy(v.copy()).long()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_semkitti_train_labels: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    print(f"host: {os.cpu_count()} cores")
    lm = {int(k): int(v) for k, v in np.load(GOLDEN)["learning_map"]}
    frames = [sk.synthetic_voxels(lm, 70 + b, "mixed") for b in range(4)]
    pre = [sk.occupancy(lab, inv, lm) for lab, inv in frames]
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)  # 256 MB > L2
    lut = torch.from_numpy(targets.semkitti_remap_lut(lm)).to(dev)
    file_mb = (targets.SEMKITTI_LABEL_BYTES + targets.SEMKITTI_INVALID_BYTES) / 2 ** 20
    vol_mb = sk.NVOX * 8 / 2 ** 20
    for kind, aug in AUGS.items():
        for B in (1, 4):
            augs = [aug] * B
            refs = np.stack([st.augment(p, aug["rotate"], aug["flip_dx"], aug["flip_dy"], aug["flip_dz"])
                             for p in pre[:B]])
            label = torch.from_numpy(np.frombuffer(b"".join(f[0] for f in frames[:B]), np.uint8).copy()).to(dev)
            invalid = torch.from_numpy(np.frombuffer(b"".join(f[1] for f in frames[:B]), np.uint8).copy()).to(dev)
            rows = torch.from_numpy(targets.semkitti_augment_rows(augs)).to(dev)
            g, (vol, bad) = graphed(lambda: ops.semkitti_labels_aug(label, invalid, B, rows, lut))
            g.replay()
            torch.cuda.synchronize()
            assert int(bad.sum()) == 0
            assert np.array_equal(vol.cpu().numpy(), refs), "differs from the restatement"
            med, lo, hi = _events(g.replay, args.iters, flush)
            moved = B * (file_mb + vol_mb) * 2 ** 20
            print(f"  {kind}, batch {B}: device {med:.4f} ms per batch (graph replay, median of {args.iters}; "
                  f"{lo:.4f} .. {hi:.4f}), {moved / (med * 1e-3) / 1e9:.0f} GB/s of files read + int64 volume written")
            call = lambda: targets.semantic_kitti_occupancy([f[0] for f in frames[:B]], [f[1] for f in frames[:B]], lm,
                                                            augment=augs)
            for _ in range(3):
                call()
            cmed, clo, chi = _host(call, args.iters, flush)
            print(f"  {kind}, batch {B}: eager call {cmed:.3f} ms per batch ({clo:.3f} .. {chi:.3f}): staging, one "
                  f"host-to-device copy of {B * file_mb:.2f} MB, the kernel and one read-back")
    torch.set_num_threads(1)
    with tempfile.TemporaryDirectory() as tmp:
        npy = os.path.join(tmp, "000000_1_1.npy")
        np.save(npy, pre[0].astype(np.float32))  # what the preprocessing writes
        for kind, aug in AUGS.items():
            run = lambda: reference_host(npy, aug)
            out = run()
            assert np.array_equal(out.numpy(), st.augment(pre[0], aug["rotate"], aug["flip_dx"], aug["flip_dy"],
                                                          aug["flip_dz"]))
            hmed, hlo, hhi = _host(run, args.iters)
            print(f"  reference per sample, {kind}: np.load + voxel_transform + .long() {hmed:.3f} ms on one host "
                  f"core ({hlo:.3f} .. {hhi:.3f})")


if __name__ == "__main__":
    main()
