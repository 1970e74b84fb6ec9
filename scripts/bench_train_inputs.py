"""What the training pipelines' camera inputs cost: image_prep.camera_inputs on the GPU (the flipped and rotated images
of occ_prepare_images_aug and CreateDepthFromLiDAR's depth maps of occ_lidar_depth) next to the reference's steps on
the host (Pillow resize + crop + flip + rotate, mmcv's imnormalize by its cv2 calls, CreateDepthFromLiDAR's torch
projection), from decoded frames and a loaded scan.

    python scripts/bench_train_inputs.py [--iters 30]

Per config (nuScenes R50: 4 samples x 6 cameras 900x1600 -> 256x704, 34 720 points each; SemanticKITTI: 4 x 1 x
376x1241 -> 384x1280, 120 000 points each):
  device   camera_inputs captured once into a CUDA graph and replayed between CUDA events, L2 flushed before each,
           median; its images and depth maps are first checked against the numpy restatement
  vpass    the two vertical passes on test-mode geometry (no flip, angle 0): occ_prepare_images and
           occ_prepare_images_aug, each as a graph, alternated
  host     one core, per sample: the reference's steps as the training loader runs them
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
from oracle import image_prep as ip  # noqa: E402
from oracle import train_inputs as ti  # noqa: E402
from gpu_bench import alternated, card, graphed  # noqa: E402

CONFIGS = {"nusc_r50": ("r50", 6, (900, 1600)), "kitti": ("kitti", 1, (376, 1241))}


def inputs(case, N, shape, B, dev):
    """B samples of N cameras: uint8 frames, collated img_inputs and img_metas as the training transforms give them"""
    np.random.seed(0)
    size, norm = ti.CASES[case][5], ti.CASES[case][6]
    frames, metas, cams = [], [], []
    for b in range(B):
        f = [ip.frame(100 * b + c, *shape) for c in range(N)]
        dr = [ti.draws(case, *shape) for _ in range(N)]
        aug = dict(resize_dims=[list(d[1]) for d in dr], crop=[list(d[2]) for d in dr], input_size=list(size),
                   flip=[d[3] for d in dr], rotate=[d[4] for d in dr], **image_prep.norm_config(norm))
        cal = [ti.calib(case, c) for c in range(N)]
        rots = torch.stack([torch.tensor(np.linalg.inv(l2c)[:3, :3]).float() for _, l2c in cal])
        trans = torch.stack([torch.tensor(np.linalg.inv(l2c)[:3, 3]).float() for _, l2c in cal])
        intr = torch.stack([torch.Tensor(K) for K, _ in cal])
        from occformer_b200.pipelines import _ImageFrames
        ph = [_ImageFrames.post_homography(d[0], d[2], d[3], d[4]) for d in dr]
        pts = torch.from_numpy(ti.scan(case, b % ti.CASES[case][1]))
        aug.update(lidar_points=pts.to(dev), lidar_inv_rots=rots.inverse().to(dev))  # staged before the capture
        frames.append(np.stack(f))
        metas.append(dict(img_aug=aug))
        cams.append((rots, trans, intr, torch.stack([p[0] for p in ph]), torch.stack([p[1] for p in ph])))
    coll = [torch.from_numpy(np.stack(frames)).to(dev)] + [torch.stack([c[k] for c in cams]).to(dev)
                                                           for k in range(5)]
    coll += [torch.zeros(B, N, 1, device=dev), torch.zeros(B, N, 4, 4, device=dev)]
    return frames, tuple(coll), metas


def host_reference(frame, aug, c, norm, pts, cam):
    """the reference's per-camera image steps and its depth projection for one camera, on the host"""
    import cv2
    from PIL import Image
    img = Image.fromarray(frame).resize(tuple(aug["resize_dims"][c])).crop(tuple(aug["crop"][c]))
    if aug["flip"][c]:
        img = img.transpose(method=Image.FLIP_LEFT_RIGHT)
    img = np.array(img.rotate(aug["rotate"][c])).astype(np.float32)
    mean = np.float64(np.array(norm["mean"], np.float32).reshape(1, -1))
    stdinv = 1 / np.float64(np.array(norm["std"], np.float32).reshape(1, -1))
    if norm["to_rgb"]:
        cv2.cvtColor(img, cv2.COLOR_BGR2RGB, img)
    cv2.subtract(img, mean, img)
    cv2.multiply(img, stdinv, img)
    torch.tensor(img).float().permute(2, 0, 1).contiguous()
    rots, trans, intr, post_rot, post_tran = cam
    p = (pts.view(-1, 1, 3) - trans.view(1, -1, 3))
    p = rots.inverse().unsqueeze(0) @ p.unsqueeze(-1)
    if intr.shape[-1] == 4:
        p = torch.cat((p, torch.ones((p.shape[0], 1, 1, 1))), dim=2)
    p = (intr.unsqueeze(0) @ p).squeeze(-1)
    d = p[..., 2:3]
    uv = (post_rot[:, :2, :2].unsqueeze(0) @ (p[..., :2] / d).unsqueeze(-1)).squeeze(-1) + post_tran[..., :2]
    fH, fW = aug["input_size"]
    ok = (uv[..., 0] >= 0) & (uv[..., 1] >= 0) & (uv[..., 0] <= fW - 1) & (uv[..., 1] <= fH - 1) & (d[..., 0] > 0)
    for i in range(uv.shape[1]):
        v = torch.cat([uv[:, i], d[:, i]], 1)[ok[:, i]]
        v = v[torch.argsort(v[:, 2], descending=True)]
        m = torch.zeros(fH, fW)
        m[v[:, 1].round().long(), v[:, 0].round().long()] = v[:, 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_inputs: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.set_num_threads(1)
    import cv2
    cv2.setNumThreads(1)
    print(f"card: {card()}")
    print(f"host: {os.cpu_count()} cores, timed on one thread")
    B = 4
    for name, (case, N, shape) in CONFIGS.items():
        frames, img_inputs, metas = inputs(case, N, shape, B, dev)
        norm = ti.CASES[case][6]
        g, out = graphed(lambda: image_prep.camera_inputs(img_inputs, metas))
        g.replay()
        torch.cuda.synchronize()
        for b in range(B):
            a = metas[b]["img_aug"]
            for c in range(N):
                ref = ti.augment(frames[b][c], a["resize_dims"][c], a["crop"][c], a["flip"][c], a["rotate"][c], norm)
                assert torch.equal(out[0][b, c].cpu().view(torch.int32), torch.from_numpy(ref).view(torch.int32))
                dref = ti.depth_map(a["lidar_points"].cpu().numpy(), a["lidar_inv_rots"][c].cpu().numpy(),
                                    *(img_inputs[k][b, c].cpu().numpy() for k in (2, 3, 4, 5)), *a["input_size"])
                assert torch.equal(out[6][b, c].cpu().view(torch.int32), torch.from_numpy(dref).view(torch.int32))
        t = alternated({"camera_inputs": g}, args.iters, 3)["camera_inputs"]
        t.sort()
        print(f"  {name} batch {B}: camera_inputs device {t[len(t) // 2]:.4f} ms (graph replay, median of "
              f"{args.iters}; {t[0]:.4f} .. {t[-1]:.4f}); images and depth maps equal the restatement")
        x = img_inputs[0]
        test = [{k: v for k, v in m["img_aug"].items() if k not in ("flip", "rotate", "lidar_points",
                                                                     "lidar_inv_rots")} for m in metas]
        flat = [dict(a, flip=[False] * N, rotate=[0.0] * N) for a in test]
        g_old, o_old = graphed(lambda: image_prep.prepare_images(x, test))
        g_new, o_new = graphed(lambda: image_prep.prepare_images(x, flat))
        g_old.replay()
        g_new.replay()
        torch.cuda.synchronize()
        assert torch.equal(o_old.view(torch.int32), o_new.view(torch.int32))
        tt = alternated({"occ_prepare_images": g_old, "occ_prepare_images_aug": g_new}, args.iters, 3)
        print("    test-mode geometry, both passes: " + ", ".join(
            f"{k} {sorted(v)[len(v) // 2]:.4f} ms" for k, v in tt.items()) + f" (median of {args.iters}, alternated)")
        ts = []
        for _ in range(2):
            t0 = time.perf_counter()
            a = metas[0]["img_aug"]
            for c in range(N):
                cam = tuple(img_inputs[k][0, c:c + 1].cpu() for k in range(1, 6))
                host_reference(frames[0][c], a, c, norm, a["lidar_points"].cpu(), cam)
            ts.append((time.perf_counter() - t0) * 1e3)
        print(f"  {name} host per sample, one thread: reference images + depth maps {min(ts):.1f} ms")


if __name__ == "__main__":
    main()
