"""What the image encoder costs on the GPU: the library forward against torch's own (cuDNN) forward of the same modules.

    python scripts/bench_image_encoder.py [--batch 4] [--iters 20] [--warmup 5]

Workload: nuScenes R50 (occformer_nusc_r50_256x704.py:65-79), ResNet(depth=50) + SECONDFPN([256, 512, 1024, 2048], [128]
* 4, [0.25, 0.5, 1, 2]) on images (batch * 6, 3, 256, 704) -> (batch * 6, 512, 16, 44), seeded synthetic weights
(synth.make_resnet_state / make_secondfpn_state).  Three arms, alternated in one process, each a CUDA-graph replay timed
with CUDA events after a 128 MiB L2 flush:
  library       ResNet / SECONDFPN forward on CUDA tensors (image_encoder.py _forward_cuda: this package's sm_90a kernels)
  torch_tf32    their _forward_torch with torch's default torch.backends.cudnn.allow_tf32 = True
  torch_fp32    the same with TF32 disabled (cuDNN and matmul)
Reports the median ms per forward, the algorithmic TF/s (FLOPs of the fp32 problem from the layer shapes, below), the max
relative error max|a-b|/max|b| of each arm's output against the torch forward in fp64 on the host (first image), the
library forward's launch count and the share of its GPU time per kind of launch (one profiled eager forward), the stem
columns' size, and the card name, power limit and max SM clock read in the same run.  Writes nothing; needs a GPU.
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from occformer_b200 import ops, synth  # noqa: E402
from occformer_b200.image_encoder import SECONDFPN, ResNet  # noqa: E402
from gpu_bench import alternated, capture, card, launch_shares, rel, torch_arms  # noqa: E402

N, H, W = 6, 256, 704
FPN = dict(in_channels=[256, 512, 1024, 2048], out_channels=[128, 128, 128, 128], upsample_strides=[0.25, 0.5, 1, 2])


def encoder_flops(n, h=H, w=W):
    """2 * MACs of every convolution of ResNet-50 + SECONDFPN at (n, 3, h, w) (the max-pool and the adds are < 0.1 %)"""
    macs = 0
    h, w = h // 2, w // 2
    macs += 147 * 64 * h * w  # stem 7x7x3 -> 64
    h, w = h // 2, w // 2     # max-pool
    cin = 64
    for stage, (blocks, planes) in enumerate(zip((3, 4, 6, 3), (64, 128, 256, 512))):
        for b in range(blocks):
            s = 2 if stage > 0 and b == 0 else 1
            ho, wo = h // s, w // s
            macs += cin * planes * h * w + 9 * planes * planes * ho * wo + planes * 4 * planes * ho * wo
            if b == 0:
                macs += cin * 4 * planes * ho * wo  # downsample
            cin, h, w = 4 * planes, ho, wo
    fh, fw = H // 16, W // 16
    macs += 16 * 256 * 128 * fh * fw + 4 * 512 * 128 * fh * fw + 1024 * 128 * fh * fw  # stride-4 / stride-2 convs, 1x1 deconv
    macs += 2048 * 4 * 128 * (fh // 2) * (fw // 2)  # 2x2 stride-2 deconv
    return 2.0 * macs * n


KINDS = (("stem_im2col", "stem_im2col"), ("maxpool", "maxpool3x3s2"), ("to_split", "split_rows"),
         ("fpn_glue", "space_to_depth|depth_to_space|head_prep"), ("gemm_conv", "gemm_bf16x3"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_image_encoder.py needs a CUDA device")
    dev = torch.device("cuda:0")
    n = args.batch * N
    sd_b, sd_n = synth.make_resnet_state(0), synth.make_secondfpn_state(seed=1, **FPN)
    backbone, neck = ResNet(50).eval(), SECONDFPN(**FPN).eval()
    backbone.load_state_dict(sd_b, strict=True)
    neck.load_state_dict(sd_n, strict=True)
    backbone, neck = backbone.to(dev), neck.to(dev)
    x_h = torch.randn(n, 3, H, W, generator=torch.Generator().manual_seed(2))
    x = x_h.to(dev)

    def library():
        return neck(list(backbone(x)))[0]

    graphs, outs = capture({"library": library,
                            **torch_arms(lambda: neck._forward_torch(list(backbone._forward_torch(x)))[0])})
    times = alternated(graphs, args.iters, args.warmup)

    launches, shares = launch_shares(library, KINDS)
    rb, rn = ResNet(50).eval(), SECONDFPN(**FPN).eval()
    rb.load_state_dict(sd_b, strict=True)
    rn.load_state_dict(sd_n, strict=True)
    with torch.no_grad():
        want = rn.double()(list(rb.double()(x_h[:1].double())))[0]
    gf = encoder_flops(n)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    res = {"card": card(), "workload": f"ResNet-50 + SECONDFPN nuScenes R50, images ({n}, 3, {H}, {W}) -> ({n}, 512, "
                                       f"{H // 16}, {W // 16})",
           "gflop_per_forward": round(gf / 1e9, 1), "iters": args.iters, "library_launches": launches,
           "stem_columns_mb": round(n * Ho * Wo * ops.STEM_COLS * 4 / 1e6, 1), "library_launch_time": shares}
    for name in graphs:
        ms = statistics.median(times[name])
        row = {"ms_median": round(ms, 4), "ms_min": round(min(times[name]), 4), "tflops": round(gf / (ms * 1e-3) / 1e12, 1),
               "rel_err": float(f"{rel(outs[name][:1], want):.3e}")}
        res[name] = row
        print(f"{name:12s} {ms:8.3f} ms  " + "  ".join(f"{k}={v}" for k, v in row.items()), file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
