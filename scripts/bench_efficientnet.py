"""What the SemanticKITTI image encoder costs on the GPU: the library forward against torch's own (cuDNN) forward of the
same modules.

    python scripts/bench_efficientnet.py [--batch 4] [--iters 20] [--warmup 5]

Workload: SemanticKITTI (occformer_kitti.py:66-80), CustomEfficientNet(arch='b7', out_indices=(2, 3, 4, 5, 6)) + SECONDFPN(
[48, 80, 224, 640, 2560], [128] * 5, [0.25, 0.5, 1, 2, 2]) on images (batch, 3, 384, 1280) -> (batch, 640, 24, 80), seeded
synthetic weights (synth.make_efficientnet_state / make_secondfpn_state).  Three arms, alternated in one process, each a
CUDA-graph replay timed with CUDA events after a 128 MiB L2 flush:
  library       CustomEfficientNet / SECONDFPN forward on CUDA tensors (efficientnet.py _forward_cuda: this package's
                sm_90a kernels)
  torch_tf32    their _forward_torch with torch's default torch.backends.cudnn.allow_tf32 = True
  torch_fp32    the same with TF32 disabled (cuDNN and matmul)
Reports the median ms per forward, the algorithmic TF/s (FLOPs of the fp32 problem from the layer shapes, below), the max
relative error max|a-b|/max|b| of each arm's output against the torch forward in fp64 (first image, on the GPU: fp64
convolutions have no TF32 path), the library forward's launch count and the share of its GPU time per kind of launch (one
profiled eager forward), and the card name, power limit and max SM clock read in the same run.  Writes nothing; needs a
GPU.
"""
import argparse
import copy
import json
import os
import statistics
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from occformer_b200 import synth  # noqa: E402
from occformer_b200.efficientnet import CustomEfficientNet  # noqa: E402
from occformer_b200.image_encoder import SECONDFPN  # noqa: E402
from gpu_bench import alternated, capture, card, launch_shares, rel, torch_arms  # noqa: E402

H, W = 384, 1280
OUTS = (2, 3, 4, 5, 6)
FPN = dict(in_channels=[48, 80, 224, 640, 2560], out_channels=[128] * 5, upsample_strides=[0.25, 0.5, 1, 2, 2])


def encoder_flops(net, neck, n, h=H, w=W):
    """2 * MACs of every convolution and SE FC of the backbone + SECONDFPN at (n, 3, h, w), from the modules' shapes
    (Swish, the SE means and the adds are < 1 %)"""
    macs = 0

    def hook(m, i, o):
        nonlocal macs
        macs += o[0].numel() * m.weight[0].numel()
    ref = copy.deepcopy(net).cpu()
    hooks = [m.register_forward_hook(hook) for m in ref.modules() if isinstance(m, nn.Conv2d)]
    with torch.no_grad():
        stages = ref._forward_torch(torch.zeros(1, 3, h, w))
    for hk in hooks:
        hk.remove()
    for t, s, c in zip(stages, neck.upsample_strides, neck.out_channels):
        # a kernel = stride = f conv or transposed conv touches every input value once per output channel
        macs += t.numel() * c
    return 2.0 * macs * n


KINDS = (("stem_im2col", "stem_im2col"), ("depthwise", "dwconv_swish"), ("se_gate", "se_gate"), ("se_scale", "se_scale"),
         ("to_split", "split_rows"), ("fpn_glue", "space_to_depth|depth_to_space|head_prep"), ("gemm", "gemm_bf16x3"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_efficientnet.py needs a CUDA device")
    dev = torch.device("cuda:0")
    n = args.batch
    sd_b = synth.make_efficientnet_state("b7", seed=0, out_indices=OUTS)
    sd_n = synth.make_secondfpn_state(seed=1, out_hw=(6, 20), **FPN)
    backbone, neck = CustomEfficientNet("b7", out_indices=OUTS).eval(), SECONDFPN(**FPN).eval()
    backbone.load_state_dict(sd_b, strict=True)
    neck.load_state_dict(sd_n, strict=True)
    gf = encoder_flops(backbone, neck, n)
    backbone, neck = backbone.to(dev), neck.to(dev)
    x_h = torch.randn(n, 3, H, W, generator=torch.Generator().manual_seed(2))
    x = x_h.to(dev)

    def library():
        return neck(list(backbone(x)))[0]

    graphs, outs = capture({"library": library,
                            **torch_arms(lambda: neck._forward_torch(list(backbone._forward_torch(x)))[0])})
    times = alternated(graphs, args.iters, args.warmup)

    launches, shares = launch_shares(library, KINDS)
    rb, rn = copy.deepcopy(backbone).double(), copy.deepcopy(neck).double()
    with torch.no_grad():
        want = rn._forward_torch(list(rb._forward_torch(x[:1].double())))[0]
    res = {"card": card(), "workload": f"CustomEfficientNet b7 + SECONDFPN SemanticKITTI, images ({n}, 3, {H}, {W}) -> "
                                       f"({n}, 640, {H // 16}, {W // 16})",
           "gflop_per_forward": round(gf / 1e9, 1), "iters": args.iters, "library_launches": launches,
           "library_launch_time": shares}
    for name in graphs:
        ms = statistics.median(times[name])
        row = {"ms_median": round(ms, 4), "ms_min": round(min(times[name]), 4), "tflops": round(gf / (ms * 1e-3) / 1e12, 1),
               "rel_err": float(f"{rel(outs[name][:1], want):.3e}")}
        res[name] = row
        print(f"{name:12s} {ms:8.3f} ms  " + "  ".join(f"{k}={v}" for k, v in row.items()), file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
