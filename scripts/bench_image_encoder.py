"""What the image encoder costs on the GPU: the library forward against torch's own (cuDNN) forward of the same modules.

    python scripts/bench_image_encoder.py [--backbone r50|r101] [--batch 4] [--iters 20] [--warmup 5]

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

--backbone r101: nuScenes R101 (occformer_nusc_r101_896x1600.py:67-84), ResNetDCN(101, style 'caffe', DCNv2 in layer3 /
layer4) + the same SECONDFPN on images (batch * 6, 3, 896, 1600) -> (batch * 6, 512, 56, 100), weights from
synth.make_resnet_dcn_state.  A fourth arm, torch_fp16, runs the torch forward under fp16 autocast (the reference runner
wraps this config with wrap_fp16_model).  The torch arms' DCNv2 is the module's own torch restatement (grid_sample
columns times the mask, then an einsum), not mmcv's CUDA op, so their times say what that restatement costs, not what
mmcv costs.  The error reference is the fp64 torch forward on the GPU (first image); the launch-time shares also split
out the modulated deformable im2col and the GEMMs of its columns (the GEMM launch right after each im2col).
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from occformer_b200 import ops, synth  # noqa: E402
from occformer_b200.image_encoder import SECONDFPN, ResNet, ResNetDCN  # noqa: E402
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


R101 = dict(style="caffe", dcn=dict(type="DCNv2", deform_groups=1, fallback_on_stride=False),
            stage_with_dcn=(False, False, True, True))
H101, W101 = 896, 1600


def r101_flops(n, h=H101, w=W101):
    """2 * MACs of every convolution of R101-DCN + SECONDFPN at (n, 3, h, w): caffe-style blocks (stride on conv1), each
    DCNv2 as its conv_offset (3x3, 27 outputs) plus the 3x3 contraction of its columns; the bilinear sampling, the
    max-pool and the adds are left out (< 0.5 %)"""
    macs = 147 * 64 * (h // 2) * (w // 2)
    h, w = h // 4, w // 4
    cin = 64
    for stage, (blocks, planes) in enumerate(zip((3, 4, 23, 3), (64, 128, 256, 512))):
        for b in range(blocks):
            s = 2 if stage > 0 and b == 0 else 1
            ho, wo = h // s, w // s
            macs += cin * planes * ho * wo + 9 * planes * planes * ho * wo + planes * 4 * planes * ho * wo
            if stage >= 2:
                macs += 9 * planes * 27 * ho * wo  # conv_offset
            if b == 0:
                macs += cin * 4 * planes * ho * wo  # downsample
            cin, h, w = 4 * planes, ho, wo
    fh, fw = H101 // 16, W101 // 16
    macs += 16 * 256 * 128 * fh * fw + 4 * 512 * 128 * fh * fw + 1024 * 128 * fh * fw
    macs += 2048 * 4 * 128 * (fh // 2) * (fw // 2)
    return 2.0 * macs * n


def dcn_shares(fn):
    """GPU time of one eager call of fn split into the modulated deformable im2col, the GEMM launched right after each
    (the contraction of its columns) and everything else, in ms (torch.profiler, device events in start order)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if str(e.device_type).endswith("CUDA")), key=lambda e: e.time_range.start)
    t = {"modulated_deform_im2col": 0.0, "dcn_column_gemm": 0.0, "other": 0.0}
    prev = ""
    for e in ev:
        ms = (e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total) / 1e3
        kind = "modulated_deform_im2col" if "deform_im2col" in e.name else \
            "dcn_column_gemm" if "gemm_bf16x3" in e.name and "deform_im2col" in prev else "other"
        t[kind] += ms
        prev = e.name
    total = sum(t.values())
    return {k: {"ms": round(v, 3), "share": round(v / total, 4)} for k, v in t.items()}


KINDS = (("stem_im2col", "stem_im2col"), ("dcn_im2col", "deform_im2col"), ("maxpool", "maxpool3x3s2"), ("to_split", "split_rows"),
         ("fpn_glue", "space_to_depth|depth_to_space|head_prep"), ("gemm_conv", "gemm_bf16x3"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backbone", choices=("r50", "r101"), default="r50")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_image_encoder.py needs a CUDA device")
    dev = torch.device("cuda:0")
    if args.backbone == "r101":
        return main_r101(args, dev)
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


def main_r101(args, dev):
    n = args.batch * N
    sd_b, sd_n = synth.make_resnet_dcn_state(0, **R101), synth.make_secondfpn_state(seed=1, **FPN)
    backbone, neck = ResNetDCN(101, **R101).eval(), SECONDFPN(**FPN).eval()
    backbone.load_state_dict(sd_b, strict=True)
    neck.load_state_dict(sd_n, strict=True)
    backbone, neck = backbone.to(dev), neck.to(dev)
    x = torch.randn(n, 3, H101, W101, generator=torch.Generator().manual_seed(2)).to(dev)

    def library():
        return neck(list(backbone(x)))[0]

    def torch_fwd():
        return neck._forward_torch(list(backbone._forward_torch(x)))[0]

    def torch_fp16():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            return torch_fwd()

    graphs, outs = capture({"library": library, **torch_arms(torch_fwd), "torch_fp16": torch_fp16})
    times = alternated(graphs, args.iters, args.warmup)
    launches, shares = launch_shares(library, KINDS)
    dcn = dcn_shares(library)
    with torch.no_grad():
        want = neck.double()._forward_torch(list(backbone.double()._forward_torch(x[:1].double())))[0]
    gf = r101_flops(n)
    rows = n * (H101 // 16) * (W101 // 16)
    res = {"card": card(), "workload": f"ResNet-101-DCN (caffe, DCNv2 in layer3/4) + SECONDFPN nuScenes R101, images "
                                       f"({n}, 3, {H101}, {W101}) -> ({n}, 512, {H101 // 16}, {W101 // 16})",
           "gflop_per_forward": round(gf / 1e9, 1), "iters": args.iters, "library_launches": launches,
           "layer3_columns_gb_per_call": round(rows * 9 * 256 * 4 / 1e9, 2), "library_launch_time": shares,
           "dcn_launch_time": dcn, "torch_dcn": "grid_sample restatement (image_encoder.ModulatedDeformConv2dPack), "
                                               "not mmcv's CUDA op"}
    for name in graphs:
        ms = statistics.median(times[name])
        row = {"ms_median": round(ms, 4), "ms_min": round(min(times[name]), 4), "tflops": round(gf / (ms * 1e-3) / 1e12, 1),
               "rel_err": float(f"{rel(outs[name][:1], want):.3e}")}
        res[name] = row
        print(f"{name:12s} {ms:8.3f} ms  " + "  ".join(f"{k}={v}" for k, v in row.items()), file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
