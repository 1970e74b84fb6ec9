"""What DepthNet costs on the GPU: the library forward against torch's own (cuDNN) forward of the same module.

    python scripts/bench_depthnet.py [--batch 4] [--iters 30] [--warmup 5]

Workload: nuScenes R50 (occformer_nusc_r50_256x704.py), DepthNet(512, 512, 128, 112, cam_channels=27) on x
(batch * 6, 512, 16, 44) and mlp_input (batch, 6, 27), seeded synthetic weights (synth.make_depthnet_state).  Three arms,
alternated in one process, each a CUDA-graph replay timed with CUDA events after a 128 MiB L2 flush:
  library       DepthNet.forward on CUDA tensors (depthnet.py _forward_cuda: this package's sm_90a kernels)
  torch_tf32    DepthNet._forward_torch with torch's default torch.backends.cudnn.allow_tf32 = True
  torch_fp32    the same with TF32 disabled (cuDNN and matmul)
Reports the median ms per forward, the algorithmic TF/s (FLOPs of the fp32 problem from the layer shapes, below), the
max relative error max|a-b|/max|b| of each arm's depth logits and context against depthnet.py's forward in fp64 on the
host (first sample), the whole view-transformer forward (library DepthNet + fused lift-splat) and the card name, power
limit and max SM clock read in the same run.  Writes nothing; needs a GPU (no CPU fallback).
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from occformer_b200 import synth  # noqa: E402
from occformer_b200.depthnet import DepthNet  # noqa: E402
from occformer_b200.view_transformer import ViewTransformerLiftSplatShootVoxel  # noqa: E402
from gpu_bench import alternated, capture, card, rel, torch_arms  # noqa: E402

CIN, MID, CTX, D, CAM, N, FH, FW = 512, 512, 128, 112, 27, 6, 16, 44


def depthnet_flops(n, H, W, cin=CIN, mid=MID, ctx=CTX, d=D):
    """2 * MACs of every convolution / contraction of DepthNet (the SE gates and the pooling branch are < 0.01 %)."""
    macs = (9 * cin * mid              # reduce_conv 3x3
            + mid * ctx                # context_conv 1x1
            + 6 * 9 * mid * mid        # three BasicBlocks, two 3x3 convs each
            + mid * mid + 3 * 9 * mid * mid  # ASPP: 1x1 + three dilated 3x3 branches
            + 5 * mid * mid            # ASPP.conv1 (5C -> C)
            + 9 * mid * 18             # DCN conv_offset 3x3
            + 9 * mid * mid // 4       # DCN, 4 groups
            + mid * d)                 # depth head 1x1
    return 2.0 * macs * n * H * W


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_depthnet.py needs a CUDA device")
    dev = torch.device("cuda:0")
    B, n = args.batch, args.batch * N
    sd = synth.make_depthnet_state(CIN, MID, CTX, D, CAM, seed=0)
    net = DepthNet(CIN, MID, CTX, D, cam_channels=CAM).eval()
    net.load_state_dict(sd, strict=True)
    net = net.to(dev)
    g = torch.Generator().manual_seed(1)
    x_h = torch.randn(n, CIN, FH, FW, generator=g)
    mlp_h = torch.randn(B, N, CAM, generator=g)
    x, mlp = x_h.to(dev), mlp_h.to(dev)

    # view transformer (library DepthNet + fused lift-splat) at the reference grid 128 x 128 x 16
    vt = ViewTransformerLiftSplatShootVoxel(grid_config=synth.grid_config("nusc_ref"), data_config={"input_size": (256, 704)},
                                            numC_input=CIN, numC_Trans=CTX, cam_channels=CAM)
    vt.depth_net.load_state_dict(sd, strict=True)
    vt = vt.to(dev).eval()
    cams = {k: v.to(dev) for k, v in synth.nusc_cameras(B, N, (256, 704)).items()}
    vt_in = [x.view(B, N, CIN, FH, FW)] + [cams[k] for k in ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")]
    vt_in.append(mlp)

    graphs, outs = capture({"library": lambda: net(x, mlp), **torch_arms(lambda: net._forward_torch(x, mlp)),
                            "view_transformer": lambda: vt(vt_in)[0]})
    times = alternated(graphs, args.iters, args.warmup)

    ref = DepthNet(CIN, MID, CTX, D, cam_channels=CAM).eval()
    ref.load_state_dict(sd, strict=True)
    with torch.no_grad():
        want = ref.double()(x_h[:N].double(), mlp_h[:1].double())
    gf = depthnet_flops(n, FH, FW)
    res = {"card": card(), "workload": f"DepthNet nuScenes R50, x ({n}, {CIN}, {FH}, {FW}), mlp_input ({B}, {N}, {CAM})",
           "gflop_per_forward": round(gf / 1e9, 1), "iters": args.iters}
    for name in graphs:
        ms = statistics.median(times[name])
        row = {"ms_median": round(ms, 4), "ms_min": round(min(times[name]), 4)}
        if name != "view_transformer":
            row["tflops"] = round(gf / (ms * 1e-3) / 1e12, 1)
            y = outs[name][:N]
            row["rel_err_depth"] = float(f"{rel(y[:, :D], want[:, :D]):.3e}")
            row["rel_err_context"] = float(f"{rel(y[:, D:], want[:, D:]):.3e}")
        res[name] = row
        print(f"{name:17s} {ms:8.3f} ms  " + "  ".join(f"{k}={v}" for k, v in row.items()), file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
