"""python tests/forward_trace.py depthnet|r50|r101|b7: one warm CUDA forward under util.trace, then the same forward
captured with scripts/gpu_bench.graphed and replayed.  depthnet: DepthNet at nuScenes R50 shapes; r50: ResNet-50 +
SECONDFPN of the nuScenes R50 config on (6, 3, 256, 704) images; r101: ResNetDCN(101) + SECONDFPN of the nuScenes R101
config on (6, 3, 896, 1600) images; b7: CustomEfficientNet b7 + SECONDFPN of the KITTI config on (2, 3, 384, 1280)
images.  Run by util.run_trace in a process of its own.  Prints one JSON line: util.trace's counts, whether the replay
equals eager bit for bit and, for b7, the launch count expected from the module's structure."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]

import torch  # noqa: E402

from util import images, trace  # noqa: E402
from occformer_b200 import synth  # noqa: E402
from occformer_b200.depthnet import DepthNet  # noqa: E402
from occformer_b200.efficientnet import CustomEfficientNet  # noqa: E402
from occformer_b200.image_encoder import SECONDFPN, ResNet, ResNetDCN  # noqa: E402
from scripts.gpu_bench import graphed  # noqa: E402

# the SECONDFPN of the nuScenes R50 and R101 configs
FPN = dict(in_channels=[256, 512, 1024, 2048], out_channels=[128] * 4, upsample_strides=[0.25, 0.5, 1, 2])


def _load(net, state, dev):
    net.eval().load_state_dict(state, strict=True)
    return net.to(dev)


def depthnet(dev):
    cin, mid, ctx, D, cam, n = 512, 512, 128, 112, 27, 6
    net = _load(DepthNet(cin, mid, ctx, D, cam_channels=cam), synth.make_depthnet_state(cin, mid, ctx, D, cam, seed=16),
                dev)
    g = torch.Generator().manual_seed(17)
    x, mlp = torch.randn(n, cin, 16, 44, generator=g).to(dev), torch.randn(1, n, cam, generator=g).to(dev)
    return lambda: net(x, mlp), {}


def r50(dev):
    backbone = _load(ResNet(50), synth.make_resnet_state(seed=30), dev)
    neck = _load(SECONDFPN(**FPN), synth.make_secondfpn_state(seed=31, **FPN), dev)
    x = images(6, 256, 704, seed=32).to(dev)
    return lambda: neck(list(backbone(x)))[0], {}


def r101(dev):
    dcn = dict(style="caffe", dcn=dict(type="DCNv2", deform_groups=1, fallback_on_stride=False),
               stage_with_dcn=(False, False, True, True))
    backbone = _load(ResNetDCN(101, **dcn), synth.make_resnet_dcn_state(seed=33, **dcn), dev)
    neck = _load(SECONDFPN(**FPN), synth.make_secondfpn_state(seed=34, **FPN), dev)
    x = images(6, 896, 1600, seed=35).to(dev)
    return lambda: neck(list(backbone(x)))[0], {}


def expected_launches(net, neck):
    """stem im2col + GEMM; per block [expand GEMM] + depthwise + SE gate + SE scale + linear GEMM [+ split_rows when the
    next op is a GEMM or the block ends an output stage]; layers.6 GEMM + split; SECONDFPN: per level space_to_depth +
    conv (stride < 1), conv (stride 1) or GEMM + depth_to_space (stride > 1)"""
    blocks = [b for layer in net.layers[1:6] for b in layer]
    n = 2
    for i, b in enumerate(blocks):
        nxt_gemm = blocks[i + 1].with_expand_conv if i + 1 < len(blocks) else True  # layers.6 follows the last block
        n += int(b.with_expand_conv) + 4 + int(nxt_gemm)
    n += 2
    return n + sum(2 if s != 1 else 1 for s in neck.upsample_strides)


def b7(dev):
    outs = (2, 3, 4, 5, 6)
    fpn = dict(in_channels=[48, 80, 224, 640, 2560], out_channels=[128] * 5, upsample_strides=[0.25, 0.5, 1, 2, 2])
    net = _load(CustomEfficientNet("b7", out_indices=outs), synth.make_efficientnet_state("b7", seed=40, out_indices=outs),
                dev)
    neck = _load(SECONDFPN(**fpn), synth.make_secondfpn_state(seed=41, out_hw=(6, 20), **fpn), dev)
    x = images(2, 384, 1280, seed=42).to(dev)
    return lambda: neck(list(net(x)))[0], {"expected": expected_launches(net, neck)}


@torch.no_grad()
def main(case):
    fwd, extra = {"depthnet": depthnet, "r50": r50, "r101": r101, "b7": b7}[case](torch.device("cuda:0"))
    eager = fwd()  # warm-up: weight preparation, module loading, workspaces
    res = dict(trace(fwd), **extra)
    graph, y = graphed(fwd)
    graph.replay()
    torch.cuda.synchronize()
    res["graph_equals_eager"] = bool(torch.equal(y.view(torch.int32), eager.view(torch.int32)))
    print(json.dumps(res))


if __name__ == "__main__":
    main(sys.argv[1])
