"""One warm CUDA forward of the SemanticKITTI image encoder (CustomEfficientNet b7 + SECONDFPN of the KITTI config on
(2, 3, 384, 1280) images) under torch.profiler, then the same forward captured into a CUDA graph and replayed.  Run as a
script by tests/test_gpu_efficientnet.py, in a process of its own (see tests/depthnet_trace.py).  Prints one JSON line:
the library's launch count over the traced forward, the occ:: kernels and memsets of the trace, any other GPU work,
whether the replay equals eager bit for bit, and the launch count expected from the module's structure."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from occformer_b200 import ops, synth  # noqa: E402
from occformer_b200.efficientnet import CustomEfficientNet  # noqa: E402
from occformer_b200.image_encoder import SECONDFPN  # noqa: E402

FPN = dict(in_channels=[48, 80, 224, 640, 2560], out_channels=[128] * 5, upsample_strides=[0.25, 0.5, 1, 2, 2])


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


@torch.no_grad()
def main():
    dev = torch.device("cuda:0")
    net = CustomEfficientNet("b7", out_indices=(2, 3, 4, 5, 6)).eval()
    net.load_state_dict(synth.make_efficientnet_state("b7", seed=40, out_indices=(2, 3, 4, 5, 6)), strict=True)
    neck = SECONDFPN(**FPN).eval()
    neck.load_state_dict(synth.make_secondfpn_state(seed=41, out_hw=(6, 20), **FPN), strict=True)
    net, neck = net.to(dev), neck.to(dev)
    x = torch.randn(2, 3, 384, 1280, generator=torch.Generator().manual_seed(42)).to(dev)

    def fwd():
        return neck(list(net(x)))[0]

    eager = fwd()  # warm-up: weight preparation, module loading
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        n0 = ops.LAUNCH_COUNT[0]
        fwd()
        torch.cuda.synchronize()
        counted = ops.LAUNCH_COUNT[0] - n0
    gpu = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA")]
    res = dict(counted=counted, kernels=sum("occ::" in e for e in gpu), memsets=sum(e.startswith("Memset") for e in gpu),
               other=sorted({e for e in gpu if "occ::" not in e and not e.startswith("Memset")}),
               expected=expected_launches(net, neck))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fwd()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = fwd()
    graph.replay()
    torch.cuda.synchronize()
    res["graph_equals_eager"] = bool(torch.equal(y.view(torch.int32), eager.view(torch.int32)))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
