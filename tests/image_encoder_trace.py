"""One warm CUDA image-encoder forward (ResNet-50 + SECONDFPN of the nuScenes R50 config on (6, 3, 256, 704) images) under
torch.profiler, then the same forward captured into a CUDA graph and replayed.  Run as a script by
tests/test_gpu_image_encoder.py, in a process of its own (see tests/depthnet_trace.py).  Prints one JSON line: the
library's launch count over the traced forward, the occ:: kernels and memsets of the trace, any other GPU work, and
whether the replay equals eager bit for bit."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from occformer_b200 import ops, synth  # noqa: E402
from occformer_b200.image_encoder import SECONDFPN, ResNet  # noqa: E402

FPN = dict(in_channels=[256, 512, 1024, 2048], out_channels=[128, 128, 128, 128], upsample_strides=[0.25, 0.5, 1, 2])


@torch.no_grad()
def main():
    dev = torch.device("cuda:0")
    backbone = ResNet(50).eval()
    backbone.load_state_dict(synth.make_resnet_state(seed=30), strict=True)
    neck = SECONDFPN(**FPN).eval()
    neck.load_state_dict(synth.make_secondfpn_state(seed=31, **FPN), strict=True)
    backbone, neck = backbone.to(dev), neck.to(dev)
    x = torch.randn(6, 3, 256, 704, generator=torch.Generator().manual_seed(32)).to(dev)

    def fwd():
        return neck(list(backbone(x)))[0]

    eager = fwd()  # warm-up: weight preparation, module loading, conv workspace
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        n0 = ops.LAUNCH_COUNT[0]
        fwd()
        torch.cuda.synchronize()
        counted = ops.LAUNCH_COUNT[0] - n0
    gpu = [e.name for e in prof.events() if str(e.device_type).endswith("CUDA")]
    res = dict(counted=counted, kernels=sum("occ::" in e for e in gpu), memsets=sum(e.startswith("Memset") for e in gpu),
               other=sorted({e for e in gpu if "occ::" not in e and not e.startswith("Memset")}))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fwd()  # the side stream's own warm-up (workspaces are per stream)
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
