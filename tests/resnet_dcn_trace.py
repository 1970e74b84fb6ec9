"""python tests/resnet_dcn_trace.py: ResNetDCN(101) + SECONDFPN of the nuScenes R101 config on (6, 3, 896, 1600) images,
one warm CUDA forward under util.trace, then the same forward captured into a CUDA graph and replayed.  Run by
tests/test_gpu_resnet_dcn.py in a process of its own (as tests/forward_trace.py is for the other encoders).  Prints one
JSON line: util.trace's counts and whether the replay equals eager bit for bit."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]

import torch  # noqa: E402

from util import images, trace  # noqa: E402
from occformer_b200 import synth  # noqa: E402
from occformer_b200.image_encoder import SECONDFPN, ResNetDCN  # noqa: E402

R101 = dict(style="caffe", dcn=dict(type="DCNv2", deform_groups=1, fallback_on_stride=False),
            stage_with_dcn=(False, False, True, True))
FPN = dict(in_channels=[256, 512, 1024, 2048], out_channels=[128] * 4, upsample_strides=[0.25, 0.5, 1, 2])


@torch.no_grad()
def main():
    dev = torch.device("cuda:0")
    backbone = ResNetDCN(101, **R101).eval()
    backbone.load_state_dict(synth.make_resnet_dcn_state(seed=33, **R101), strict=True)
    neck = SECONDFPN(**FPN).eval()
    neck.load_state_dict(synth.make_secondfpn_state(seed=34, **FPN), strict=True)
    backbone, neck = backbone.to(dev), neck.to(dev)
    x = images(6, 896, 1600, seed=35).to(dev)

    def fwd():
        return neck(list(backbone(x)))[0]

    eager = fwd()  # warm-up: weight preparation, module loading, workspaces
    res = trace(fwd)
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
