"""python tests/detector_trace.py: the nuScenes R50 OccupancyFormer (tests/golden/detector_cfg_nusc_r50.json, synthetic
weights) on one sample of six 256x704 images, without LiDAR points.  Run by tests/test_gpu_detector.py in a process of
its own (its profiler session and graph capture must not change what a later profiler session of the test process
records).  Prints one JSON line:

  counted / kernels / memsets   util.trace of one warm simple_test call
  per_module                    the library's launch count of each stage called by hand in the reference's order
  other, unexpected             GPU work that is not the library's: every name, and those that are not one of
                                SMALL_TORCH_OPS
  other_ms, total_ms            their GPU time and the call's
  graph_equals_eager            simple_test captured with scripts/gpu_bench.graphed replays bit for bit ...
  graph_within_gate             ... or within the 1e-3 gate, label agreement > 0.9999 (the pooled sums' order)
"""
import collections
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [ROOT, HERE]

import torch  # noqa: E402

from util import images, trace  # noqa: E402
from occformer_b200 import DETECTORS, ops, synth  # noqa: E402
from scripts.gpu_bench import graphed  # noqa: E402

# torch's kernels on tensors of a few hundred bytes: the glue's get_mlp_input (stack, cat, repeat copies) and the fills
# of the modules' small zero-initialised buffers
SMALL_TORCH_OPS = ("CatArrayBatchedCopy", "direct_copy_kernel", "FillFunctor")


def kernel_times(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    t = collections.defaultdict(float)
    for e in prof.events():
        if str(e.device_type).endswith("CUDA"):
            t[e.name] += (e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total) / 1e3
    return t


@torch.no_grad()
def main():
    dev = torch.device("cuda:0")
    cfg = json.load(open(os.path.join(HERE, "golden", "detector_cfg_nusc_r50.json")))
    model = DETECTORS.build(cfg).eval()
    cams = synth.workload_cameras("nusc_ref", 1)
    model.load_state_dict(synth.make_detector_state(cfg, seed=60, cams=cams), strict=True)
    model = model.to(dev)
    img_inputs = [images(6, 256, 704, seed=61).view(1, 6, 3, 256, 704)]
    img_inputs += [cams[k] for k in ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")]
    img_inputs = [t.to(dev) for t in img_inputs]
    metas = [dict(occ_size=[256, 256, 32], pc_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0])]

    def fwd():
        return model.simple_test(metas, img_inputs)

    eager = fwd()  # warm-up: weight preparation, module loading, workspaces
    eager = {k: eager[k].clone() for k in ("output_voxels", "output_labels")}
    res = trace(fwd)
    times = kernel_times(fwd)
    res["unexpected"] = sorted(n for n in res["other"] if not any(p in n for p in SMALL_TORCH_OPS))
    res["other_ms"] = round(sum(v for n, v in times.items() if n in res["other"]), 4)
    res["total_ms"] = round(sum(times.values()), 3)

    per = {}

    def count(name, f):
        n0 = ops.LAUNCH_COUNT[0]
        y = f()
        per[name] = ops.LAUNCH_COUNT[0] - n0
        return y

    imgs = img_inputs[0]
    B, N, C, H, W = imgs.shape
    x = count("img_backbone", lambda: model.img_backbone(imgs.view(B * N, C, H, W)))
    x = count("img_neck", lambda: model.img_neck(x))[0]
    x = x.view(B, N, *x.shape[1:])
    mlp = count("get_mlp_input", lambda: model.img_view_transformer.get_mlp_input(*img_inputs[1:7]))
    bev, _ = count("img_view_transformer", lambda: model.img_view_transformer([x] + img_inputs[1:7] + [mlp]))
    enc = count("img_bev_encoder_backbone", lambda: model.img_bev_encoder_backbone(bev))
    feats = count("img_bev_encoder_neck", lambda: model.img_bev_encoder_neck(enc))
    count("pts_bbox_head", lambda: model.pts_bbox_head.simple_test(feats, metas))
    res["per_module"] = per

    graph, out = graphed(fwd)
    graph.replay()
    torch.cuda.synchronize()
    a, b = out["output_voxels"], eager["output_voxels"]
    res["graph_equals_eager"] = bool(torch.equal(a.view(torch.int32), b.view(torch.int32))
                                     and torch.equal(out["output_labels"], eager["output_labels"]))
    d, r = (a - b).double(), b.double()
    rel = float(d.abs().max() / r.abs().max())
    agree = float((out["output_labels"] == eager["output_labels"]).double().mean())
    res["graph_rel_max"], res["graph_label_agreement"] = rel, agree
    res["graph_within_gate"] = rel <= 1e-3 and agree > 0.9999
    print(json.dumps(res))


if __name__ == "__main__":
    main()
