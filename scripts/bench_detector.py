"""What the whole model costs on the GPU: OccupancyFormer from normalised camera images to simple_test's outputs.

    python scripts/bench_detector.py [--config nusc_r50|nusc_r101|nusc_panoptic|kitti] [--batch 4] [--iters 20] [--warmup 5]

The detector is built from the unmodified config's ``model`` dict (tests/golden/detector_cfg_<config>.json) with seeded
synthetic weights (synth.make_detector_state) and run on seeded N(0, 1) images of the config's size (nuScenes: batch x 6
x 256x704, R101: batch x 6 x 896x1600, KITTI: batch x 1 x 384x1280) with the synthetic cameras of occformer_b200.synth,
without LiDAR points (the lidarseg tail's host synchronisation is evaluation, not inference).  simple_test is captured in
one CUDA graph (scripts/gpu_bench.graphed) and replayed after a 128 MiB L2 flush, timed with CUDA events.

Prints one JSON line: the median ms per forward and samples/s; gpu_launches, the library's launch count of one eager
call; the GPU time of each stage (image encoder = backbone + neck, view transformer including DepthNet, occupancy
encoder, pixel decoder, head), each stage called by hand and profiled on its own; the relative error max|a-b|/max|b| of
the replayed output_voxels against a seeded eager call; and the card name, power limit and max SM clock read in the same
run.  Writes nothing; needs a GPU.
"""
import argparse
import collections
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from occformer_b200 import DETECTORS, ops, synth  # noqa: E402
from gpu_bench import alternated, card, graphed, rel  # noqa: E402

WL = {"nusc_r50": "nusc_ref", "nusc_r101": "nusc_ref", "nusc_panoptic": "nusc_ref", "kitti": "kitti"}


def cameras(config, vt, B):
    if config == "kitti":
        return synth.kitti_camera(B, tuple(vt.data_config["input_size"]))
    return synth.nusc_cameras(B, 6, tuple(vt.data_config["input_size"]))


def gpu_ms(fn):
    """GPU time of the kernels of one call of fn, in ms (torch.profiler)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    ms = sum((e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total) / 1e3
             for e in prof.events() if str(e.device_type).endswith("CUDA"))
    return out, ms


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=tuple(WL), default="nusc_r50")
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    B = a.batch
    cfg = json.load(open(os.path.join(ROOT, "tests", "golden", f"detector_cfg_{a.config}.json")))
    model = DETECTORS.build(cfg).eval()
    vt = model.img_view_transformer
    model.load_state_dict(synth.make_detector_state(cfg, seed=0, cams=cameras(a.config, vt, 1)), strict=True)
    model = model.to(dev)
    cams = cameras(a.config, vt, B)
    N = cams["rots"].shape[1]
    H, W = vt.data_config["input_size"]
    g = torch.Generator().manual_seed(1)
    img_inputs = [torch.randn(B, N, 3, H, W, generator=g)]
    img_inputs += [cams[k] for k in ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")]
    img_inputs = [t.to(dev) for t in img_inputs]
    wl = synth.WORKLOADS[WL[a.config]]
    metas = [dict(occ_size=list(wl["occ"]), pc_range=list(wl["pc"])) for _ in range(B)]

    def fwd():
        return model.simple_test(metas, img_inputs)

    def voxels(out):
        v = out["output_voxels"]
        if isinstance(v, list):  # the panoptic head's [(semantic, panoptic)] ids
            v = v[0][0]
        return v

    eager = voxels(fwd()).clone()
    n0 = ops.LAUNCH_COUNT[0]
    fwd()
    torch.cuda.synchronize()
    launches = ops.LAUNCH_COUNT[0] - n0

    # GPU time by stage, each stage called by hand on the previous stage's output
    split = collections.OrderedDict()
    imgs = img_inputs[0]
    x, split["image_encoder"] = gpu_ms(lambda: model.img_neck(model.img_backbone(imgs.flatten(0, 1)))[0])
    x = x.view(B, N, *x.shape[1:])
    mlp = vt.get_mlp_input(*img_inputs[1:7])
    (bev, _), split["view_transformer"] = gpu_ms(lambda: vt([x] + img_inputs[1:7] + [mlp]))
    enc, split["encoder"] = gpu_ms(lambda: model.img_bev_encoder_backbone(bev))
    feats, split["pixel_decoder"] = gpu_ms(lambda: model.img_bev_encoder_neck(enc))
    _, split["head"] = gpu_ms(lambda: model.pts_bbox_head.simple_test(feats, metas))
    total = sum(split.values())

    graph, out = graphed(fwd)
    graph.replay()
    torch.cuda.synchronize()
    err = rel(voxels(out).float(), eager.float())
    times = alternated({"detector": graph}, a.iters, a.warmup)["detector"]
    ms = statistics.median(times)
    print(json.dumps({
        "config": a.config, "batch": B, "images": [B, N, 3, H, W], "ms_per_forward": round(ms, 3),
        "samples_per_s": round(1e3 * B / ms, 2), "gpu_launches": launches,
        "stage_gpu_ms": {k: round(v, 3) for k, v in split.items()},
        "stage_share": {k: round(v / total, 4) for k, v in split.items()},
        "rel_err_graph_vs_eager": err, "card": card()}))


if __name__ == "__main__":
    main()
