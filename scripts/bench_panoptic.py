"""What the panoptic head costs on the GPU (nuScenes panoptic workload, synth.WORKLOADS["nusc_panoptic"]).

    python scripts/bench_panoptic.py [--batch 4] [--steps 10] [--rounds 3]

1. The connected step (view transformer -> encoder -> neck -> head.simple_test) at the reference grid 128x128x16 ->
   occ 256x256x32, timed as bench.py times it (CUDA graph replay, CUDA events, L2 flushed between steps): the panoptic
   head (150 queries) and the semantic head (100 queries) alternate in one run.
2. The panoptic tail alone (occ_panoptic_voxels on the last layer's native logits), with its algorithmic bytes over the
   time against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), next to the semantic tail (occ_classmix).
Prints the card name, power limit and max SM clock with the numbers.  Needs a GPU; there is no CPU fallback.
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from occformer_b200 import HEADS, ops, synth  # noqa: E402
from occformer_b200.head import head_cfg  # noqa: E402
from gpu_bench import card  # noqa: E402

HBM_TBS = 3.35


def build_head(dev, wl, queries):
    w = synth.WORKLOADS[wl]
    kw = dict(thing_indices=w["thing_indices"]) if "thing_indices" in w else {}
    head = HEADS.build(dict(type=w["head"], **head_cfg(bench.EMBED, queries, w["classes"], bench.DEC_LAYERS, bench.HEADS,
                                                       w["pc"]), **kw))
    head.load_state_dict(synth.make_head_state(bench.EMBED, queries, w["classes"], bench.DEC_LAYERS, 3, seed=1), strict=True)
    return head.to(dev).eval()


def graphed_step(dev, vt, enc, neck, head, inp, metas):
    mats = [inp[k] for k in ("rots", "trans", "intrins", "post_rots", "post_trans", "bda")]

    @torch.no_grad()
    def step():
        voxel, _ = vt([inp["x"]] + mats + [None])
        return head.simple_test(neck(enc(voxel)), metas)

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    torch.cuda.synchronize()
    return g


def time_graph(g, steps, flush):
    ms = []
    for i in range(steps):
        flush.fill_(float(i))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return sum(ms) / len(ms)


def time_fn(fn, iters, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ms = []
    for i in range(iters):
        flush.fill_(float(i))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return sum(ms) / len(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_panoptic: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B = args.batch
    print(f"card: {card()}")
    bench.set_workload("nusc_ref")  # the panoptic config's grid and occupancy size
    vt, enc, neck, _ = bench.build_b200(dev)
    w = synth.WORKLOADS["nusc_panoptic"]
    heads = {"panoptic Q=150": build_head(dev, "nusc_panoptic", w["queries"]),
             "semantic Q=100": build_head(dev, "nusc_ref", 100)}
    inp = {k: v.to(dev) for k, v in bench.host_inputs(B, seed=0).items()}
    metas = [dict(occ_size=w["occ"], pc_range=w["pc"])] * B
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)  # 256 MB > L2
    graphs = {k: graphed_step(dev, vt, enc, neck, h, inp, metas) for k, h in heads.items()}
    res = {k: [] for k in graphs}
    for _ in range(args.rounds):
        for k, g in graphs.items():
            res[k].append(time_graph(g, args.steps, flush))
    print(f"connected step, batch {B}, grid 128x128x16 -> occ 256x256x32 (CUDA graph, L2 flushed):")
    for k, v in res.items():
        print(f"  {k}: {min(v):.1f} .. {max(v):.1f} ms/step  ({B * 1000 / max(v):.2f} .. {B * 1000 / min(v):.2f} samples/s)")

    # ---- the tails alone, on native-resolution logits of the workload's shape
    X, Y, Z = 128, 128, 16
    Xo, Yo, Zo = w["occ"]
    Q, Qs, NC = w["queries"], (w["queries"] + 3) // 4 * 4, w["classes"] + 1
    gen = torch.Generator(device=dev).manual_seed(0)
    mask = torch.randn(B, X * Y * Z, Qs, device=dev, generator=gen)
    cls = torch.randn(B, Q, NC, device=dev, generator=gen)
    thing = ops.thing_mask(w["thing_indices"])
    pan_ms = time_fn(lambda: ops.panoptic_voxels(mask, cls, B, (X, Y, Z), (Xo, Yo, Zo), Q, thing), 10, flush)
    Vo = Xo * Yo * Zo
    pan_bytes = B * X * Y * Z * Qs * 4 + B * Vo * (16 + 2)  # logits once, two int64 ids, query index write + read
    mask100 = mask[..., :100].contiguous()
    cls100 = cls[:, :100].contiguous()
    sem_ms = time_fn(lambda: ops.classmix(mask100, cls100, B, (X, Y, Z), (Xo, Yo, Zo), 100, NC, with_labels=True), 10,
                     flush)
    sem_bytes = B * X * Y * Z * 100 * 4 + B * Vo * ((NC - 1) * 4 + 1)
    print(f"tails alone, batch {B}, native 128x128x16 -> occ 256x256x32 (CUDA events, L2 flushed):")
    for name, ms, nb in (("occ_panoptic_voxels Q=150", pan_ms, pan_bytes), ("occ_classmix Q=100 (semantic)", sem_ms,
                                                                            sem_bytes)):
        bw = nb / (ms * 1e-3) / 1e12
        print(f"  {name}: {ms:.2f} ms, {nb / 1e6:.0f} MB algorithmic, {bw:.2f} TB/s = {100 * bw / HBM_TBS:.0f} % of "
              f"{HBM_TBS} TB/s (data sheet, not measured)")


if __name__ == "__main__":
    main()
