"""What the occupancy ground truth costs on the GPU (occformer_b200.targets, occ_lidarseg_occupancy), next to the
reference loaders' algorithm on the host (float64 voxel index, np.lexsort, then a per-voxel loop with a fresh 256- or
65 536-entry counter, loading_nusc_occ.py:95-138 / loading_nusc_panoptic_occ.py:120-166, restated here and jitted with
numba when it is importable).

    python scripts/bench_occ_targets.py [--iters 50]

Inputs: synthetic 34 720-point scans spread uniformly over the configs' range [-51.2, -51.2, -5, 51.2, 51.2, 3], 256x256x32
voxels, semantic labels 0..16 or panoptic ids; batch 1 and 4.  Device time per batch: the call captured once into a CUDA
graph and replayed between CUDA events, so the GPU does not wait for the host's enqueue; call time: CUDA events around
the eager Python call (allocation, ctypes marshalling and five enqueues included); L2 flushed before every timed run,
median.  Host time per sample of the restatement, best of three semantic / one panoptic run (the compiling call not
counted).  Prints the card name, power limit and max SM clock, the host's core count and the occupied-voxel counts with
the numbers.  Needs a GPU; there is no CPU fallback.
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from occformer_b200 import ops  # noqa: E402
from oracle import occ_targets as ot  # noqa: E402
from gpu_bench import card, graphed  # noqa: E402

R, G = ot.NUSC_RANGE, ot.NUSC_GRID


def scan(n, seed, panoptic):
    rng = np.random.default_rng(seed)
    lo, hi = np.array(R[:3]), np.array(R[3:])
    xyz = lo + (hi - lo) * rng.random((n, 3))
    cls = rng.integers(0, 17, n)
    ids = np.where(cls <= 10, cls * 1000 + rng.integers(0, 20, n), cls * 1000) if panoptic else cls
    return np.concatenate([xyz, ids[:, None]], axis=1).astype(np.float32)


def _walk(processed, pairs, size, drop_zero):
    """the per-voxel counter loop over the lexsorted (x, y, z, id) rows"""
    counter = np.zeros(size, dtype=np.uint16)
    counter[pairs[0, 3]] = 1
    cur = pairs[0, :3]
    for i in range(1, pairs.shape[0]):
        ind = pairs[i, :3]
        if ind[0] != cur[0] or ind[1] != cur[1] or ind[2] != cur[2]:
            if drop_zero:
                counter[0] = 0
            processed[cur[0], cur[1], cur[2]] = np.argmax(counter)
            counter = np.zeros(size, dtype=np.uint16)
            cur = ind
        counter[pairs[i, 3]] += 1
    processed[cur[0], cur[1], cur[2]] = np.argmax(counter)
    return processed


try:
    import numba
    _walk_fn = numba.njit(cache=False)(_walk)
except ImportError:
    _walk_fn = None


def host_reference(pts, panoptic):
    """the loader's gt_occ of one scan by its own algorithm -> int64 (X, Y, Z)"""
    idx = ot.voxel_index(pts[:, :3], R, G)
    pairs = np.concatenate([idx, pts[:, 3:4].astype(np.int64)], axis=1)
    pairs = pairs[np.lexsort((idx[:, 0], idx[:, 1], idx[:, 2]))]
    empty = 17000 if panoptic else 17
    processed = np.full(G, empty, dtype=np.int64)
    processed = _walk_fn(processed, pairs, 65536 if panoptic else 256, panoptic)
    processed[processed == 0] = 65535 if panoptic else 255
    processed[processed == empty] = 0
    return processed


def _timed(run, iters, flush):
    """median, min, max of `iters` event-timed runs, L2 flushed before each"""
    ms = []
    for i in range(iters):
        flush.fill_(float(i))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return ms[len(ms) // 2], ms[0], ms[-1]


def device_ms(pts, counts, panoptic, iters, flush):
    """-> (device time: the call's five operations and the counter's fill replayed as one CUDA graph, so the GPU never
    waits for the host; call time: events around the eager Python call, host enqueue included; the volume)"""
    args = (pts, counts, R, G, panoptic, 17000 if panoptic else 17, 65535 if panoptic else 255)
    g, (out, invalid) = graphed(lambda: ops.lidarseg_occupancy(*args))
    g.replay()
    torch.cuda.synchronize()
    assert int(invalid.item()) == 0
    device = _timed(g.replay, iters, flush)
    for _ in range(3):
        ops.lidarseg_occupancy(*args)
    call = _timed(lambda: ops.lidarseg_occupancy(*args), iters, flush)
    return device, call, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--n", type=int, default=34720)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_occ_targets: needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(f"card: {card()}")
    print(f"host: {os.cpu_count()} cores, numba {'yes' if _walk_fn else 'not importable'}")
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device=dev)  # 256 MB > L2
    for panoptic in (False, True):
        mode = "panoptic" if panoptic else "semantic"
        scans = [scan(args.n, 7 + b, panoptic) for b in range(4)]
        occ = [int((ot.occupancy(s, G, R, panoptic) != 0).sum()) for s in scans]
        for B in (1, 4):
            pts = torch.from_numpy(np.concatenate(scans[:B])).to(dev)
            (med, lo, hi), (cmed, clo, chi), out = device_ms(pts, [args.n] * B, panoptic, args.iters, flush)
            ref = np.stack([ot.occupancy(s, G, R, panoptic) for s in scans[:B]])
            assert np.array_equal(out.cpu().numpy(), ref), "device volume differs from the restatement"
            print(f"  {mode} batch {B} ({args.n} points per sample, occupied voxels {occ[:B]}): device {med:.4f} ms "
                  f"per batch (graph replay, median of {args.iters}; {lo:.4f} .. {hi:.4f}), call {cmed:.4f} ms "
                  f"(eager, host enqueue included; {clo:.4f} .. {chi:.4f})")
        if _walk_fn is None:
            print(f"  {mode} host reference algorithm: not run (numba not importable)")
            continue
        host_reference(scans[0][:100], panoptic)  # compile
        ts = []
        for _ in range(1 if panoptic else 3):  # the panoptic walk takes seconds per sample
            t = time.perf_counter()
            got = host_reference(scans[0], panoptic)
            ts.append((time.perf_counter() - t) * 1e3)
        assert np.array_equal(got, ot.occupancy(scans[0], G, R, panoptic)), "host reference differs from restatement"
        print(f"  {mode} host reference algorithm (index + lexsort + counter loop, numba, one core): "
              f"{min(ts):.1f} ms per sample ({occ[0]} occupied voxels)")


if __name__ == "__main__":
    main()
