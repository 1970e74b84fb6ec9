"""The per-stream workspaces of the input pipeline's and the evaluation's wrappers (ops._stream_workspace): when a call
needs more workspace than the stream's buffer holds, the buffer grows, and a CUDA graph captured before still points at
the old one, so the cache keeps the superseded buffer referenced (as test_gpu_voxel_pool does for the pooling
workspace)."""
import gc
import weakref

import numpy as np
import pytest
import torch

from util import GOLDEN
from occformer_b200 import image_prep, ops

pytestmark = pytest.mark.gpu


def _panoptic_eval(dev, large):
    n, K = (100_000 if large else 1000), 4
    ids = torch.arange(n, device=dev) % K
    state = torch.zeros(K * K + 6 * K + 1, dtype=torch.int64, device=dev)
    ops.panoptic_eval(ids, ids, ids, ids, K, 1, 0, state)


def _lidarseg_occupancy(dev, large):
    n = 100_000 if large else 1000
    pts = torch.rand(n, 4, device=dev) * torch.tensor([40.0, 40.0, 4.0, 0.0], device=dev)
    ops.lidarseg_occupancy(pts, [n], (0, 0, 0, 40, 40, 4), (32, 32, 8), False, 17, 255)


def _prepare_images(dev, large):
    M = 4 if large else 1
    frames = torch.zeros(M * 90 * 160 * 3, dtype=torch.uint8, device=dev)
    norm = image_prep.norm_config(None)
    ops.prepare_images(frames, [m * 90 * 160 * 3 for m in range(M)], [(90, 160, 70, 39, 0, 14)] * M, (25, 70),
                       norm["mean"], norm["std"], norm["to_rgb"])


def _decode_jpeg(dev, large):
    from oracle import jpeg as oj
    g = np.load(f"{GOLDEN}/jpeg.npz")
    files = [g[f"full_{i}_bytes"].tobytes() for i in range(len(oj.FULL))] if large else [g["small_0_bytes"].tobytes()]
    image_prep.decode_jpeg([[f] for f in files])


def _decode_png(dev, large):
    g = np.load(f"{GOLDEN}/png.npz")
    files = [g[f"file_{i}"].tobytes() for i in range(int(g["count"]))]
    image_prep.decode_png([[f] for f in files] if large else [files[:1]])


CASES = {"occ_panoptic_eval": _panoptic_eval, "occ_lidarseg_occupancy": _lidarseg_occupancy,
         "occ_prepare_images": _prepare_images, "occ_decode_jpeg": _decode_jpeg, "occ_decode_png": _decode_png}


def _fresh_stream(kernel, dev):
    """a stream on which kernel has no workspace yet: the small call then creates it and the large one grows it"""
    for _ in range(64):
        s = torch.cuda.Stream(dev)
        if (kernel, str(dev), s.cuda_stream) not in ops._stream_ws:
            return s
    raise AssertionError(f"every pool stream already has a workspace of {kernel}")


@pytest.mark.parametrize("kernel", sorted(CASES))
def test_workspace_growth_keeps_superseded_buffers_alive(cuda, kernel):
    s = _fresh_stream(kernel, cuda)
    key = (kernel, str(cuda), s.cuda_stream)
    with torch.cuda.stream(s):
        CASES[kernel](cuda, False)
        old = weakref.ref(ops._stream_ws[key][0])
        CASES[kernel](cuda, True)
    s.synchronize()
    new = ops._stream_ws[key][0]
    gc.collect()
    assert old() is not None, "the superseded workspace was freed"
    assert old().data_ptr() != new.data_ptr(), "the larger call did not grow the workspace"
