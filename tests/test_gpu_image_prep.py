"""Camera images from the decoded frames on the H100 (occformer_b200.image_prep, csrc/image_prep.cu), bit for bit: against
the reference transforms' images (SHA-256 in tests/golden/image_prep.npz, frames regenerated from their hash) and against
the numpy restatement (oracle/image_prep.py, itself checked against Pillow and the reference); launches, graph replay,
argument errors, the output bounds; then the detector from frames."""
import ctypes
import os

import numpy as np
import pytest
import torch

from util import GOLDEN, assert_close, graph_replay, launches, rejected, same_bits, sentinel, untouched
from oracle import image_prep as ip
from occformer_b200 import image_prep, ops

pytestmark = pytest.mark.gpu


def _aug(name, frames):
    """the img_aug meta the new transforms give one sample of a case"""
    _, _, size, norm = ip.CASES[name]
    aug = [ip.test_augmentation(f.shape[0], f.shape[1], size) for f in frames]
    return dict(resize_dims=[list(a[1]) for a in aug], crop=[list(a[2]) for a in aug], input_size=list(size),
                **image_prep.norm_config(norm))


def _sha(t):
    return ip.sha(t.cpu().numpy())


@pytest.mark.parametrize("name", list(ip.CASES))
def test_golden_hashes(cuda, name):
    g = np.load(os.path.join(GOLDEN, "image_prep.npz"))
    samples = ip.case_frames(name)
    augs = [_aug(name, s) for s in samples]
    for s, a in enumerate(augs):
        assert a["resize_dims"] == g[f"{name}_{s}_resize_dims"].tolist() and a["crop"] == g[f"{name}_{s}_crop"].tolist()
    frames = [torch.from_numpy(np.stack(s)).to(cuda) for s in samples]
    if len({tuple(f.shape) for f in frames}) == 1:
        frames = torch.stack(frames)  # one (B, N, H, W, 3) tensor; KITTI's mixed sizes go as a list, in one call
    n0 = ops.LAUNCH_COUNT[0]
    out = image_prep.prepare_images(frames, augs)
    assert ops.LAUNCH_COUNT[0] - n0 == 2
    assert out.shape == (len(samples), len(samples[0]), 3, *ip.CASES[name][2]) and out.dtype == torch.float32
    got = [_sha(im) for im in out.reshape(-1, *out.shape[2:])]
    assert got == [str(h) for h in g[f"{name}_sha"]]
    if name == "small":
        same_bits(out[0], torch.from_numpy(g["small_0_img"]).to(cuda), "small case")


def _one(cuda, frame, size, box, norm):
    fH, fW = box[3] - box[1], box[2] - box[0]
    aug = dict(resize_dims=[list(size)], crop=[list(box)], input_size=[fH, fW], **image_prep.norm_config(norm))
    return image_prep.prepare_images(torch.from_numpy(frame[None, None]).to(cuda), [aug])[0, 0]


def test_sweep_equals_the_restatement(cuda):
    from test_cpu_image_prep import SWEEP
    for i, (H, W, size, box) in enumerate(SWEEP):
        f = ip.frame(500 + i, H, W)
        for norm in (ip.NORM_R50, ip.NORM_R101):
            ref = ip.prepare(f, size, box, norm)
            got = _one(cuda, f, size, box, norm)
            same_bits(got, torch.from_numpy(ref).to(cuda), f"sweep {i} {(H, W, size, box)}")


def _raw(cuda, geoms, fH, fW, norm=ip.NORM_R50):
    """the C-ABI arguments of M frames with these geometries (H, W, rW, rH, x0, y0) -> (args, out)"""
    frames = [torch.from_numpy(ip.frame(900 + m, g[0], g[1])).reshape(-1) for m, g in enumerate(geoms)]
    offsets = np.cumsum([0] + [f.numel() for f in frames])[:-1].tolist()
    flat = torch.cat(frames).to(cuda)
    tables = []
    for H, W, rW, rH, _, _ in geoms:
        tables += [ops._prep_table(cuda, W, rW).data_ptr(), ops._prep_table(cuda, H, rH).data_ptr()]
    M = len(geoms)
    geom = (ctypes.c_int * (6 * M))(*[v for g in geoms for v in g])
    nbytes = ops.lib().occ_prepare_images_workspace_bytes(geom, M, fH, fW)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=cuda)
    norm_t = torch.from_numpy(image_prep.normalize_table(norm["mean"], norm["std"], norm["to_rgb"])).to(cuda)
    out = sentinel(M * 3 * fH, fW, cuda)
    args = [flat, flat.numel(), (ctypes.c_longlong * M)(*offsets), geom, M, fH, fW,
            (ctypes.c_longlong * (2 * M))(*tables), norm_t, int(norm["to_rgb"]), ws, ws.numel(), out]
    return args, out


def test_launch_count_is_constant(cuda):
    counts = set()
    for M in (1, 24):
        args, _ = _raw(cuda, [(90, 160, 70, 39, 0, 14)] * M, 25, 70)
        counts.add(launches("occ_prepare_images", *args))
    args, _ = _raw(cuda, [(37, 124, 128, 38, 0, 0), (37, 122, 128, 38, 0, 0), (36, 121, 128, 38, 0, 0)], 38, 128)
    counts.add(launches("occ_prepare_images", *args))
    assert counts == {2}


def test_graph_replay_equals_eager(cuda):
    samples = ip.case_frames("r50")[:2]
    frames = torch.from_numpy(np.stack([np.stack(s) for s in samples])).to(cuda)
    augs = [_aug("r50", s) for s in samples]
    eager = image_prep.prepare_images(frames, augs)  # builds the tables before the capture
    outs = []
    graph_replay(lambda: outs.append(image_prep.prepare_images(frames, augs)), outs)
    same_bits(outs[0], eager, "graph replay")


def test_output_bounds_untouched(cuda):
    """a view into a sentinel buffer: only the (M, 3, fH, fW) output is written"""
    geoms = [(60, 100, 44, 26, 0, -3), (60, 100, 44, 26, 5, 10), (61, 99, 44, 26, 30, 30)]
    args, out = _raw(cuda, geoms, 20, 44)
    big = sentinel(out.shape[0] + 64, out.shape[1], cuda)
    inner = big[32:32 + out.shape[0]]
    args[-1] = inner
    ops._call("occ_prepare_images", *args)
    torch.cuda.synchronize()
    untouched(big[:32], "rows before the output")
    untouched(big[32 + out.shape[0]:], "rows after the output")
    got = inner.view(3, 3, 20, 44)
    for m, (H, W, rW, rH, x0, y0) in enumerate(geoms):
        ref = ip.prepare(ip.frame(900 + m, H, W), (rW, rH), (x0, y0, x0 + 44, y0 + 20), ip.NORM_R50)
        same_bits(got[m], torch.from_numpy(ref).to(cuda), f"image {m}")


def test_argument_errors(cuda):
    good = [(90, 160, 70, 39, 0, 14), (90, 160, 70, 39, 0, 14)]
    args, out = _raw(cuda, good, 25, 70)
    ops._call("occ_prepare_images", *args)  # the arguments are right
    torch.cuda.synchronize()

    def bad(i, value, geoms=good, rc=-1):
        a, o = _raw(cuda, geoms, 25, 70)
        a[i] = value
        rejected("occ_prepare_images", *a, buffers=[o], rc=rc)

    M = len(good)
    bad(4, 0)                                                          # M = 0
    bad(4, 257)                                                        # M above the bound
    bad(5, 0)                                                          # fH = 0
    bad(6, -1)                                                         # fW < 0
    bad(1, 90 * 160 * 3 * M - 1)                                       # the last frame runs past frame_bytes
    bad(2, (ctypes.c_longlong * M)(0, 90 * 160 * 3 + 1))               # an offset past the frame buffer
    bad(2, (ctypes.c_longlong * M)(-1, 0))                             # a negative offset
    bad(7, (ctypes.c_longlong * (2 * M))(*([0] * (2 * M))))            # null tables
    bad(9, 2)                                                          # swap_rb not 0 / 1
    bad(11, 0)                                                         # workspace too short
    for g in [(0, 160, 70, 39, 0, 0), (90, 0, 70, 39, 0, 0), (90, 160, 0, 39, 0, 0), (90, 160, 70, -1, 0, 0),
              (90, 160, 70, 39, 1 << 30, 0), (90, 160, 70, 39, 0, -(1 << 30))]:
        a, o = _raw(cuda, good, 25, 70)
        a[3] = (ctypes.c_int * (6 * M))(*(list(g) + list(good[1])))
        rejected("occ_prepare_images", *a, buffers=[o], rc=-1)
    # a downscale by more than 32 needs more than 129 taps
    a, o = _raw(cuda, [(90, 3300, 100, 39, 0, 0)], 25, 70)
    rejected("occ_prepare_images", *a, buffers=[o], rc=-2)
    a, o = _raw(cuda, [(90, 3200, 100, 39, 0, 0)], 25, 70)             # by exactly 32: 129 taps, accepted
    ops._call("occ_prepare_images", *a)
    ref = ip.prepare(ip.frame(900, 90, 3200), (100, 39), (0, 0, 70, 25), ip.NORM_R50)
    same_bits(o.view(3, 25, 70), torch.from_numpy(ref).to(cuda), "downscale by 32")


def test_cpu_frames_raise(cuda):
    aug = _aug("small", ip.case_frames("small")[0])
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        image_prep.prepare_images(torch.zeros(1, 2, 90, 160, 3, dtype=torch.uint8), [aug])


# ---------------------------------------------------------------------------------------------- the detector
def test_detector_from_frames(cuda):
    from test_gpu_detector import detector, inputs
    model, _ = detector("nusc_r50", cuda)
    metas, img_inputs, _, _ = inputs("nusc_r50", 2, cuda)
    B, N = img_inputs[0].shape[:2]
    assert tuple(img_inputs[0].shape[3:]) == (256, 704) and N <= 6
    samples = [[ip.frame(7000 + 10 * b + c, 900, 1600) for c in range(N)] for b in range(B)]
    augs = [_aug("r50", s) for s in samples]
    ref_imgs = torch.from_numpy(np.stack([np.stack([ip.prepare(f, a["resize_dims"][c], a["crop"][c], ip.NORM_R50)
                                                    for c, f in enumerate(s)]) for s, a in zip(samples, augs)]))
    frames = torch.from_numpy(np.stack([np.stack(s) for s in samples])).to(cuda)
    seen = []
    hook = model.img_backbone.register_forward_pre_hook(lambda mod, args: seen.append(args[0].clone()))
    try:
        ref = model.simple_test(metas, [ref_imgs.to(cuda)] + img_inputs[1:])
        out = model.simple_test([dict(m, img_aug=a) for m, a in zip(metas, augs)], [frames] + img_inputs[1:])
    finally:
        hook.remove()
    assert len(seen) == 2 and seen[1].dtype == torch.float32
    assert tuple(seen[1].shape) == (B * N, 3, 256, 704)
    same_bits(seen[0], ref_imgs.view(B * N, 3, 256, 704).to(cuda), "image encoder input from normalised images")
    same_bits(seen[1], seen[0], "image encoder input from frames")
    with pytest.raises(ValueError, match="img_aug"):
        model.simple_test(metas, [frames] + img_inputs[1:])
    assert set(out) == set(ref)
    for k in ref:
        if torch.is_tensor(ref[k]) and ref[k].is_floating_point():
            assert_close(out[k], ref[k], what=f"detector {k}")
        elif torch.is_tensor(ref[k]):
            assert out[k].shape == ref[k].shape
