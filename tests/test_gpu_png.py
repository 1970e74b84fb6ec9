"""Camera frames from their PNG files on the H100 (image_prep.decode_png, csrc/png_decode.cu), bit for bit: against
cv2.imdecode (SHA-256 in tests/golden/png.npz) and, PNG being lossless, against the pixels the test-side writer
(oracle/png.py) encoded; every zlib level and strategy, IDAT splits, mixed frame sizes, launches, graph replay, the
output bounds, corrupt streams, argument errors; then the detector from PNG bytes."""
import ctypes

import numpy as np
import pytest
import torch

from util import GOLDEN, assert_close, launches, rejected, same_bits
from oracle import image_prep as ip
from oracle import png as op
from occformer_b200 import image_prep, ops, png

pytestmark = pytest.mark.gpu
SENT = 0xA5
KH, KW = 376, 1241


def _fixture():
    g = np.load(f"{GOLDEN}/png.npz")
    return [(str(g[f"name_{i}"]), g[f"file_{i}"].tobytes(), str(g[f"sha_{i}"])) for i in range(int(g["count"]))]


def _src(seed, H=KH, W=KW):
    return op.content(H, W, seed)


def test_fixture_frames(cuda):
    fx = _fixture()
    out = image_prep.decode_png([[f] for _, f, _ in fx])  # every small kind and the three KITTI sizes: the list form
    assert isinstance(out, list) and len(out) == len(fx)
    for (name, f, sha), o in zip(fx, out):
        assert op.sha(o[0].cpu().numpy()) == sha, name


@pytest.mark.parametrize("level", [1, 6, 9])
def test_writer_frames_every_strategy(cuda, level):
    strategies = ["default", "filtered", "huffman", "rle", "fixed"]
    srcs = [_src(300 + level * 10 + k) for k in range(len(strategies))]
    files = [op.write(s, level=level, strategy=st) for s, st in zip(srcs, strategies)]
    if level == 1:  # all stored blocks
        srcs.append(_src(399))
        files.append(op.write(srcs[-1], level=0))
    out = image_prep.decode_png([files])
    assert out.shape == (1, len(files), KH, KW, 3)
    for k, s in enumerate(srcs):
        assert np.array_equal(out[0, k].cpu().numpy(), s), f"level {level} file {k}"


def test_idat_splits(cuda):
    srcs = [_src(501, 40, 97), _src(502), _src(503)]
    files = [op.write(srcs[0], idat=1), op.write(srcs[1], idat=[1, 7, 8191, 8193, 3]),
             op.write(srcs[2], idat=65537)]
    out = image_prep.decode_png([[f] for f in files])
    for o, s in zip(out, srcs):
        assert np.array_equal(o[0].cpu().numpy(), s)


def test_mixed_sizes_list_form(cuda):
    fx = _fixture()
    full = [f for _, f, _ in fx[-3:]]
    lst = image_prep.decode_png([[full[0]], [full[1]], [full[2]]])
    assert [tuple(x.shape) for x in lst] == [(1, 376, 1241, 3), (1, 370, 1226, 3), (1, 375, 1242, 3)]
    for x, (_, _, sha) in zip(lst, fx[-3:]):
        assert op.sha(x[0].cpu().numpy()) == sha
    t = image_prep.decode_png([[full[0]], [full[0]]])
    assert torch.is_tensor(t) and t.shape == (2, 1, 376, 1241, 3)


def _raw(files, out_pad=64):
    """the C-ABI arguments of these files -> (args, big, inner, status): the frames go into inner, a view of the
    sentinel buffer big with out_pad bytes on either side"""
    headers = [png.parse(f) for f in files]
    streams = [b"".join(f[o:o + n] for o, n in h.idat) for f, h in zip(files, headers)]
    offsets = np.cumsum([0] + [len(s) for s in streams]).tolist()
    data = torch.from_numpy(np.frombuffer(b"".join(streams), np.uint8).copy()).to("cuda")
    starts = sum((np.cumsum([0] + [n for _, n in h.idat])[:-1].tolist() for h in headers), [])
    idat = torch.tensor(starts, dtype=torch.int32, device="cuda")
    M = len(files)
    geom, out_off, total = [], [], 0
    for h in headers:
        geom += [h.height, h.width, h.stream_len, h.cinfo]
        out_off.append(total)
        total += h.height * h.width * 3
    streams_c = (ctypes.c_longlong * M)(*offsets[:-1])
    geom = (ctypes.c_int * (4 * M))(*geom)
    counts = (ctypes.c_int * M)(*[len(h.idat) for h in headers])
    nbytes = ops.lib().occ_decode_png_workspace_bytes(streams_c, geom, counts, M)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    big = torch.full(((total + 2 * out_pad + 3) // 4 * 4,), SENT, dtype=torch.uint8, device="cuda")
    inner = big[out_pad:out_pad + total]
    status = torch.full((M, 2), -7, dtype=torch.int32, device="cuda")
    args = [data, data.numel(), streams_c, geom, counts, idat, idat.numel(), (ctypes.c_longlong * M)(*out_off), M,
            ws, ws.numel(), inner, inner.numel(), status]
    return args, big, inner, status


def _outside_untouched(big, inner, pad=64):
    assert bool((big[:pad] == SENT).all()) and bool((big[pad + inner.numel():] == SENT).all()), \
        "written outside the output"


def test_launch_count_is_constant(cuda):
    fx = _fixture()
    counts = set()
    for files in ([fx[3][1]], [f for _, f, _ in fx], [op.write(_src(7, 30, 40), level=0)]):
        args, _, _, _ = _raw(files)
        counts.add(launches("occ_decode_png", *args))
    assert counts == {ops.PNG_LAUNCHES}


def test_graph_replay_equals_eager(cuda):
    files = [f for _, f, _ in _fixture()[-2:]] + [op.write(_src(8, 50, 60), strategy="fixed")]
    args, _, inner, status = _raw(files)
    ops._call("occ_decode_png", *args)
    torch.cuda.synchronize()
    eager = inner.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        ops._call("occ_decode_png", *args)
    torch.cuda.current_stream().wait_stream(s)
    inner.fill_(SENT)
    status.fill_(-7)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(inner, eager) and int(status[:, 0].abs().sum()) == 0


def test_fixture_frames_link_without_serial_decodes(cuda):
    """the scan and the probe find every block of cv2's full-size files: the link jumps over all of them (a miss would
    only cost speed, so only this count shows it)"""
    args, _, _, status = _raw([f for _, f, _ in _fixture()[-3:]])
    ops._call("occ_decode_png", *args)
    torch.cuda.synchronize()
    st = status.cpu()
    assert int(st[:, 0].abs().sum()) == 0 and st[:, 1].tolist() == [0, 0, 0]


def test_output_bounds_untouched(cuda):
    fx = _fixture()
    files = [fx[0][1], fx[10][1], fx[-1][1]]
    args, big, inner, status = _raw(files)
    ops._call("occ_decode_png", *args)
    torch.cuda.synchronize()
    _outside_untouched(big, inner)
    assert int(status[:, 0].abs().sum()) == 0


@pytest.mark.parametrize("case", range(len(op.corrupt_files())))
def test_corrupt_streams_raise(cuda, case):
    name, bad, bit = op.corrupt_files()[case]
    good = op.write(_src(11, 24, 33))
    with pytest.raises(ValueError, match="cam_b: cv2 would not decode it"):
        image_prep.decode_png([[good], [bad]], names=[["cam_a"], ["cam_b"]])
    args, big, inner, status = _raw([good, bad, good])
    ops._call("occ_decode_png", *args)
    torch.cuda.synchronize()
    _outside_untouched(big, inner)
    st = status.cpu()
    assert int(st[1, 0]) & bit, f"{name}: status {int(st[1, 0])}"
    assert int(st[0, 0]) == 0 and int(st[2, 0]) == 0
    ref = _src(11, 24, 33)
    assert np.array_equal(inner[:ref.size].cpu().numpy().reshape(ref.shape), ref)
    assert np.array_equal(inner[-ref.size:].cpu().numpy().reshape(ref.shape), ref)


def test_benign_streams_decode(cuda):
    cases = op.benign_files()
    out = image_prep.decode_png([[f] for _, f, _ in cases])
    for (name, _, src), o in zip(cases, out):
        assert np.array_equal(o[0].cpu().numpy(), src), name


def test_argument_errors(cuda):
    files = [_fixture()[0][1], _fixture()[6][1]]
    args, big, inner, status = _raw(files)
    ops._call("occ_decode_png", *args)
    torch.cuda.synchronize()

    def bad(i, value):
        a, b, _, st = _raw(files)
        a[i] = value
        rejected("occ_decode_png", *a, buffers=[b.view(torch.int32), st], rc=-1)

    geom = list(args[3])
    bad(1, args[1] - 1)                                                  # the last stream runs past data_bytes
    bad(2, (ctypes.c_longlong * 2)(-1, args[2][1]))                      # a negative stream offset
    for k, v in ((0, 0), (1, 16385), (2, 6), (3, 8)):
        gg = list(geom)
        gg[k] = v
        bad(3, (ctypes.c_int * 8)(*gg))
    bad(4, (ctypes.c_int * 2)(0, 1))                                     # no IDAT chunk
    bad(6, args[6] - 1)                                                  # a short idat array
    bad(7, (ctypes.c_longlong * 2)(0, args[12] - 1))                     # an output past out_bytes
    bad(8, 0)                                                            # M = 0
    bad(8, 97)                                                           # M above the bound
    bad(10, args[10] - 1)                                                # workspace too short
    a, b, _, st = _raw(files)
    a[9] = a[9][1:]                                                      # misaligned workspace
    a[10] -= 1
    rejected("occ_decode_png", *a, buffers=[b.view(torch.int32), st], rc=-1)


def test_rejected_files_raise_on_the_host(cuda):
    src = _src(12, 16, 16)
    trns = op.write(src, ancillary=[(b"tRNS", b"\0\1\0\2\0\3")])
    n0 = ops.LAUNCH_COUNT[0]
    with pytest.raises(ValueError, match="cam_x: .*tRNS"):
        image_prep.decode_png([[trns]], names=[["cam_x"]])
    assert ops.LAUNCH_COUNT[0] == n0


# ---------------------------------------------------------------------------------------------- the detector
def test_detector_from_png(cuda):
    from test_gpu_detector import detector, inputs
    model, _ = detector("kitti", cuda)
    metas, img_inputs, _, _ = inputs("kitti", 2, cuda)
    B, N = img_inputs[0].shape[:2]
    size = list(img_inputs[0].shape[-2:])
    srcs = [_src(7000 + b) for b in range(B)]
    files = [[op.write(s, level=1)] for s in srcs]
    frames = torch.from_numpy(np.stack([s[None] for s in srcs])).to(cuda)
    augs = []
    for _ in range(B):
        a = ip.test_augmentation(KH, KW, tuple(size))
        augs.append(dict(resize_dims=[list(a[1])], crop=[list(a[2])], input_size=size,
                         **image_prep.norm_config(ip.NORM_R50)))
    seen = []
    hook = model.img_backbone.register_forward_pre_hook(lambda mod, args: seen.append(args[0].clone()))
    try:
        ref = model.simple_test([dict(m, img_aug=a) for m, a in zip(metas, augs)], [frames] + img_inputs[1:])
        placeholder = torch.zeros((B, N, 0), dtype=torch.uint8, device=cuda)
        out = model.simple_test([dict(m, img_aug=dict(a, png=s)) for m, a, s in zip(metas, augs, files)],
                                [placeholder] + img_inputs[1:])
    finally:
        hook.remove()
    same_bits(seen[1], seen[0], "image encoder input from PNG bytes")
    with pytest.raises(ValueError, match="'jpeg' files"):
        model.simple_test([dict(m, img_aug=a) for m, a in zip(metas, augs)], [placeholder] + img_inputs[1:])
    assert set(out) == set(ref)
    for k in ref:
        if torch.is_tensor(ref[k]) and ref[k].is_floating_point():
            assert_close(out[k], ref[k], what=f"detector {k}")
