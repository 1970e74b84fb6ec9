"""Camera frames from their JPEG files on the H100 (image_prep.decode_jpeg, csrc/jpeg_decode.cu), bit for bit: against
cv2.imdecode (SHA-256 in tests/golden/jpeg.npz) and against the numpy restatement (oracle/jpeg.py, itself checked
against cv2); batches of mixed sizes and samplings, the tuning knobs of the parallel Huffman decode, launches, graph
replay, the output bounds, corrupt streams, argument errors; then the detector from JPEG bytes."""
import ctypes

import numpy as np
import pytest
import torch

from util import GOLDEN, assert_close, launches, rejected, same_bits
from oracle import image_prep as ip
from oracle import jpeg as oj
from occformer_b200 import image_prep, jpeg, ops

pytestmark = pytest.mark.gpu
SENT = 0xA5


def _fixture():
    return np.load(f"{GOLDEN}/jpeg.npz")


def _small(g):
    return [g[f"small_{i}_bytes"].tobytes() for i in range(len(oj.SMALL))]


def _full(g):
    """the fixture's full-size files (4:2:0; 4:2:2 with restart markers) and a high-quality 4:4:4 one encoded here"""
    return [g[f"full_{i}_bytes"].tobytes() for i in range(len(oj.FULL))] + [oj.hq_case()]


def _shas(frames):
    return [oj.sha(f.cpu().numpy()) for f in frames]


def test_fixture_frames(cuda):
    g = _fixture()
    small = _small(g)
    out = image_prep.decode_jpeg([[f] for f in small])  # 84 sizes and samplings in one call: the list form
    assert isinstance(out, list) and len(out) == len(small)
    assert _shas([o[0] for o in out]) == [str(g[f"small_{i}_sha"]) for i in range(len(small))]
    for i, (f, o) in enumerate(zip(small, out)):
        assert np.array_equal(o[0].cpu().numpy(), oj.decode(f)), f"small case {i} {oj.SMALL[i]}"
    files = _full(g)
    full = image_prep.decode_jpeg([files])  # 4:2:0, 4:2:2 with restarts, 4:4:4, one 900 x 1600 size
    assert torch.is_tensor(full) and full.shape == (1, 3, 900, 1600, 3) and full.dtype == torch.uint8
    n = len(oj.FULL)
    assert _shas(full[0, :n]) == [str(g[f"full_{i}_sha"]) for i in range(n)]
    assert np.array_equal(full[0, n].cpu().numpy(), oj.cv2_decode(files[n]))


def test_mixed_batches(cuda):
    g = _fixture()
    small, full = _small(g), _full(g)
    ref = {f: oj.cv2_decode(f) for f in small[:12] + full}
    t = image_prep.decode_jpeg([[full[0], full[1]], [full[2], full[0]]])
    assert t.shape == (2, 2, 900, 1600, 3)
    for got, f in zip(t.reshape(4, 900, 1600, 3), [full[0], full[1], full[2], full[0]]):
        assert np.array_equal(got.cpu().numpy(), ref[f])
    samples = [[small[0], small[0]], [full[1]], [small[5], small[5], small[5]]]
    lst = image_prep.decode_jpeg(samples)
    assert [tuple(x.shape) for x in lst] == [(2, 29, 37, 3), (1, 900, 1600, 3), (3, 29, 37, 3)]
    for x, s in zip(lst, samples):
        for got, f in zip(x, s):
            assert np.array_equal(got.cpu().numpy(), ref[f])
    with pytest.raises(ValueError, match="one frame size"):
        image_prep.decode_jpeg([[small[0], small[-1]]])


def _status(files, S, R):
    headers = [jpeg.parse(f) for f in files]
    offsets = np.cumsum([0] + [len(f) for f in files]).tolist()
    data = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).to("cuda")
    out, status = ops.decode_jpeg(data, offsets[:-1], headers, S, R)
    torch.cuda.synchronize()
    return out, status.cpu()


def test_tuning_does_not_change_the_result(cuda):
    g = _fixture()
    files = _small(g)[::7] + _full(g)
    ref, st = _status(files, ops.JPEG_SEQ_BITS, ops.JPEG_SYNC_ROUNDS)
    assert int(st[:, 0].abs().sum()) == 0
    for S in (32, 1024, ops.JPEG_SEQ_BITS):
        for R in (0, ops.JPEG_SYNC_ROUNDS):
            out, st = _status(files, S, R)
            assert int(st[:, 0].abs().sum()) == 0
            assert torch.equal(out, ref), f"S {S} R {R}: not bit-identical"
            if R == 0:  # every subsequence but each interval's first went through the serial fix-up
                assert bool((st[:, 1] > 0).all()), f"S {S}: the fix-up did not run"
    # short subsequences and one round: some chains have not synchronised, and the fix-up repairs them
    out, st = _status(_full(g), 32, 1)
    assert int(st[:, 0].abs().sum()) == 0 and int(st[:, 1].sum()) > 0
    assert torch.equal(out, ref[-out.numel():]), "S 32 R 1: not bit-identical"


def _raw(files, out_pad=64, S=ops.JPEG_SEQ_BITS, R=ops.JPEG_SYNC_ROUNDS):
    """the C-ABI arguments of these files -> (args, big, inner): the frames go into inner, a view of the sentinel buffer
    big with out_pad bytes on either side"""
    headers = [jpeg.parse(f) for f in files]
    offsets = np.cumsum([0] + [len(f) for f in files]).tolist()
    data = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).to("cuda")
    M = len(files)
    scan, geom, tables, out_off, total = [], [], [], [], 0
    for off, h in zip(offsets, headers):
        scan += [off + h.scan_off, h.scan_len]
        geom += [h.height, h.width, h.hs, h.vs, h.restart]
        tables += [ops._jpeg_table(data.device, *t).data_ptr() for t in h.qt + h.dc + h.ac]
        out_off.append(total)
        total += h.height * h.width * 3
    scan = (ctypes.c_longlong * (2 * M))(*scan)
    geom = (ctypes.c_int * (5 * M))(*geom)
    nbytes = ops.lib().occ_decode_jpeg_workspace_bytes(scan, geom, M, S)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    big = torch.full(((total + 2 * out_pad + 3) // 4 * 4,), SENT, dtype=torch.uint8, device="cuda")
    inner = big[out_pad:out_pad + total]
    status = torch.full((M, 2), -7, dtype=torch.int32, device="cuda")
    args = [data, data.numel(), scan, geom, (ctypes.c_longlong * (9 * M))(*tables), (ctypes.c_longlong * M)(*out_off),
            M, S, R, ws, ws.numel(), inner, inner.numel(), status]
    return args, big, inner, status


def _outside_untouched(big, inner, pad=64):
    assert bool((big[:pad] == SENT).all()) and bool((big[pad + inner.numel():] == SENT).all()), \
        "written outside the output"


def test_launch_count_is_constant(cuda):
    g = _fixture()
    small, full = _small(g), _full(g)
    counts = set()
    for files in ([small[3]], (small * 2)[:20] + full + [small[1]]):
        args, _, _, _ = _raw(files)
        counts.add(launches("occ_decode_jpeg", *args))
    assert counts == {11 + ops.JPEG_SYNC_ROUNDS}
    args, _, _, _ = _raw([small[3]], R=0)
    assert launches("occ_decode_jpeg", *args) == 11


def test_graph_replay_equals_eager(cuda):
    g = _fixture()
    files = _full(g)[:2] + _small(g)[:5]
    headers = [jpeg.parse(f) for f in files]
    offsets = np.cumsum([0] + [len(f) for f in files]).tolist()
    data = torch.from_numpy(np.frombuffer(b"".join(files), np.uint8).copy()).to(cuda)
    eager, _ = ops.decode_jpeg(data, offsets[:-1], headers)  # uploads the tables
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.decode_jpeg(data, offsets[:-1], headers)  # sizes the capture stream's workspace
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        out, status = ops.decode_jpeg(data, offsets[:-1], headers)
    torch.cuda.current_stream().wait_stream(s)
    out.fill_(SENT)
    status.fill_(-7)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager) and int(status[:, 0].abs().sum()) == 0


def test_output_bounds_untouched(cuda):
    g = _fixture()
    files = [_small(g)[i] for i in (0, 40, 60)] + [_full(g)[2]]
    args, big, inner, status = _raw(files)
    ops._call("occ_decode_jpeg", *args)
    torch.cuda.synchronize()
    _outside_untouched(big, inner)
    assert int(status[:, 0].abs().sum()) == 0
    o = 0
    for f in files:
        ref = oj.cv2_decode(f)
        assert np.array_equal(inner[o:o + ref.size].cpu().numpy().reshape(ref.shape), ref)
        o += ref.size


def _corrupt():
    """(name, file, status bit) of streams the decoder must refuse"""
    base = oj.encode(oj.content("noise", 48, 64, 3), 90, "420")
    rst = oj.encode(oj.content("noise", 48, 64, 4), 90, "420", restart=2)
    h = jpeg.parse(base)
    s0, n = h.scan_off, h.scan_len
    out = [("truncated", base[:s0 + n // 2], 8),
           ("truncated to the header", base[:s0 + 3], 8),
           ("marker inside the scan", base[:s0 + n // 2] + b"\xff\xc4" + base[s0 + n // 2:], 1),
           ("all-ones codes", base[:s0 + n // 3] + b"\xff\x00" * 12 + base[s0 + n // 3 + 24:], 4)]
    hr = jpeg.parse(rst)
    seg = rst[hr.scan_off:hr.scan_off + hr.scan_len]
    k = seg.find(b"\xff\xd0")
    out.append(("restart markers out of order", rst[:hr.scan_off + k + 1] + b"\xd3" + rst[hr.scan_off + k + 2:], 2))
    k2 = seg.find(b"\xff\xd1")
    out.append(("restart marker missing", rst[:hr.scan_off + k2] + rst[hr.scan_off + k2 + 2:], 2))
    # an AC table whose end-of-block symbol reads as (run 15, size 1): runs past coefficient 63
    i = base.find(b"\xff\xc4")
    while base[i + 4] >> 4 != 1:
        i = base.find(b"\xff\xc4", i + 2)
    counts = base[i + 5:i + 21]
    vals = bytearray(base[i + 21:i + 21 + sum(counts)])
    vals[vals.index(0x00)] = 0xF1
    out.append(("run past 63", base[:i + 21] + bytes(vals) + base[i + 21 + len(vals):], 4))
    return out


@pytest.mark.parametrize("case", range(7))
def test_corrupt_streams_raise(cuda, case):
    name, bad, bit = _corrupt()[case]
    good = oj.encode(oj.content("smooth", 48, 64, 1), 90, "420")
    with pytest.raises(ValueError, match="cam_b: corrupt entropy-coded data"):
        image_prep.decode_jpeg([[good], [bad]], names=[["cam_a"], ["cam_b"]])
    args, big, inner, status = _raw([good, bad, good])
    ops._call("occ_decode_jpeg", *args)
    torch.cuda.synchronize()
    _outside_untouched(big, inner)
    st = status.cpu()
    assert int(st[1, 0]) & bit, f"{name}: status {int(st[1, 0])}"
    assert int(st[0, 0]) == 0 and int(st[2, 0]) == 0
    ref = oj.cv2_decode(good)
    assert np.array_equal(inner[:ref.size].cpu().numpy().reshape(ref.shape), ref)
    assert np.array_equal(inner[-ref.size:].cpu().numpy().reshape(ref.shape), ref)


def test_argument_errors(cuda):
    g = _fixture()
    files = [_small(g)[0], _small(g)[30]]
    args, big, inner, status = _raw(files)
    ops._call("occ_decode_jpeg", *args)
    torch.cuda.synchronize()
    M = 2

    def bad(i, value, rc=-1):
        a, b, _, st = _raw(files)
        a[i] = value
        rejected("occ_decode_jpeg", *a, buffers=[b.view(torch.int32), st], rc=rc)

    h = [jpeg.parse(f) for f in files]
    geom = [h[0].height, h[0].width, h[0].hs, h[0].vs, h[0].restart, h[1].height, h[1].width, h[1].hs, h[1].vs, 0]
    scan = list(args[2])
    bad(1, args[2][2] + args[2][3] - 1)                                       # the last segment runs past data_bytes
    bad(2, (ctypes.c_longlong * 4)(-1, scan[1], *scan[2:]))                   # a negative segment offset
    bad(2, (ctypes.c_longlong * 4)(scan[0], 1 << 28, *scan[2:]))              # a segment of 2^28 bytes
    for k, v in ((0, 0), (1, 0), (0, 16385), (2, 3), (3, 2), (4, -1), (4, 65536)):
        gg = list(geom)
        gg[k] = v
        if k == 3:
            gg[2] = 1                                                         # sampling (1, 2)
        bad(3, (ctypes.c_int * 10)(*gg))
    bad(4, (ctypes.c_longlong * 18)(*([0] * 18)))                             # null tables
    bad(4, (ctypes.c_longlong * 18)(*[t + 2 for t in args[4]]))               # misaligned tables
    bad(5, (ctypes.c_longlong * M)(0, args[12] - 1))                          # an output past out_bytes
    bad(5, (ctypes.c_longlong * M)(-3, 0))                                    # a negative output offset
    bad(6, 0)                                                                 # M = 0
    bad(6, 97)                                                                # M above the bound
    bad(7, 31)                                                                # S below 32
    bad(7, (1 << 20) + 1)                                                     # S above 2^20
    bad(8, -1)                                                                # R < 0
    bad(8, 65)                                                                # R above 64
    bad(10, args[10] - 1)                                                     # workspace too short
    a, b, _, st = _raw(files)
    a[9] = a[9][1:]                                                           # misaligned workspace
    a[10] -= 1
    rejected("occ_decode_jpeg", *a, buffers=[b.view(torch.int32), st], rc=-1)
    assert ops.lib().occ_decode_jpeg_workspace_bytes(args[2], args[3], M, 31) == 0


def test_rejected_files_raise_on_the_host(cuda):
    import cv2
    gray = cv2.imencode(".jpg", np.zeros((16, 16), np.uint8))[1].tobytes()
    prog = cv2.imencode(".jpg", oj.content("noise", 16, 16, 0), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
    n0 = ops.LAUNCH_COUNT[0]
    for f, what in ((gray, "1-component"), (prog, "progressive")):
        with pytest.raises(ValueError, match=f"cam_x: .*{what}"):
            image_prep.decode_jpeg([[f]], names=[["cam_x"]])
    assert ops.LAUNCH_COUNT[0] == n0


# ---------------------------------------------------------------------------------------------- the detector
def test_detector_from_jpeg(cuda):
    from test_gpu_detector import detector, inputs
    model, _ = detector("nusc_r50", cuda)
    metas, img_inputs, _, _ = inputs("nusc_r50", 2, cuda)
    B, N = img_inputs[0].shape[:2]
    files = [[oj.encode(ip.frame(7000 + 10 * b + c, 900, 1600), 95, "420") for c in range(N)] for b in range(B)]
    frames = torch.from_numpy(np.stack([np.stack([oj.cv2_decode(f) for f in s]) for s in files])).to(cuda)
    augs = []
    for s in files:
        aug = [ip.test_augmentation(900, 1600, (256, 704)) for _ in s]
        augs.append(dict(resize_dims=[list(a[1]) for a in aug], crop=[list(a[2]) for a in aug], input_size=[256, 704],
                         **image_prep.norm_config(ip.NORM_R50)))
    seen = []
    hook = model.img_backbone.register_forward_pre_hook(lambda mod, args: seen.append(args[0].clone()))
    try:
        ref = model.simple_test([dict(m, img_aug=a) for m, a in zip(metas, augs)], [frames] + img_inputs[1:])
        placeholder = torch.zeros((B, N, 0), dtype=torch.uint8, device=cuda)
        out = model.simple_test([dict(m, img_aug=dict(a, jpeg=s)) for m, a, s in zip(metas, augs, files)],
                                [placeholder] + img_inputs[1:])
    finally:
        hook.remove()
    same_bits(seen[1], seen[0], "image encoder input from JPEG bytes")
    with pytest.raises(ValueError, match="'jpeg' files"):
        model.simple_test([dict(m, img_aug=a) for m, a in zip(metas, augs)], [placeholder] + img_inputs[1:])
    assert set(out) == set(ref)
    # the image encoder sees the same bits; the rest of the model is not bit-reproducible from run to run (the ASPP
    # image-pooling branch sums in fp64 atomics), so its outputs are compared as test_gpu_image_prep compares them
    for k in ref:
        if torch.is_tensor(ref[k]) and ref[k].is_floating_point():
            assert_close(out[k], ref[k], what=f"detector {k}")
