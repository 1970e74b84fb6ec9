"""PNG decoding without a GPU: the host-side parser (occformer_b200.png) accepts and refuses each kind of file with cv2's
verdict beside it, cv2's edge cases are pinned, the restatement (oracle/png.py) equals cv2 and zlib on the fixture and
on writer-generated files, the scan predicate accepts every true dynamic block start, the loader transform, and the
header entry."""
import os
import struct
import zlib

import numpy as np
import pytest

from oracle import png as op
from occformer_b200 import png

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "png.npz")
cv2 = pytest.importorskip("cv2")


def _fixture():
    g = np.load(GOLDEN)
    return [(str(g[f"name_{i}"]), g[f"file_{i}"].tobytes(), str(g[f"sha_{i}"])) for i in range(int(g["count"]))]


def _flip(stream):
    return stream[:-4] + struct.pack(">I", struct.unpack(">I", stream[-4:])[0] ^ 1)


def test_fixture_is_cv2s_decode_of_the_written_pixels():
    g = np.load(GOLDEN)
    assert str(g["opencv"]) and str(g["libpng"])
    for (name, f, sha), src in zip(_fixture(), op.small_files() + [(n, None) for n in range(3)]):
        dec = op.cv2_decode(f)
        assert op.sha(dec) == sha, name
        assert png.frame_size(f) == dec.shape[:2]
        if src[1] is not None:
            assert src[1] == f, f"{name}: the writer no longer reproduces the fixture"


@pytest.mark.parametrize("level", [0, 1, 6, 9])
@pytest.mark.parametrize("strategy", sorted(op.STRATEGIES))
def test_cv2_decodes_the_writers_pixels_in_bgr(level, strategy):
    src = op.content(21, 34, level * 7 + len(strategy))
    f = op.write(src, level=level, strategy=strategy, idat=[7, 1, 50])
    assert np.array_equal(op.cv2_decode(f), src)
    assert np.array_equal(op.decode(f), src)


def test_oracle_against_zlib_and_cv2_on_the_fixture():
    for name, f, sha in _fixture():
        s = op.idat_stream(f)
        blocks, raw, _ = op.walk(s)
        assert raw == zlib.decompress(s), name
        assert op.adler32(raw) == zlib.adler32(raw)
        assert op.sha(op.decode(f)) == sha, name
        assert sum(b["out"] for b in blocks) == len(raw) and blocks[-1]["final"] == 1
    kinds = {b["type"] for _, f, _ in _fixture() for b in op.walk(op.idat_stream(f))[0]}
    assert kinds == {0, 1, 2}


def test_predicate_accepts_every_true_dynamic_block_start():
    total_bits, false = 0, 0
    for name, f, _ in _fixture():
        s = op.idat_stream(f)
        blocks, _, _ = op.walk(s)
        cand = set(op.candidates(s))
        bits = op.Bits(s[2:])
        for b in blocks:
            if b["type"] == 2:
                assert b["start"] in cand, f"{name}: dynamic block at bit {b['start']} not found"
                assert op.dynamic_header_ok(bits, b["start"])
        true = {b["start"] for b in blocks if b["type"] == 2}
        false += len(cand - true)
        total_bits += 8 * len(s)
    print(f"false candidates: {false} in {total_bits / 8e6:.2f} MB ({false / (total_bits / 8e6):.0f} per MB)")


# ---------------------------------------------------------------------------------------------- the parser
def _ihdr(W=8, H=4, depth=8, colour=2, interlace=0):
    return struct.pack(">IIBBBBB", W, H, depth, colour, 0, 0, interlace)


def _base(H=4, W=8, **kw):
    src = op.content(H, W, 3)
    raw = op.filter_rows(src[..., ::-1], [0] * H).tobytes()
    return src, zlib.compress(raw)


def _zhead(cmf, flags):
    """a zlib header with CMF cmf and FLG flags | the FCHECK that makes it valid"""
    return bytes([cmf, flags | (31 - ((cmf << 8) | flags) % 31) % 31])


def _cv2_refuses_or_other(f):
    d = op.cv2_decode(f)
    return d is None or d.ndim != 3 or d.shape[2] != 3 or d.dtype != np.uint8


REFUSED = [
    ("16-bit", lambda s: op.assemble(4, 8, zlib.compress(bytes(4 * (1 + 48))), ihdr=_ihdr(depth=16)), "bit depth 16"),
    ("grayscale", lambda s: op.assemble(4, 8, zlib.compress(bytes(4 * 9)), ihdr=_ihdr(colour=0)), "grayscale"),
    ("gray+alpha", lambda s: op.assemble(4, 8, zlib.compress(bytes(4 * 17)), ihdr=_ihdr(colour=4)), "grayscale \\+ alpha"),
    ("RGBA", lambda s: op.assemble(4, 8, zlib.compress(bytes(4 * 33)), ihdr=_ihdr(colour=6)), "RGBA"),
    ("palette", lambda s: op.assemble(4, 8, zlib.compress(bytes(4 * 9)), ihdr=_ihdr(colour=3),
                                      ancillary=[(b"PLTE", bytes(3))]), "palette"),
    ("tRNS", lambda s: op.assemble(4, 8, s, ancillary=[(b"tRNS", b"\0\1\0\2\0\3")]), "tRNS"),
    ("interlaced", lambda s: op.assemble(4, 8, s, ihdr=_ihdr(interlace=1)), "Adam7"),
    ("APNG", lambda s: op.assemble(4, 8, s, ancillary=[(b"acTL", struct.pack(">II", 1, 0))]), "APNG"),
    ("CM 7", lambda s: op.assemble(4, 8, _zhead(0x77, 0) + s[2:]), "method"),
    ("CINFO 8", lambda s: op.assemble(4, 8, _zhead(0x88, 0) + s[2:]), "CINFO"),
    ("bad FCHECK", lambda s: op.assemble(4, 8, bytes([s[0], s[1] ^ 1]) + s[2:]), "FCHECK"),
    ("FDICT", lambda s: op.assemble(4, 8, _zhead(0x78, 0x20) + b"\0\0\0\1" + s[2:]), "FDICT"),
    ("no IDAT", lambda s: op.assemble(4, 8, b""), "IDAT missing"),
    ("bad IDAT CRC", lambda s: (lambda f: f[:f.find(b"IDAT") + 4 + len(s)] + bytes([f[f.find(b"IDAT") + 4 + len(s)] ^ 1])
                                + f[f.find(b"IDAT") + 5 + len(s):])(op.assemble(4, 8, s)), "bad CRC"),
    ("no IEND", lambda s: op.assemble(4, 8, s, iend=False), "IEND"),
]


@pytest.mark.parametrize("case", REFUSED, ids=lambda r: r[0])
def test_refused_files(case):
    name, make, what = case
    _, s = _base()
    f = make(s)
    with pytest.raises(png.PngError, match=what):
        png.parse(f)
    # cv2 expands a palette file to B, G, R and shows an APNG's default image; both are out of the device's scope
    assert _cv2_refuses_or_other(f) == (name not in ("palette", "APNG")), f"{name}: cv2's verdict changed"


def test_idat_chunks_apart_are_refused():
    src, s = _base()
    f = op.assemble(4, 8, s, idat=[3, len(s)])
    i = f.find(b"IDAT", f.find(b"IDAT") + 4) - 4
    g = f[:i] + op.chunk(b"tEXt", b"a\0b") + f[i:]
    with pytest.raises(png.PngError, match="not consecutive"):
        png.parse(g)
    assert op.cv2_decode(g) is None


def test_ignored_chunks():
    src, s = _base()
    anc = [(b"gAMA", struct.pack(">I", 45455)), (b"sRGB", b"\0"), (b"iCCP", b"x\0\0" + zlib.compress(b"profile")),
           (b"sBIT", b"\x08\x08\x08"), (b"pHYs", struct.pack(">IIB", 1, 1, 1)), (b"tEXt", b"k\0v"),
           (b"tIME", struct.pack(">HBBBBB", 2026, 1, 1, 0, 0, 0)), (b"PLTE", bytes(range(12)))]
    f = op.assemble(4, 8, s, ancillary=anc)
    assert png.frame_size(f) == (4, 8)
    f = bytearray(f)
    i = f.find(b"gAMA")
    f[i + 4] ^= 1  # a bad CRC on an ancillary chunk
    f = bytes(f)
    assert png.parse(f).stream_len == len(s)
    assert np.array_equal(op.cv2_decode(f), src)


def test_cv2_edge_cases():
    """what cv2.imdecode (OpenCV 4.13.0, libpng 1.6.53) returns: the device decoder follows these verdicts"""
    H, W = 20, 30
    src = op.content(H, W, 1)
    raw = op.filter_rows(src[..., ::-1], [y % 5 for y in range(H)]).tobytes()
    s = zlib.compress(raw)
    none = {"wrong Adler-32": op.assemble(H, W, _flip(s)),
            "cut before the trailer": op.assemble(H, W, s[:-4]),
            "truncated": op.assemble(H, W, s[:len(s) // 2]),
            "too little image data": op.assemble(H, W, zlib.compress(raw[:-5])),
            "filter type 5": op.assemble(H, W, zlib.compress(raw[:3 * (1 + 3 * W)] + b"\x05" + raw[3 * (1 + 3 * W) + 1:])),
            "no IEND": op.assemble(H, W, s, iend=False)}
    for name, f in none.items():
        assert op.cv2_decode(f) is None, name
    extra = zlib.compress(raw + bytes(50))
    same = {"too much image data": op.assemble(H, W, extra),
            "too much image data and a wrong Adler-32": op.assemble(H, W, _flip(extra)),
            "bytes after the stream": op.assemble(H, W, s + b"junk"),
            "wrong Adler-32 read after the rows (trailer in its own IDAT)": op.assemble(H, W, _flip(s),
                                                                                      idat=[len(s) - 4, 4]),
            "wrong Adler-32 read after the rows (1-byte IDATs)": op.assemble(H, W, _flip(s), idat=1)}
    for name, f in same.items():
        assert np.array_equal(op.cv2_decode(f), src), name
    # libpng reads an IDAT chunk 8192 bytes at a time: a wrong Adler-32 fails only when its trailer arrives in the same
    # read as the last row's bytes
    row = np.random.default_rng(0).integers(0, 256, (1, 2728, 3), dtype=np.uint8)
    st = zlib.compress(op.filter_rows(row[..., ::-1], [0]).tobytes(), 0)
    assert len(st) == 8196  # the last row byte at 8191, the trailer at 8192..8195
    assert op.cv2_decode(op.assemble(1, 2728, _flip(st))) is not None
    assert op.cv2_decode(op.assemble(1, 2728, _flip(st), idat=[8000, 8000])) is None


def test_cv2_verdicts_on_the_device_tests_files():
    """every corrupt file of the GPU tests is refused by cv2, every defective file they expect decoded is decoded to
    its source pixels; an invalid code right after the last row's byte fails (zlib decodes it in the call that fills
    the last row), one literal later it does not (zlib stops for want of output first)"""
    for name, f, _ in op.corrupt_files():
        png.parse(f)
        assert op.cv2_decode(f) is None, name
    for name, f, src in op.benign_files():
        png.parse(f)
        assert np.array_equal(op.cv2_decode(f), src), name


def test_parser_takes_only_streams_the_device_takes():
    src, s = _base()
    f = op.assemble(4, 8, s, idat=[5, 0, 0, 3, 0, len(s)])
    h = png.parse(f)  # the empty IDAT chunks are dropped
    assert [n for _, n in h.idat] == [5, 3, len(s) - 8] and h.stream_len == len(s)
    for n in (2, 6):
        f = op.assemble(4, 8, s[:n])
        with pytest.raises(png.PngError, match="too short"):
            png.parse(f)
        assert op.cv2_decode(f) is None
    assert png.MAX_STREAM == (1 << 27) - 1  # occ_decode_png takes streams below 2^27 bytes


# ---------------------------------------------------------------------------------------------- the transform
def test_png_bytes_transform_matches_the_frame_transform(tmp_path):
    from occformer_b200.pipelines import LoadMultiViewImageFrames_SemanticKitti, LoadMultiViewPngBytes_SemanticKitti
    _, f, _ = _fixture()[-1]
    path = str(tmp_path / "000000.png")
    open(path, "wb").write(f)
    cfg = dict(data_config=dict(input_size=(384, 1280), resize=(0.0, 0.0), rot=(0.0, 0.0), flip=False,
                                crop_h=(0.0, 0.0), resize_test=0.0, cams=["cam0"], Ncams=1, src_size=(376, 1241)))

    def results():
        return dict(img_filename=[path], cam_intrinsic=[np.eye(3).tolist()], lidar2cam=[np.eye(4).tolist()])

    ref = LoadMultiViewImageFrames_SemanticKitti(**cfg)(results())
    got = LoadMultiViewPngBytes_SemanticKitti(**cfg)(results())
    assert "raw_img" in ref and "raw_img" not in got
    assert got["img_inputs"][0].shape == (1, 0) and got["img_inputs"][0].dtype.is_floating_point is False
    for a, b in zip(ref["img_inputs"][1:], got["img_inputs"][1:]):
        assert a.shape == b.shape and bool((a == b).all())
    aug = dict(got["img_aug"])
    assert aug.pop("png") == [f] and aug.pop("png_files") == [path]
    assert aug == ref["img_aug"]
    bad = str(tmp_path / "rgba.png")
    open(bad, "wb").write(op.assemble(4, 8, zlib.compress(bytes(4 * 33)), ihdr=_ihdr(colour=6)))
    with pytest.raises(ValueError, match="rgba.png: RGBA"):
        LoadMultiViewPngBytes_SemanticKitti(**cfg)(dict(results(), img_filename=[bad]))
    with pytest.raises(ValueError, match="is_train"):
        LoadMultiViewPngBytes_SemanticKitti(is_train=True, **cfg)


def test_header_entry_is_bound_and_checked():
    from occformer_b200._lib import parameters
    p = dict(parameters())
    assert [n for n, _ in p["occ_decode_png"]] == ["data", "data_bytes", "streams", "geom", "idat_counts", "idat",
                                                   "idat_len", "out_offsets", "M", "ws", "ws_bytes", "out",
                                                   "out_bytes", "status", "stream"]
    assert dict(p["occ_decode_png"])["idat"] == "int" and dict(p["occ_decode_png"])["out"] == "unsigned char"
    assert [n for n, _ in p["occ_decode_png_workspace_bytes"]] == ["streams", "geom", "idat_counts", "M"]
