"""JPEG decoding without a GPU: the numpy restatement (oracle/jpeg.py) equals cv2.imdecode bit for bit, the host-side
parser (occformer_b200.jpeg) refuses every unsupported kind with a clear error and reads the frame size as cv2 does, and
the JPEG-bytes loader transform describes the same augmentation as the frame transform."""
import os

import numpy as np
import pytest
import torch

from oracle import jpeg as oj
from occformer_b200 import jpeg

cv2 = pytest.importorskip("cv2")


@pytest.mark.parametrize("start", range(0, len(oj.SMALL), 12))
def test_oracle_equals_cv2(start):
    for i in range(start, min(start + 12, len(oj.SMALL))):
        data = oj.small_case(i)
        assert np.array_equal(oj.decode(data), oj.cv2_decode(data)), f"case {i} {oj.SMALL[i]}"


def test_fixture_is_what_cv2_decodes():
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg.npz"))
    for i in range(len(oj.SMALL)):
        data = g[f"small_{i}_bytes"].tobytes()
        assert oj.sha(oj.cv2_decode(data)) == str(g[f"small_{i}_sha"])
        assert oj.sha(oj.decode(data)) == str(g[f"small_{i}_sha"])
    for i in range(len(oj.FULL)):
        assert oj.sha(oj.cv2_decode(g[f"full_{i}_bytes"].tobytes())) == str(g[f"full_{i}_sha"])


def test_idct_output_is_clamped_as_cv2_clamps_it(monkeypatch):
    """requantised streams push IDCT outputs to +-512 and beyond, where libjpeg's portable wrap-around table and
    clamping disagree: cv2 clamps, and so does the restatement"""
    cases = [oj.requant(oj.encode(oj.content(k, 29, 37, 1), q, s), 8)
             for q, k in ((100, "noise"), (90, "checker")) for s in oj.SAMPLINGS]
    for data in cases:
        assert np.array_equal(oj.decode(data), oj.cv2_decode(data))
    monkeypatch.setattr(oj, "range_limit", oj.range_limit_wrap)
    assert sum(not np.array_equal(oj.decode(d), oj.cv2_decode(d)) for d in cases) == len(cases)


def test_frame_size_agrees_with_cv2():
    for i in range(0, len(oj.SMALL), 5):
        data = oj.small_case(i)
        assert jpeg.frame_size(data) == oj.cv2_decode(data).shape[:2]
    h = jpeg.parse(oj.small_case(0))
    assert (h.hs, h.vs, h.restart) == (1, 1, 0)


def _base():
    return oj.encode(oj.content("noise", 16, 24, 0), 90, "420")


def _segment(data, marker):
    i = data.find(bytes([0xFF, marker]))
    assert i > 0
    return i


def _with_sof(data, **edit):
    """the file with fields of its SOF0 marker changed: precision, height, kind (the marker byte)"""
    b = bytearray(data)
    i = _segment(data, 0xC0)
    if "kind" in edit:
        b[i + 1] = edit["kind"]
    if "precision" in edit:
        b[i + 4] = edit["precision"]
    if "height" in edit:
        b[i + 5:i + 7] = edit["height"].to_bytes(2, "big")
    if "ids" in edit:  # in the SOF and the SOS marker
        j = _segment(data, 0xDA)
        for c, v in enumerate(edit["ids"]):
            b[i + 10 + 3 * c] = v
            b[j + 5 + 2 * c] = v
    return bytes(b)


def _without_app0(data):
    i = _segment(data, 0xE0)
    n = (data[i + 2] << 8) | data[i + 3]
    return data[:i] + data[i + 2 + n:]


def _before_sos(data, seg):
    i = _segment(data, 0xDA)
    return data[:i] + seg + data[i:]


def _single_component_scan(data):
    """the header with a first scan of one component (as a multi-scan baseline file starts)"""
    i = _segment(data, 0xDA)
    return data[:i] + b"\xff\xda\x00\x08\x01\x01\x00\x00\x3f\x00" + data[i + 14:]


REJECTED = {
    "progressive": (lambda: cv2.imencode(".jpg", oj.content("noise", 16, 16, 0), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1]
                    .tobytes(), "progressive"),
    "grayscale": (lambda: cv2.imencode(".jpg", np.zeros((16, 16), np.uint8))[1].tobytes(), "1-component"),
    "411": (lambda: oj.encode(oj.content("noise", 16, 32, 0), 90, "420")[:0] + cv2.imencode(
        ".jpg", oj.content("noise", 16, 32, 0), [cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                                  cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411])[1].tobytes(), "sampling"),
    "440": (lambda: cv2.imencode(".jpg", oj.content("noise", 16, 32, 0), [
        cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440])[1].tobytes(), "sampling"),
    "12-bit": (lambda: _with_sof(_base(), precision=12), "12-bit samples"),
    "lossless": (lambda: _with_sof(_base(), kind=0xC3), "lossless"),
    "arithmetic": (lambda: _with_sof(_base(), kind=0xC9), "arithmetic"),
    "arithmetic conditioning": (lambda: _before_sos(_base(), b"\xff\xcc\x00\x04\x00\x10"), "arithmetic"),
    "height from DNL": (lambda: _with_sof(_base(), height=0), "DNL"),
    "DNL marker": (lambda: _before_sos(_base(), b"\xff\xdc\x00\x04\x00\x10"), "DNL"),
    "multi-scan": (lambda: _single_component_scan(_base()), "multi-scan"),
    "Adobe RGB": (lambda: _before_sos(_base(), b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00"), "Adobe transform 0"),
    "RGB ids": (lambda: _with_sof(_without_app0(_base()), ids=(82, 71, 66)), "'R', 'G', 'B'"),
    "not a JPEG": (lambda: b"\x89PNG\r\n\x1a\n" + bytes(64), "no SOI"),
    "no scan": (lambda: _base()[:_segment(_base(), 0xDA)], "ends before the scan"),
}


@pytest.mark.parametrize("kind", list(REJECTED))
def test_parser_rejects(kind):
    make, what = REJECTED[kind]
    with pytest.raises(ValueError, match=what):
        jpeg.parse(make())


def test_parser_accepts_what_it_should():
    base = _base()
    assert jpeg.frame_size(_before_sos(base, b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x01")) == (16, 24)
    assert jpeg.frame_size(_with_sof(base, kind=0xC1)) == (16, 24)          # SOF1 with 8-bit samples
    assert jpeg.frame_size(_with_sof(base, ids=(82, 71, 66))) == (16, 24)   # JFIF: YCbCr whatever the ids
    h = jpeg.parse(oj.encode(oj.content("noise", 40, 24, 0), 90, "422", restart=3))
    assert (h.height, h.width, h.hs, h.vs, h.restart) == (40, 24, 2, 1, 3)
    data = oj.encode(oj.content("noise", 40, 24, 0), 90, "420")
    h = jpeg.parse(data)
    assert data[h.scan_off + h.scan_len:] == b"\xff\xd9"


def test_huffman_table_matches_the_canonical_codes():
    data = oj.small_case(1)
    _, _, ht, _, _, _ = oj._markers(data)
    for (tc, th), (counts, values) in ht.items():
        t = jpeg.huff_table(counts, values, tc == 0)
        for (length, code), sym in oj._codes(counts, values).items():
            if length <= jpeg.LOOKAHEAD:
                e = t[code << (jpeg.LOOKAHEAD - length)]
                assert (e >> 8, e & 255) == (length, sym)
            else:
                assert t[512 + length] >= code and t[547 + code + t[530 + length]] == sym
    with pytest.raises(ValueError, match="overflow"):
        jpeg.huff_table([2] + [0] * 15, [0, 1], True)
    with pytest.raises(ValueError, match="DC symbol"):
        jpeg.huff_table([1] + [0] * 15, [16], True)


def test_jpeg_bytes_transform_matches_the_frame_transform(tmp_path):
    from oracle import image_prep as ip
    from occformer_b200.pipelines import LoadMultiViewImageFrames_OccFormer, LoadMultiViewJpegBytes_OccFormer
    frames = [ip.frame(40 + c, 90, 160) for c in range(2)]
    paths = []
    for c, f in enumerate(frames):
        p = tmp_path / f"cam{c}.jpg"
        p.write_bytes(oj.encode(f, 95, "420"))
        paths.append(str(p))
    cams = ip.NUSC_CAMS[:2]
    cal = [ip.calib(c) for c in range(2)]

    def results():
        return dict(curr=dict(cams={cam: dict(data_path=p, cam_intrinsic=cal[c][0].tolist())
                                    for c, (cam, p) in enumerate(zip(cams, paths))}),
                    lidar2cam_dic={cam: cal[c][1].tolist() for c, cam in enumerate(cams)})

    kw = dict(data_config=ip.data_config((48, 72), cams), img_norm_cfg=ip.NORM_R50)
    ref = LoadMultiViewImageFrames_OccFormer(**kw)(results())
    got = LoadMultiViewJpegBytes_OccFormer(**kw)(results())
    aug = dict(got["img_aug"])
    assert aug.pop("jpeg") == [open(p, "rb").read() for p in paths] and aug.pop("jpeg_files") == paths
    assert aug == ref["img_aug"]
    assert got["img_inputs"][0].dtype == torch.uint8 and tuple(got["img_inputs"][0].shape) == (2, 0)
    assert len(got["img_inputs"]) == len(ref["img_inputs"])
    for a, b in zip(got["img_inputs"][1:], ref["img_inputs"][1:]):
        assert torch.equal(a, b)
    with pytest.raises(ValueError, match="is_train"):
        LoadMultiViewJpegBytes_OccFormer(is_train=True, **kw)
    (tmp_path / "cam0.jpg").write_bytes(cv2.imencode(".jpg", frames[0], [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes())
    with pytest.raises(ValueError, match="cam0.jpg: progressive"):
        LoadMultiViewJpegBytes_OccFormer(**kw)(results())
