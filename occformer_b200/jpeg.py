"""JPEG headers on the host, for the device decoder of csrc/jpeg_decode.cu (ops.decode_jpeg, image_prep.decode_jpeg).

The camera files of the nuScenes loader are baseline JPEGs that the reference decodes with cv2.imdecode (mmcv.imread's
cv2 backend, libjpeg-turbo).  This module reads the markers of one file and refuses, with a ValueError naming the
feature, everything the device decoder does not implement:

    accepted   SOF0, or SOF1 with 8-bit samples; Huffman coding; three components Y, Cb, Cr (JFIF, an Adobe marker with
               transform 1, or neither with component ids other than 'R', 'G', 'B'); luma sampling 1x1, 2x1 or 2x2 with
               chroma 1x1 (4:4:4, 4:2:2, 4:2:0); one interleaved scan of all three components in frame order, Ss = 0,
               Se = 63, Ah = Al = 0; 8- and 16-bit quantisation tables; any restart interval; sides up to MAX_SIDE.
    refused    progressive, lossless, hierarchical and arithmetic-coded frames, 12- and 16-bit samples, grayscale, CMYK,
               RGB (Adobe transform 0), other samplings, a first scan of fewer components (multi-scan files), a frame
               height of 0 (height from a DNL marker), DNL itself.

Markers after the first scan are not read: the entropy-coded segment runs from the end of the SOS header to the last
EOI marker of the file, or to the end of the file when it has none, and the device rejects any marker other than RSTn
inside it.  EXIF orientation is ignored, as cv2.IMREAD_UNCHANGED ignores it.

The Huffman tables are handed to the device in a flat int32 form (HUFF_INTS entries, see huff_table), the quantisation
tables as 64 int32 in natural order.  Both are keyed by their marker bytes so that ops caches each distinct table once.
"""
import numpy as np

MAX_SIDE = 16384              # largest accepted width and height
MAX_FILE = 1 << 28            # largest accepted file: bit positions of a scan stay below 2^31
LOOKAHEAD = 9                 # bits of the device's first-level Huffman lookup
HUFF_INTS = 804               # lookup[512] | maxcode[18] | valoff[17] | huffval[256] | pad

# natural (row-major) index of the k-th zig-zag coefficient, ITU T.81 figure A.6
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63], dtype=np.int32)

_SOF_KINDS = {0xC2: "progressive (SOF2)", 0xC3: "lossless (SOF3)", 0xC5: "differential sequential (SOF5)",
              0xC6: "differential progressive (SOF6)", 0xC7: "differential lossless (SOF7)",
              0xC9: "arithmetic-coded sequential (SOF9)", 0xCA: "arithmetic-coded progressive (SOF10)",
              0xCB: "arithmetic-coded lossless (SOF11)", 0xCD: "arithmetic-coded differential (SOF13)",
              0xCE: "arithmetic-coded differential progressive (SOF14)",
              0xCF: "arithmetic-coded differential lossless (SOF15)"}


class JpegError(ValueError):
    pass


class Header:
    """what the device needs of one file: size, sampling, tables and the entropy-coded segment"""
    __slots__ = ("height", "width", "hs", "vs", "restart", "scan_off", "scan_len", "qt", "dc", "ac")

    @property
    def mcus(self):
        return -(-self.width // (8 * self.hs)), -(-self.height // (8 * self.vs))


def huff_table(counts, values, is_dc):
    """DHT counts (16 code lengths) and values -> the flat int32 table of the device decoder:
    [0, 512)    lookup of the next 9 bits: length << 8 | symbol, or 0 for a longer code
    [512, 530)  maxcode[l], l = 0..17: the largest code of length l, -1 if none
    [530, 547)  valoff[l]: index in huffval of the first code of length l, minus that code
    [547, 803)  huffval
    The code assignment is ITU T.81 Annex C; a table whose codes overflow their length (or that would assign the
    all-ones code) is refused, as libjpeg refuses it."""
    counts = [int(c) for c in counts]
    values = [int(v) for v in values]
    if sum(counts) > 256 or sum(counts) != len(values):
        raise JpegError("bad Huffman table: more than 256 codes")
    if is_dc and any(v > 15 for v in values):
        raise JpegError("bad Huffman table: DC symbol above 15")
    t = np.zeros(HUFF_INTS, np.int32)
    maxcode = t[512:530]
    valoff = t[530:547]
    maxcode[:] = -1
    code, k = 0, 0
    for length in range(1, 17):
        n = counts[length - 1]
        if n:
            valoff[length] = k - code
            for _ in range(n):
                if length <= LOOKAHEAD:
                    lo = code << (LOOKAHEAD - length)
                    t[lo:lo + (1 << (LOOKAHEAD - length))] = (length << 8) | values[k]
                code += 1
                k += 1
            maxcode[length] = code - 1
        if code >= (1 << length):
            raise JpegError("bad Huffman table: codes overflow their length")
        code <<= 1
    t[547:547 + len(values)] = values
    return t


_huff_cache = {}  # DHT bytes (class, id, counts, values) -> huff_table


def _u16(data, i):
    return (data[i] << 8) | data[i + 1]


def parse(data):
    """file bytes (bytes-like) -> Header; JpegError (a ValueError) for anything the decoder does not take"""
    raw = data if isinstance(data, (bytes, bytearray)) else bytes(data)
    data = memoryview(raw).cast("B")
    n = len(data)
    if n > MAX_FILE:
        raise JpegError(f"file of {n} bytes is above the {MAX_FILE}-byte bound")
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise JpegError("not a JPEG file (no SOI marker)")
    qts, dcs, acs = {}, {}, {}
    frame = None
    restart = 0
    jfif = adobe = False
    transform = None
    i = 2
    while True:
        if i < n and data[i] != 0xFF:
            raise JpegError(f"garbage where a marker should be, at byte {i}")
        while i < n and data[i] == 0xFF:
            i += 1
        if i >= n:
            raise JpegError("file ends before the scan")
        m = data[i]
        i += 1
        if m == 0xD8 or 0xD0 <= m <= 0xD7 or m == 0x01:
            continue
        if m == 0xD9:
            raise JpegError("EOI before any scan")
        if i + 2 > n:
            raise JpegError("file ends inside a marker")
        seg = _u16(data, i)
        if seg < 2 or i + seg > n:
            raise JpegError(f"marker 0xFF{m:02X} has a bad length")
        body = data[i + 2:i + seg]
        i += seg
        if m in _SOF_KINDS:
            raise JpegError(f"{_SOF_KINDS[m]} JPEG is not supported (baseline or extended sequential Huffman only)")
        if m in (0xC0, 0xC1):
            if frame is not None:
                raise JpegError("more than one SOF marker")
            if len(body) < 6:
                raise JpegError("short SOF marker")
            prec, H, W, nc = body[0], _u16(body, 1), _u16(body, 3), body[5]
            if prec != 8:
                raise JpegError(f"{prec}-bit samples are not supported (8-bit only)")
            if nc != 3:
                raise JpegError(f"{nc}-component JPEG is not supported (three components, YCbCr, only)")
            if len(body) != 6 + 3 * nc:
                raise JpegError("bad SOF length")
            if H == 0:
                raise JpegError("frame height 0 (height from a DNL marker) is not supported")
            if W == 0:
                raise JpegError("frame width 0")
            if H > MAX_SIDE or W > MAX_SIDE:
                raise JpegError(f"{W} x {H} frame is above the {MAX_SIDE}-pixel bound per side")
            comps = [(body[6 + 3 * c], body[7 + 3 * c] >> 4, body[7 + 3 * c] & 15, body[8 + 3 * c]) for c in range(3)]
            frame = (H, W, comps)
        elif m == 0xC4:
            j = 0
            while j < len(body):
                if j + 17 > len(body):
                    raise JpegError("short DHT marker")
                tc, th = body[j] >> 4, body[j] & 15
                counts = list(body[j + 1:j + 17])
                total = sum(counts)
                if tc > 1 or th > 3 or j + 17 + total > len(body):
                    raise JpegError("bad DHT marker")
                key = bytes(body[j:j + 17 + total])
                if key not in _huff_cache:
                    _huff_cache[key] = huff_table(counts, body[j + 17:j + 17 + total], tc == 0)
                (dcs if tc == 0 else acs)[th] = (key, _huff_cache[key])
                j += 17 + total
        elif m == 0xCC:
            raise JpegError("arithmetic coding (DAC marker) is not supported")
        elif m == 0xDB:
            j = 0
            while j < len(body):
                pq, tq = body[j] >> 4, body[j] & 15
                size = 64 * (pq + 1)
                if pq > 1 or tq > 3 or j + 1 + size > len(body):
                    raise JpegError("bad DQT marker")
                vals = np.frombuffer(bytes(body[j + 1:j + 1 + size]), np.uint8 if pq == 0 else ">u2").astype(np.int32)
                q = np.zeros(64, np.int32)
                q[ZIGZAG] = vals
                qts[tq] = (bytes(body[j:j + 1 + size]), q)
                j += 1 + size
        elif m == 0xDD:
            if len(body) != 2:
                raise JpegError("bad DRI marker")
            restart = _u16(body, 0)
        elif m == 0xDC:
            raise JpegError("DNL marker is not supported")
        elif m == 0xE0:
            jfif = jfif or bytes(body[:5]) == b"JFIF\0"
        elif m == 0xEE:
            if bytes(body[:5]) == b"Adobe" and len(body) >= 12:
                adobe, transform = True, body[11]
        elif m == 0xDA:
            if frame is None:
                raise JpegError("SOS before SOF")
            H, W, comps = frame
            ns = body[0] if len(body) else 0
            if ns != 3:
                raise JpegError(f"a first scan of {ns} component(s) (multi-scan JPEG) is not supported")
            if len(body) != 4 + 2 * ns:
                raise JpegError("bad SOS length")
            ids = [body[1 + 2 * c] for c in range(3)]
            if ids != [c[0] for c in comps]:
                raise JpegError("scan components out of frame order are not supported")
            ss, se, ahal = body[7], body[8], body[9]
            if ss != 0 or se != 63 or ahal != 0:
                raise JpegError("a sequential scan needs Ss = 0, Se = 63, Ah = Al = 0")
            if adobe and transform == 0:
                raise JpegError("RGB / CMYK JPEG (Adobe transform 0) is not supported (YCbCr only)")
            if not jfif and not adobe and ids == [82, 71, 66]:
                raise JpegError("RGB JPEG (component ids 'R', 'G', 'B') is not supported (YCbCr only)")
            (_, hs, vs, _), c1, c2 = comps
            if (hs, vs) not in ((1, 1), (2, 1), (2, 2)) or c1[1:3] != (1, 1) or c2[1:3] != (1, 1):
                raise JpegError(f"sampling {[c[1:3] for c in comps]} is not supported (4:4:4, 4:2:2, 4:2:0 only)")
            h = Header()
            h.height, h.width, h.hs, h.vs, h.restart = H, W, hs, vs, restart
            h.qt, h.dc, h.ac = [], [], []
            for c in range(3):
                td, ta = body[2 + 2 * c] >> 4, body[2 + 2 * c] & 15
                tq = comps[c][3]
                if tq not in qts:
                    raise JpegError(f"component {c} uses undefined quantisation table {tq}")
                if td not in dcs or ta not in acs:
                    raise JpegError(f"component {c} uses an undefined Huffman table")
                h.qt.append(qts[tq])
                h.dc.append(dcs[td])
                h.ac.append(acs[ta])
            h.scan_off = i
            end = raw.rfind(b"\xff\xd9", i)
            h.scan_len = (n if end < 0 else end) - i
            return h
        # APPn, COM and any other marker with a length: skipped


def frame_size(data):
    """(H, W) of a JPEG file from its SOF marker (the file is checked as parse checks it)"""
    h = parse(data)
    return h.height, h.width
