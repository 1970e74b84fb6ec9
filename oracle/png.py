"""TEST INFRASTRUCTURE ONLY (oracle) -- 8-bit RGB PNG decoding as cv2.imdecode(buf, IMREAD_UNCHANGED) does it (mmcv.imread's
cv2 backend, which the reference's LoadMultiViewImageFromFiles_SemanticKitti calls), restated in Python and numpy from
RFC 1950 (zlib), RFC 1951 (DEFLATE) and the PNG specification (ISO/IEC 15948):

    blocks       walk(stream): every DEFLATE block's start bit, type, BFINAL and output length, by a serial decode
    predicate    dynamic_header_ok(bits, pos): could a dynamic-Huffman block start at bit pos?  zlib's own
                 validity rules (HLIT, HDIST <= 29, complete code-length code, no repeat past the end, complete
                 literal/length and distance codes or zlib's one-code exception, a nonzero length for code 256) -- the
                 test of the device's scan pass
    Adler-32     adler32(data)
    unfilter     unfilter(raw, H, W): the five filter types of PNG section 9, -> (H, W, 3) R, G, B

The inflated bytes themselves are checked against Python's zlib, the library libpng uses.  write() is the test-side
writer (numpy + zlib): each row's filter, the zlib level and strategy, the IDAT split and ancillary chunks are chosen
by the caller.

    python -m oracle.png gen     # tests/golden/png.npz
"""
import hashlib
import os
import struct
import zlib

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "png.npz")
SIGNATURE = b"\x89PNG\r\n\x1a\n"
STRATEGIES = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman": zlib.Z_HUFFMAN_ONLY,
              "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}

# RFC 1951 3.2.5: base and extra bits of the length codes 257..285 and the distance codes 0..29
LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227,
            258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097,
             6145, 8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [k for k in range(1, 14) for _ in range(2)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


# =============================================================================
# chunks and the writer
# =============================================================================
def chunk(kind, body, crc=None):
    c = zlib.crc32(kind + body) if crc is None else crc
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", c & 0xFFFFFFFF)


def filter_rows(rgb, filters):
    """(H, W, 3) uint8 R, G, B and one filter type (0..4) per row -> the filtered bytes H * (1 + 3W)"""
    H, W, _ = rgb.shape
    x = rgb.reshape(H, 3 * W).astype(np.int32)
    out = np.zeros((H, 1 + 3 * W), np.uint8)
    for y in range(H):
        f = int(filters[y])
        cur = x[y]
        up = x[y - 1] if y > 0 else np.zeros_like(cur)
        left = np.concatenate([np.zeros(3, np.int32), cur[:-3]])
        ul = np.concatenate([np.zeros(3, np.int32), up[:-3]])
        if f == 0:
            pred = np.zeros_like(cur)
        elif f == 1:
            pred = left
        elif f == 2:
            pred = up
        elif f == 3:
            pred = (left + up) >> 1
        else:
            pred = paeth(left, up, ul)
        out[y, 0] = f
        out[y, 1:] = (cur - pred) & 0xFF
    return out.reshape(-1)


def paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def write(bgr, filters=None, level=6, strategy="default", idat=None, ancillary=(), wbits=15):
    """(H, W, 3) uint8 B, G, R (cv2's order) -> PNG bytes, 8-bit RGB.  filters: one type per row, or an int for all
    rows (default: row y gets y % 5); level 0 writes stored blocks; idat: None (one chunk), an int (chunks of that many
    bytes) or a list of chunk sizes, the last repeated; ancillary: (chunk type, body) pairs written before IDAT"""
    H, W, _ = bgr.shape
    if filters is None:
        filters = [y % 5 for y in range(H)]
    elif isinstance(filters, int):
        filters = [filters] * H
    raw = filter_rows(bgr[..., ::-1], filters).tobytes()
    co = zlib.compressobj(level, zlib.DEFLATED, wbits, 8, STRATEGIES[strategy])
    return assemble(H, W, co.compress(raw) + co.flush(), idat, ancillary)


def assemble(H, W, stream, idat=None, ancillary=(), ihdr=None, iend=True):
    """the chunks of a PNG around one zlib stream (see write)"""
    body = ihdr if ihdr is not None else struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)
    out = [SIGNATURE, chunk(b"IHDR", body)]
    out += [chunk(k, b) for k, b in ancillary]
    sizes = [len(stream)] if idat is None else ([idat] if isinstance(idat, int) else list(idat))
    i, k = 0, 0
    while i < len(stream):
        n = sizes[min(k, len(sizes) - 1)]
        out.append(chunk(b"IDAT", stream[i:i + n]))
        i += n
        k += 1
    if iend:
        out.append(chunk(b"IEND", b""))
    return b"".join(out)


def idat_stream(data):
    """the concatenated IDAT payloads of a PNG"""
    i, out = 8, []
    while i + 8 <= len(data):
        n = struct.unpack(">I", data[i:i + 4])[0]
        if data[i + 4:i + 8] == b"IDAT":
            out.append(data[i + 8:i + 8 + n])
        i += 12 + n
    return b"".join(out)


def fixed_block(literals, tail=()):
    """a zlib stream of one final fixed-Huffman block: the bytes literals as literal codes, then tail, a list of
    (code, bits) written MSB first as Huffman codes are (e.g. (0b11000110, 8), the invalid literal/length code 286),
    then end-of-block and a zero Adler-32 -- for streams no encoder writes"""
    bits = [1, 1, 0]
    for v in literals:
        code, n = (0x30 + v, 8) if v < 144 else (0x190 + v - 144, 9)
        bits += [(code >> (n - 1 - i)) & 1 for i in range(n)]
    for code, n in tail:
        bits += [(code >> (n - 1 - i)) & 1 for i in range(n)]
    bits += [0] * 7
    bits += [0] * (-len(bits) % 8)
    body = bytes(sum(bits[i + k] << k for k in range(8)) for i in range(0, len(bits), 8))
    return b"\x78\x01" + body + b"\0\0\0\0"


# =============================================================================
# DEFLATE
# =============================================================================
class Bits:
    def __init__(self, data):
        self.b = np.unpackbits(np.frombuffer(bytes(data), np.uint8), bitorder="little").tolist()
        self.n = len(self.b)

    def get(self, pos, k):
        """k bits LSB first from bit pos (bits past the end read as 0) -> int"""
        v = 0
        for i in range(k):
            if pos + i < self.n and self.b[pos + i]:
                v |= 1 << i
        return v


def code_counts(lengths):
    bl = [0] * 16
    for L in lengths:
        bl[L] += 1
    return bl


def kraft_left(lengths):
    """zlib's inflate_table check: < 0 over-subscribed, 0 complete, > 0 incomplete (codes of length 1..15)"""
    bl = code_counts(lengths)
    left = 1
    for L in range(1, 16):
        left = 2 * left - bl[L]
        if left < 0:
            return -1
    return left


def decoder(lengths):
    """canonical Huffman code (RFC 1951 3.2.2) -> {(length, code read MSB first): symbol}"""
    bl = code_counts(lengths)
    bl[0] = 0
    code, nxt = 0, [0] * 16
    for L in range(1, 16):
        code = (code + bl[L - 1]) << 1
        nxt[L] = code
    table = {}
    for s, L in enumerate(lengths):
        if L:
            table[(L, nxt[L])] = s
            nxt[L] += 1
    return table


def read_sym(bits, pos, table):
    code = 0
    for L in range(1, 16):
        code = (code << 1) | (bits.b[pos + L - 1] if pos + L - 1 < bits.n else 0)
        s = table.get((L, code))
        if s is not None:
            return s, pos + L
    raise ValueError(f"invalid Huffman code at bit {pos}")


def read_dynamic_header(bits, pos):
    """the code lengths of the dynamic block whose HLIT field starts at bit pos -> (lit lengths, dist lengths, pos after
    the header), or a ValueError naming the rule it breaks (zlib's inflate.c checks, in its order)"""
    hlit, hdist, hclen = bits.get(pos, 5) + 257, bits.get(pos + 5, 5) + 1, bits.get(pos + 10, 4) + 4
    pos += 14
    if hlit > 286 or hdist > 30:
        raise ValueError("too many length or distance symbols")
    cl = [0] * 19
    for i in range(hclen):
        cl[CL_ORDER[i]] = bits.get(pos, 3)
        pos += 3
    if kraft_left(cl) != 0:
        raise ValueError("invalid code lengths set")
    t = decoder(cl)
    lens = []
    while len(lens) < hlit + hdist:
        s, pos = read_sym(bits, pos, t)
        if s < 16:
            lens.append(s)
        elif s == 16:
            if not lens:
                raise ValueError("invalid bit length repeat")
            n = 3 + bits.get(pos, 2)
            pos += 2
            lens += [lens[-1]] * n
        else:
            n = (3 + bits.get(pos, 3)) if s == 17 else (11 + bits.get(pos, 7))
            pos += 3 if s == 17 else 7
            lens += [0] * n
        if len(lens) > hlit + hdist:
            raise ValueError("invalid bit length repeat")
    lit, dist = lens[:hlit], lens[hlit:]
    if lit[256] == 0:
        raise ValueError("invalid code -- missing end-of-block")
    left = kraft_left(lit)
    if left < 0 or (left > 0 and max(lit) != 1):  # zlib: incomplete only as a single 1-bit code
        raise ValueError("invalid literal/lengths set")
    left = kraft_left(dist)
    if left < 0 or (left > 0 and max(dist) > 1):  # ... or no distance code at all
        raise ValueError("invalid distances set")
    return lit, dist, pos


def dynamic_header_ok(bits, pos):
    """could a dynamic-Huffman block (BTYPE 10, either BFINAL) start at bit pos?  The device's scan predicate."""
    if bits.get(pos, 3) >> 1 != 0b10:
        return False
    try:
        read_dynamic_header(bits, pos + 3)
    except (ValueError, IndexError):
        return False
    return True


def candidates(stream):
    """every bit offset of the zlib payload (after the 2-byte header) where dynamic_header_ok holds, relative to the
    payload's first bit; numpy narrows by the first 17 bits, the full predicate runs on the rest"""
    payload = stream[2:]
    bits = Bits(payload)
    b = np.asarray(bits.b + [0] * 32, np.int64)
    n = bits.n
    idx = np.arange(n)
    ok = (b[idx + 1] == 0) & (b[idx + 2] == 1)
    hlit = sum(b[idx + 3 + i] << i for i in range(5))
    hdist = sum(b[idx + 8 + i] << i for i in range(5))
    ok &= (hlit <= 29) & (hdist <= 29)
    return [int(p) for p in np.nonzero(ok)[0] if dynamic_header_ok(bits, int(p))]


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30


def walk(stream):
    """a zlib stream -> (blocks, inflated bytes, bit position after the last block): blocks is a list of dicts with
    the start bit (in the payload after the 2-byte header), type (0 stored, 1 fixed, 2 dynamic), BFINAL and the
    output length of each DEFLATE block"""
    bits = Bits(stream[2:])
    pos, out, blocks = 0, bytearray(), []
    while True:
        start, final, btype = pos, bits.get(pos, 1), bits.get(pos + 1, 2)
        pos += 3
        n0 = len(out)
        if btype == 0:
            pos = (pos + 7) & ~7
            ln, nln = bits.get(pos, 16), bits.get(pos + 16, 16)
            if ln != (~nln & 0xFFFF):
                raise ValueError("invalid stored block lengths")
            pos += 32
            out += bytes(bits.get(pos + 8 * i, 8) for i in range(ln))
            pos += 8 * ln
        elif btype == 3:
            raise ValueError("invalid block type")
        else:
            if btype == 1:
                lit, dist = FIXED_LIT, FIXED_DIST
            else:
                lit, dist, pos = read_dynamic_header(bits, pos)
            lt, dt = decoder(lit), decoder(dist)
            while True:
                s, pos = read_sym(bits, pos, lt)
                if s < 256:
                    out.append(s)
                    continue
                if s == 256:
                    break
                if s > 285:
                    raise ValueError("invalid literal/length code")
                L = LEN_BASE[s - 257] + bits.get(pos, LEN_EXTRA[s - 257])
                pos += LEN_EXTRA[s - 257]
                d, pos = read_sym(bits, pos, dt)
                if d > 29:
                    raise ValueError("invalid distance code")
                D = DIST_BASE[d] + bits.get(pos, DIST_EXTRA[d])
                pos += DIST_EXTRA[d]
                if D > len(out):
                    raise ValueError("invalid distance too far back")
                for _ in range(L):
                    out.append(out[-D])
        blocks.append(dict(start=start, type=btype, final=final, out=len(out) - n0))
        if final:
            return blocks, bytes(out), pos


def adler32(data):
    a, b = 1, 0
    arr = np.frombuffer(bytes(data), np.uint8).astype(np.int64)
    for i in range(0, len(arr), 4096):  # chunks short enough that the int64 sums cannot overflow
        c = arr[i:i + 4096]
        n = len(c)
        b = (b + n * a + int(((n - np.arange(n)) * c).sum())) % 65521
        a = (a + int(c.sum())) % 65521
    return (b << 16) | a


def unfilter(raw, H, W):
    """H * (1 + 3W) filtered bytes -> (H, W, 3) uint8 R, G, B (PNG section 9); a filter type above 4 raises"""
    rows = np.frombuffer(bytes(raw[:H * (1 + 3 * W)]), np.uint8).reshape(H, 1 + 3 * W)
    out = np.zeros((H, 3 * W), np.int32)
    prev = np.zeros(3 * W, np.int32)
    for y in range(H):
        f, r = int(rows[y, 0]), rows[y, 1:].astype(np.int32)
        if f > 4:
            raise ValueError(f"bad filter type {f} in row {y}")
        if f == 0:
            cur = r
        elif f == 2:
            cur = (r + prev) & 0xFF
        else:
            cur = np.zeros(3 * W, np.int32)
            for x in range(3 * W):
                a = cur[x - 3] if x >= 3 else 0
                c = prev[x - 3] if x >= 3 else 0
                p = a if f == 1 else ((a + prev[x]) >> 1 if f == 3 else int(paeth(np.int32(a), prev[x], c)))
                cur[x] = (r[x] + p) & 0xFF
        out[y] = cur
        prev = cur
    return out.reshape(H, W, 3).astype(np.uint8)


def decode(data):
    """PNG bytes -> (H, W, 3) B, G, R by the restatement (walk + Adler-32 + unfilter)"""
    W, H = struct.unpack(">II", data[16:24])
    s = idat_stream(data)
    _, raw, pos = walk(s)
    if len(raw) < H * (1 + 3 * W):
        raise ValueError("not enough image data")
    end = 2 + (pos + 7) // 8
    if adler32(raw) != struct.unpack(">I", s[end:end + 4])[0]:
        raise ValueError("incorrect data check")
    return np.ascontiguousarray(unfilter(raw, H, W)[..., ::-1])


def cv2_decode(data):
    import cv2
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_UNCHANGED)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


# =============================================================================
# content and the fixture
# =============================================================================
def content(H, W, seed):
    """seeded photo-like (H, W, 3) uint8: smooth gradients, a few hard edges and noise"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    img = np.zeros((H, W, 3))
    for c in range(3):
        fx, fy, ph = rng.uniform(0.001, 0.006), rng.uniform(0.001, 0.006), rng.uniform(0, 6.3)
        img[..., c] = 128 + 90 * np.sin(fx * x + fy * y + ph)
    for _ in range(6):
        x0, y0 = rng.integers(0, W), rng.integers(0, H)
        w, h = rng.integers(1, max(2, W // 3)), rng.integers(1, max(2, H // 3))
        img[y0:y0 + h, x0:x0 + w] += rng.uniform(-80, 80, 3)
    y0, x0 = rng.integers(0, max(1, H - H // 8)), rng.integers(0, max(1, W - W // 8))
    img[y0:y0 + H // 8, x0:x0 + W // 8] += rng.normal(0, 3, img[y0:y0 + H // 8, x0:x0 + W // 8].shape)  # a textured patch
    img += rng.normal(0, 0.35, img.shape) * (rng.random((H, W, 1)) < 0.05)  # sparse sensor noise
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


KITTI_SIZES = [(376, 1241), (370, 1226), (375, 1242)]


def _flip_adler(stream):
    return stream[:-4] + struct.pack(">I", struct.unpack(">I", stream[-4:])[0] ^ 1)


def _stored_row():
    """a 1 x 2728 frame as one stored block: its last row byte at stream byte 8191, the trailer at 8192..8195"""
    row = np.random.default_rng(0).integers(0, 256, (1, 2728, 3), dtype=np.uint8)
    return row, zlib.compress(filter_rows(row[..., ::-1], [0]).tobytes(), 0)


def corrupt_files():
    """(name, file, status bit of occ_decode_png) of files cv2.imdecode refuses (OpenCV 4.13.0, libpng 1.6.53)"""
    H, W = 20, 30
    raw = filter_rows(content(H, W, 9)[..., ::-1], [y % 5 for y in range(H)]).tobytes()
    s = zlib.compress(raw, 6)
    r5 = bytearray(raw)
    r5[(1 + 3 * W) * 3] = 5
    h, w = 4, 5  # a frame whose whole stream is one fixed block: codes placed right after the last row's byte
    tiny = filter_rows(content(h, w, 2)[..., ::-1], [0] * h).tobytes()
    row, st = _stored_row()
    return [("wrong Adler-32", assemble(H, W, _flip_adler(s)), 4),
            ("cut before the trailer", assemble(H, W, s[:-4]), 2),
            ("truncated", assemble(H, W, s[:len(s) // 2]), 2),
            ("too little image data", assemble(H, W, zlib.compress(raw[:-5])), 2),
            ("filter type 5", assemble(H, W, zlib.compress(bytes(r5))), 8),
            ("distance too far back", assemble(H, W, fixed_block(raw[:10], [(1, 7), (10, 5), (0, 4)])), 1),
            ("invalid distance code", assemble(H, W, fixed_block(raw[:10], [(1, 7), (30, 5)])), 1),
            ("wrong Adler-32 in the last row's read", assemble(1, 2728, _flip_adler(st), idat=[8000, 8000]), 4),
            ("invalid literal/length code right after the rows", assemble(h, w, fixed_block(tiny, [(0b11000110, 8)])),
             1),
            ("invalid distance code right after the rows", assemble(h, w, fixed_block(tiny, [(1, 7), (30, 5)])), 1)]


def benign_files():
    """(name, file, source pixels) of defective files that cv2.imdecode decodes normally"""
    H, W = 20, 30
    src = content(H, W, 10)
    raw = filter_rows(src[..., ::-1], [y % 5 for y in range(H)]).tobytes()
    s = zlib.compress(raw, 6)
    extra = zlib.compress(raw + bytes(100))
    h, w = 4, 5
    tsrc = content(h, w, 2)
    tiny = filter_rows(tsrc[..., ::-1], [0] * h).tobytes()
    row, st = _stored_row()
    return [("too much image data", assemble(H, W, extra), src),
            ("too much data and a wrong Adler-32", assemble(H, W, _flip_adler(extra)), src),
            ("bytes after the stream", assemble(H, W, s + b"\x01\x02junk"), src),
            ("wrong Adler-32 in its own IDAT", assemble(H, W, _flip_adler(s), idat=[len(s) - 4, 4]), src),
            ("wrong Adler-32 across an 8192-byte read", assemble(1, 2728, _flip_adler(st)), row),
            ("a literal, then an invalid literal/length code",
             assemble(h, w, fixed_block(tiny, [(0x30, 8), (0b11000110, 8)])), tsrc),
            ("a literal, then an invalid distance code", assemble(h, w, fixed_block(tiny, [(0x30, 8), (1, 7), (30, 5)])),
             tsrc),
            ("a distance too far back right after the rows",
             assemble(h, w, fixed_block(tiny, [(1, 7), (10, 5), (0, 4)])), tsrc),
            ("empty IDAT chunks", assemble(H, W, s, idat=[5, 0, 0, 3, 0, len(s)]), src)]


def small_files():
    """(name, PNG bytes) of the fixture's small files: every filter type, every block type, long matches across block
    and IDAT boundaries, sides of 1, ignored ancillary chunks"""
    rng = np.random.default_rng(5)
    out = []
    for f in range(5):
        out.append((f"filter {f}", write(content(23, 31, 10 + f), filters=f, level=6)))
    out.append(("mixed filters", write(content(40, 37, 20), level=9)))
    out.append(("stored", write(content(19, 29, 21), level=0)))
    out.append(("fixed", write(content(30, 40, 22), strategy="fixed")))
    out.append(("huffman only", write(content(30, 40, 23), strategy="huffman")))
    out.append(("rle", write(content(30, 40, 24), strategy="rle")))
    out.append(("1 x 1", write(content(1, 1, 25))))
    out.append(("1 x 57", write(content(1, 57, 26))))
    out.append(("61 x 1", write(content(61, 1, 27))))
    row = np.zeros(3 * 11400, np.uint8)  # one row: a random run and its copy 32768 bytes later, zeros between
    row[100:1100] = rng.integers(0, 256, 1000, dtype=np.uint8)
    row[100 + 32768:1100 + 32768] = row[100:1100]
    out.append(("distance 32768", write(row.reshape(1, 11400, 3), filters=0, level=9, idat=997)))
    flat = np.zeros((50, 400, 3), np.uint8)
    flat[::7] = 200
    out.append(("length 258", write(flat, filters=0, level=9, idat=[5, 1, 3000])))
    anc = [(b"gAMA", struct.pack(">I", 45455)), (b"sRGB", b"\x00"), (b"pHYs", struct.pack(">IIB", 2835, 2835, 1)),
           (b"tEXt", b"Comment\x00occformer"), (b"tIME", struct.pack(">HBBBBB", 2026, 1, 2, 3, 4, 5)),
           (b"sBIT", b"\x08\x08\x08"), (b"PLTE", bytes(range(48)))]
    out.append(("ancillary chunks", write(content(17, 19, 28), ancillary=anc)))
    return out


def full_files():
    import cv2
    return [(f"{W} x {H}", cv2.imencode(".png", content(H, W, 100 + i))[1].tobytes())
            for i, (H, W) in enumerate(KITTI_SIZES)]


def gen():
    import cv2
    files = small_files() + full_files()
    arrs = {}
    for i, (name, f) in enumerate(files):
        dec = cv2_decode(f)
        assert dec is not None and dec.shape[2] == 3, name
        arrs[f"file_{i}"] = np.frombuffer(f, np.uint8)
        arrs[f"name_{i}"] = np.array(name)
        arrs[f"sha_{i}"] = np.array(sha(dec))
    arrs["count"] = np.array(len(files))
    arrs["opencv"] = np.array(cv2.__version__)
    arrs["libpng"] = np.array(libpng_version())
    np.savez_compressed(GOLDEN, **arrs)
    print(f"wrote {GOLDEN}: {len(files)} files, {os.path.getsize(GOLDEN)} bytes")


def libpng_version():
    import cv2
    for line in cv2.getBuildInformation().splitlines():
        if line.strip().startswith("PNG:"):
            return line.split("(ver", 1)[-1].strip(" )") if "(ver" in line else line.split(":", 1)[1].strip()
    return "unknown"


if __name__ == "__main__":
    import sys
    if sys.argv[1:] == ["gen"]:
        gen()
