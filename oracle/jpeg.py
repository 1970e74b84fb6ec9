"""TEST INFRASTRUCTURE ONLY (oracle) -- baseline JPEG decoding as cv2.imdecode(buf, IMREAD_UNCHANGED) does it (mmcv.imread's
cv2 backend, which the reference's LoadMultiViewImageFromFiles_OccFormer calls), restated in numpy from the published
JPEG specification (ITU T.81) and libjpeg's documented integer arithmetic:

    entropy decoding   T.81 Annex C (code assignment) and F.2.2 (DECODE, RECEIVE, EXTEND), serial, restart intervals
                       resetting the DC predictions (F.2.1.3.1)
    IDCT               libjpeg's "islow" (JDCT_ISLOW): the scaled-integer Loeffler-Ligtenberg-Moschytz 8-point IDCT with
                       13-bit constants and 2 extra bits between the passes, then the output + 128 clamped to [0, 255].
                       libjpeg's portable C code indexes a range-limit table by the output & 1023 (RANGE_MASK), which
                       wraps an output of 512 or more (or below -512) around to the other end; the x86-64 SIMD IDCT that cv2's
                       libjpeg-turbo runs saturates instead.  Streams requantised to reach that region (requant below)
                       show cv2 clamping, so clamping is the rule here
    upsampling         libjpeg's "fancy" triangle filter: h2v1 (3 * nearer + farther) / 4 with alternating +1 / +2
                       rounding; h2v2 the same on column sums 3 * nearer row + farther row, / 16 with +8 / +7; edges
                       replicated at the component's real (downsampled) size
    colour             libjpeg's YCbCr -> RGB tables with 16 fractional bits (jdcolor.c's constants 1.402, 1.772,
                       0.71414, 0.34414), clamped to [0, 255]; cv2 returns B, G, R

tests/test_cpu_jpeg.py checks it against the installed cv2 bit for bit.  It is also the fixture writer:

    python -m oracle.jpeg gen     # tests/golden/jpeg.npz

The fixture records the OpenCV and libjpeg-turbo versions that wrote it (OpenCV 4.13.0 with its bundled libjpeg-turbo 3.1.2).  The
reference environment pins opencv-python 4.7.0.72, which bundles an older libjpeg-turbo; its 8-bit islow IDCT, fancy
upsampling and colour tables are believed unchanged, but that is unverified.
"""
import hashlib
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "jpeg.npz")

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63])


# =============================================================================
# markers
# =============================================================================
def _markers(data):
    """-> (frame (H, W, [(id, h, v, tq)]), {tq: natural-order table}, {(class, id): (counts, values)}, restart,
    [(comp index, td, ta)], entropy-coded bytes up to EOI)"""
    i, qt, ht, restart = 2, {}, {}, 0
    while True:
        while data[i] == 0xFF:
            i += 1
        m = data[i]
        i += 1
        n = (data[i] << 8) | data[i + 1]
        body = data[i + 2:i + n]
        i += n
        if m in (0xC0, 0xC1):
            H, W = (body[1] << 8) | body[2], (body[3] << 8) | body[4]
            comps = [(body[6 + 3 * c], body[7 + 3 * c] >> 4, body[7 + 3 * c] & 15, body[8 + 3 * c]) for c in range(body[5])]
            frame = (H, W, comps)
        elif m == 0xDB:
            j = 0
            while j < len(body):
                pq, tq = body[j] >> 4, body[j] & 15
                raw = np.frombuffer(body[j + 1:j + 1 + 64 * (pq + 1)], np.uint8 if pq == 0 else ">u2").astype(np.int64)
                q = np.zeros(64, np.int64)
                q[ZIGZAG] = raw
                qt[tq] = q
                j += 1 + 64 * (pq + 1)
        elif m == 0xC4:
            j = 0
            while j < len(body):
                counts = list(body[j + 1:j + 17])
                ht[(body[j] >> 4, body[j] & 15)] = (counts, list(body[j + 17:j + 17 + sum(counts)]))
                j += 17 + sum(counts)
        elif m == 0xDD:
            restart = (body[0] << 8) | body[1]
        elif m == 0xDA:
            ids = [c[0] for c in frame[2]]
            scan = [(ids.index(body[1 + 2 * c]), body[2 + 2 * c] >> 4, body[2 + 2 * c] & 15) for c in range(body[0])]
            end = data.rfind(b"\xff\xd9", i)
            return frame, qt, ht, restart, scan, data[i:end if end >= 0 else len(data)]


def _codes(counts, values):
    """T.81 Annex C: (length, code) -> symbol"""
    table, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            table[(length, code)] = values[k]
            code += 1
            k += 1
        code <<= 1
    return table


# =============================================================================
# entropy decoding
# =============================================================================
class _Bits:
    """the entropy-coded data of one restart interval, FF00 stuffing removed"""

    def __init__(self, seg):
        self.bits = np.unpackbits(np.frombuffer(seg.replace(b"\xff\x00", b"\xff"), np.uint8))
        self.p = 0

    def get(self, n):
        if self.p + n > len(self.bits):
            raise ValueError("entropy-coded data ends early")
        v = 0
        for b in self.bits[self.p:self.p + n]:
            v = (v << 1) | int(b)
        self.p += n
        return v

    def decode(self, table):
        code = 0
        for length in range(1, 17):
            code = (code << 1) | self.get(1)
            if (length, code) in table:
                return table[(length, code)]
        raise ValueError("invalid Huffman code")


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def coefficients(data):
    """-> (frame, qt, per-component int64 coefficient arrays (blocks_y, blocks_x, 64) in natural order, DC restored)"""
    frame, qt, ht, restart, scan, ecs = _markers(data)
    H, W, comps = frame
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    mx, my = -(-W // (8 * hmax)), -(-H // (8 * vmax))
    coef = [np.zeros((my * c[2], mx * c[1], 64), np.int64) for c in comps]
    tables = [(_codes(*ht[(0, td)]), _codes(*ht[(1, ta)])) for _, td, ta in scan]
    # restart intervals: RSTn markers split the segment
    segs, j, start = [], 0, 0
    while True:
        k = ecs.find(b"\xff", j)
        if k < 0 or k + 1 >= len(ecs):
            break
        if 0xD0 <= ecs[k + 1] <= 0xD7:
            segs.append(ecs[start:k])
            start = j = k + 2
        else:
            j = k + 2
    segs.append(ecs[start:])
    per = restart if restart else mx * my
    for u in range(mx * my):
        if u % per == 0:
            bits = _Bits(segs[u // per])
            pred = [0, 0, 0]
        for si, (ci, _, _) in enumerate(scan):
            _, h, v, _ = comps[ci]
            dct, act = tables[si]
            for by in range(v):
                for bx in range(h):
                    blk = coef[ci][(u // mx) * v + by, (u % mx) * h + bx]
                    s = bits.decode(dct)
                    pred[ci] += _extend(bits.get(s), s)
                    blk[0] = pred[ci]
                    k = 1
                    while k < 64:
                        rs = bits.decode(act)
                        r, s = rs >> 4, rs & 15
                        if s:
                            k += r
                            if k > 63:
                                raise ValueError("coefficient run past 63")
                            blk[ZIGZAG[k]] = _extend(bits.get(s), s)
                            k += 1
                        elif r == 15:
                            k += 16
                        else:
                            break
    return frame, qt, coef


# =============================================================================
# islow IDCT, range limit
# =============================================================================
CONST_BITS, PASS1_BITS = 13, 2
F0298, F0390, F0541, F0765 = 2446, 3196, 4433, 6270
F0899, F1175, F1501, F1847 = 7373, 9633, 12299, 15137
F1961, F2053, F2562, F3072 = 16069, 16819, 20995, 25172


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(c0, c1, c2, c3, c4, c5, c6, c7):
    """one 8-point pass on int64 arrays -> (even + odd, ...) before descaling, in output order 0..7"""
    z1 = (c2 + c6) * F0541
    tmp2 = z1 - c6 * F1847
    tmp3 = z1 + c2 * F0765
    tmp0 = (c0 + c4) << CONST_BITS
    tmp1 = (c0 - c4) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    o0, o1, o2, o3 = c7, c5, c3, c1
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * F1175
    o0, o1, o2, o3 = o0 * F0298, o1 * F2053, o2 * F3072, o3 * F1501
    z1, z2, z3, z4 = -z1 * F0899, -z2 * F2562, -z3 * F1961 + z5, -z4 * F0390 + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    return [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]


def range_limit(x):
    """IDCT output -> sample: x + 128 clamped to [0, 255] (see the module docstring)"""
    return (np.clip(x, -128, 127) + 128).astype(np.uint8)


def range_limit_wrap(x):
    """libjpeg's portable range-limit table indexed by x & 1023, for the tests that tell the two rules apart"""
    u = x & 1023
    return np.where(u < 128, u + 128, np.where(u < 512, 255, np.where(u < 896, 0, u - 896))).astype(np.uint8)


def idct_islow(coef, q):
    """(..., 64) natural-order coefficients, (64,) table -> (..., 8, 8) uint8 samples"""
    q = q.astype(np.int64).astype(np.int16).astype(np.int64)  # libjpeg's multiplier table is 16-bit
    d = (coef * q).reshape(coef.shape[:-1] + (8, 8))
    cols = _idct_1d(*[d[..., k, :] for k in range(8)])        # pass 1 down the columns
    ws = np.stack([_descale(c, CONST_BITS - PASS1_BITS) for c in cols], axis=-2)
    rows = _idct_1d(*[ws[..., :, k] for k in range(8)])       # pass 2 along the rows
    out = np.stack([_descale(r, CONST_BITS + PASS1_BITS + 3) for r in rows], axis=-1)
    return range_limit(out)


def planes(data):
    """-> (frame, per-component uint8 planes at their MCU-padded size)"""
    frame, qt, coef = coefficients(data)
    out = []
    for (_, _, _, tq), c in zip(frame[2], coef):
        s = idct_islow(c, qt[tq])                     # (by, bx, 8, 8)
        out.append(s.transpose(0, 2, 1, 3).reshape(c.shape[0] * 8, c.shape[1] * 8))
    return frame, out


# =============================================================================
# fancy upsampling, colour
# =============================================================================
def _h2(c):
    """h2v1 fancy upsampling of (rows, w) int64 -> (rows, 2w) along the last axis, edge replicated"""
    left = np.concatenate([c[:, :1], c[:, :-1]], axis=1)
    right = np.concatenate([c[:, 1:], c[:, -1:]], axis=1)
    out = np.empty((c.shape[0], 2 * c.shape[1]), np.int64)
    out[:, 0::2] = (3 * c + left + 1) >> 2
    out[:, 1::2] = (3 * c + right + 2) >> 2
    return out


def _h2v2(c):
    above = np.concatenate([c[:1], c[:-1]], axis=0)
    below = np.concatenate([c[1:], c[-1:]], axis=0)
    out = np.empty((2 * c.shape[0], 2 * c.shape[1]), np.int64)
    for r, nb in ((0, above), (1, below)):
        cs = 3 * c + nb
        left = np.concatenate([cs[:, :1], cs[:, :-1]], axis=1)
        right = np.concatenate([cs[:, 1:], cs[:, -1:]], axis=1)
        out[r::2, 0::2] = (3 * cs + left + 8) >> 4
        out[r::2, 1::2] = (3 * cs + right + 7) >> 4
    return out


SCALEBITS = 16


def _fix(x):
    return int(x * (1 << SCALEBITS) + 0.5)


def colour_tables():
    """jdcolor.c's build_ycc_rgb_table: (Cr->R, Cb->B, Cr->G, Cb->G) over x = 0..255"""
    x = np.arange(256, dtype=np.int64) - 128
    half = 1 << (SCALEBITS - 1)
    return ((_fix(1.40200) * x + half) >> SCALEBITS, (_fix(1.77200) * x + half) >> SCALEBITS,
            -_fix(0.71414) * x, -_fix(0.34414) * x + half)


def decode(data):
    """file bytes -> uint8 (H, W, 3) BGR, as cv2.imdecode(buf, cv2.IMREAD_UNCHANGED)"""
    data = bytes(data)
    (H, W, comps), pl = planes(data)
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    full = []
    for (_, h, v, _), p in zip(comps, pl):
        dh, dw = -(-H * v // vmax), -(-W * h // hmax)  # the component's real (downsampled) size
        c = p[:dh, :dw].astype(np.int64)
        if (h, v) == (hmax, vmax):
            f = c
        elif (hmax // h, vmax // v) == (2, 1):
            f = _h2(c)
        else:
            f = _h2v2(c)
        full.append(f[:H, :W])
    y, cb, cr = full
    crr, cbb, crg, cbg = colour_tables()
    r = np.clip(y + crr[cr], 0, 255)
    g = np.clip(y + ((cbg[cb] + crg[cr]) >> SCALEBITS), 0, 255)
    b = np.clip(y + cbb[cb], 0, 255)
    return np.stack([b, g, r], axis=-1).astype(np.uint8)


# =============================================================================
# test images and the fixture
# =============================================================================
SAMPLINGS = {"444": 0x111111, "422": 0x211111, "420": 0x221111}


def encode(img, quality=95, sampling="420", restart=0):
    """cv2.imencode of a uint8 (H, W, 3) BGR image -> bytes"""
    import cv2
    ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                         SAMPLINGS[sampling], cv2.IMWRITE_JPEG_RST_INTERVAL, restart])
    assert ok
    return buf.tobytes()


def cv2_decode(data):
    import cv2
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_UNCHANGED)


def content(kind, H, W, seed):
    """uint8 (H, W, 3): 'smooth' ramps, 'noise' (uniform, saturating), 'checker' (0 / 255 cells of 1 to 3 pixels)"""
    y = np.arange(H)[:, None, None]
    x = np.arange(W)[None, :, None]
    c = np.arange(3)[None, None, :]
    if kind == "smooth":
        v = (x * 255 // max(W - 1, 1) + y * 97 // max(H - 1, 1) + c * 60 + seed * 13) % 256
    elif kind == "noise":
        v = np.random.default_rng(seed).integers(0, 256, (H, W, 3))
    else:
        s = 1 + seed % 3
        v = (((y // s) + (x // s) + c * (seed & 1)) % 2) * 255 + 0 * c
    return np.broadcast_to(v, (H, W, 3)).astype(np.uint8)


# the small cases: (H, W, sampling, quality, restart, content)
SMALL = []
for _s in SAMPLINGS:
    for _q in (10, 75, 95, 100):
        for _k in ("smooth", "noise", "checker"):
            SMALL.append((29, 37, _s, _q, 0, _k))
    for _r in (1, 7):
        SMALL.append((29, 37, _s, 90, _r, "noise"))
    for _hw in ((1, 1), (8, 17), (17, 8), (2, 2), (3, 5), (16, 16), (40, 24)):
        SMALL.append(_hw + (_s, 95, 0, "noise"))
        SMALL.append(_hw + (_s, 100, 3, "checker"))


def small_case(i):
    H, W, s, q, r, k = SMALL[i]
    return encode(content(k, H, W, i), q, s, r)


# full-size frames stored in the fixture: (sampling, quality, restart, seed of oracle.image_prep.frame).  Low qualities
# keep them at about 100 KB each; hq_case, a high-quality frame of about 1.4 MB, is encoded when a test runs instead.
FULL = [("420", 10, 0, 11), ("422", 15, 64, 13)]


def full_case(i):
    from . import image_prep
    s, q, r, seed = FULL[i]
    return encode(image_prep.frame(seed, 900, 1600), q, s, r)


def requant(data, scale):
    """the file with every quantisation value multiplied by scale (capped at 255): the same coefficients dequantise to
    larger values, past the IDCT's clamping range.  libjpeg-turbo's 16-bit SIMD arithmetic holds dequantised values in
    the range 8-bit images produce (about +-2^11); scale 8 on the test images stays inside it."""
    b, i = bytearray(data), 2
    while True:
        while b[i] == 0xFF:
            i += 1
        m, n = b[i], (b[i + 1] << 8) | b[i + 2]
        i += 1
        if m == 0xDB:
            j = i + 2
            while j < i + n:
                for k in range(64):
                    b[j + 1 + k] = min(255, b[j + 1 + k] * scale)
                j += 65
        if m == 0xDA:
            return bytes(b)
        i += n


def hq_case():
    """a 900 x 1600 quality-95 4:4:4 file of oracle.image_prep.frame(12), encoded by the installed cv2 (not stored: it
    alone would be 1.4 MB); compare its decode against cv2_decode"""
    from . import image_prep
    return encode(image_prep.frame(12, 900, 1600), 95, "444")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint8).tobytes()).hexdigest()


def gen():
    """tests/golden/jpeg.npz: the bytes of every small and full-size case and the SHA-256 of cv2's decode of each"""
    import cv2
    import re
    turbo = re.findall(r"JPEG:\s*(.*)", cv2.getBuildInformation())
    out = dict(cv2_version=np.array(cv2.__version__), cv2_jpeg=np.array(turbo[0].strip() if turbo else "unknown"))
    for name, n, make in (("small", len(SMALL), small_case), ("full", len(FULL), full_case)):
        for i in range(n):
            data = make(i)
            out[f"{name}_{i}_bytes"] = np.frombuffer(data, np.uint8)
            out[f"{name}_{i}_sha"] = np.array(sha(cv2_decode(data)))
    np.savez_compressed(GOLDEN, **out)
    print(GOLDEN, os.path.getsize(GOLDEN), "bytes")


if __name__ == "__main__":
    import sys
    {"gen": gen}[sys.argv[1] if len(sys.argv) > 1 else "gen"]()
