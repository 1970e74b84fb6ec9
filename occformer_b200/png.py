"""PNG chunks on the host, for the device decoder of csrc/png_decode.cu (ops.decode_png, image_prep.decode_png).

The camera frames of the SemanticKITTI loader are 8-bit RGB PNGs that the reference decodes with cv2.imdecode
(mmcv.imread(..., 'unchanged'), loading_kitti_imgs.py:103; libpng + zlib).  This module walks the chunks of one file
and refuses, with a ValueError naming the feature, everything the device decoder does not implement:

    accepted   the PNG signature, IHDR first; bit depth 8, colour type 2 (RGB), compression 0, filter method 0,
               interlace 0; sides up to MAX_SIDE; consecutive IDAT chunks holding a zlib stream of MIN_STREAM to
               MAX_STREAM bytes with CM 8, CINFO <= 7, a valid FCHECK and no preset dictionary; an IEND chunk.
    refused    other bit depths; grayscale, grayscale + alpha, RGBA and palette files; tRNS (cv2 returns 4 channels);
               Adam7 interlace; APNG (acTL); a bad zlib header; IDAT chunks that are missing, empty in total or not
               consecutive; a bad CRC on a critical chunk; a file without IEND (cv2 returns None).
    ignored    ancillary chunks (gAMA, sRGB, iCCP, sBIT, pHYs, tEXt, tIME, ...), bad CRCs on them included, and a
               suggested PLTE in an RGB file, as libpng ignores them.

The concatenated IDAT payloads are the zlib stream; Header gives each non-empty chunk's payload offset and length in
the file, so that the staging copy lays the streams out back to back.  Empty IDAT chunks are dropped: they change
neither the stream nor where libpng's reads of it start.
"""
import struct
import zlib

MAX_SIDE = 16384              # largest accepted width and height
MAX_STREAM = (1 << 27) - 1    # largest accepted zlib stream: bit positions stay below 2^31
MIN_STREAM = 7                # a shorter zlib stream cannot hold a header, a block and the Adler-32 (cv2 refuses it)
SIGNATURE = b"\x89PNG\r\n\x1a\n"
_COLOUR = {0: "grayscale", 3: "palette", 4: "grayscale + alpha", 6: "RGBA"}


class PngError(ValueError):
    pass


class Header:
    """what the device needs of one file: size, the zlib window and the IDAT payloads (offset, length) in the file"""
    __slots__ = ("height", "width", "cinfo", "idat")

    @property
    def stream_len(self):
        return sum(n for _, n in self.idat)


def _chunks(data):
    if bytes(data[:8]) != SIGNATURE:
        raise PngError("not a PNG file (bad signature)")
    i, n = 8, len(data)
    while i < n:
        if i + 12 > n:
            raise PngError("truncated chunk")
        length, kind = struct.unpack(">I4s", data[i:i + 8])
        if i + 12 + length > n:
            raise PngError(f"truncated {kind.decode('latin-1')} chunk")
        crc = struct.unpack(">I", data[i + 8 + length:i + 12 + length])[0]
        yield kind, i + 8, length, crc == zlib.crc32(data[i + 4:i + 8 + length])
        i += 12 + length


def parse(data):
    """PNG bytes -> Header; raises PngError naming the feature the device decoder does not take"""
    data = memoryview(data).cast("B")
    h, seen_ihdr, seen_idat, idat_done, iend = Header(), False, False, False, False
    h.idat = []
    for kind, off, length, crc_ok in _chunks(data):
        critical = not (kind[0] & 0x20)
        if not seen_ihdr:
            if kind != b"IHDR" or length != 13:
                raise PngError("IHDR is not the first chunk")
        if critical and not crc_ok:
            raise PngError(f"bad CRC on the critical {kind.decode('latin-1')} chunk")
        if kind == b"IHDR":
            if seen_ihdr:
                raise PngError("a second IHDR chunk")
            seen_ihdr = True
            W, H, depth, colour, comp, filt, interlace = struct.unpack(">IIBBBBB", data[off:off + 13])
            if colour != 2:
                raise PngError(f"{_COLOUR.get(colour, f'colour type {colour}')} PNG (only 8-bit RGB is decoded)")
            if depth != 8:
                raise PngError(f"bit depth {depth} (only 8-bit RGB is decoded)")
            if comp != 0 or filt != 0:
                raise PngError("unknown compression or filter method")
            if interlace != 0:
                raise PngError("Adam7-interlaced PNG (only non-interlaced files are decoded)")
            if not (1 <= W <= MAX_SIDE and 1 <= H <= MAX_SIDE):
                raise PngError(f"frame {W} x {H} outside 1..{MAX_SIDE}")
            h.width, h.height = W, H
        elif kind == b"IDAT":
            if idat_done:
                raise PngError("IDAT chunks are not consecutive")
            if length:  # an empty IDAT adds no data and no read boundary of its own
                h.idat.append((off, length))
            seen_idat = True
        elif kind == b"IEND":
            iend = True
            break
        else:
            if seen_idat:
                idat_done = True
            if kind == b"tRNS":
                raise PngError("tRNS chunk (cv2 decodes the file with an alpha channel)")
            if kind in (b"acTL", b"fcTL", b"fdAT"):
                raise PngError("animated PNG (APNG)")
            if critical and kind != b"PLTE":
                raise PngError(f"unknown critical chunk {kind.decode('latin-1')}")
    if not h.idat or h.stream_len == 0:
        raise PngError("no image data (IDAT missing or empty)")
    if not iend:
        raise PngError("no IEND chunk (cv2 refuses the file)")
    if h.stream_len > MAX_STREAM:
        raise PngError(f"zlib stream of {h.stream_len} bytes (at most {MAX_STREAM})")
    if h.stream_len < MIN_STREAM:
        raise PngError(f"zlib stream of {h.stream_len} bytes, too short to be complete (cv2 refuses it)")
    head = bytes(data[h.idat[0][0]:h.idat[0][0] + 2]) if h.idat[0][1] >= 2 else bytes(
        b"".join(bytes(data[o:o + n]) for o, n in h.idat)[:2])
    if len(head) < 2:
        raise PngError("zlib stream shorter than its header")
    cmf, flg = head
    if cmf & 15 != 8:
        raise PngError(f"zlib compression method {cmf & 15} (only deflate)")
    if cmf >> 4 > 7:
        raise PngError(f"zlib window CINFO {cmf >> 4} above 7")
    if ((cmf << 8) | flg) % 31:
        raise PngError("bad zlib header check (FCHECK)")
    if flg & 0x20:
        raise PngError("zlib preset dictionary (FDICT), which PNG forbids")
    h.cinfo = cmf >> 4
    return h


def frame_size(data):
    """(H, W) of an accepted PNG file, as cv2.imdecode returns it"""
    h = parse(data)
    return h.height, h.width
