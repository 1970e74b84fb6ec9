// 8-bit RGB PNG decoding on the device, bit for bit as cv2.imdecode(buf, IMREAD_UNCHANGED) (libpng + zlib) -- the camera
// frames of LoadMultiViewImageFromFiles_SemanticKitti (P/datasets/pipelines/loading_kitti_imgs.py:103, mmcv.imread(...,
// 'unchanged') with its cv2 backend).  include/occ_b200.h states the semantics; occformer_b200/png.py walks the chunks
// on the host and stages every image's zlib stream (its IDAT payloads back to back).
//
// DEFLATE is serial by construction: a block's start is known only once the previous block has been decoded.  Dynamic
// Huffman blocks (what zlib writes for photos) carry a header that random bits rarely satisfy, so the starts are found
// speculatively and the true chain is linked afterwards:
//   scan     one thread per bit of a stream: could a dynamic-Huffman block (BTYPE 10, either BFINAL) start here?  zlib's
//            own rules: HLIT, HDIST <= 29, a complete code-length code, code lengths without an overrun of a repeat,
//            complete literal/length and distance codes (or zlib's one-code exception), a nonzero length for code
//            256.  Survivors go into a per-image hash table keyed by bit position (PD_CANDIDATES at most)
//   probe    one thread per table slot decodes its candidate to end-of-block without writing: end bit and output bytes,
//            or "unknown" on an invalid symbol or past PD_PROBE_SYMBOLS symbols
//   link     one thread per image walks the true chain from the first block: a stored block is skipped by its LEN, a
//            probed candidate jumped over, anything else (fixed blocks, unknown or unlisted candidates) decoded
//            serially to its end.  Records every block's start, type and output offset, the total output, the first
//            error, and whether the trailer is present
//   inflate  one warp per true block (lane 0) decodes it again: literals as they are, each byte of a match as the
//            position of its source, folded so that it lies before the match when the distance is shorter than the
//            length
//   resolve  PD_RESOLVE_ROUNDS rounds of pointer jumping turn every source position into its literal
//   finish   one block per image: Adler-32 of the rows' bytes, the status as cv2 decides it (below), then the unfilter
//            as a wavefront (one warp per 32 rows, lane l owns a row and lags lane l - 1 by one pixel; above and
//            above-left arrive by shuffle, the last row of the previous warp through the frame and a progress word in
//            shared memory) writing B, G, R
// plus two memsets (status words; the candidate tables and per-image counters): 7 + PD_RESOLVE_ROUNDS operations
// whatever the data and the number of images, no host synchronisation, capturable in a CUDA graph.  The candidate
// capacity, the probe's symbol cap and the encoder's block sizes change only the speed: a stream of fixed or stored
// blocks alone decodes on the link thread.
//
// cv2's verdict (libpng 1.6 reading rows through zlib; libpng feeds zlib each IDAT chunk in reads of PD_READ_SIZE
// bytes).  An error before the rows are complete fails the image, and so does data that ends early anywhere.  The call
// that fills the last row goes on while it needs no output and has input: an invalid literal/length or distance code,
// or an invalid block header, met there with no byte past the rows produced yet and within the same read as the
// last row's bytes fails the image, and so does a wrong Adler-32 when the stream holds exactly the rows' bytes and its
// trailer is in that read.  Every other error after the rows (a distance too far back included: zlib stops for want of
// output before it checks one) is benign for libpng, and the frame is decoded.
#include "occ_common.cuh"

namespace occ {

constexpr int PD_MAX_IMAGES = 96;
constexpr int PD_CANDIDATES = 8192;            // candidate block starts per image (hash table of twice as many slots)
constexpr int PD_SLOTS = 2 * PD_CANDIDATES;
constexpr int PD_PROBE_SYMBOLS = 1 << 16;      // symbols a probe decodes before giving up
constexpr int PD_RESOLVE_ROUNDS = 30;          // 2^30 > the longest chain of back-references in a frame
constexpr int PD_READ_SIZE = 8192;             // libpng's IDAT read size (PNG_IDAT_READ_SIZE)
constexpr int PD_THREADS = 256;
constexpr int PD_INFLATE_CTAS = 16;            // inflate blocks per image: 128 warps
constexpr unsigned PD_LIT = 0x80000000u;       // a resolved byte: PD_LIT | value; else the index of its source

// status bits (include/occ_b200.h)
constexpr int PD_E_DATA = 1;      // invalid DEFLATE data before the rows are complete
constexpr int PD_E_SHORT = 2;     // the stream ends early, or holds fewer bytes than the rows
constexpr int PD_E_ADLER = 4;     // Adler-32 mismatch where libpng treats it as an error
constexpr int PD_E_FILTER = 8;    // a filter type above 4

// per-image counters (int, zeroed by the memset)
enum { PM_NCAND, PM_NBLK, PM_TOTAL, PM_ERR, PM_ERR_OUT, PM_ERR_BIT, PM_TRAILER, PM_FAR, PM_HORIZON, PM_SERIAL,
       PM_COUNT = 16 };

struct PdImage {
  long long src;                 // byte offset of the zlib stream in `data`
  long long out;                 // byte offset of the (H, W, 3) frame in `out`
  long long o_keys, o_meta;      // workspace byte offsets (zeroed area)
  long long o_res, o_blk, o_refs;
  int len;                       // stream bytes
  int H, W, raw;                 // raw = H * (1 + 3W) filtered bytes
  int wsize;                     // LZ77 window of the zlib header, 2^(CINFO + 8)
  int nblk;                      // capacity of the block list
  int idat0, nidat;              // the image's IDAT chunk starts in `idat`
  int scan0, probe0, inf0, res0; // the image's first block in each grid
};

struct PdParams {
  PdImage img[PD_MAX_IMAGES];
  int M;
};

#define PD_FIND(P, field, b)                                        \
  ([&]() {                                                          \
    int lo__ = 0, hi__ = (P).M - 1;                                 \
    while (lo__ < hi__) {                                           \
      const int mid__ = (lo__ + hi__ + 1) >> 1;                     \
      if ((P).img[mid__].field <= (int)(b)) lo__ = mid__; else hi__ = mid__ - 1; \
    }                                                               \
    return lo__;                                                    \
  }())

template <typename T>
__device__ __forceinline__ T* pd_at(void* ws, long long off) {
  return reinterpret_cast<T*>(static_cast<unsigned char*>(ws) + off);
}

// ------------------------------------------------------------------------------------------------ bits and codes
// at least 32 bits of the stream from bit pos, LSB first; bits past the end read as 0
__device__ __forceinline__ unsigned pd_peek(const unsigned char* s, int len, int pos) {
  const int b = pos >> 3;
  unsigned long long w = 0;
#pragma unroll
  for (int i = 0; i < 5; ++i)
    if (b + i < len) w |= (unsigned long long)__ldg(s + b + i) << (8 * i);
  return (unsigned)(w >> (pos & 7));
}

// a canonical Huffman code (RFC 1951 3.2.2): codes per length and the symbols in code order, and (pd_lut) a lookup of
// the next PD_LUT_BITS stream bits: length << 9 | symbol for the codes of at most that length, 0 for longer ones
constexpr int PD_LUT_BITS = 9;
struct PdHuff {
  unsigned short count[16];
  unsigned short sym[288];
  unsigned short lut[1 << PD_LUT_BITS];
};

// lengths[0, n) -> h; returns the unused code space (< 0 over-subscribed, 0 complete) and the longest length in *maxl
__device__ int pd_build(PdHuff& h, const unsigned char* lengths, int n, int* maxl) {
  for (int l = 0; l < 16; ++l) h.count[l] = 0;
  for (int i = 0; i < n; ++i) h.count[lengths[i]]++;
  int left = 1, mx = 0;
  for (int l = 1; l < 16; ++l) {
    left = 2 * left - h.count[l];
    if (left < 0) return -1;
    if (h.count[l]) mx = l;
  }
  unsigned short offs[16];
  offs[1] = 0;
  for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + h.count[l];
  for (int i = 0; i < n; ++i)
    if (lengths[i]) h.sym[offs[lengths[i]]++] = (unsigned short)i;
  *maxl = mx;
  return left;
}

// the next symbol of code h in bits (LSB first) -> symbol, *used = its length; -1 for a code not in h
__device__ __forceinline__ int pd_decode(const PdHuff& h, unsigned bits, int* used) {
  int code = 0, first = 0, index = 0;
  for (int l = 1; l < 16; ++l) {
    code |= (bits >> (l - 1)) & 1;
    const int count = h.count[l];
    if (code - first < count) {
      *used = l;
      return h.sym[index + code - first];
    }
    index += count;
    first = (first + count) << 1;
    code <<= 1;
  }
  return -1;
}

// fills h.lut from h.count and h.sym: each code of length l <= PD_LUT_BITS, bit-reversed (the stream sends a code's
// first bit first, LSB first), in every entry whose low l bits it matches
__device__ void pd_lut(PdHuff& h) {
  for (int i = 0; i < (1 << PD_LUT_BITS); ++i) h.lut[i] = 0;
  int code = 0, idx = 0;
  for (int l = 1; l <= PD_LUT_BITS; ++l) {
    for (int n = 0; n < h.count[l]; ++n, ++code, ++idx) {
      const unsigned short e = (unsigned short)(l << 9 | h.sym[idx]);
      for (int k = (int)(__brev((unsigned)code) >> (32 - l)); k < (1 << PD_LUT_BITS); k += 1 << l) h.lut[k] = e;
    }
    code <<= 1;
  }
}

// pd_decode through the lookup (pd_lut must have run), falling back to the code counts for longer codes
__device__ __forceinline__ int pd_decode_lut(const PdHuff& h, unsigned bits, int* used) {
  const int e = h.lut[bits & ((1 << PD_LUT_BITS) - 1)];
  if (e) {
    *used = e >> 9;
    return e & 511;
  }
  return pd_decode(h, bits, used);
}

__constant__ unsigned char pd_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
__constant__ unsigned short pd_len_base[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                               31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ unsigned char pd_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5,
                                               5, 5, 5, 0};
__constant__ unsigned short pd_dist_base[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,
                                                97,  129, 193, 257, 385, 513,  769,  1025, 1537, 2049, 3073, 4097,
                                                6145, 8193, 12289, 16385, 24577};
__constant__ unsigned char pd_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2,  3,  3,  4,  4,  5,  5,  6,
                                                6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

// the dynamic header whose HLIT field starts at bit pos -> the bit after it, or -1 where zlib would refuse it
__device__ int pd_dynamic(const unsigned char* s, int len, int pos, PdHuff& lit, PdHuff& dist) {
  unsigned w = pd_peek(s, len, pos);
  const int hlit = (w & 31) + 257, hdist = ((w >> 5) & 31) + 1, hclen = ((w >> 10) & 15) + 4;
  if (hlit > 286 || hdist > 30) return -1;
  pos += 14;
  unsigned char lengths[320];
  for (int i = 0; i < 19; ++i) lengths[i] = 0;
  for (int i = 0; i < hclen; ++i) lengths[pd_cl_order[i]] = (pd_peek(s, len, pos + 3 * i) & 7);
  pos += 3 * hclen;
  int mx;
  if (pd_build(lit, lengths, 19, &mx) != 0 || mx == 0) return -1;  // the code-length code must be complete
  const int n = hlit + hdist;
  for (int i = 0; i < n;) {
    int used;
    w = pd_peek(s, len, pos);
    const int sym = pd_decode(lit, w, &used);
    if (sym < 0) return -1;
    pos += used;
    w >>= used;
    if (sym < 16) {
      lengths[i++] = (unsigned char)sym;
      continue;
    }
    int rep, v = 0;
    if (sym == 16) {
      if (i == 0) return -1;
      v = lengths[i - 1];
      rep = 3 + (w & 3);
      pos += 2;
    } else if (sym == 17) {
      rep = 3 + (w & 7);
      pos += 3;
    } else {
      rep = 11 + (w & 127);
      pos += 7;
    }
    if (i + rep > n) return -1;
    while (rep--) lengths[i++] = (unsigned char)v;
  }
  if (lengths[256] == 0) return -1;
  int left = pd_build(lit, lengths, hlit, &mx);
  if (left < 0 || (left > 0 && mx != 1)) return -1;
  left = pd_build(dist, lengths + hlit, hdist, &mx);
  if (left < 0 || (left > 0 && mx > 1)) return -1;
  if (pos > 8 * len) return -1;
  return pos;
}

__device__ void pd_fixed(PdHuff& lit, PdHuff& dist) {
  unsigned char lengths[288];
  for (int i = 0; i < 288; ++i) lengths[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
  int mx;
  pd_build(lit, lengths, 288, &mx);
  for (int i = 0; i < 30; ++i) lengths[i] = 5;
  pd_build(dist, lengths, 30, &mx);
}

// outcome of decoding one block's symbols
enum { PD_OK = 0, PD_BAD = 1, PD_EARLY = 2, PD_CAP = 3, PD_FAR = 4 };

struct PdRun {
  int pos;       // bit after end-of-block, or where the failing element starts
  int out;       // bytes produced
  int err;       // PD_OK, ...
};

// the symbols of a Huffman block from bit pos.  out0 >= 0: the block's first output byte; then distances that reach
// before the stream's start are refused and, with refs, every byte below raw is written (see the file comment) and
// *horizon gets the bit after the symbol that produces byte raw - 1.  out0 < 0 (a probe): at most cap symbols.
__device__ PdRun pd_body(const unsigned char* s, int len, int pos, const PdHuff& lit, const PdHuff& dist, int out0,
                         int wsize, int cap, unsigned* refs, int raw, int* horizon) {
  PdRun r{pos, 0, PD_OK};
  const int end = 8 * len;
  for (int n = 0;; ++n) {
    if (cap && n >= cap) { r.err = PD_CAP; return r; }
    const int start = pos;
    unsigned w = pd_peek(s, len, pos);
    int used;
    const int sym = pd_decode_lut(lit, w, &used);
    if (sym < 0 || sym > 285) { r.pos = start; r.err = PD_BAD; return r; }
    pos += used;
    if (sym < 256) {
      if (pos > end) { r.pos = start; r.err = PD_EARLY; return r; }
      if (refs) {
        const int o = out0 + r.out;
        if (o < raw) refs[o] = PD_LIT | sym;
        if (o == raw - 1) *horizon = pos;
      }
      r.out++;
      continue;
    }
    if (sym == 256) {
      if (pos > end) { r.pos = start; r.err = PD_EARLY; return r; }
      r.pos = pos;
      return r;
    }
    w = pd_peek(s, len, pos);
    const int k = sym - 257;
    const int L = pd_len_base[k] + (w & ((1u << pd_len_extra[k]) - 1));
    pos += pd_len_extra[k];
    w = pd_peek(s, len, pos);
    const int dsym = pd_decode_lut(dist, w, &used);
    if (dsym < 0 || dsym > 29) { r.pos = start; r.err = PD_BAD; return r; }
    pos += used;
    const int D = pd_dist_base[dsym] + ((w >> used) & ((1u << pd_dist_extra[dsym]) - 1));
    pos += pd_dist_extra[dsym];
    if (pos > end) { r.pos = start; r.err = PD_EARLY; return r; }
    if (D > wsize || (out0 >= 0 && D > out0 + r.out)) { r.pos = start; r.err = PD_FAR; return r; }
    if (refs) {
      const int o = out0 + r.out;
      const int lim = min(L, raw - o);
      for (int i = 0; i < lim; ++i) refs[o + i] = (unsigned)(o - D + (D >= L ? i : i % D));
      if (o <= raw - 1 && raw - 1 < o + L) *horizon = pos;
    }
    r.out += L;
  }
}

__device__ __forceinline__ unsigned pd_hash(int key) { return ((unsigned)key * 2654435761u) >> 18; }  // 14 bits

// ------------------------------------------------------------------------------------------------ scan
__global__ void __launch_bounds__(PD_THREADS)
pd_scan_kernel(const __grid_constant__ PdParams P, const unsigned char* __restrict__ data, void* ws) {
  const int m = PD_FIND(P, scan0, blockIdx.x);
  const PdImage& d = P.img[m];
  const int pos = 16 + (blockIdx.x - d.scan0) * PD_THREADS + threadIdx.x;  // bits after the 2-byte zlib header
  if (pos + 17 > 8 * d.len) return;
  const unsigned char* s = data + d.src;
  const unsigned w = pd_peek(s, d.len, pos);
  if (((w >> 1) & 3) != 2 || (w >> 3 & 31) > 29 || (w >> 8 & 31) > 29) return;
  PdHuff lit, dist;
  if (pd_dynamic(s, d.len, pos + 3, lit, dist) < 0) return;
  int* meta = pd_at<int>(ws, d.o_meta);
  if (atomicAdd(meta + PM_NCAND, 1) >= PD_CANDIDATES) return;  // overflow: the link decodes the block serially
  int* keys = pd_at<int>(ws, d.o_keys);
  for (unsigned h = pd_hash(pos);; h = (h + 1) & (PD_SLOTS - 1))
    if (atomicCAS(keys + h, 0, pos + 1) == 0) return;
}

// ------------------------------------------------------------------------------------------------ probe
__global__ void __launch_bounds__(PD_THREADS)
pd_probe_kernel(const __grid_constant__ PdParams P, const unsigned char* __restrict__ data, void* ws) {
  const int m = PD_FIND(P, probe0, blockIdx.x);
  const PdImage& d = P.img[m];
  const int slot = (blockIdx.x - d.probe0) * PD_THREADS + threadIdx.x;
  const int key = pd_at<int>(ws, d.o_keys)[slot];
  if (key == 0) return;
  const unsigned char* s = data + d.src;
  PdHuff lit, dist;
  const int pos = pd_dynamic(s, d.len, key - 1 + 3, lit, dist);
  if (pos < 0) { pd_at<int2>(ws, d.o_res)[slot] = make_int2(-1, 0); return; }
  pd_lut(lit);
  pd_lut(dist);
  const PdRun r = pd_body(s, d.len, pos, lit, dist, -1, d.wsize, PD_PROBE_SYMBOLS, nullptr, 0, nullptr);
  pd_at<int2>(ws, d.o_res)[slot] = r.err == PD_OK ? make_int2(r.pos, r.out) : make_int2(-1, 0);
}

// ------------------------------------------------------------------------------------------------ link
// block record: x start bit, y type | final << 2 | (failing block) << 3, z output offset
__global__ void __launch_bounds__(32) pd_link_kernel(const __grid_constant__ PdParams P,
                                                     const unsigned char* __restrict__ data, void* ws) {
  if (threadIdx.x) return;
  const PdImage& d = P.img[blockIdx.x];
  const unsigned char* s = data + d.src;
  const int* keys = pd_at<int>(ws, d.o_keys);
  const int2* res = pd_at<int2>(ws, d.o_res);
  int4* blk = pd_at<int4>(ws, d.o_blk);
  int* meta = pd_at<int>(ws, d.o_meta);
  const int end = 8 * d.len;
  int pos = 16, out = 0, nb = 0, serial = 0, err = PD_OK, err_pos = 0, err_out = 0, trailer = 0;
  for (;;) {
    if (nb >= d.nblk || pos + 3 > end) { err = PD_EARLY; err_pos = pos; err_out = out; break; }
    const unsigned w = pd_peek(s, d.len, pos);
    const int final = w & 1, type = (w >> 1) & 3;
    blk[nb] = make_int4(pos, type | final << 2, out, 0);
    if (type == 3) { err = PD_BAD; err_pos = pos; err_out = out; blk[nb++].y |= 8; break; }
    int n = 0, next = -1;
    if (type == 0) {
      const int b = (pos + 3 + 7) >> 3;
      if (8 * (b + 4) > end) { err = PD_EARLY; err_pos = pos; err_out = out; blk[nb++].y |= 8; break; }
      const int ln = s[b] | s[b + 1] << 8, nln = s[b + 2] | s[b + 3] << 8;
      if (ln != (~nln & 0xFFFF)) { err = PD_BAD; err_pos = pos; err_out = out; blk[nb++].y |= 8; break; }
      if (8 * (b + 4 + ln) > end) { err = PD_EARLY; err_pos = pos; err_out = out + (end / 8 - b - 4);
                                    blk[nb++].y |= 8; break; }
      n = ln;
      next = 8 * (b + 4 + ln);
    } else {
      if (type == 2) {
        for (unsigned h = pd_hash(pos), i = 0; i < PD_SLOTS; h = (h + 1) & (PD_SLOTS - 1), ++i) {
          const int k = keys[h];
          if (k == 0) break;
          if (k == pos + 1) {
            if (res[h].x >= 0) { next = res[h].x; n = res[h].y; }
            break;
          }
        }
      }
      if (next < 0) {  // decode serially
        PdHuff lit, dist;
        int p = pos + 3;
        if (type == 1) {
          pd_fixed(lit, dist);
        } else {
          p = pd_dynamic(s, d.len, p, lit, dist);
        }
        if (p < 0) { err = PD_BAD; err_pos = pos; err_out = out; blk[nb++].y |= 8; break; }
        pd_lut(lit);
        pd_lut(dist);
        const PdRun r = pd_body(s, d.len, p, lit, dist, out, d.wsize, 0, nullptr, 0, nullptr);
        if (r.err != PD_OK) {
          err = r.err; err_pos = r.pos; err_out = out + r.out; blk[nb++].y |= 8;
          break;
        }
        next = r.pos;
        n = r.out;
        ++serial;
      }
    }
    ++nb;
    out += n;
    pos = next;
    if (final) {
      const int b = (pos + 7) >> 3;
      if (b + 4 > d.len) { err = PD_EARLY; err_pos = pos; err_out = out; }
      else trailer = b;
      break;
    }
  }
  meta[PM_NBLK] = nb;
  meta[PM_TOTAL] = out;
  meta[PM_ERR] = err;
  meta[PM_ERR_OUT] = err_out;
  meta[PM_ERR_BIT] = err_pos;
  meta[PM_TRAILER] = trailer;
  meta[PM_SERIAL] = serial;
}

// ------------------------------------------------------------------------------------------------ inflate
// one true block k (see pd_link_kernel): its bytes below raw into refs
__device__ void pd_inflate_block(const PdImage& d, const unsigned char* __restrict__ data, void* ws, int* meta, int4 k) {
  const unsigned char* s = data + d.src;
  unsigned* refs = pd_at<unsigned>(ws, d.o_refs);
  const int type = k.y & 3, out0 = k.z;
  if (out0 >= d.raw) return;
  int horizon = -1;
  if (type == 0) {
    if (k.y & 8) return;
    const int bb = (k.x + 3 + 7) >> 3;
    const int ln = s[bb] | s[bb + 1] << 8;
    const int lim = min(ln, d.raw - out0);
    for (int i = 0; i < lim; ++i) refs[out0 + i] = PD_LIT | s[bb + 4 + i];
    if (out0 + ln >= d.raw) horizon = 8 * (bb + 4 + d.raw - out0);
  } else if (type != 3) {
    PdHuff lit, dist;
    int p = k.x + 3;
    if (type == 1) pd_fixed(lit, dist);
    else p = pd_dynamic(s, d.len, p, lit, dist);
    if (p < 0) return;
    pd_lut(lit);
    pd_lut(dist);
    const PdRun r = pd_body(s, d.len, p, lit, dist, out0, d.wsize, 0, refs, d.raw, &horizon);
    if (r.err == PD_FAR) atomicMax(meta + PM_FAR, 0x7FFFFFFF - (out0 + r.out));
  }
  if (horizon >= 0) meta[PM_HORIZON] = horizon;
}

// each warp of the image's PD_INFLATE_CTAS blocks takes true blocks warp, warp + 128, ...; lane 0 decodes: the serial
// decodes diverge, so two of them in one warp would run in turn
__global__ void __launch_bounds__(PD_THREADS)
pd_inflate_kernel(const __grid_constant__ PdParams P, const unsigned char* __restrict__ data, void* ws) {
  const int m = PD_FIND(P, inf0, blockIdx.x);
  const PdImage& d = P.img[m];
  if (threadIdx.x & 31) return;
  int* meta = pd_at<int>(ws, d.o_meta);
  const int nb = meta[PM_NBLK];
  for (int b = (blockIdx.x - d.inf0) * (PD_THREADS / 32) + (threadIdx.x >> 5); b < nb;
       b += PD_INFLATE_CTAS * (PD_THREADS / 32))
    pd_inflate_block(d, data, ws, meta, pd_at<int4>(ws, d.o_blk)[b]);
}

// ------------------------------------------------------------------------------------------------ resolve
__global__ void __launch_bounds__(PD_THREADS) pd_resolve_kernel(const __grid_constant__ PdParams P, void* ws) {
  const int m = PD_FIND(P, res0, blockIdx.x);
  const PdImage& d = P.img[m];
  const int i = (blockIdx.x - d.res0) * PD_THREADS + threadIdx.x;
  if (i >= d.raw) return;
  unsigned* refs = pd_at<unsigned>(ws, d.o_refs);
  const unsigned v = refs[i];
  if (v & PD_LIT) return;
  // a source at or after i is a byte no block wrote (a failed image): a literal 0 keeps every read in bounds
  refs[i] = v < (unsigned)i ? __ldcg(refs + v) : PD_LIT;
}

// ------------------------------------------------------------------------------------------------ finish
__device__ __forceinline__ long long pd_piece(const int* starts, int n, int byte) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (starts[mid] <= byte) lo = mid; else hi = mid - 1;
  }
  return ((long long)lo << 32) | ((byte - starts[lo]) / PD_READ_SIZE);
}

__global__ void __launch_bounds__(1024)
pd_finish_kernel(const __grid_constant__ PdParams P, const unsigned char* __restrict__ data,
                 const int* __restrict__ idat, void* ws, unsigned char* __restrict__ out, int* status) {
  __shared__ unsigned long long sa[32], sb[32];
  __shared__ volatile int progress[32];
  const PdImage& d = P.img[blockIdx.x];
  const int* meta = pd_at<int>(ws, d.o_meta);
  const unsigned* refs = pd_at<unsigned>(ws, d.o_refs);
  const int T = meta[PM_TOTAL], raw = d.raw;
  // Adler-32 of the rows' bytes: thread t sums a contiguous run (s1 = sum, s2 = sum of (run end - index) * byte)
  const int per = (raw + blockDim.x - 1) / blockDim.x;
  const int i0 = min(raw, (int)threadIdx.x * per), i1 = min(raw, i0 + per);
  unsigned long long s1 = 0, s2 = 0;
  if (T >= raw && meta[PM_ERR] == PD_OK) {
    for (int i = i0; i < i1; ++i) {
      const unsigned v = refs[i] & 0xFF;
      s1 += v;
      s2 += (unsigned long long)(i1 - i) * v;
    }
  }
  s1 %= 65521;
  s2 = (s2 + s1 * (unsigned long long)(raw - i1)) % 65521;  // weight of the bytes after the run
  for (int o = 16; o; o >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if ((threadIdx.x & 31) == 0) { sa[threadIdx.x >> 5] = s1; sb[threadIdx.x >> 5] = s2; }
  if (threadIdx.x < 32) progress[threadIdx.x] = 0;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long A = 1, B = raw;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) { A += sa[k]; B += sb[k]; }
    A %= 65521;
    B %= 65521;
    int st = 0;
    const int err = meta[PM_ERR], far = meta[PM_FAR];
    int eo = err != PD_OK ? meta[PM_ERR_OUT] : 0x7FFFFFFF;
    const int fo = far ? 0x7FFFFFFF - far : 0x7FFFFFFF;
    const int* starts = idat + d.idat0;
    const int hz = meta[PM_HORIZON];
    if (fo < eo && fo < raw) {
      st = PD_E_DATA;
    } else if (fo < eo) {
      // a distance too far back once the rows are complete: benign for libpng
    } else if (err != PD_OK) {
      if (eo < raw) st = err == PD_EARLY ? PD_E_SHORT : PD_E_DATA;
      else if (err == PD_EARLY) st = PD_E_SHORT;
      else if (err == PD_BAD && eo == raw &&
               pd_piece(starts, d.nidat, meta[PM_ERR_BIT] >> 3) == pd_piece(starts, d.nidat, (hz - 1) >> 3))
        st = PD_E_DATA;  // zlib decodes the bad symbol or header in the call that fills the last row
    } else if (T < raw) {
      st = PD_E_SHORT;
    } else if (T == raw) {
      const int t = meta[PM_TRAILER];
      const unsigned char* s = data + d.src + t;
      const unsigned want = (unsigned)s[0] << 24 | (unsigned)s[1] << 16 | (unsigned)s[2] << 8 | s[3];
      if (want != (unsigned)(B << 16 | A) &&
          pd_piece(starts, d.nidat, t + 3) == pd_piece(starts, d.nidat, (hz - 1) >> 3))
        st = PD_E_ADLER;
    }
    status[2 * blockIdx.x] = st;
    status[2 * blockIdx.x + 1] = meta[PM_SERIAL];
  }
  __syncthreads();
  // unfilter: warp w takes rows 32 (w + nw k) + lane for k = 0, 1, ...; lane l handles pixel x at step x + l
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int W = d.W, stride = 1 + 3 * W;
  unsigned char* frame = out + d.out;
  int bad = 0;
  for (int g = 0; 32 * (wid + nw * g) < d.H; ++g) {
    const int grp = wid + nw * g;
    const int y = 32 * grp + lane;
    const bool live = y < d.H;
    const int f = live ? (refs[(long long)y * stride] & 0xFF) : 0;
    if (f > 4) bad = 1;
    const unsigned* row = refs + (long long)y * stride + 1;
    int l0 = 0, l1 = 0, l2 = 0;      // left pixel (this row)
    int u0 = 0, u1 = 0, u2 = 0;      // last pixel this lane produced: the next lane's "above"
    int q0 = 0, q1 = 0, q2 = 0;      // the one before: the next lane's "above-left"
    const int prev_warp = (wid + nw - 1) % nw;
    for (int step = 0; step < W + 31; ++step) {
      const int x = step - lane;
      // above and above-left from lane - 1 (its pixels x and x - 1 of the row above)
      int a0 = __shfl_up_sync(0xffffffffu, u0, 1), a1 = __shfl_up_sync(0xffffffffu, u1, 1),
          a2 = __shfl_up_sync(0xffffffffu, u2, 1);
      int c0 = __shfl_up_sync(0xffffffffu, q0, 1), c1 = __shfl_up_sync(0xffffffffu, q1, 1),
          c2 = __shfl_up_sync(0xffffffffu, q2, 1);
      if (live && x >= 0 && x < W) {
        if (lane == 0) {
          if (y == 0) {
            a0 = a1 = a2 = c0 = c1 = c2 = 0;
          } else {
            const int want = (grp - 1) * (W + 1) + x + 1;
            while (progress[prev_warp] < want) {}
            __threadfence_block();
            const volatile unsigned char* up = frame + ((long long)(y - 1) * W + x) * 3;
            a2 = up[0]; a1 = up[1]; a0 = up[2];
            if (x > 0) { c2 = up[-3]; c1 = up[-2]; c0 = up[-1]; }
            else c0 = c1 = c2 = 0;
          }
        }
        if (x == 0) c0 = c1 = c2 = 0;
        const int r0 = row[3 * x] & 0xFF, r1 = row[3 * x + 1] & 0xFF, r2 = row[3 * x + 2] & 0xFF;
        int v[3];
        const int rr[3] = {r0, r1, r2}, aa[3] = {a0, a1, a2}, cc[3] = {c0, c1, c2}, ll[3] = {l0, l1, l2};
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int left = ll[c], upv = aa[c], ul = cc[c];
          int p;
          if (f == 0) p = 0;
          else if (f == 1) p = left;
          else if (f == 2) p = upv;
          else if (f == 3) p = (left + upv) >> 1;
          else {
            const int pp = left + upv - ul, pa = abs(pp - left), pb = abs(pp - upv), pc = abs(pp - ul);
            p = (pa <= pb && pa <= pc) ? left : (pb <= pc ? upv : ul);
          }
          v[c] = (rr[c] + p) & 0xFF;
        }
        unsigned char* o = frame + ((long long)y * W + x) * 3;
        o[0] = (unsigned char)v[2];
        o[1] = (unsigned char)v[1];
        o[2] = (unsigned char)v[0];
        q0 = u0; q1 = u1; q2 = u2;
        u0 = l0 = v[0]; u1 = l1 = v[1]; u2 = l2 = v[2];
        if (lane == 31 || y == d.H - 1) {
          __threadfence_block();
          progress[wid] = grp * (W + 1) + x + 1;
        }
      }
    }
  }
  bad = __any_sync(0xffffffffu, bad);
  if (bad && lane == 0) atomicOr(status + 2 * blockIdx.x, PD_E_FILTER);
}

// ------------------------------------------------------------------------------------------------ host side
inline long long pd_align(long long n) { return (n + 15) & ~15LL; }

// geom (M, 4): H, W, stream bytes, CINFO; streams (M): byte offset in data; idat_counts (M): IDAT chunks per image
inline int pd_layout(const long long* streams, const int* geom, const int* idat_counts, int M, PdParams* P,
                     size_t* bytes, long long* zero_bytes, long long* grids /*scan, probe, inflate, resolve*/) {
  if (!streams || !geom || !idat_counts || M < 1 || M > PD_MAX_IMAGES) return OCC_EINVAL;
  long long zero = 0, rest = 0, g[4] = {0, 0, 0, 0}, ic = 0;
  for (int m = 0; m < M; ++m) {
    PdImage& d = P->img[m];
    const int H = geom[4 * m], W = geom[4 * m + 1], len = geom[4 * m + 2], cinfo = geom[4 * m + 3];
    if (H < 1 || W < 1 || H > 16384 || W > 16384 || len < 7 || len >= (1 << 27) || cinfo < 0 || cinfo > 7 ||
        streams[m] < 0 || idat_counts[m] < 1 || idat_counts[m] > len)
      return OCC_EINVAL;
    d.src = streams[m];
    d.H = H; d.W = W; d.len = len; d.wsize = 1 << (cinfo + 8);
    d.raw = H * (1 + 3 * W);
    d.nblk = (int)((8LL * len) / 10 + 2);  // every block takes at least 10 bits (a fixed block's header and EOB)
    d.idat0 = (int)ic; d.nidat = idat_counts[m];
    ic += idat_counts[m];
    d.o_keys = zero; zero += 4LL * PD_SLOTS;
    d.o_meta = zero; zero += 4LL * PM_COUNT;
    d.o_res = rest;  rest += 8LL * PD_SLOTS;
    d.o_blk = rest;  rest += 16LL * d.nblk;
    d.o_refs = rest; rest += pd_align(4LL * d.raw);
    d.scan0 = (int)g[0];  g[0] += (8LL * (len - 2) + PD_THREADS - 1) / PD_THREADS;
    d.probe0 = (int)g[1]; g[1] += PD_SLOTS / PD_THREADS;
    d.inf0 = (int)g[2];   g[2] += PD_INFLATE_CTAS;
    d.res0 = (int)g[3];   g[3] += (d.raw + PD_THREADS - 1) / PD_THREADS;
  }
  for (int k = 0; k < 4; ++k) {
    if (g[k] >= (1LL << 31)) return OCC_EINVAL;
    if (grids) grids[k] = g[k];
  }
  for (int m = 0; m < M; ++m) {
    P->img[m].o_res += zero; P->img[m].o_blk += zero; P->img[m].o_refs += zero;
  }
  P->M = M;
  *zero_bytes = zero;
  *bytes = (size_t)(zero + rest);
  return OCC_OK;
}

}  // namespace occ

using namespace occ;

extern "C" size_t occ_decode_png_workspace_bytes(const long long* streams, const int* geom, const int* idat_counts,
                                                 int M) {
  PdParams P;
  size_t bytes = 0;
  long long zero;
  return pd_layout(streams, geom, idat_counts, M, &P, &bytes, &zero, nullptr) == OCC_OK ? bytes : 0;
}

extern "C" int occ_decode_png(const unsigned char* data, long long data_bytes, const long long* streams,
                              const int* geom, const int* idat_counts, const int* idat, long long idat_len,
                              const long long* out_offsets, int M, void* ws, size_t ws_bytes, unsigned char* out,
                              long long out_bytes, int* status, cudaStream_t stream) {
  OCC_REQUIRE(data && streams && geom && idat_counts && idat && out_offsets && out && status && ws);
  OCC_REQUIRE(data_bytes >= 0 && out_bytes >= 0 && idat_len >= 0);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 15) == 0);
  PdParams P;
  size_t need = 0;
  long long grids[4], zero = 0;
  const int rc = pd_layout(streams, geom, idat_counts, M, &P, &need, &zero, grids);
  if (rc != OCC_OK) {
    fprintf(stderr, "occ_b200: occ_decode_png: bad image count, geometry, stream length or IDAT count\n");
    return rc;
  }
  OCC_REQUIRE(ws_bytes >= need);
  long long nidat = 0;
  for (int m = 0; m < M; ++m) {
    PdImage& d = P.img[m];
    OCC_REQUIRE(d.src + d.len <= data_bytes);
    OCC_REQUIRE(out_offsets[m] >= 0 && out_offsets[m] <= out_bytes &&
                (long long)d.H * d.W * 3 <= out_bytes - out_offsets[m]);
    d.out = out_offsets[m];
    nidat += d.nidat;
  }
  OCC_REQUIRE(nidat <= idat_len);
  OCC_MEMSET(status, 0, sizeof(int) * 2 * M, stream);
  OCC_MEMSET(ws, 0, (size_t)zero, stream);
  pd_scan_kernel<<<(unsigned)grids[0], PD_THREADS, 0, stream>>>(P, data, ws);
  OCC_LAUNCH_CHECK();
  pd_probe_kernel<<<(unsigned)grids[1], PD_THREADS, 0, stream>>>(P, data, ws);
  OCC_LAUNCH_CHECK();
  pd_link_kernel<<<M, 32, 0, stream>>>(P, data, ws);
  OCC_LAUNCH_CHECK();
  pd_inflate_kernel<<<(unsigned)grids[2], PD_THREADS, 0, stream>>>(P, data, ws);
  OCC_LAUNCH_CHECK();
  for (int r = 0; r < PD_RESOLVE_ROUNDS; ++r) {
    pd_resolve_kernel<<<(unsigned)grids[3], PD_THREADS, 0, stream>>>(P, ws);
    OCC_LAUNCH_CHECK();
  }
  pd_finish_kernel<<<M, 1024, 0, stream>>>(P, data, idat, ws, out, status);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
