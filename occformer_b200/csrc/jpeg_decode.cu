// Baseline JPEG decoding on the device, bit for bit as cv2.imdecode(buf, IMREAD_UNCHANGED) (libjpeg-turbo: islow IDCT,
// fancy upsampling, integer YCbCr -> RGB) -- the camera files of LoadMultiViewImageFromFiles_OccFormer
// (P/datasets/pipelines/loading_nusc_imgs.py:181-195, mmcv.imread's cv2 backend).  include/occ_b200.h states the
// semantics; occformer_b200/jpeg.py parses the headers and builds the tables on the host.
//
// Every image's entropy-coded segment goes through these launches, all images of the call together:
//   count    per 4 KB chunk of a segment: bytes kept after removing FF00 stuffing, RSTn markers and fill bytes, and the
//            number of RSTn markers; any other marker flags the image
//   scan     per image: exclusive prefix sums of the chunk counts; the RSTn count must be the interval count - 1
//   compact  per chunk: the kept bytes to the image's unstuffed stream, and each RSTn's position there (the start of
//            the next restart interval); RSTn numbers must run 0..7 in order
//   plan     per image: every restart interval (the whole scan without DRI) is cut into subsequences of S bits; prefix
//            sums give each interval's first subsequence
//   sync     R rounds, one thread per subsequence.  The decoder state at a bit position is (position, block in MCU,
//            zig-zag index).  Round 0 starts every subsequence but an interval's first at its first bit with
//            (block 0, index 0), a guess; round r starts subsequence i at the state where i - 1 ended in round r - 1.
//            Each round records where every subsequence ends and how many blocks start in it.  An interval's first
//            subsequence starts exactly, so when every subsequence starts where its predecessor ended the states are
//            exact by induction.  Huffman codes resynchronise after a few symbols, but the block-in-MCU index only by chance
//            (its tables differ between luma and chroma), so subsequences are long (4096 bits by default) and the
//            rounds several (6).
//   fixup    one warp per interval walks its subsequences in order: a run whose start agrees with its predecessor's
//            exit in the last round is taken as it is, any other subsequence is decoded again on one thread from the
//            exact exit of its predecessor.  The result is exact for every stream, whatever R; only streams that
//            resynchronise slowly (or R = 0) decode serially.  Prefix sums of the block counts give every subsequence's
//            first output block; an interval with fewer blocks than its MCUs need flags the image
//   decode   one thread per subsequence from its exact start: de-zigzagged int16 coefficients (DC differences) into
//            the zeroed coefficient buffer; invalid codes, runs past coefficient 63 and blocks that run past the end of
//            their interval's data flag the image, and nothing is written outside the image's own blocks
//   dc       per (image, component): segmented prefix sum of the DC differences, restarting at every interval
//   idct     8 threads per block: dequantisation and the islow IDCT, output + 128 clamped to [0, 255] (libjpeg-turbo's
//            SIMD IDCT saturates; its portable C table would wrap from +-512 on), into MCU-padded component planes
//   colour   per output pixel: fancy h2v1 / h2v2 chroma upsampling with the edges replicated at the component's real
//            (downsampled) size, libjpeg's YCbCr -> RGB, written as B, G, R
// plus two memsets (status words, coefficients): 11 + R operations whatever the data and the number of images, no host
// synchronisation, capturable in a CUDA graph.
#include "occ_common.cuh"

namespace occ {

constexpr int JD_MAX_IMAGES = 96;
constexpr int JD_CHUNK = 4096;                    // stuffed bytes per count / compact block
constexpr int JD_CHUNK_THREADS = 256;             // 16 bytes per thread
constexpr int JD_SEQ_THREADS = 128;               // subsequences per sync / decode block
constexpr int JD_FIX_WARPS = 4;                   // intervals per fixup block
constexpr int JD_IDCT_BLOCKS = 32;                // 8 x 8 blocks per idct block (8 threads each)
constexpr int JD_COLOUR_THREADS = 256;

// status bits (include/occ_b200.h)
constexpr int JD_E_MARKER = 1;     // a marker other than RSTn inside the entropy-coded segment
constexpr int JD_E_RESTART = 2;    // RSTn markers missing, surplus or out of order
constexpr int JD_E_CODE = 4;       // an invalid Huffman code or a run past coefficient 63
constexpr int JD_E_SHORT = 8;      // the data of an interval ends before its last MCU

__constant__ unsigned char jd_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                            12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                            35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                            58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct JdImage {
  long long src;                 // byte offset of the entropy-coded segment in `data`
  long long out;                 // byte offset of the (H, W, 3) frame in `out`
  const int* qt[3];              // quantisation tables, 64 ints in natural order
  const int* huff[3][2];         // [component][DC, AC] flat Huffman tables (occformer_b200.jpeg.HUFF_INTS ints)
  long long o_blk, o_u, o_q, o_sb, o_meta, o_e0, o_e1, o_f, o_cnt, o_base, o_pl[3];  // workspace byte offsets
  long long coef;                // first block of the image in the coefficient area (blocks)
  int len;                       // segment bytes
  int W, H, hs, vs, ri, nint, mcux, mcuy, bpm, cap;
  int chunk0, seq0, fix0, idct0, col0;  // the image's first block in each grid
};

struct JdParams {
  JdImage img[JD_MAX_IMAGES];
  int M;
};

// the image whose first block (field `f` of JdImage) is the largest not above b
#define JD_FIND(P, field, b)                                        \
  ([&]() {                                                          \
    int lo__ = 0, hi__ = (P).M - 1;                                 \
    while (lo__ < hi__) {                                           \
      const int mid__ = (lo__ + hi__ + 1) >> 1;                     \
      if ((P).img[mid__].field <= (int)(b)) lo__ = mid__; else hi__ = mid__ - 1; \
    }                                                               \
    return lo__;                                                    \
  }())

template <typename T>
__device__ __forceinline__ T* jd_at(void* ws, long long off) {
  return reinterpret_cast<T*>(static_cast<unsigned char*>(ws) + off);
}

// ------------------------------------------------------------------------------------------------ block scans
// inclusive sum over the block of v (all threads must call); *total = the block's sum
template <int NT>
__device__ __forceinline__ int jd_block_scan(int v, int* sh, int* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int o = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v += o;
  }
  if (lane == 31) sh[w] = v;
  __syncthreads();
  if (w == 0) {
    int s = lane < NT / 32 ? sh[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += o;
    }
    if (lane < NT / 32) sh[lane] = s;
  }
  __syncthreads();
  const int r = v + (w ? sh[w - 1] : 0);
  *total = sh[NT / 32 - 1];
  __syncthreads();
  return r;
}

// ------------------------------------------------------------------------------------------------ unstuffing
// byte i of the segment s[0, n): kept, an RSTn (at its FF), or a bad marker
__device__ __forceinline__ void jd_classify(const unsigned char* s, int n, int i, bool* keep, int* rst, bool* bad) {
  const int c = s[i];
  *keep = false;
  *rst = -1;
  *bad = false;
  if (c == 0xFF) {
    const int nx = i + 1 < n ? s[i + 1] : 0xFF;  // the segment ends at the EOI marker's FF (or the end of the file)
    if (nx == 0x00) *keep = true;
    else if (nx >= 0xD0 && nx <= 0xD7) *rst = nx & 7;
    else if (nx != 0xFF) *bad = true;           // FF FF: a fill byte
  } else {
    *keep = !(i > 0 && s[i - 1] == 0xFF);       // the byte after an FF: stuffing or a marker number
  }
}

__global__ void __launch_bounds__(JD_CHUNK_THREADS)
jd_count_kernel(const __grid_constant__ JdParams P, const unsigned char* __restrict__ data, void* ws, int* status) {
  __shared__ int sh[32];
  const int m = JD_FIND(P, chunk0, blockIdx.x);
  const JdImage& d = P.img[m];
  const int c = blockIdx.x - d.chunk0;
  const unsigned char* s = data + d.src;
  int keep = 0, rst = 0, bad = 0;
  const int i0 = c * JD_CHUNK + threadIdx.x * (JD_CHUNK / JD_CHUNK_THREADS);
  for (int t = 0; t < JD_CHUNK / JD_CHUNK_THREADS; ++t) {
    const int i = i0 + t;
    if (i >= d.len) break;
    bool k, b;
    int r;
    jd_classify(s, d.len, i, &k, &r, &b);
    keep += k;
    rst += r >= 0;
    bad |= b;
  }
  if (bad) atomicOr(status + 2 * m, JD_E_MARKER);
  int tk, tr;
  jd_block_scan<JD_CHUNK_THREADS>(keep, sh, &tk);
  jd_block_scan<JD_CHUNK_THREADS>(rst, sh, &tr);
  if (threadIdx.x == 0) {
    int* blk = jd_at<int>(ws, d.o_blk);
    blk[2 * c] = tk;
    blk[2 * c + 1] = tr;
  }
}

// one block per image: exclusive prefix sums of the chunk counts; q[0] = 0, q[nint] = unstuffed length
__global__ void __launch_bounds__(1024) jd_scan_kernel(const __grid_constant__ JdParams P, void* ws, int* status) {
  __shared__ int sh[32];
  const int m = blockIdx.x;
  const JdImage& d = P.img[m];
  int* blk = jd_at<int>(ws, d.o_blk);
  const int n = (d.len + JD_CHUNK - 1) / JD_CHUNK;
  int ck = 0, cr = 0;
  for (int b0 = 0; b0 < n; b0 += 1024) {
    const int i = b0 + threadIdx.x;
    const int k = i < n ? blk[2 * i] : 0, r = i < n ? blk[2 * i + 1] : 0;
    int tk, tr;
    const int ik = jd_block_scan<1024>(k, sh, &tk);
    const int ir = jd_block_scan<1024>(r, sh, &tr);
    if (i < n) {
      blk[2 * i] = ck + ik - k;
      blk[2 * i + 1] = cr + ir - r;
    }
    ck += tk;
    cr += tr;
  }
  if (threadIdx.x == 0) {
    int* q = jd_at<int>(ws, d.o_q);
    q[0] = 0;
    q[d.nint] = ck;
    jd_at<int>(ws, d.o_meta)[0] = ck;
    if (cr != d.nint - 1) atomicOr(status + 2 * m, JD_E_RESTART);
  }
}

__global__ void __launch_bounds__(JD_CHUNK_THREADS)
jd_compact_kernel(const __grid_constant__ JdParams P, const unsigned char* __restrict__ data, void* ws, int* status) {
  __shared__ int sh[32];
  const int m = JD_FIND(P, chunk0, blockIdx.x);
  const JdImage& d = P.img[m];
  const int c = blockIdx.x - d.chunk0;
  const unsigned char* s = data + d.src;
  constexpr int PER = JD_CHUNK / JD_CHUNK_THREADS;
  const int i0 = c * JD_CHUNK + threadIdx.x * PER;
  unsigned keepmask = 0, rstmask = 0;
  int keep = 0, rst = 0;
  for (int t = 0; t < PER; ++t) {
    const int i = i0 + t;
    if (i >= d.len) break;
    bool k, b;
    int r;
    jd_classify(s, d.len, i, &k, &r, &b);
    keepmask |= (unsigned)k << t;
    rstmask |= (unsigned)(r >= 0) << t;
    keep += k;
    rst += r >= 0;
  }
  int tk, tr;
  const int* blk = jd_at<int>(ws, d.o_blk);
  int pk = blk[2 * c] + jd_block_scan<JD_CHUNK_THREADS>(keep, sh, &tk) - keep;
  int pr = blk[2 * c + 1] + jd_block_scan<JD_CHUNK_THREADS>(rst, sh, &tr) - rst;
  unsigned char* u = jd_at<unsigned char>(ws, d.o_u);
  int* q = jd_at<int>(ws, d.o_q);
  for (int t = 0; t < PER; ++t) {
    const int i = i0 + t;
    if (keepmask >> t & 1) u[pk++] = s[i];
    if (rstmask >> t & 1) {
      if ((s[i + 1] & 7) != (pr & 7)) atomicOr(status + 2 * m, JD_E_RESTART);
      if (pr + 1 < d.nint) q[pr + 1] = pk;
      ++pr;
    }
  }
}

// one block per image: subsequences per interval and their prefix sums (nothing to decode after an unstuffing error)
__global__ void __launch_bounds__(1024) jd_plan_kernel(const __grid_constant__ JdParams P, void* ws, const int* status,
                                                       int S) {
  __shared__ int sh[32];
  const int m = blockIdx.x;
  const JdImage& d = P.img[m];
  const bool ok = status[2 * m] == 0;
  const int* q = jd_at<int>(ws, d.o_q);
  int* sb = jd_at<int>(ws, d.o_sb);
  int carry = 0;
  for (int k0 = 0; k0 < d.nint; k0 += 1024) {
    const int k = k0 + threadIdx.x;
    int n = 0;
    if (k < d.nint && ok) {
      const long long bits = 8LL * (q[k + 1] - q[k]);
      n = bits <= S ? 1 : (int)((bits + S - 1) / S);
    }
    int t;
    const int inc = jd_block_scan<1024>(n, sh, &t);
    if (k < d.nint) sb[k] = carry + inc - n;
    carry += t;
  }
  if (threadIdx.x == 0) {
    sb[d.nint] = carry;
    jd_at<int>(ws, d.o_meta)[1] = carry <= d.cap ? carry : 0;
  }
}

// ------------------------------------------------------------------------------------------------ Huffman decoding
struct JdHuff {
  unsigned short lut[512];
  int maxcode[18];
  int valoff[17];
  unsigned char val[256];
};

struct JdTables {
  JdHuff h[3][2];  // [component][DC, AC]
};

__device__ void jd_load_tables(const JdImage& d, JdTables& T) {
  for (int t = 0; t < 6; ++t) {
    const int* g = d.huff[t >> 1][t & 1];
    JdHuff& h = T.h[t >> 1][t & 1];
    for (int i = threadIdx.x; i < 512; i += blockDim.x) h.lut[i] = (unsigned short)__ldg(g + i);
    for (int i = threadIdx.x; i < 18; i += blockDim.x) h.maxcode[i] = __ldg(g + 512 + i);
    for (int i = threadIdx.x; i < 17; i += blockDim.x) h.valoff[i] = __ldg(g + 530 + i);
    for (int i = threadIdx.x; i < 256; i += blockDim.x) h.val[i] = (unsigned char)__ldg(g + 547 + i);
  }
  __syncthreads();
}

typedef unsigned long long JdState;  // (block in MCU << 8 | zig-zag index) << 32 | bit position

__device__ __forceinline__ JdState jd_state(unsigned p, int b, int z) {
  return ((JdState)(unsigned)((b << 8) | z) << 32) | p;
}

// big-endian 32-bit word w of the unstuffed stream u[0, n), zero past its end
__device__ __forceinline__ unsigned jd_word(const unsigned char* u, int n, int w) {
  const int b = 4 * w;
  if (b >= n) return 0;
  const unsigned x = __byte_perm(*reinterpret_cast<const unsigned*>(u + b), 0, 0x0123);
  return b + 4 <= n ? x : x & (0xFFFFFFFFu << (8 * (b + 4 - n)));
}

__device__ __forceinline__ unsigned jd_peek(const unsigned char* u, int n, unsigned p) {
  const int w = (int)(p >> 5), sh = p & 31;
  const unsigned hi = jd_word(u, n, w);
  return sh ? (hi << sh) | (jd_word(u, n, w + 1) >> (32 - sh)) : hi;
}

struct JdWrite {           // what the decode pass needs to write and check
  short* coef;             // the interval's first block
  int rel;                 // block (relative to the interval) of the first block that starts in the subsequence
  int expected;            // blocks of the interval
  unsigned iend;           // bit where the interval's data ends
  int* err;                // the image's status word
};

// Decodes the symbols that start in [p, end) from state (p, b, z) -> the state after them; *blocks = DC symbols
// decoded.  Without W (sync, fixup) an invalid code or run is taken as the end of its block, so that any start state
// yields some exit state; with W (decode) the same happens, and within the interval's real blocks it flags the image.
template <bool W>
__device__ JdState jd_walk(const JdTables& T, const unsigned char* u, int n, unsigned p, int b, int z, unsigned end,
                           int bpm, int ny, int* blocks, const JdWrite* wr) {
  int count = 0;
  int blk = W ? wr->rel - 1 : 0;  // the block being decoded (relative to the interval)
  while (p < end) {
    const int comp = b < ny ? 0 : b - ny + 1;
    const JdHuff& h = T.h[comp][z ? 1 : 0];
    const unsigned v = jd_peek(u, n, p);
    int len, sym;
    const unsigned e = h.lut[v >> 23];
    if (e) {
      len = e >> 8;
      sym = e & 255;
    } else {
      len = 0;
      sym = 0;
#pragma unroll 1
      for (int l = 10; l <= 16; ++l) {
        const int code = (int)(v >> (32 - l));
        if (code <= h.maxcode[l]) {
          len = l;
          sym = h.val[(code + h.valoff[l]) & 255];
          break;
        }
      }
    }
    if (z == 0) {
      ++count;
      if (W) ++blk;
    }
    const bool real = W && blk >= 0 && blk < wr->expected;
    if (len == 0) {  // invalid code
      if (real) atomicOr(wr->err, JD_E_CODE);
      p += 1;
      z = 0;
      b = b + 1 == bpm ? 0 : b + 1;
      continue;
    }
    const int s = sym & 15, r = z ? sym >> 4 : 0;
    const int val = s ? (int)((v << len) >> (32 - s)) : 0;
    const int x = s && val < (1 << (s - 1)) ? val - (1 << s) + 1 : val;
    p += len + s;
    if (real && p > wr->iend) atomicOr(wr->err, JD_E_SHORT);
    if (z == 0) {
      if (real) wr->coef[(long long)blk * 64] = (short)x;
      z = 1;
    } else if (s) {
      z += r;
      if (z > 63) {
        if (real) atomicOr(wr->err, JD_E_CODE);
        z = 64;
      } else {
        if (real) wr->coef[(long long)blk * 64 + jd_zigzag[z]] = (short)x;
        ++z;
      }
    } else if (r == 15) {
      z += 16;
      if (z > 64) {
        if (real) atomicOr(wr->err, JD_E_CODE);
        z = 64;
      }
    } else {
      z = 64;  // EOB
    }
    if (z == 64) {
      z = 0;
      b = b + 1 == bpm ? 0 : b + 1;
    }
  }
  *blocks = count;
  return jd_state(p, b, z);
}

struct JdInterval {
  int k, a, b;            // interval, its subsequences [a, b) (image-local)
  unsigned start, end;    // its data in bits
  int expected;           // its blocks
  long long first;        // its first block (image-local)
};

__device__ __forceinline__ JdInterval jd_interval(const JdImage& d, void* ws, int k) {
  const int* q = jd_at<int>(ws, d.o_q);
  const int* sb = jd_at<int>(ws, d.o_sb);
  JdInterval I;
  I.k = k;
  I.a = sb[k];
  I.b = sb[k + 1];
  I.start = 8u * (unsigned)q[k];
  I.end = 8u * (unsigned)q[k + 1];
  const int per = d.ri ? d.ri : d.mcux * d.mcuy;
  const long long mcu0 = (long long)k * per;
  const long long left = (long long)d.mcux * d.mcuy - mcu0;
  I.expected = (int)((left < per ? left : per) * d.bpm);
  I.first = mcu0 * d.bpm;
  return I;
}

// the interval of image-local subsequence i
__device__ __forceinline__ int jd_interval_of(const JdImage& d, void* ws, int i) {
  const int* sb = jd_at<int>(ws, d.o_sb);
  int lo = 0, hi = d.nint - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (sb[mid] <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ unsigned jd_sub_end(const JdInterval& I, int i, int S) {
  const long long e = (long long)I.start + (long long)(i - I.a + 1) * S;
  return e < I.end ? (unsigned)e : I.end;
}

__device__ __forceinline__ JdState jd_guess(const JdInterval& I, int i, int S) {
  return jd_state(I.start + (unsigned)(i - I.a) * (unsigned)S, 0, 0);
}

// round r of the synchronisation: reads the exits of round r - 1 (e_in), writes exits and block counts
__global__ void __launch_bounds__(JD_SEQ_THREADS)
jd_sync_kernel(const __grid_constant__ JdParams P, void* ws, int S, int r) {
  __shared__ JdTables T;
  const int m = JD_FIND(P, seq0, blockIdx.x);
  const JdImage& d = P.img[m];
  jd_load_tables(d, T);
  const int i = (blockIdx.x - d.seq0) * JD_SEQ_THREADS + threadIdx.x;
  const int nseq = jd_at<int>(ws, d.o_meta)[1];
  if (i >= nseq) return;
  const JdInterval I = jd_interval(d, ws, jd_interval_of(d, ws, i));
  const JdState* e_in = jd_at<JdState>(ws, (r & 1) ? d.o_e1 : d.o_e0);
  JdState* e_out = jd_at<JdState>(ws, (r & 1) ? d.o_e0 : d.o_e1);
  const JdState st = i == I.a ? jd_state(I.start, 0, 0) : (r == 0 ? jd_guess(I, i, S) : e_in[i - 1]);
  int blocks;
  e_out[i] = jd_walk<false>(T, jd_at<unsigned char>(ws, d.o_u), jd_at<int>(ws, d.o_meta)[0], (unsigned)st,
                            (int)(st >> 40), (int)(st >> 32) & 255, jd_sub_end(I, i, S), d.bpm, d.hs * d.vs, &blocks,
                            nullptr);
  jd_at<int>(ws, d.o_cnt)[i] = blocks;
}

// one warp per interval: exact start states and block offsets of its subsequences
__global__ void __launch_bounds__(32 * JD_FIX_WARPS)
jd_fixup_kernel(const __grid_constant__ JdParams P, void* ws, int* status, int S, int R) {
  __shared__ JdTables T;
  const int m = JD_FIND(P, fix0, blockIdx.x);
  const JdImage& d = P.img[m];
  jd_load_tables(d, T);
  const int k = (blockIdx.x - d.fix0) * JD_FIX_WARPS + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const int nseq = jd_at<int>(ws, d.o_meta)[1];
  if (k >= d.nint || nseq == 0) return;
  const JdInterval I = jd_interval(d, ws, k);
  const unsigned char* u = jd_at<unsigned char>(ws, d.o_u);
  const int ulen = jd_at<int>(ws, d.o_meta)[0];
  const JdState* e_in = jd_at<JdState>(ws, ((R - 1) & 1) ? d.o_e1 : d.o_e0);   // starts of the last round
  const JdState* e_out = jd_at<JdState>(ws, (R & 1) ? d.o_e1 : d.o_e0);        // exits of the last round
  JdState* F = jd_at<JdState>(ws, d.o_f);
  int* cnt = jd_at<int>(ws, d.o_cnt);
  // the start subsequence j had in the last round
  auto used = [&](int j) -> JdState {
    return j == I.a ? jd_state(I.start, 0, 0) : (R == 1 ? jd_guess(I, j, S) : e_in[j - 1]);
  };
  JdState cur = jd_state(I.start, 0, 0);  // the exact start of subsequence i
  int i = I.a, redone = 0;
  while (i < I.b) {
    if (lane == 0) F[i] = cur;
    if (R > 0 && used(i) == cur) {
      // the last round decoded i from its exact start: follow the run of subsequences that start where their
      // predecessor ended
      int j = i + 1;
      while (j < I.b) {
        const int t = j + lane;
        const bool agree = t < I.b && used(t) == e_out[t - 1];
        if (t < I.b && agree) F[t] = used(t);
        const unsigned miss = __ballot_sync(0xffffffffu, !agree);
        if (miss) {
          j += __ffs(miss) - 1;
          break;
        }
        j += 32;
      }
      if (j >= I.b) break;
      cur = e_out[j - 1];
      i = j;
    } else {
      JdState next = 0;
      if (lane == 0) {
        int blocks;
        next = jd_walk<false>(T, u, ulen, (unsigned)cur, (int)(cur >> 40), (int)(cur >> 32) & 255,
                              jd_sub_end(I, i, S), d.bpm, d.hs * d.vs, &blocks, nullptr);
        cnt[i] = blocks;
      }
      cur = __shfl_sync(0xffffffffu, next, 0);
      ++redone;
      ++i;
    }
  }
  __syncwarp();
  // block offsets: exclusive prefix sums of the counts over the interval
  int* base = jd_at<int>(ws, d.o_base);
  int carry = 0;
  for (int j0 = I.a; j0 < I.b; j0 += 32) {
    const int j = j0 + lane;
    const int c = j < I.b ? cnt[j] : 0;
    int v = c;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, v, s);
      if (lane >= s) v += o;
    }
    if (j < I.b) base[j] = carry + v - c;
    carry += __shfl_sync(0xffffffffu, v, 31);
  }
  if (lane == 0) {
    if (carry < I.expected) atomicOr(status + 2 * m, JD_E_SHORT);
    if (redone) atomicAdd(status + 2 * m + 1, redone);
  }
}

__global__ void __launch_bounds__(JD_SEQ_THREADS)
jd_decode_kernel(const __grid_constant__ JdParams P, void* ws, short* __restrict__ coef, int* status, int S) {
  __shared__ JdTables T;
  const int m = JD_FIND(P, seq0, blockIdx.x);
  const JdImage& d = P.img[m];
  jd_load_tables(d, T);
  const int i = (blockIdx.x - d.seq0) * JD_SEQ_THREADS + threadIdx.x;
  const int nseq = jd_at<int>(ws, d.o_meta)[1];
  if (i >= nseq) return;
  const JdInterval I = jd_interval(d, ws, jd_interval_of(d, ws, i));
  const JdState st = jd_at<JdState>(ws, d.o_f)[i];
  JdWrite w;
  w.coef = coef + (d.coef + I.first) * 64;
  w.rel = jd_at<int>(ws, d.o_base)[i];
  w.expected = I.expected;
  w.iend = I.end;
  w.err = status + 2 * m;
  int blocks;
  jd_walk<true>(T, jd_at<unsigned char>(ws, d.o_u), jd_at<int>(ws, d.o_meta)[0], (unsigned)st, (int)(st >> 40),
                (int)(st >> 32) & 255, jd_sub_end(I, i, S), d.bpm, d.hs * d.vs, &blocks, &w);
}

// ------------------------------------------------------------------------------------------------ DC prediction
// grid (M, 3): segmented inclusive sum of component c's DC differences in coding order, restarting at every interval
__global__ void __launch_bounds__(1024) jd_dc_kernel(const __grid_constant__ JdParams P, short* __restrict__ coef) {
  __shared__ int shv[32], shf[32];
  const JdImage& d = P.img[blockIdx.x];
  const int c = blockIdx.y;
  const int ny = d.hs * d.vs;
  const int nc = c == 0 ? ny : 1;                // blocks of the component per MCU
  const int off = c == 0 ? 0 : ny + c - 1;       // its first block in the MCU
  const int per = d.ri ? d.ri : d.mcux * d.mcuy;
  const long long total = (long long)d.mcux * d.mcuy * nc;
  short* base = coef + d.coef * 64;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int carry = 0;
  for (long long s0 = 0; s0 < total; s0 += 1024) {
    const long long s = s0 + threadIdx.x;
    int v = 0, f = 0;
    long long n = 0;
    if (s < total) {
      const long long mcu = s / nc;
      const int t = (int)(s % nc);
      n = mcu * d.bpm + off + t;
      v = base[n * 64];
      f = t == 0 && mcu % per == 0;
    }
    // segmented scan: (f1, v1) + (f2, v2) = (f1 | f2, f2 ? v2 : v1 + v2)
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) {
      const int ov = __shfl_up_sync(0xffffffffu, v, k), of = __shfl_up_sync(0xffffffffu, f, k);
      if (lane >= k) {
        if (!f) v += ov;
        f |= of;
      }
    }
    if (lane == 31) { shv[w] = v; shf[w] = f; }
    __syncthreads();
    if (w == 0) {
      int sv = shv[lane], sf = shf[lane];
#pragma unroll
      for (int k = 1; k < 32; k <<= 1) {
        const int ov = __shfl_up_sync(0xffffffffu, sv, k), of = __shfl_up_sync(0xffffffffu, sf, k);
        if (lane >= k) {
          if (!sf) sv += ov;
          sf |= of;
        }
      }
      shv[lane] = sv;
      shf[lane] = sf;
    }
    __syncthreads();
    if (w > 0 && !f) { v += shv[w - 1]; f = shf[w - 1]; }
    if (!f) v += carry;
    if (s < total) base[n * 64] = (short)v;  // libjpeg keeps the prediction in an int and stores it as JCOEF
    __syncthreads();
    if (threadIdx.x == 1023) shv[0] = v;
    __syncthreads();
    carry = shv[0];
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ IDCT
constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
              F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

// one 8-point pass of the islow IDCT on c[0..7] -> o[0..7] before descaling
__device__ __forceinline__ void jd_idct8(const int* c, int* o) {
  const int z1 = (c[2] + c[6]) * F0541;
  const int tmp2 = z1 - c[6] * F1847, tmp3 = z1 + c[2] * F0765;
  const int tmp0 = (c[0] + c[4]) * 8192, tmp1 = (c[0] - c[4]) * 8192;
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int o0 = c[7], o1 = c[5], o2 = c[3], o3 = c[1];
  const int y1 = o0 + o3, y2 = o1 + o2, y3 = o0 + o2, y4 = o1 + o3;
  const int z5 = (y3 + y4) * F1175;
  o0 *= F0298; o1 *= F2053; o2 *= F3072; o3 *= F1501;
  const int w1 = -y1 * F0899, w2 = -y2 * F2562, w3 = -y3 * F1961 + z5, w4 = -y4 * F0390 + z5;
  o0 += w1 + w3; o1 += w2 + w4; o2 += w2 + w3; o3 += w1 + w4;
  o[0] = t10 + o3; o[7] = t10 - o3;
  o[1] = t11 + o2; o[6] = t11 - o2;
  o[2] = t12 + o1; o[5] = t12 - o1;
  o[3] = t13 + o0; o[4] = t13 - o0;
}

__global__ void __launch_bounds__(8 * JD_IDCT_BLOCKS)
jd_idct_kernel(const __grid_constant__ JdParams P, const short* __restrict__ coef, void* ws) {
  __shared__ int wsh[JD_IDCT_BLOCKS][64];
  const int m = JD_FIND(P, idct0, blockIdx.x);
  const JdImage& d = P.img[m];
  const int lb = threadIdx.x >> 3, c = threadIdx.x & 7;
  const long long n = (long long)(blockIdx.x - d.idct0) * JD_IDCT_BLOCKS + lb;
  const long long nblocks = (long long)d.mcux * d.mcuy * d.bpm;
  if (n >= nblocks) return;  // whole groups of 8 threads leave together
  const long long u = n / d.bpm;
  const int t = (int)(n % d.bpm), ny = d.hs * d.vs;
  const int comp = t < ny ? 0 : t - ny + 1;
  int bx, by, pw;
  if (comp == 0) {
    bx = (int)(u % d.mcux) * d.hs + t % d.hs;
    by = (int)(u / d.mcux) * d.vs + t / d.hs;
    pw = d.mcux * d.hs * 8;
  } else {
    bx = (int)(u % d.mcux);
    by = (int)(u / d.mcux);
    pw = d.mcux * 8;
  }
  const short* in = coef + (d.coef + n) * 64;
  const int* q = d.qt[comp];
  int col[8], o[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) col[k] = (int)in[k * 8 + c] * (int)(short)__ldg(q + k * 8 + c);  // 16-bit multipliers
  jd_idct8(col, o);
#pragma unroll
  for (int k = 0; k < 8; ++k) wsh[lb][k * 8 + c] = (o[k] + (1 << 10)) >> 11;  // CONST_BITS - PASS1_BITS
  __syncwarp(0xffu << (threadIdx.x & 24));
  int row[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) row[k] = wsh[lb][c * 8 + k];
  jd_idct8(row, o);
  unsigned lo = 0, hi = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int v = (o[k] + (1 << 17)) >> 18;  // CONST_BITS + PASS1_BITS + 3
    v = (v < -128 ? -128 : (v > 127 ? 127 : v)) + 128;
    if (k < 4) lo |= (unsigned)v << (8 * k); else hi |= (unsigned)v << (8 * (k - 4));
  }
  unsigned char* pl = jd_at<unsigned char>(ws, d.o_pl[comp]);
  *reinterpret_cast<uint2*>(pl + (long long)(by * 8 + c) * pw + bx * 8) = make_uint2(lo, hi);
}

// ------------------------------------------------------------------------------------------------ upsampling, colour
__device__ __forceinline__ int jd_chroma(const unsigned char* pl, int pw, int cw, int ch, int hs, int vs, int y, int x) {
  if (hs == 1) return pl[(long long)y * pw + x];
  const int j = x >> 1, odd = x & 1;
  const int jn = odd ? min(j + 1, cw - 1) : max(j - 1, 0);
  if (vs == 1) {
    const unsigned char* r = pl + (long long)y * pw;
    return (3 * r[j] + r[jn] + (odd ? 2 : 1)) >> 2;
  }
  const int rr = y >> 1;
  const int rn = (y & 1) ? min(rr + 1, ch - 1) : max(rr - 1, 0);
  const unsigned char* a = pl + (long long)rr * pw;
  const unsigned char* b = pl + (long long)rn * pw;
  const int cs = 3 * a[j] + b[j], cn = 3 * a[jn] + b[jn];
  return (3 * cs + cn + (odd ? 7 : 8)) >> 4;
}

__global__ void __launch_bounds__(JD_COLOUR_THREADS)
jd_colour_kernel(const __grid_constant__ JdParams P, void* ws, unsigned char* __restrict__ out) {
  const int m = JD_FIND(P, col0, blockIdx.x);
  const JdImage& d = P.img[m];
  const int xt = (d.W + JD_COLOUR_THREADS - 1) / JD_COLOUR_THREADS;
  const int local = blockIdx.x - d.col0;
  const int y = local / xt, x = (local % xt) * JD_COLOUR_THREADS + threadIdx.x;
  if (y >= d.H || x >= d.W) return;
  const int pwy = d.mcux * d.hs * 8, pwc = d.mcux * 8;
  const int cw = (d.W + d.hs - 1) / d.hs, ch = (d.H + d.vs - 1) / d.vs;  // the chroma planes' real size
  const int Y = jd_at<unsigned char>(ws, d.o_pl[0])[(long long)y * pwy + x];
  const int cb = jd_chroma(jd_at<unsigned char>(ws, d.o_pl[1]), pwc, cw, ch, d.hs, d.vs, y, x) - 128;
  const int cr = jd_chroma(jd_at<unsigned char>(ws, d.o_pl[2]), pwc, cw, ch, d.hs, d.vs, y, x) - 128;
  // jdcolor.c's tables: FIX(1.402) = 91881, FIX(1.772) = 116130, FIX(0.71414) = 46802, FIX(0.34414) = 22554
  const int R = Y + ((91881 * cr + 32768) >> 16);
  const int G = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
  const int B = Y + ((116130 * cb + 32768) >> 16);
  unsigned char* o = out + d.out + ((long long)y * d.W + x) * 3;
  o[0] = (unsigned char)min(max(B, 0), 255);
  o[1] = (unsigned char)min(max(G, 0), 255);
  o[2] = (unsigned char)min(max(R, 0), 255);
}

// ------------------------------------------------------------------------------------------------ host side
inline long long jd_align(long long b) { return (b + 15) & ~15LL; }

// image m's descriptor and workspace layout from its geometry; *ws_end advances past its workspace, *coef_blocks past
// its coefficient blocks.  0 or -1.
inline int jd_describe(const long long* scan, const int* geom, int m, int S, JdImage* d, long long* ws_end,
                       long long* coef_blocks) {
  const long long len = scan[2 * m + 1];
  const int H = geom[5 * m], W = geom[5 * m + 1], hs = geom[5 * m + 2], vs = geom[5 * m + 3], ri = geom[5 * m + 4];
  if (scan[2 * m] < 0 || len < 0 || len >= (1LL << 28)) return OCC_EINVAL;
  if (H < 1 || W < 1 || H > 16384 || W > 16384 || ri < 0 || ri > 65535) return OCC_EINVAL;
  if (!((hs == 1 && vs == 1) || (hs == 2 && vs == 1) || (hs == 2 && vs == 2))) return OCC_EINVAL;
  d->src = scan[2 * m];
  d->len = (int)len;
  d->W = W; d->H = H; d->hs = hs; d->vs = vs; d->ri = ri;
  d->mcux = (W + 8 * hs - 1) / (8 * hs);
  d->mcuy = (H + 8 * vs - 1) / (8 * vs);
  d->bpm = hs * vs + 2;
  const long long mcus = (long long)d->mcux * d->mcuy;
  d->nint = ri ? (int)((mcus + ri - 1) / ri) : 1;
  d->cap = (int)((8 * len + S - 1) / S) + d->nint;
  const long long nchunks = (len + JD_CHUNK - 1) / JD_CHUNK;
  long long o = *ws_end;
  d->o_blk = o;  o += jd_align(8 * nchunks);
  d->o_u = o;    o += jd_align(len) + 32;
  d->o_q = o;    o += jd_align(4LL * (d->nint + 1));
  d->o_sb = o;   o += jd_align(4LL * (d->nint + 1));
  d->o_meta = o; o += 16;
  d->o_e0 = o;   o += 8LL * d->cap;
  d->o_e1 = o;   o += 8LL * d->cap;
  d->o_f = o;    o += 8LL * d->cap;
  d->o_cnt = o;  o += jd_align(4LL * d->cap);
  d->o_base = o; o += jd_align(4LL * d->cap);
  const long long pwy = (long long)d->mcux * hs * 8, phy = (long long)d->mcuy * vs * 8;
  d->o_pl[0] = o; o += jd_align(pwy * phy);
  d->o_pl[1] = o; o += jd_align((long long)d->mcux * 8 * d->mcuy * 8);
  d->o_pl[2] = o; o += jd_align((long long)d->mcux * 8 * d->mcuy * 8);
  *ws_end = o;
  d->coef = *coef_blocks;
  *coef_blocks += mcus * d->bpm;
  return OCC_OK;
}

// the whole layout: workspace bytes (coefficients first) and the grids' per-image first blocks
inline int jd_layout(const long long* scan, const int* geom, int M, int S, JdParams* P, size_t* bytes,
                     long long* coef_area, long long* grids /*chunks, seq, fix, idct, colour blocks*/) {
  if (!scan || !geom || M < 1 || M > JD_MAX_IMAGES || S < 32 || S > (1 << 20)) return OCC_EINVAL;
  long long coef_blocks = 0, ws_end = 0;
  for (int m = 0; m < M; ++m) {
    if (jd_describe(scan, geom, m, S, &P->img[m], &ws_end, &coef_blocks) != OCC_OK) return OCC_EINVAL;
  }
  const long long coef_bytes = jd_align(coef_blocks * 128);
  long long g[5] = {0, 0, 0, 0, 0};
  for (int m = 0; m < M; ++m) {
    JdImage& d = P->img[m];
    d.o_blk += coef_bytes; d.o_u += coef_bytes; d.o_q += coef_bytes; d.o_sb += coef_bytes; d.o_meta += coef_bytes;
    d.o_e0 += coef_bytes; d.o_e1 += coef_bytes; d.o_f += coef_bytes; d.o_cnt += coef_bytes; d.o_base += coef_bytes;
    for (int c = 0; c < 3; ++c) d.o_pl[c] += coef_bytes;
    d.chunk0 = (int)g[0]; g[0] += (d.len + JD_CHUNK - 1) / JD_CHUNK;
    d.seq0 = (int)g[1];   g[1] += (d.cap + JD_SEQ_THREADS - 1) / JD_SEQ_THREADS;
    d.fix0 = (int)g[2];   g[2] += (d.nint + JD_FIX_WARPS - 1) / JD_FIX_WARPS;
    d.idct0 = (int)g[3];  g[3] += ((long long)d.mcux * d.mcuy * d.bpm + JD_IDCT_BLOCKS - 1) / JD_IDCT_BLOCKS;
    d.col0 = (int)g[4];   g[4] += (long long)d.H * ((d.W + JD_COLOUR_THREADS - 1) / JD_COLOUR_THREADS);
  }
  for (int k = 0; k < 5; ++k) {
    if (g[k] >= (1LL << 31)) return OCC_EINVAL;
    if (grids) grids[k] = g[k];
  }
  P->M = M;
  *coef_area = coef_bytes;
  *bytes = (size_t)(coef_bytes + ws_end);
  return OCC_OK;
}

}  // namespace occ

using namespace occ;

extern "C" size_t occ_decode_jpeg_workspace_bytes(const long long* scan, const int* geom, int M, int seq_bits) {
  JdParams P;
  size_t bytes = 0;
  long long coef_bytes;
  return jd_layout(scan, geom, M, seq_bits, &P, &bytes, &coef_bytes, nullptr) == OCC_OK ? bytes : 0;
}

extern "C" int occ_decode_jpeg(const unsigned char* data, long long data_bytes, const long long* scan, const int* geom,
                               const long long* tables, const long long* out_offsets, int M, int seq_bits,
                               int sync_rounds, void* ws, size_t ws_bytes, unsigned char* out, long long out_bytes,
                               int* status, cudaStream_t stream) {
  OCC_REQUIRE(data && scan && geom && tables && out_offsets && out && status && ws);
  OCC_REQUIRE(sync_rounds >= 0 && sync_rounds <= 64 && data_bytes >= 0 && out_bytes >= 0);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 15) == 0);
  JdParams P;
  size_t need = 0;
  long long grids[5], coef_bytes = 0;
  const int rc = jd_layout(scan, geom, M, seq_bits, &P, &need, &coef_bytes, grids);
  if (rc != OCC_OK) {
    fprintf(stderr, "occ_b200: occ_decode_jpeg: bad image count, subsequence length or geometry\n");
    return rc;
  }
  OCC_REQUIRE(ws_bytes >= need);
  for (int m = 0; m < M; ++m) {
    JdImage& d = P.img[m];
    OCC_REQUIRE(d.src + d.len <= data_bytes);
    OCC_REQUIRE(out_offsets[m] >= 0 && out_offsets[m] <= out_bytes &&
                (long long)d.H * d.W * 3 <= out_bytes - out_offsets[m]);
    d.out = out_offsets[m];
    for (int c = 0; c < 3; ++c) {
      const long long qa = tables[9 * m + c], da = tables[9 * m + 3 + c], aa = tables[9 * m + 6 + c];
      OCC_REQUIRE(qa != 0 && da != 0 && aa != 0 && (qa & 3) == 0 && (da & 3) == 0 && (aa & 3) == 0);
      d.qt[c] = reinterpret_cast<const int*>(qa);
      d.huff[c][0] = reinterpret_cast<const int*>(da);
      d.huff[c][1] = reinterpret_cast<const int*>(aa);
    }
  }
  short* coef = static_cast<short*>(ws);
  OCC_MEMSET(status, 0, sizeof(int) * 2 * M, stream);
  OCC_MEMSET(ws, 0, (size_t)coef_bytes, stream);
  if (grids[0] > 0) {
    jd_count_kernel<<<(unsigned)grids[0], JD_CHUNK_THREADS, 0, stream>>>(P, data, ws, status);
    OCC_LAUNCH_CHECK();
  }
  jd_scan_kernel<<<M, 1024, 0, stream>>>(P, ws, status);
  OCC_LAUNCH_CHECK();
  if (grids[0] > 0) {
    jd_compact_kernel<<<(unsigned)grids[0], JD_CHUNK_THREADS, 0, stream>>>(P, data, ws, status);
    OCC_LAUNCH_CHECK();
  }
  jd_plan_kernel<<<M, 1024, 0, stream>>>(P, ws, status, seq_bits);
  OCC_LAUNCH_CHECK();
  for (int r = 0; r < sync_rounds; ++r) {
    jd_sync_kernel<<<(unsigned)grids[1], JD_SEQ_THREADS, 0, stream>>>(P, ws, seq_bits, r);
    OCC_LAUNCH_CHECK();
  }
  jd_fixup_kernel<<<(unsigned)grids[2], 32 * JD_FIX_WARPS, 0, stream>>>(P, ws, status, seq_bits, sync_rounds);
  OCC_LAUNCH_CHECK();
  jd_decode_kernel<<<(unsigned)grids[1], JD_SEQ_THREADS, 0, stream>>>(P, ws, coef, status, seq_bits);
  OCC_LAUNCH_CHECK();
  jd_dc_kernel<<<dim3(M, 3), 1024, 0, stream>>>(P, coef);
  OCC_LAUNCH_CHECK();
  jd_idct_kernel<<<(unsigned)grids[3], 8 * JD_IDCT_BLOCKS, 0, stream>>>(P, coef, ws);
  OCC_LAUNCH_CHECK();
  jd_colour_kernel<<<(unsigned)grids[4], JD_COLOUR_THREADS, 0, stream>>>(P, ws, out);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
