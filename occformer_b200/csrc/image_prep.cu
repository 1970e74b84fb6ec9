// Camera images from the decoded uint8 BGR frames, on the device: the resize, crop and normalisation of the test loaders
//
//   LoadMultiViewImageFromFiles_OccFormer.img_transform_core + mmlabNormalize   P/datasets/pipelines/loading_nusc_imgs.py:34-62,181-195
//   LoadMultiViewImageFromFiles_SemanticKitti.img_transform_core                P/datasets/pipelines/loading_kitti_imgs.py:35-65
//
// bit for bit (include/occ_b200.h states the semantics).  Pillow's bicubic resample is integer arithmetic on coefficient
// tables the host computes (occformer_b200.image_prep), and imnormalize of a uint8 value is a 256-entry table per channel,
// so the device runs integer multiply-adds and one table lookup per output value:
//   hpass  per (image, source row the vertical taps read, resized column the crop reads): the source row's span of
//          pixels is staged in shared memory, then (1 << 21) + sum w * p per channel, clipped >> 22 -> three uint8 planes
//          in the workspace
//   vpass  per output pixel of the crop: (1 << 21) + sum w * p down the planes (0 outside the resized image), clipped
//          >> 22, then norm[c][v] -> float NCHW
// Two launches per call whatever M; the per-image descriptors travel in the kernel parameters (up to 256 images).
//
// occ_prepare_images_aug adds the training loaders' flip and rotation (img_transform_core: resize, crop, FLIP_LEFT_RIGHT,
// Image.rotate).  Both only move pixels inside the crop window, so hpass is unchanged; vpass_aug maps each output pixel
// through Pillow's 16.16 fixed-point nearest gather, the mirror and the crop offset to a resized (row, column), and
// reads that row's vertical taps per thread.
#include "occ_common.cuh"

namespace occ {

constexpr int IP_MAX_IMAGES = 256;
constexpr int IP_MAX_TAPS = 129;                  // Pillow's ksize for a downscale by 32: 2 * ceil(2 * 32) + 1
constexpr int IP_THREADS = 256;                   // resized columns per hpass block, output columns per vpass block
constexpr int IP_MAX_SPAN = 259 * 32 + 2;         // source pixels one hpass block reads: <= 255 f + 2 * 2 f + 1 at f <= 32

struct IpImage {
  long long src;        // byte offset of the frame in `frames`
  long long ws;         // byte offset of its three (nr, nc) uint8 planes in the workspace
  const int* ht;        // horizontal table (W -> rW)
  const int* vt;        // vertical table (H -> rH)
  int W, rW, rH, x0, y0;
  int c0, nc;           // resized columns [c0, c0 + nc) the crop reads
  int r0, nr;           // source rows [r0, r0 + nr) the vertical taps of the cropped rows read
};

struct IpParams {
  IpImage img[IP_MAX_IMAGES];
};

__device__ __forceinline__ int ip_clip8(int acc) {
  const int v = acc >> 22;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// grid (column chunks, rows, M); block (m, row r0 + blockIdx.y, resized columns c0 + 256 * blockIdx.x + [0, 256))
__global__ void __launch_bounds__(IP_THREADS)
ip_hpass_kernel(const __grid_constant__ IpParams P, const unsigned char* __restrict__ frames,
                unsigned char* __restrict__ ws) {
  __shared__ unsigned char s[IP_MAX_SPAN * 3];
  const IpImage& d = P.img[blockIdx.z];
  const int r = blockIdx.y;
  const int jb = blockIdx.x * IP_THREADS;
  if (r >= d.nr || jb >= d.nc) return;
  const int j0 = d.c0 + jb;
  const int j1 = min(j0 + IP_THREADS, d.c0 + d.nc) - 1;
  const int first = __ldg(d.ht + 2 * j0);
  int span = __ldg(d.ht + 2 * j1) + __ldg(d.ht + 2 * j1 + 1) - first;
  span = span < 0 ? 0 : (span > IP_MAX_SPAN ? IP_MAX_SPAN : span);  // the host checked the bound on its own bounds
  const unsigned char* row = frames + d.src + ((long long)(d.r0 + r) * d.W + first) * 3;
  for (int i = threadIdx.x; i < span * 3; i += IP_THREADS) s[i] = row[i];
  __syncthreads();
  const int j = j0 + threadIdx.x;
  if (j > j1) return;
  const int lo = __ldg(d.ht + 2 * j) - first;
  const int n = min(__ldg(d.ht + 2 * j + 1), span - lo);
  const int* w = d.ht + 2 * d.rW + j;
  int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
  for (int k = 0; k < n; ++k) {
    const int wk = __ldg(w + (long long)k * d.rW);
    const unsigned char* p = s + (lo + k) * 3;
    a0 += wk * p[0];
    a1 += wk * p[1];
    a2 += wk * p[2];
  }
  const long long plane = (long long)d.nr * d.nc;
  unsigned char* o = ws + d.ws + (long long)r * d.nc + (j - d.c0);
  o[0] = (unsigned char)ip_clip8(a0);
  o[plane] = (unsigned char)ip_clip8(a1);
  o[2 * plane] = (unsigned char)ip_clip8(a2);
}

// grid (column chunks, fH, M); block (m, output row blockIdx.y, output columns 256 * blockIdx.x + [0, 256))
__global__ void __launch_bounds__(IP_THREADS)
ip_vpass_kernel(const __grid_constant__ IpParams P, const unsigned char* __restrict__ ws,
                const float* __restrict__ norm, int swap_rb, int fH, int fW, float* __restrict__ out) {
  const IpImage& d = P.img[blockIdx.z];
  const int y = blockIdx.y;
  const int x = blockIdx.x * IP_THREADS + threadIdx.x;
  if (x >= fW) return;
  const int R = d.y0 + y, X = d.x0 + x;
  int v0 = 0, v1 = 0, v2 = 0;
  if (R >= 0 && R < d.rH && X >= 0 && X < d.rW) {
    // the host sized [r0, r0 + nr) and [c0, c0 + nc) from these taps; the clamps only keep a foreign table in bounds
    const int lo = __ldg(d.vt + 2 * R) - d.r0;
    const int n = min(__ldg(d.vt + 2 * R + 1), d.nr - lo);
    const int col = X - d.c0;
    if (lo >= 0 && col < d.nc) {
      const long long plane = (long long)d.nr * d.nc;
      const unsigned char* p = ws + d.ws + (long long)lo * d.nc + col;
      const int* w = d.vt + 2 * d.rH + R;
      int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
      for (int k = 0; k < n; ++k) {
        const int wk = __ldg(w + (long long)k * d.rH);
        const unsigned char* q = p + (long long)k * d.nc;
        a0 += wk * __ldg(q);
        a1 += wk * __ldg(q + plane);
        a2 += wk * __ldg(q + 2 * plane);
      }
      v0 = ip_clip8(a0);
      v1 = ip_clip8(a1);
      v2 = ip_clip8(a2);
    }
  }
  const long long hw = (long long)fH * fW;
  float* o = out + (long long)blockIdx.z * 3 * hw + (long long)y * fW + x;
  o[0] = __ldg(norm + (swap_rb ? v2 : v0));
  o[hw] = __ldg(norm + 256 + v1);
  o[2 * hw] = __ldg(norm + 512 + (swap_rb ? v0 : v2));
}

struct IpRotate {
  int a[6];             // Pillow's affine_fixed coefficients a0..a5 (16.16) of Image.rotate on the fW x fH crop
  int flip;             // 1: FLIP_LEFT_RIGHT of the crop before the rotation
};

struct IpRotateParams {
  IpRotate img[IP_MAX_IMAGES];
};

// grid (column chunks, fH, M); block (m, output row blockIdx.y, output columns 256 * blockIdx.x + [0, 256)).  Output
// pixel (x, y) of the rotated crop reads crop pixel ((a2 + y a1 + x a0) >> 16, (a5 + y a4 + x a3) >> 16) (0 outside the
// crop), mirrored when flipped, i.e. resized pixel (x0 + column, y0 + row) (0 outside the resized image).  The host
// checked that no intermediate leaves int32, as Pillow's int accumulation assumes.
__global__ void __launch_bounds__(IP_THREADS)
ip_vpass_aug_kernel(const __grid_constant__ IpParams P, const __grid_constant__ IpRotateParams Q,
                    const unsigned char* __restrict__ ws, const float* __restrict__ norm, int swap_rb, int fH, int fW,
                    float* __restrict__ out) {
  const IpImage& d = P.img[blockIdx.z];
  const IpRotate& q = Q.img[blockIdx.z];
  const int y = blockIdx.y;
  const int x = blockIdx.x * IP_THREADS + threadIdx.x;
  if (x >= fW) return;
  const int xs = (int)((q.a[2] + (long long)y * q.a[1] + (long long)x * q.a[0]) >> 16);
  const int ys = (int)((q.a[5] + (long long)y * q.a[4] + (long long)x * q.a[3]) >> 16);
  int v0 = 0, v1 = 0, v2 = 0;
  if (xs >= 0 && xs < fW && ys >= 0 && ys < fH) {
    const int R = d.y0 + ys, X = d.x0 + (q.flip ? fW - 1 - xs : xs);
    if (R >= 0 && R < d.rH && X >= 0 && X < d.rW) {
      const int lo = __ldg(d.vt + 2 * R) - d.r0;
      const int n = min(__ldg(d.vt + 2 * R + 1), d.nr - lo);
      const int col = X - d.c0;
      if (lo >= 0 && col < d.nc) {
        const long long plane = (long long)d.nr * d.nc;
        const unsigned char* p = ws + d.ws + (long long)lo * d.nc + col;
        const int* w = d.vt + 2 * d.rH + R;
        int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
        for (int k = 0; k < n; ++k) {
          const int wk = __ldg(w + (long long)k * d.rH);
          const unsigned char* r = p + (long long)k * d.nc;
          a0 += wk * __ldg(r);
          a1 += wk * __ldg(r + plane);
          a2 += wk * __ldg(r + 2 * plane);
        }
        v0 = ip_clip8(a0);
        v1 = ip_clip8(a1);
        v2 = ip_clip8(a2);
      }
    }
  }
  const long long hw = (long long)fH * fW;
  float* o = out + (long long)blockIdx.z * 3 * hw + (long long)y * fW + x;
  o[0] = __ldg(norm + (swap_rb ? v2 : v0));
  o[hw] = __ldg(norm + 256 + v1);
  o[2 * hw] = __ldg(norm + 512 + (swap_rb ? v0 : v2));
}

// Pillow's precompute_coeffs (resample.c) for one output index: ksize and the tap window [first, first + count), in the
// same float64 operations the host's table builder uses
inline int ip_ksize(int in, int n) {
  const double scale = (double)in / (double)n;
  const double support = 2.0 * (scale < 1.0 ? 1.0 : scale);
  return (int)ceil(support) * 2 + 1;
}

inline void ip_window(int in, int n, int i, int* first, int* count) {
  const double scale = (double)in / (double)n;
  const double support = 2.0 * (scale < 1.0 ? 1.0 : scale);
  const double center = (i + 0.5) * scale;
  int lo = (int)(center - support + 0.5);
  int hi = (int)(center + support + 0.5);
  lo = lo < 0 ? 0 : lo;
  hi = hi > in ? in : hi;
  *first = lo;
  *count = hi - lo;
}

inline size_t ip_align(size_t b) { return (b + 15) & ~(size_t)15; }

// image m's descriptor without its pointers and offsets -> 0, -1 (argument error) or -2 (too many taps)
inline int ip_describe(const int* g, int fH, int fW, IpImage* d) {
  const int H = g[0], W = g[1], rW = g[2], rH = g[3], x0 = g[4], y0 = g[5];
  if (H < 1 || W < 1 || rW < 1 || rH < 1 || fH < 1 || fW < 1) return OCC_EINVAL;
  if (x0 <= -(1 << 30) || x0 >= (1 << 30) || y0 <= -(1 << 30) || y0 >= (1 << 30)) return OCC_EINVAL;
  if (ip_ksize(W, rW) > IP_MAX_TAPS || ip_ksize(H, rH) > IP_MAX_TAPS) return OCC_EUNSUPPORTED;
  d->W = W; d->rW = rW; d->rH = rH; d->x0 = x0; d->y0 = y0;
  const int cx0 = x0 > 0 ? x0 : 0, cx1 = x0 + fW < rW ? x0 + fW : rW;  // resized columns / rows inside the crop
  const int cy0 = y0 > 0 ? y0 : 0, cy1 = y0 + fH < rH ? y0 + fH : rH;
  d->c0 = d->nc = d->r0 = d->nr = 0;
  if (cx0 < cx1 && cy0 < cy1) {
    int f0, n0, f1, n1;
    ip_window(H, rH, cy0, &f0, &n0);
    ip_window(H, rH, cy1 - 1, &f1, &n1);
    d->c0 = cx0;
    d->nc = cx1 - cx0;
    d->r0 = f0;
    d->nr = f1 + n1 - f0;
  }
  return OCC_OK;
}

}  // namespace occ

using namespace occ;

extern "C" size_t occ_prepare_images_workspace_bytes(const int* geom, int M, int fH, int fW) {
  if (!geom || M < 1 || M > IP_MAX_IMAGES) return 0;
  size_t total = 0;
  for (int m = 0; m < M; ++m) {
    IpImage d;
    if (ip_describe(geom + 6 * m, fH, fW, &d) != OCC_OK) return 0;
    total += ip_align((size_t)3 * d.nr * d.nc);
  }
  return total;
}

// the descriptors of both entries' M images -> 0 or the entry's error code; *ws_need, *max_nr, *max_nc for the launch
static int ip_setup(const char* fn, long long frame_bytes, const long long* offsets, const int* geom, int M, int fH,
                    int fW, const long long* tables, IpParams* P, size_t* ws_need, int* max_nr, int* max_nc) {
  size_t ws_off = 0;
  *max_nr = *max_nc = 0;
  for (int m = 0; m < M; ++m) {
    IpImage& d = P->img[m];
    const int rc = ip_describe(geom + 6 * m, fH, fW, &d);
    if (rc != OCC_OK) {
      if (rc == OCC_EINVAL) fprintf(stderr, "occ_b200: %s: bad geometry of image %d\n", fn, m);
      return rc;
    }
    const int H = geom[6 * m];
    OCC_REQUIRE(offsets[m] >= 0 && offsets[m] <= frame_bytes &&
                (long long)H * d.W * 3 <= frame_bytes - offsets[m]);
    OCC_REQUIRE(tables[2 * m] != 0 && tables[2 * m + 1] != 0);
    OCC_REQUIRE(d.nr < 65536);
    d.src = offsets[m];
    d.ht = reinterpret_cast<const int*>(tables[2 * m]);
    d.vt = reinterpret_cast<const int*>(tables[2 * m + 1]);
    d.ws = (long long)ws_off;
    ws_off += ip_align((size_t)3 * d.nr * d.nc);
    *max_nr = d.nr > *max_nr ? d.nr : *max_nr;
    *max_nc = d.nc > *max_nc ? d.nc : *max_nc;
  }
  *ws_need = ws_off;
  return OCC_OK;
}

extern "C" int occ_prepare_images(const unsigned char* frames, long long frame_bytes, const long long* offsets,
                                  const int* geom, int M, int fH, int fW, const long long* tables, const float* norm,
                                  int swap_rb, void* ws, size_t ws_bytes, float* out, cudaStream_t stream) {
  OCC_REQUIRE(frames && offsets && geom && tables && norm && out && M >= 1 && M <= IP_MAX_IMAGES);
  OCC_REQUIRE(fH >= 1 && fW >= 1 && (swap_rb == 0 || swap_rb == 1) && frame_bytes >= 0);
  OCC_REQUIRE((long long)fH * fW <= (1LL << 31) && (long long)fH < 65536);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 15) == 0);
  IpParams P;  // 18 KB of kernel parameters (sm_90 takes up to 32 KB)
  size_t ws_off = 0;
  int max_nr = 0, max_nc = 0;
  const int rc = ip_setup("occ_prepare_images", frame_bytes, offsets, geom, M, fH, fW, tables, &P, &ws_off, &max_nr,
                          &max_nc);
  if (rc != OCC_OK) return rc;
  OCC_REQUIRE(ws_bytes >= ws_off && (ws_off == 0 || ws));
  if (max_nr > 0) {
    const dim3 grid((unsigned)((max_nc + IP_THREADS - 1) / IP_THREADS), (unsigned)max_nr, (unsigned)M);
    ip_hpass_kernel<<<grid, IP_THREADS, 0, stream>>>(P, frames, static_cast<unsigned char*>(ws));
    OCC_LAUNCH_CHECK();
  }
  const dim3 grid((unsigned)((fW + IP_THREADS - 1) / IP_THREADS), (unsigned)fH, (unsigned)M);
  ip_vpass_kernel<<<grid, IP_THREADS, 0, stream>>>(P, static_cast<const unsigned char*>(ws), norm, swap_rb, fH, fW,
                                                   out);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_prepare_images_aug(const unsigned char* frames, long long frame_bytes, const long long* offsets,
                                      const int* geom, const int* aug, int M, int fH, int fW, const long long* tables,
                                      const float* norm, int swap_rb, void* ws, size_t ws_bytes, float* out,
                                      cudaStream_t stream) {
  OCC_REQUIRE(frames && offsets && geom && aug && tables && norm && out && M >= 1 && M <= IP_MAX_IMAGES);
  OCC_REQUIRE(fH >= 1 && fW >= 1 && (swap_rb == 0 || swap_rb == 1) && frame_bytes >= 0);
  OCC_REQUIRE((long long)fH * fW <= (1LL << 31) && (long long)fH < 65536);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 15) == 0);
  for (int m = 0; m < M; ++m) {
    const int* g = aug + 7 * m;
    OCC_REQUIRE(g[0] == 0 || g[0] == 1);
    // every intermediate of a + y * a1 + x * a0 at the crop's corners (hence everywhere inside) fits in int32
    for (int c = 0; c < 2; ++c) {
      const long long a0 = g[1 + 3 * c], a1 = g[2 + 3 * c], a2 = g[3 + 3 * c];
      const long long lo = a2 + (a1 < 0 ? a1 * (fH - 1) : 0) + (a0 < 0 ? a0 * (fW - 1) : 0);
      const long long hi = a2 + (a1 > 0 ? a1 * (fH - 1) : 0) + (a0 > 0 ? a0 * (fW - 1) : 0);
      OCC_REQUIRE(lo >= INT32_MIN && hi <= INT32_MAX);
    }
  }
  IpParams P;
  size_t ws_off = 0;
  int max_nr = 0, max_nc = 0;
  const int rc = ip_setup("occ_prepare_images_aug", frame_bytes, offsets, geom, M, fH, fW, tables, &P, &ws_off,
                          &max_nr, &max_nc);
  if (rc != OCC_OK) return rc;
  OCC_REQUIRE(ws_bytes >= ws_off && (ws_off == 0 || ws));
  IpRotateParams R;  // 7 KB beside P's 18 KB of kernel parameters
  for (int m = 0; m < M; ++m) {
    const int* g = aug + 7 * m;
    R.img[m].flip = g[0];
    for (int k = 0; k < 6; ++k) R.img[m].a[k] = g[1 + k];
  }
  if (max_nr > 0) {
    const dim3 grid((unsigned)((max_nc + IP_THREADS - 1) / IP_THREADS), (unsigned)max_nr, (unsigned)M);
    ip_hpass_kernel<<<grid, IP_THREADS, 0, stream>>>(P, frames, static_cast<unsigned char*>(ws));
    OCC_LAUNCH_CHECK();
  }
  const dim3 grid((unsigned)((fW + IP_THREADS - 1) / IP_THREADS), (unsigned)fH, (unsigned)M);
  ip_vpass_aug_kernel<<<grid, IP_THREADS, 0, stream>>>(P, R, static_cast<const unsigned char*>(ws), norm, swap_rb, fH,
                                                       fW, out);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
