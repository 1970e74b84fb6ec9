// Depth maps from the LiDAR scan, on the device: CreateDepthFromLiDAR of the training pipelines
//
//   CreateDepthFromLiDAR.project_points + __call__   P/datasets/pipelines/lidar2depth.py:15-82
//
// bit for bit as the reference computes it in a loader worker (one torch thread; include/occ_b200.h states the
// semantics).  Every product, sum and quotient is one IEEE round-to-nearest fp32 operation in the reference's order, so
// the arithmetic uses the _rn intrinsics (no contraction into FMA).  The reference sorts the valid points by descending
// depth and writes them in that order, so the nearest point of a pixel wins: here each (point, camera) thread takes the
// atomicMin of its depth's bits (positive floats order as their bits) over a map of all ones bits, and a finishing pass
// turns the pixels no point reached into 0.
//   memset  out = 0xff bytes
//   scatter per (point, camera): project, test, round half-even, atomicMin
//   finish  per pixel: all ones -> 0.0f
// Three launches and memsets per call whatever the scans; the per-sample point ranges travel in the kernel parameters.
#include "occ_common.cuh"

namespace occ {

constexpr int LD_MAX_SAMPLES = 256;
constexpr int LD_THREADS = 256;

struct LdOffsets {
  long long off[LD_MAX_SAMPLES + 1];  // sample b's points are rows [off[b], off[b + 1]) of pts
};

// row i of a 3 x 3 matrix times v, summed left to right
__device__ __forceinline__ float ld_dot3(const float* m, float v0, float v1, float v2) {
  return __fadd_rn(__fadd_rn(__fmul_rn(__ldg(m), v0), __fmul_rn(__ldg(m + 1), v1)), __fmul_rn(__ldg(m + 2), v2));
}

// grid (point chunks, N, B); block (sample blockIdx.z, camera blockIdx.y, its points 256 * blockIdx.x + [0, 256))
__global__ void __launch_bounds__(LD_THREADS)
ld_scatter_kernel(const __grid_constant__ LdOffsets O, const float* __restrict__ pts, const float* __restrict__ inv_rots,
                  const float* __restrict__ trans, const float* __restrict__ intrins, int kd,
                  const float* __restrict__ post_rots, const float* __restrict__ post_trans, int fH, int fW,
                  unsigned* __restrict__ out) {
  const int b = blockIdx.z;
  const long long cam = (long long)b * gridDim.y + blockIdx.y;
  const long long p = O.off[b] + (long long)blockIdx.x * LD_THREADS + threadIdx.x;
  if (p >= O.off[b + 1]) return;
  const float* t = trans + 3 * cam;
  const float q0 = __fsub_rn(__ldg(pts + 3 * p), __ldg(t));
  const float q1 = __fsub_rn(__ldg(pts + 3 * p + 1), __ldg(t + 1));
  const float q2 = __fsub_rn(__ldg(pts + 3 * p + 2), __ldg(t + 2));
  const float* R = inv_rots + 9 * cam;
  const float c0 = ld_dot3(R, q0, q1, q2), c1 = ld_dot3(R + 3, q0, q1, q2), c2 = ld_dot3(R + 6, q0, q1, q2);
  const float* K = intrins + (long long)kd * kd * cam;
  float x = ld_dot3(K, c0, c1, c2), y = ld_dot3(K + kd, c0, c1, c2), d = ld_dot3(K + 2 * kd, c0, c1, c2);
  if (kd == 4) {  // KITTI's 4 x 4 intrinsics act on (c, 1): the fourth product is the fourth column itself
    x = __fadd_rn(x, __ldg(K + 3));
    y = __fadd_rn(y, __ldg(K + 7));
    d = __fadd_rn(d, __ldg(K + 11));
  }
  const float u = __fdiv_rn(x, d), v = __fdiv_rn(y, d);
  const float* A = post_rots + 9 * cam;
  const float* s = post_trans + 3 * cam;
  const float pu = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(A), u), __fmul_rn(__ldg(A + 1), v)), __ldg(s));
  const float pv = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(A + 3), u), __fmul_rn(__ldg(A + 4), v)), __ldg(s + 1));
  // the reference's comparisons: false for NaN, so a NaN coordinate or depth never passes
  if (!(pu >= 0.f && pv >= 0.f && pu <= (float)(fW - 1) && pv <= (float)(fH - 1) && d > 0.f)) return;
  const int px = (int)rintf(pu), py = (int)rintf(pv);
  atomicMin(out + (cam * fH + py) * fW + px, __float_as_uint(d));
}

__global__ void __launch_bounds__(LD_THREADS) ld_finish_kernel(unsigned* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * LD_THREADS + threadIdx.x; i < n; i += (long long)gridDim.x * LD_THREADS)
    if (out[i] == 0xffffffffu) out[i] = 0u;
}

}  // namespace occ

using namespace occ;

extern "C" int occ_lidar_depth(const float* pts, const long long* offsets, int B, int N, const float* inv_rots,
                               const float* trans, const float* intrins, int intrin_dim, const float* post_rots,
                               const float* post_trans, int fH, int fW, float* out, cudaStream_t stream) {
  OCC_REQUIRE(offsets && inv_rots && trans && intrins && post_rots && post_trans && out);
  OCC_REQUIRE(B >= 1 && B <= LD_MAX_SAMPLES && N >= 1 && N <= 65535 && (intrin_dim == 3 || intrin_dim == 4));
  OCC_REQUIRE(fH >= 1 && fW >= 1 && fH <= (1 << 24) && fW <= (1 << 24) && (long long)fH * fW <= (1LL << 31));
  LdOffsets O;
  long long most = 0;
  OCC_REQUIRE(offsets[0] == 0);
  for (int b = 0; b < B; ++b) {
    OCC_REQUIRE(offsets[b + 1] >= offsets[b] && offsets[b + 1] < (1LL << 40));
    O.off[b] = offsets[b];
    most = offsets[b + 1] - offsets[b] > most ? offsets[b + 1] - offsets[b] : most;
  }
  O.off[B] = offsets[B];
  OCC_REQUIRE(pts || offsets[B] == 0);
  OCC_REQUIRE((most + LD_THREADS - 1) / LD_THREADS < (1LL << 31));
  const long long n = (long long)B * N * fH * fW;
  unsigned* o = reinterpret_cast<unsigned*>(out);
  OCC_MEMSET(o, 0xff, (size_t)n * sizeof(float), stream);
  const dim3 grid((unsigned)(most > 0 ? (most + LD_THREADS - 1) / LD_THREADS : 1), (unsigned)N, (unsigned)B);
  ld_scatter_kernel<<<grid, LD_THREADS, 0, stream>>>(O, pts, inv_rots, trans, intrins, intrin_dim, post_rots,
                                                     post_trans, fH, fW, o);
  OCC_LAUNCH_CHECK();
  const long long blocks = (n + LD_THREADS - 1) / LD_THREADS;
  ld_finish_kernel<<<(unsigned)(blocks < 132 * 16 ? blocks : 132 * 16), LD_THREADS, 0, stream>>>(o, n);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
