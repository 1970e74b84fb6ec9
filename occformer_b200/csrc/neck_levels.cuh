// The level pyramid of the pixel decoder's level-major token rows (csrc/neck_ops.cu), shared by its kernels: the per-level
// grid, the first token of each level, and the mapping of a global row back to (level, sample, local voxel).
#pragma once
#include "occ_common.cuh"

namespace occ {

constexpr int NK_MAX_LEVELS = 4;
constexpr int NK_PX = 4, NK_PY = 4;  // query patch of the deformable gather: NK_PX x NK_PY x Z_l tokens of one level

struct NeckLevels {
  int L, B;
  int X[NK_MAX_LEVELS], Y[NK_MAX_LEVELS], Z[NK_MAX_LEVELS];
  int start[NK_MAX_LEVELS];  // first token of the level inside one sample's Nq tokens (levels coarse -> fine)
  int n[NK_MAX_LEVELS];      // X*Y*Z
  float stride[NK_MAX_LEVELS];
  int pstart[NK_MAX_LEVELS]; // first query patch of the level (deformable gather grid), all samples
  int npatches;
  long long rows;            // B * Nq
};

// global row -> (level, sample, local voxel index)
__device__ __forceinline__ void nk_locate(const NeckLevels& g, long long row, int& lvl, int& b, int& local) {
  lvl = 0;
#pragma unroll
  for (int l = 1; l < NK_MAX_LEVELS; ++l)
    if (l < g.L && row >= (long long)g.B * g.start[l]) lvl = l;
  const long long r = row - (long long)g.B * g.start[lvl];
  b = (int)(r / g.n[lvl]);
  local = (int)(r - (long long)b * g.n[lvl]);
}

inline int fill_levels(NeckLevels& g, int L, int B, const int* grids, const float* strides) {
  if (L < 1 || L > NK_MAX_LEVELS || B < 1) return OCC_EINVAL;
  g.L = L; g.B = B;
  int start = 0;
  for (int l = 0; l < NK_MAX_LEVELS; ++l) {
    if (l < L) {
      g.X[l] = grids[3 * l]; g.Y[l] = grids[3 * l + 1]; g.Z[l] = grids[3 * l + 2];
      if (g.X[l] < 1 || g.Y[l] < 1 || g.Z[l] < 1) return OCC_EINVAL;
      g.n[l] = g.X[l] * g.Y[l] * g.Z[l];
      g.start[l] = start;
      g.stride[l] = strides ? strides[l] : 1.f;
      start += g.n[l];
    } else {
      g.X[l] = g.Y[l] = g.Z[l] = 1; g.n[l] = 1; g.start[l] = 0x3fffffff; g.stride[l] = 1.f;
    }
  }
  g.rows = (long long)B * start;
  int ps = 0;
  for (int l = 0; l < NK_MAX_LEVELS; ++l) {
    g.pstart[l] = l < L ? ps : 0x3fffffff;
    if (l < L) ps += B * ((g.X[l] + NK_PX - 1) / NK_PX) * ((g.Y[l] + NK_PY - 1) / NK_PY);
  }
  g.npatches = ps;
  return OCC_OK;
}

}  // namespace occ
