// Shared geometry and softmax / P V core of the two window-attention kernels (window_attn.cu: q/k/v from HBM;
// swin_attn_fused.cu: QKV projection inside the kernel): 7x7 windows over the B*(Z+1) X-Y images, token -> global row,
// shift-mask regions.
#pragma once
#include "occ_common.cuh"
#include "occ_ptx.cuh"

namespace occ {

constexpr int WS = 7;
constexpr int WT = WS * WS;  // 49 tokens
constexpr int HD = 32;       // head dim (multihead_base_channel, dualpath_block.py:32)
constexpr int WA_STAGES = 4;
constexpr int WA_TILE = 128 * HD * 4;                  // 16 KB: 128 rows x 128 B
constexpr int WA_BIAS_FLOATS = 2404;                   // 49*49 padded to a 16-byte multiple
constexpr int WA_OFF_SRC = 3 * WA_TILE;                // 49152: per row, the global source pointer of its q slice (8 B)
constexpr int WA_STAGE_BYTES = 49 * 1024;              // 50176 = 49152 + 128 * 8, multiple of 1024
constexpr int WA_BIAS_LD = 52;                         // padded bias row pitch (floats): 13 conflict-free LDS.128 per row
constexpr int WA_BIAS_BYTES = 10240;                   // resident bias of this CTA's head, (49, 52) floats, * log2(e)
constexpr int WA_THREADS = 384;                        // two consumer warpgroups (one window each) + four loader warps

struct WinGeom {
  int B, X, Y, Z, C, heads, shift;
  int head_major;  // qkv columns ordered [head][q|k|v][32] instead of the reference's [q|k|v][head][32]
  int Xp, Yp, nWx, nWy;
  long long vox_rows;  // B*X*Y*Z
  long long nwin;
  int passes;  // tensor-core passes per 32-k block (occ_common.cuh: mma_passes)
};

// token t of window (img, wx, wy) -> global token row (or -1 for a pad token) and shift-mask region id
__device__ __forceinline__ long long window_token_row(const WinGeom& g, int img, int wx, int wy, int t, int* region) {
  const int i = t / WS, j = t % WS;
  const int xs = wx * WS + i, ys = wy * WS + j;
  int x = xs, y = ys;
  if (g.shift) {
    x = xs + 3; if (x >= g.Xp) x -= g.Xp;
    y = ys + 3; if (y >= g.Yp) y -= g.Yp;
    const int rx = xs < g.Xp - WS ? 0 : (xs < g.Xp - 3 ? 1 : 2);
    const int ry = ys < g.Yp - WS ? 0 : (ys < g.Yp - 3 ? 1 : 2);
    *region = rx * 3 + ry;
  } else {
    *region = 0;
  }
  if (x >= g.X || y >= g.Y) return -1;
  if (img < g.B * g.Z) {
    const int b = img / g.Z, z = img % g.Z;
    return (((long long)b * g.X + x) * g.Y + y) * g.Z + z;
  }
  const int b = img - g.B * g.Z;
  return g.vox_rows + ((long long)b * g.X + x) * g.Y + y;
}

// Inverse of window_token_row for real tokens: token (img, x, y) -> row of the WINDOW-LAYOUT buffer, window * 64 + t with
// window = (wx * nWy + wy) * n_images + img (the
// 49 tokens of a window are 49 consecutive rows, windows are 64 rows apart, rows 49..63 stay zero; a pair of windows is
// one 128-row MMA tile that a single TMA box fetches).  Window pad tokens (positions >= X or >= Y of the padded image)
// have no source token: their rows are never written and stay zero.
__device__ __forceinline__ long long window_layout_row(const WinGeom& g, int img, int x, int y) {
  int xs = x, ys = y;
  if (g.shift) {
    xs = x - 3; if (xs < 0) xs += g.Xp;
    ys = y - 3; if (ys < 0) ys += g.Yp;
  }
  const int wx = xs / WS, wy = ys / WS;
  const int t = (xs - wx * WS) * WS + (ys - wy * WS);
  // window index = (wx, wy) major, image minor: the Z + 1 images of a (b, x, y) column -- which the producer handles
  // together -- land 32 KB apart instead of one whole image (27 MB at 200 x 200) apart, and a pair of windows is the
  // same (wx, wy) in two adjacent height slices, whose output rows are neighbours in token order
  return (((long long)wx * g.nWy + wy) * ((long long)g.B * (g.Z + 1)) + img) * 64 + t;
}

// Key-region mask of a window: bit k (k < 49) set iff key k lies in shift-mask region `reg` (all 49 bits for an
// un-shifted partition).  Regions are separable: region = rx(window row) * 3 + ry(window column).
__device__ __forceinline__ uint64_t window_same_mask(const WinGeom& g, int wx, int wy, int reg) {
  if (!g.shift) return (1ull << WT) - 1;
  uint32_t xeq = 0, yeq = 0;
#pragma unroll
  for (int i = 0; i < WS; ++i) {
    const int xs = wx * WS + i, ys = wy * WS + i;
    const int rx = xs < g.Xp - WS ? 0 : (xs < g.Xp - 3 ? 1 : 2);
    const int ry = ys < g.Yp - WS ? 0 : (ys < g.Yp - 3 ? 1 : 2);
    xeq |= (uint32_t)(rx == reg / 3) << i;
    yeq |= (uint32_t)(ry == reg % 3) << i;
  }
  uint64_t m = 0;
#pragma unroll
  for (int i = 0; i < WS; ++i)
    if ((xeq >> i) & 1u) m |= (uint64_t)yeq << (WS * i);
  return m;
}

// Softmax and P V of one window and head on a warpgroup (the window's 64 query rows, wgmma fragment layout of
// occ_ptx.cuh: this thread holds rows t[0] = 16 (warp % 4) + lane / 4 and t[1] = t[0] + 8, key columns 8j + 2 (lane % 4)
// + {0, 1}).  s: raw scores Q K^T (keys >= 49 are ignored); sb: relative-position bias (49, WA_BIAS_LD) * log2 e;
// diff[r]: keys outside the row's shift-mask region (additive -100, as the reference).  The probabilities are split into
// hi / lo register A fragments and multiplied with the V tile (vdesc: MN-major SWIZZLE_128B, 64 key rows of
// [hi | lo] of the head dim = N 64): o[:, :32] + o[:, 32:] = unnormalised P V; sum[r] = softmax denominators.
template <int PASSES>
__device__ __forceinline__ void wa_softmax_pv(float (&s)[32], const float* __restrict__ sb, const int (&t)[2],
                                              const uint64_t (&diff)[2], uint64_t vdesc, float (&o)[32],
                                              float (&sum)[2]) {
  const int q = threadIdx.x & 3;
  const float sl2 = 0.17677669529663687f * 1.4426950408889634f;  // 32^-0.5 * log2 e: scores live in the log2 domain
  const float neg = -100.0f * 1.4426950408889634f;
  const float* brow[2] = {sb + (t[0] < WT ? t[0] : 0) * WA_BIAS_LD, sb + (t[1] < WT ? t[1] : 0) * WA_BIAS_LD};
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int r = (j >> 1) & 1, c = 8 * (j >> 2) + 2 * q + (j & 1);
    if (c < WT) {
      float z = fmaf(s[j], sl2, brow[r][c]);
      if ((diff[r] >> c) & 1ull) z += neg;
      s[j] = z;
      mx[r] = fmaxf(mx[r], z);
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
    mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    sum[r] = 0.f;
  }
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int r = (j >> 1) & 1, c = 8 * (j >> 2) + 2 * q + (j & 1);
    const float pj = c < WT ? ex2_approx(s[j] - mx[r]) : 0.f;
    sum[r] += pj;
    s[j] = pj;
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
  }
  uint32_t ph[4][4], pl[4][4];
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) split_frag_k16(&s[8 * kk], ph[kk], pl[kk]);
#pragma unroll
  for (int j = 0; j < 32; ++j) o[j] = 0.f;
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {  // 16 keys per wgmma = two 8-key (1024 B) atoms of V rows
    wgmma_rs<64, 1>(o, ph[kk], vdesc + (uint64_t)(kk * 128), kk != 0);           // P_hi [V_hi | V_lo]
    if constexpr (PASSES == 3) wgmma_rs<64, 1>(o, pl[kk], vdesc + (uint64_t)(kk * 128), 1u);  // P_lo [V_hi | V_lo]
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_fence_regs(o);
}

// o / sum of wa_softmax_pv -> the head's 32 output channels of the thread's two rows, as (parts of) one S32 chunk per row
// (A operand of the projection GEMM).  row[r] < 0 (window pad token, MMA padding row) and t[r] >= 49 are not written.
__device__ __forceinline__ void wa_store_rows(const float (&o)[32], const float (&sum)[2], const long long (&row)[2],
                                              const int (&t)[2], float* __restrict__ out, int C, int h) {
  const int q = threadIdx.x & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    if (t[r] < WT && row[r] >= 0) {
      const float inv = 1.0f / sum[r];
      uint8_t* dst = reinterpret_cast<uint8_t*>(out + row[r] * C + h * HD);
#pragma unroll
      for (int nb = 0; nb < 4; ++nb) {
        const float a = (o[4 * nb + 2 * r] + o[4 * (nb + 4) + 2 * r]) * inv;
        const float b = (o[4 * nb + 2 * r + 1] + o[4 * (nb + 4) + 2 * r + 1]) * inv;
        uint32_t hi, lo;
        split_pair(a, b, hi, lo);
        const int d = 8 * nb + 2 * q;
        *reinterpret_cast<uint32_t*>(dst + 2 * d) = hi;
        *reinterpret_cast<uint32_t*>(dst + 64 + 2 * d) = lo;
      }
    }
  }
}

inline WinGeom make_win_geom(int B, int X, int Y, int Z, int C, int heads, int shift) {
  WinGeom g;
  g.B = B; g.X = X; g.Y = Y; g.Z = Z; g.C = C; g.heads = heads; g.shift = shift ? 1 : 0;
  g.head_major = 1;
  g.nWx = (X + WS - 1) / WS; g.nWy = (Y + WS - 1) / WS;
  g.Xp = g.nWx * WS; g.Yp = g.nWy * WS;
  g.vox_rows = (long long)B * X * Y * Z;
  g.nwin = (long long)B * (Z + 1) * g.nWx * g.nWy;
  g.passes = mma_passes();
  return g;
}

}  // namespace occ
