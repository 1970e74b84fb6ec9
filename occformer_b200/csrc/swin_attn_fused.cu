// Shifted-window attention with the QKV projection fused in (C = 128): the kernel reads the LayerNorm'ed tokens once
// (S32, 512 B per token) instead of a materialised q/k/v tensor (1.5 KB per token written by a GEMM and read back).
//
//   WindowMSA.forward: qkv = Linear(C -> 3C)(x) ... attn = softmax(q k^T * scale + bias [+ mask]) v
//   (projects/mmdet3d_plugin/occformer/backbones/modules/window_attention.py:69-107), ShiftWindowMSA pad / roll / mask /
//   partition / reverse (:168-242) as index arithmetic, exactly as in window_attn.cu (same geometry header).
//
// Work unit = (pair of windows, head), one head per CTA (gridDim.x is a multiple of the head count): the head's 96 x 128
// slice of the qkv weight (rows [q | k | v] x 32, head-major) stays resident in shared memory for the whole kernel.
//   loader (warp 8)        one TMA box (32 channels x 128 rows) per k-block into a ring of SF_NSLOT slots (two units):
//                          the tokens arrive in WINDOW LAYOUT (window_geom.cuh: the LayerNorm producer writes token
//                          (img, x, y) to row window * 64 + t), so a pair of windows is a contiguous tile.
//   warps 0-3 / 4-7        one warpgroup per window of the pair, per unit:
//       M1      : D[64 x 96] = A W_h^T (4 k-blocks x 6 wgmma 64x96x16: three bf16 passes), + qkv bias
//       operands: k and v rows -> S32 K / V tiles of the warpgroup in shared memory; q stays in registers as the A
//                 fragments of QK^T
//       QK      : S = Q K^T (6 wgmma 64x64x16, A from registers)
//       softmax / PV / epilogue: as window_attn.cu (window_geom.cuh: wa_softmax_pv, wa_store_rows)
#include "window_geom.cuh"

namespace occ {

constexpr int SF_C = 128;
constexpr int SF_KB = SF_C / 32;                      // k-blocks of the projection
constexpr int SF_W_BYTES = SF_KB * 96 * 128;          // 49152: W_h as 4 K-major SWIZZLE_128B tiles of 96 rows
constexpr int SF_SLOT = 128 * 128;                    // 16384: one k-block of the token tile (128 rows x 128 B)
constexpr int SF_NSLOT = 8;                           // ring of k-block slots = 2 token tiles
constexpr int SF_THREADS = 288;                       // two consumer warpgroups + the loader warp
constexpr int SF_OFF_A = SF_W_BYTES;                                    // 49152
constexpr int SF_OFF_KV = SF_OFF_A + SF_NSLOT * SF_SLOT;                // 180224: per warpgroup a K and a V tile (64 rows)
constexpr int SF_OFF_BIAS = SF_OFF_KV + 2 * 2 * 64 * 128;               // 212992: relative-position bias (49, 52) * log2 e
constexpr int SF_OFF_QB = SF_OFF_BIAS + WA_BIAS_BYTES;                  // 223232: this head's 96 qkv bias values
constexpr int SF_OFF_BAR = SF_OFF_QB + 384;                             // 223616
constexpr int SF_SMEM = SF_OFF_BAR + 2 * SF_NSLOT * 8 + 1024;           // 224768 <= 232448 (227 KB)

template <int PASSES>  // tensor-core passes per 32-k block, fixed so that each wgmma batch is one straight line
__global__ void __launch_bounds__(SF_THREADS, 1)
swin_qkv_attn_kernel(const __grid_constant__ CUtensorMap tmap_tok /*window-layout tokens (npairs*128, 128) S32, box 32 x 128*/,
                     const float* __restrict__ wqkv /*(384, 128) S32,
                     head-major rows*/, const float* __restrict__ bqkv /*(384) fp32, head-major*/,
                     const float* __restrict__ bias_pad /*(heads, 2404)*/, float* __restrict__ out, const WinGeom g) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sw = smem;
  uint8_t* sa = smem + SF_OFF_A;
  float* sb = reinterpret_cast<float*>(smem + SF_OFF_BIAS);
  float* sqb = reinterpret_cast<float*>(smem + SF_OFF_QB);
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + SF_OFF_BAR);  // [SF_NSLOT] k-block slot filled
  uint64_t* a_empty = a_full + SF_NSLOT;                              // [SF_NSLOT] k-block slot consumed by M1

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long npairs = (g.nwin + 1) / 2;
  const int H = g.heads;
  const int h = blockIdx.x % H;
  const int pair0 = blockIdx.x / H, pair_stride = gridDim.x / H;
  const long long n_units = (npairs > pair0) ? (npairs - pair0 + pair_stride - 1) / pair_stride : 0;

  // resident operands of this head: W_h (96 rows of the head-major qkv weight) as 4 K-major swizzled k-blocks, its bias,
  // the relative-position bias table (log2 domain)
  for (int i = threadIdx.x; i < 96 * 32; i += SF_THREADS) {  // 16-byte chunks: row r, chunk cc of the 512-byte row
    const int r = i >> 5, cc = i & 31;
    const int kb = cc >> 3, c = cc & 7;
    const float4 v = __ldg(reinterpret_cast<const float4*>(wqkv + ((size_t)h * 96 + r) * SF_C) + cc);
    *reinterpret_cast<float4*>(sw + kb * (96 * 128) + r * 128 + ((c ^ (r & 7)) << 4)) = v;
  }
  if (threadIdx.x < 96) sqb[threadIdx.x] = bqkv[h * 96 + threadIdx.x];
  for (int i = threadIdx.x; i < WT * WA_BIAS_LD; i += SF_THREADS) {
    const int r = i / WA_BIAS_LD, c = i % WA_BIAS_LD;
    sb[i] = c < WT ? bias_pad[(size_t)h * WA_BIAS_FLOATS + r * WT + c] * 1.4426950408889634f : 0.f;
  }
  if (warp == 8 && lane == 0) {
    for (int i = 0; i < SF_NSLOT; ++i) {
      mbar_init(&a_full[i], 1);   // expect_tx by the loader
      mbar_init(&a_empty[i], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  fence_proxy_async_smem();  // W_h was written with generic stores; the wgmmas read it through the async proxy
  __syncthreads();

  if (warp == 8) {
    // ===================================================================== loader: one TMA box per k-block
    if (lane == 0) {
      uint32_t slot = 0, par = 1;  // parity of the "slot is empty" phase to wait for (fresh barriers pass parity 1)
      for (uint32_t u = 0; u < (uint32_t)n_units; ++u) {
        const int row0 = (int)((pair0 + (long long)u * pair_stride) * 128);
#pragma unroll 1
        for (int kb = 0; kb < SF_KB; ++kb) {
          mbar_wait(&a_empty[slot], par);
          mbar_expect_tx(&a_full[slot], SF_SLOT);
          tma_load_2d(sa + (size_t)slot * SF_SLOT, &tmap_tok, &a_full[slot], kb * 32, row0);
          if (++slot == SF_NSLOT) { slot = 0; par ^= 1; }
        }
      }
    }
  } else {
    // ===================================================================== one warpgroup per window of the pair
    const int half = warp >> 2;
    const int q4 = lane & 3;
    const int t[2] = {(warp & 3) * 16 + (lane >> 2), (warp & 3) * 16 + (lane >> 2) + 8};  // window token of my rows
    uint8_t* ktile = smem + SF_OFF_KV + half * (2 * 64 * 128);
    uint8_t* vtile = ktile + 64 * 128;
    const uint64_t kdesc = make_sw128_desc(smem_u32(ktile), 1024, 16);
    const uint64_t vdesc = make_sw128_desc(smem_u32(vtile), 1024, 1024);
    const uint64_t wdesc0 = make_sw128_desc(smem_u32(sw), 1024, 16);
    uint32_t slot = 0, par = 0;
    for (long long u = 0; u < n_units; ++u) {
      // ---- M1: q | k | v of my window's 64 rows
      float d[48];
#pragma unroll
      for (int j = 0; j < 48; ++j) d[j] = 0.f;
      int prev = -1;
#pragma unroll 1
      for (int kb = 0; kb < SF_KB; ++kb) {
        mbar_wait(&a_full[slot], par);
        wgmma_fence();
        wgmma_bf16x3_ss<96, PASSES>(d, make_sw128_desc(smem_u32(sa + (size_t)slot * SF_SLOT) + half * (64 * 128), 1024, 16),
                                    wdesc0 + (uint64_t)(kb * ((96 * 128) >> 4)), kb != 0);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && lane == 0) mbar_arrive(&a_empty[prev]);
        prev = (int)slot;
        if (++slot == SF_NSLOT) { slot = 0; par ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      if (lane == 0) mbar_arrive(&a_empty[prev]);
#pragma unroll
      for (int j = 0; j < 48; ++j) d[j] += sqb[8 * (j >> 2) + 2 * q4 + (j & 1)];
      // ---- metadata of my rows: global token row, keys outside the row's shift-mask region
      long long row[2] = {-2, -2};
      uint64_t diff[2] = {0, 0};
      {
        const long long win = 2 * (pair0 + u * pair_stride) + half;
        if (win < g.nwin) {
          const int nimg = g.B * (g.Z + 1);  // window index = (wx * nWy + wy) * n_images + img (window_geom.cuh)
          const int img = (int)(win % nimg), w2 = (int)(win / nimg);
          const int wx = w2 / g.nWy, wy = w2 % g.nWy;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            int reg = 0;
            if (t[r] < WT) {
              row[r] = window_token_row(g, img, wx, wy, t[r], &reg);
              diff[r] = ~window_same_mask(g, wx, wy, reg) & ((1ull << WT) - 1);
            }
          }
        }
      }
      // ---- k, v rows -> the S32 K / V tiles (K-major SWIZZLE_128B: 16-byte chunk c of row r at c ^ (r & 7))
      named_bar_sync(1 + half, 128);  // the previous unit's QK^T / PV of this warpgroup have read the tiles
#pragma unroll
      for (int r = 0; r < 2; ++r) {
#pragma unroll
        for (int nb = 4; nb < 12; ++nb) {
          uint32_t hi, lo;
          split_pair(d[4 * nb + 2 * r], d[4 * nb + 2 * r + 1], hi, lo);
          uint8_t* trow = (nb < 8 ? ktile : vtile) + t[r] * 128;
          const int bh = 2 * (8 * (nb & 3) + 2 * q4), bl = 64 + bh;
          *reinterpret_cast<uint32_t*>(trow + ((((bh >> 4) ^ (t[r] & 7)) << 4) | (bh & 15))) = hi;
          *reinterpret_cast<uint32_t*>(trow + ((((bl >> 4) ^ (t[r] & 7)) << 4) | (bl & 15))) = lo;
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1 + half, 128);
      // ---- QK^T with q as register A fragments (head dim k = 16 h .. 16 h + 15)
      uint32_t qh[2][4], ql[2][4];
      split_frag_k16(&d[0], qh[0], ql[0]);
      split_frag_k16(&d[8], qh[1], ql[1]);
      float sc[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) sc[j] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        wgmma_rs<64, 0>(sc, qh[hh], kdesc + 2 * hh, hh != 0);                 // hi * hi
        if constexpr (PASSES == 3) {
          wgmma_rs<64, 0>(sc, ql[hh], kdesc + 2 * hh, 1u);                    // lo * hi
          wgmma_rs<64, 0>(sc, qh[hh], kdesc + 2 * (2 + hh), 1u);              // hi * lo
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sc);
      float o[32], sum[2];
      wa_softmax_pv<PASSES>(sc, sb, t, diff, vdesc, o, sum);
      wa_store_rows(o, sum, row, t, out, g.C, h);
    }
  }
}

}  // namespace occ

using namespace occ;

// tokn (occ_window_layout_rows(B,X,Y,Z), 128) S32 = LayerNorm1'ed tokens in the WINDOW LAYOUT of this block's partition
// (shift), zero where no token lands (occ_gn_relu_zmean_ln with win_shift = shift writes it); wqkv (384, 128) S32 and
// bqkv (384) fp32 with HEAD-MAJOR rows [head][q|k|v][32]; bias_pad as occ_window_attention; out (rows, 128) S32.
// Returns -2 (unsupported) for C != 128: the caller then runs occ_gemm_bf16x3 + occ_window_attention.
extern "C" int occ_swin_qkv_attention(const float* tokn, const float* wqkv, const float* bqkv, const float* bias_pad,
                                      float* out, int B, int X, int Y, int Z, int C, int heads, int shift,
                                      cudaStream_t stream) {
  OCC_REQUIRE(tokn && wqkv && bqkv && bias_pad && out);
  OCC_REQUIRE(B > 0 && X > 0 && Y > 0 && Z > 0 && heads > 0 && C == heads * HD);
  if (C != SF_C) return OCC_EUNSUPPORTED;
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(tokn) & 15) == 0 && (reinterpret_cast<uintptr_t>(wqkv) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(bias_pad) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0);
  const WinGeom g = make_win_geom(B, X, Y, Z, C, heads, shift);
  OCC_REQUIRE(g.nwin < (1ll << 31));
  static_assert(SF_SMEM <= 227 * 1024, "shared memory budget");
  const long long npairs = (g.nwin + 1) / 2;
  long long groups = sm_count() / heads;
  if (groups > npairs) groups = npairs;
  if (groups < 1) groups = 1;
  CUtensorMap tm;
  {
    const long long rows = (g.nwin + 1) / 2 * 128;  // occ_window_layout_rows
    const uint64_t dims[2] = {(uint64_t)SF_C, (uint64_t)rows}, strides[1] = {(uint64_t)SF_C * 4};
    const uint32_t box[2] = {32, 128};
    OCC_REQUIRE(make_tmap_f32(&tm, tokn, 2, dims, strides, box, nullptr) == OCC_OK);
  }
  auto launch = [&](auto passes) {
    constexpr int P = decltype(passes)::value;
    OCC_ENSURE_SMEM(swin_qkv_attn_kernel<P>, SF_SMEM);
    swin_qkv_attn_kernel<P><<<(int)(groups * heads), SF_THREADS, SF_SMEM, stream>>>(tm, wqkv, bqkv, bias_pad, out, g);
    OCC_LAUNCH_CHECK();
    return OCC_OK;
  };
  return g.passes == 1 ? launch(std::integral_constant<int, 1>{}) : launch(std::integral_constant<int, 3>{});
}
