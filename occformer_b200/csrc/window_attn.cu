// Shifted-window multi-head self-attention core over the B*(Z+1) X-Y images of the dual-path encoder, on the Hopper
// tensor cores (wgmma on split-bf16 operands, three passes per contraction = fp32-faithful, see occ_ptx.cuh; scores and
// probabilities in registers).  qkv arrives in the S32 split format (one 128-byte chunk per (token, head, q|k|v)), the
// output is written in S32 (A operand of the projection GEMM).
//
// Replaces ShiftWindowMSA.forward's pad / roll / mask build / window_partition / window_reverse / roll back /
// crop and WindowMSA.forward's score pipeline (q*scale, QK^T, + relative-position bias, + shift mask, softmax,
// PV) -- projects/mmdet3d_plugin/occformer/backbones/modules/window_attention.py:168-242 and :69-107 -- with
// index arithmetic: the kernel gathers the 49 tokens of a (possibly shifted, possibly padded) window straight
// from the token-ordered qkv tensor and scatters the result back to token order.  No (nW,49,49) mask tensor,
// no score tensor in HBM.
//
// Semantics kept (SURVEY.md Appendix D.5-D.8):
//   * padding to a multiple of 7 happens AFTER LayerNorm: pad tokens are zeros, so their q/k/v equal the qkv
//     bias and they take part in the softmax as real keys; their outputs are cropped.
//   * shifted blocks: roll(-3,-3); region ids from slices (0,-7),(-7,-3),(-3,None) on the padded extent;
//     additive mask -100.0 (not -inf) where ids differ.
//   * relative-position bias added after the q*scale product.
//
// Work unit = (pair of windows, head): 128 tile rows (window A in rows 0..63, window B in rows 64..127, 49 real rows
// each).  Persistent CTA, 384 threads:
//   warps 8-11  loaders : cp.async gather of the Q / K / V head slices (128 B per token) into 128B-swizzled tiles, a
//                         ring of WA_STAGES units
//   warps 0-3 / 4-7     : one warpgroup per window of the pair: S = Q K^T (6 wgmma 64x64x16: hi*hi + lo*hi + hi*lo over
//                         the 32-wide head dim), scale, bias, shift mask, softmax in registers, O' = [P_hi; P_lo]
//                         [V_hi | V_lo] (8 wgmma 64x64x16, P as register A fragments, the V rows as an MN-major
//                         SWIZZLE_128B operand, N = 64 = hi | lo halves of the head dim -- no transpose of V anywhere),
//                         O = O'[:, :32] + O'[:, 32:], normalise, scatter 128 B per (token, head) to global.
#include "window_geom.cuh"

namespace occ {

template <int PASSES>  // tensor-core passes per 32-k block, fixed so that each wgmma batch is one straight line
__global__ void __launch_bounds__(WA_THREADS, 1)
window_attn_tc_kernel(const float* __restrict__ qkv, const float* __restrict__ qkv_bias,
                      const float* __restrict__ bias_pad /*(heads, 2404)*/, float* __restrict__ out, const WinGeom g) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  float* sb = reinterpret_cast<float*>(smem + WA_STAGES * WA_STAGE_BYTES);  // bias of head h, resident
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + WA_STAGES * WA_STAGE_BYTES + WA_BIAS_BYTES);
  uint64_t* empty_bar = full_bar + WA_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long npairs = (g.nwin + 1) / 2;
  const int H = g.heads;
  // One head per CTA (gridDim.x is a multiple of H): CTA c works on head c % H of the window pairs c / H,
  // + gridDim.x / H, ...  The H CTAs of a group walk the same pairs at the same time, so the 12 128-byte segments of
  // every qkv token row (one DRAM page) are fetched together, and the head's bias table stays resident in smem.
  const int h = blockIdx.x % H;
  // head-major qkv: the head's q, k, v slices are one contiguous 384-byte run per token (three adjacent lines of one
  // DRAM page); reference order: three 128-byte slices C floats apart
  const int h_off = g.head_major ? h * 3 * HD : h * HD;
  const int kv_step = g.head_major ? HD : g.C;
  const int pair0 = blockIdx.x / H, pair_stride = gridDim.x / H;
  const long long n_units = (npairs > pair0) ? (npairs - pair0 + pair_stride - 1) / pair_stride : 0;
  for (int i = threadIdx.x; i < WT * WA_BIAS_LD; i += WA_THREADS) {  // scores live in the log2 domain (exp2 softmax)
    const int r = i / WA_BIAS_LD, c = i % WA_BIAS_LD;
    sb[i] = c < WT ? bias_pad[(size_t)h * WA_BIAS_FLOATS + r * WT + c] * 1.4426950408889634f : 0.f;
  }
  if (warp == 8 && lane == 0) {
    for (int i = 0; i < WA_STAGES; ++i) {
      mbar_init(&full_bar[i], 256); // per loader thread: one asynchronous cp.async arrival + one release arrival
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // ===================================================================== loaders
    const int l = threadIdx.x - 8 * 32;  // 0..127
    const int C = g.C;
    for (long long u = 0; u < n_units; ++u) {
      const int s = (int)(u % WA_STAGES);
      const long long pair = pair0 + u * pair_stride;
      uint8_t* st = smem + (size_t)s * WA_STAGE_BYTES;
      mbar_wait(&empty_bar[s], (uint32_t)(((u / WA_STAGES) & 1) ^ 1));
      {  // source of row l: window = 2*pair + l/64, token = l%64; pad tokens read the qkv bias, MMA padding rows are zero
        const long long win = 2 * pair + (l >> 6);
        const int t = l & 63;
        long long r = -2;
        if (t < WT && win < g.nwin) {
          long long w = win;
          const int wy = (int)(w % g.nWy); w /= g.nWy;
          const int wx = (int)(w % g.nWx); w /= g.nWx;
          int reg;
          r = window_token_row(g, (int)w, wx, wy, t, &reg);
        }
        // global address of this token's q head-slice (k / v follow at +kv_step / +2 kv_step floats)
        reinterpret_cast<const float**>(st + WA_OFF_SRC)[l] =
            r >= 0 ? qkv + r * 3 * C + h_off : (r == -1 ? qkv_bias + h_off : nullptr);
      }
      named_bar_sync(2, 128);
      // thread l copies 16-byte chunk c = l & 7 of rows (l >> 3) + 16*rr, rr = 0..7, for the three tiles.  (r & 7) does
      // not depend on rr, so the swizzled chunk offset is a per-thread constant:
      //   Q, K: K-major SWIZZLE_128B (16-byte chunk c ^ (r & 7)); V: MN-major bf16 operand, N = 64 (hi | lo of the head
      //   dim) = one 128-byte row per key, 8-key atoms -- the same SWIZZLE_128B chunk pattern
      {
        const int c = l & 7, rb = l >> 3;
        const int off = (c ^ (rb & 7)) << 4;
        const float* const* srcp = reinterpret_cast<const float* const*>(st + WA_OFF_SRC);
#pragma unroll
        for (int rr = 0; rr < 8; ++rr) {
          const int r = rb + 16 * rr;
          uint8_t* drow = st + r * 128;
          const float* src = srcp[r];
          if (src == nullptr) {
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            *reinterpret_cast<float4*>(drow + off) = z;
            *reinterpret_cast<float4*>(drow + WA_TILE + off) = z;
            *reinterpret_cast<float4*>(drow + 2 * WA_TILE + off) = z;
          } else {
            cp_async_16(drow + off, src + c * 4);
            cp_async_16(drow + WA_TILE + off, src + kv_step + c * 4);
            cp_async_16(drow + 2 * WA_TILE + off, src + 2 * kv_step + c * 4);
          }
        }
      }
      cp_async_mbar_arrive_noinc(&full_bar[s]);  // fires when this thread's copies of the unit have landed
      mbar_arrive(&full_bar[s]);                 // release: zero-fill stores
    }
    // the loaders never wait for their own copies: up to WA_STAGES units of gathers are in flight per CTA
    cp_async_wait<0>();
  } else {
    // ===================================================================== one warpgroup per window of the pair
    const int half = warp >> 2;
    const int t[2] = {(warp & 3) * 16 + (lane >> 2), (warp & 3) * 16 + (lane >> 2) + 8};  // window token of my rows
    for (long long u = 0; u < n_units; ++u) {
      const int s = (int)(u % WA_STAGES);
      const long long win = 2 * (pair0 + u * pair_stride) + half;
      // metadata of my rows (while the gathers land): global token row, keys outside the row's shift-mask region
      long long row[2] = {-2, -2};
      uint64_t diff[2] = {0, 0};
      if (win < g.nwin) {
        long long w = win;
        const int wy = (int)(w % g.nWy); w /= g.nWy;
        const int wx = (int)(w % g.nWx); w /= g.nWx;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          int reg = 0;
          if (t[r] < WT) {
            row[r] = window_token_row(g, (int)w, wx, wy, t[r], &reg);
            diff[r] = ~window_same_mask(g, wx, wy, reg) & ((1ull << WT) - 1);
          }
        }
      }
      mbar_wait(&full_bar[s], (uint32_t)((u / WA_STAGES) & 1));
      fence_proxy_async_smem();  // cp.async / st.shared (generic proxy) -> wgmma operand reads (async proxy)
      const uint32_t base = smem_u32(smem + (size_t)s * WA_STAGE_BYTES) + half * (64 * 128);
      float sc[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) sc[j] = 0.f;
      wgmma_fence();
      wgmma_bf16x3_ss<64, PASSES>(sc, make_sw128_desc(base, 1024, 16), make_sw128_desc(base + WA_TILE, 1024, 16), 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sc);
      float o[32], sum[2];
      wa_softmax_pv<PASSES>(sc, sb, t, diff, make_sw128_desc(base + 2 * WA_TILE, 1024, 1024), o, sum);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);
      wa_store_rows(o, sum, row, t, out, g.C, h);
    }
  }
}

}  // namespace occ

using namespace occ;

// qkv (rows, 3C) with rows = B*X*Y*(Z+1) token-ordered (voxel tokens then BEV tokens); out (rows, C) in S32 (A operand of the projection GEMM); qkv and qkv_bias in S32.
// bias_pad = relative_position_bias_table[relative_position_index] arranged (heads, 49*49 padded to 2404 floats).
extern "C" int occ_window_attention(const float* qkv, const float* qkv_bias, const float* bias_pad, float* out, int B,
                                    int X, int Y, int Z, int C, int heads, int shift, int qkv_head_major,
                                    cudaStream_t stream) {
  OCC_REQUIRE(qkv && qkv_bias && bias_pad && out);
  OCC_REQUIRE(B > 0 && X > 0 && Y > 0 && Z > 0 && heads > 0 && C == heads * HD);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(qkv_bias) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(bias_pad) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0);
  WinGeom g = make_win_geom(B, X, Y, Z, C, heads, shift);
  g.head_major = qkv_head_major ? 1 : 0;
  OCC_REQUIRE(g.nwin < (1ll << 31));
  const size_t smem = (size_t)WA_STAGES * WA_STAGE_BYTES + WA_BIAS_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  static_assert((size_t)WA_STAGES * WA_STAGE_BYTES + WA_BIAS_BYTES + 1024 + 256 <= 227 * 1024, "shared memory budget");
  const long long npairs = (g.nwin + 1) / 2;
  OCC_REQUIRE(heads <= sm_count());
  long long groups = sm_count() / heads;  // CTA groups of `heads` CTAs, one head each
  if (groups > npairs) groups = npairs;
  const int grid = (int)(groups * heads);
  auto launch = [&](auto passes) {
    constexpr int P = decltype(passes)::value;
    OCC_ENSURE_SMEM(window_attn_tc_kernel<P>, smem);
    window_attn_tc_kernel<P><<<grid, WA_THREADS, smem, stream>>>(qkv, qkv_bias, bias_pad, out, g);
    OCC_LAUNCH_CHECK();
    return OCC_OK;
  };
  return g.passes == 1 ? launch(std::integral_constant<int, 1>{}) : launch(std::integral_constant<int, 3>{});
}
