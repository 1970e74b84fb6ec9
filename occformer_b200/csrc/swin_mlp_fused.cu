// Swin block tail for C = 128 tokens in one kernel: attention output projection + residual, LayerNorm2, FFN
// (Linear - GELU - Linear) + residual.  Three chained 128x128x128 GEMMs per 128-token tile on the wgmma tensor cores
// (split-bf16 operands, three passes = fp32-faithful, occ_ptx.cuh); the intermediate activations never leave the SM
// (registers / shared memory).
//
// Reference: mmdet SwinBlock.forward (swin.py) as used by projects/mmdet3d_plugin/occformer/backbones/
// dualpath_block.py:57-70 (shared_transformer on every Z slice and on the BEV slice):
//     x = identity + attn.proj(att)          (window_attention.py WindowMSA.proj, ShiftWindowMSA residual)
//     x = x + ffn(norm2(x))                  (FFN: Linear(C, C) -> GELU(erf) -> Linear(C, C))
// Unfused this is proj GEMM (R att, R tok, W y1) + LayerNorm (R y1, W y1n) + FFN1 (R y1n, W h) + FFN2 (R h, R y1, W y2):
// 2.4 GB of HBM traffic for the 680k tokens of a 200x200x16 grid; fused: R att, R tok, W y2 = 1.04 GB.
//
//   warp 8    : producer -- one ring of 16 KB k-blocks in the exact order the consumers read them: per tile
//               (att, Wp) x 4 k-blocks, W1 x 4, W2 x 4 (att from HBM, the weights from L2)
//   warps 0-7 : two consumer warpgroups, rows 64g .. 64g+63 of every 128-token tile, fp32 accumulators in registers:
//               M1 = att Wp^T (wgmma, both operands in shared memory) -> y1 = tok + M1 + bp (y1 + b2 parked in shared
//               memory) -> LayerNorm2 with quad shuffles (a row is spread over four lanes) -> split into register A
//               fragments -> M2 = LN2(y1) W1^T -> GELU(+ b1) -> register A fragments -> M3 accumulates h W2^T onto
//               y1 + b2 (the residual add is done by the tensor core) -> out.
#include "occ_common.cuh"
#include "occ_ptx.cuh"

namespace occ {

constexpr int SMF_THREADS = 288;
constexpr int SMF_C = 128;
constexpr int SMF_SLOT = 128 * 32 * 4;  // 16 KB k-block: 128 rows x 32 floats, K-major SWIZZLE_128B
constexpr int SMF_SLOTS = 8;
constexpr int SMF_PER_TILE = 16;        // k-blocks per tile in the ring: 4 x (att, Wp), 4 x W1, 4 x W2
constexpr int SMF_STASH = 64 * SMF_C * 4;  // per warpgroup: y1 + b2 of its 64 rows, fragment order
constexpr float SMF_EPS = 1e-5f;

struct SwinMlpParams {
  const float* tok;  // (M, 128) identity of the attention residual
  const float *bp, *lnw, *lnb, *b1, *b2;
  float* out;        // (M, 128)
  long long M;
  int n_tiles;
  int passes;  // tensor-core passes per 32-k block (occ_common.cuh: mma_passes)
};

// GELU(x) = x * Phi(x) with erfc(z) = P(t) exp(-z^2), t = 1 / (1 + p z) (Abramowitz-Stegun 7.1.26, |err| <= 1.5e-7):
// branch-free, 2 MUFU + ~14 FP32 ops instead of erff's ~30.
__device__ __forceinline__ float smf_gelu(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  const float t = __fdividef(1.0f, fmaf(0.3275911f, z, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float e = ex2_approx(-1.4426950408889634f * z * z);
  const float half_q = 0.5f * poly * t * e;               // 0.5 * erfc(z)
  const float phi = 0.5f + copysignf(0.5f - half_q, x);   // x >= 0: 1 - q/2 ; x < 0: q/2
  return x * phi;
}

template <int PASSES>  // tensor-core passes per 32-k block, fixed so that each wgmma batch is one straight line
__global__ void __launch_bounds__(SMF_THREADS, 1)
swin_mlp_fused_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmWp,
                      const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmW2,
                      const SwinMlpParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* ring = smem;
  float* stash = reinterpret_cast<float*>(ring + SMF_SLOTS * SMF_SLOT);
  float* vecs = stash + 2 * SMF_STASH / 4;  // bp | lnw | lnb | b1 | b2
  uint64_t* full = reinterpret_cast<uint64_t*>(vecs + 5 * SMF_C);
  uint64_t* empty = full + SMF_SLOTS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_my = (p.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmWp);
    tma_prefetch_desc(&tmW1);
    tma_prefetch_desc(&tmW2);
    for (int i = 0; i < SMF_SLOTS; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 5 * SMF_C; i += SMF_THREADS) {
    const int which = i / SMF_C, c = i % SMF_C;
    const float* src = which == 0 ? p.bp : which == 1 ? p.lnw : which == 2 ? p.lnb : which == 3 ? p.b1 : p.b2;
    vecs[i] = __ldg(src + c);
  }
  __syncthreads();

  if (warp == 8) {
    // ===================================================================== producer (consumption order)
    if (lane == 0) {
      int it = 0;
      for (int i = 0; i < n_my; ++i) {
        const int tile = blockIdx.x + i * gridDim.x;
        for (int k = 0; k < SMF_PER_TILE; ++k, ++it) {
          const int s = it % SMF_SLOTS;
          mbar_wait(&empty[s], (uint32_t)(((it / SMF_SLOTS) & 1) ^ 1));
          mbar_expect_tx(&full[s], SMF_SLOT);
          uint8_t* dst = ring + (size_t)s * SMF_SLOT;
          if (k < 8) {
            if (k & 1) tma_load_2d(dst, &tmWp, &full[s], (k >> 1) * 32, 0);
            else tma_load_2d(dst, &tmA, &full[s], (k >> 1) * 32, tile * 128);
          } else {
            tma_load_2d(dst, k < 12 ? &tmW1 : &tmW2, &full[s], (k & 3) * 32, 0);
          }
        }
      }
    }
  } else {
    // ===================================================================== consumer warpgroups
    const int cg = warp >> 2;
    const int q4 = lane & 3;
    const int r0 = cg * 64 + (warp & 3) * 16 + (lane >> 2);  // my rows of the tile: r0, r0 + 8
    const float *s_bp = vecs, *s_lnw = vecs + SMF_C, *s_lnb = vecs + 2 * SMF_C, *s_b1 = vecs + 3 * SMF_C,
                *s_b2 = vecs + 4 * SMF_C;
    float2* my_stash = reinterpret_cast<float2*>(stash + cg * (SMF_STASH / 4)) + (threadIdx.x & 127);
    int it = 0;
    auto slot_addr = [&](int k) { return smem_u32(ring + (size_t)((it + k) % SMF_SLOTS) * SMF_SLOT); };
    auto wait_slot = [&](int k) { mbar_wait(&full[(it + k) % SMF_SLOTS], (uint32_t)(((it + k) / SMF_SLOTS) & 1)); };
    auto free_slot = [&](int k) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[(it + k) % SMF_SLOTS]);
    };
    // x[64] (cols 16 ks .. 16 ks + 15 of my rows) as register A fragments times the 4 W k-blocks at ring positions
    // k0 .. k0 + 3 -> d (three passes per K = 16 step: hi*hi + lo*hi + hi*lo)
    auto gemm_rs = [&](const uint32_t (&ah)[8][4], const uint32_t (&al)[8][4], float (&d)[64], int k0, uint32_t acc0) {
#pragma unroll
      for (int kb = 0; kb < 4; ++kb) {
        wait_slot(k0 + kb);
        const uint64_t bdesc = make_sw128_desc(slot_addr(k0 + kb), 1024, 16);
        wgmma_fence();
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int ks = 2 * kb + hh;
          wgmma_rs<128, 0>(d, ah[ks], bdesc + 2 * hh, (kb | hh) ? 1u : acc0);
          if constexpr (PASSES == 3) {
            wgmma_rs<128, 0>(d, al[ks], bdesc + 2 * hh, 1u);
            wgmma_rs<128, 0>(d, ah[ks], bdesc + 2 * (2 + hh), 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(d);
        free_slot(k0 + kb);
      }
    };
    for (int i = 0; i < n_my; ++i, it += SMF_PER_TILE) {
      const long long row0 = (long long)(blockIdx.x + i * gridDim.x) * 128 + r0;
      // ---- M1: att Wp^T
      float acc[64];
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] = 0.f;
#pragma unroll 1
      for (int kb = 0; kb < 4; ++kb) {
        wait_slot(2 * kb);
        wait_slot(2 * kb + 1);
        wgmma_fence();
        wgmma_bf16x3_ss<128, PASSES>(acc, make_sw128_desc(slot_addr(2 * kb) + cg * (64 * 128), 1024, 16),
                                     make_sw128_desc(slot_addr(2 * kb + 1), 1024, 16), kb != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        free_slot(2 * kb);
        free_slot(2 * kb + 1);
      }
      // ---- y1 = tok + D1 + bp; y1 + b2 parked for M3; LayerNorm2 (two-pass: mean, then centred sum of squares)
      float sum[2] = {0.f, 0.f};
#pragma unroll
      for (int nb = 0; nb < 16; ++nb) {
        const int c = 8 * nb + 2 * q4;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const long long row = row0 + 8 * r;
          const float2 tk = __ldg(reinterpret_cast<const float2*>(p.tok + (row < p.M ? row : 0) * SMF_C + c));
          float& y0 = acc[4 * nb + 2 * r];
          float& y1 = acc[4 * nb + 2 * r + 1];
          y0 += tk.x + s_bp[c];
          y1 += tk.y + s_bp[c + 1];
          sum[r] += y0 + y1;
          my_stash[(2 * nb + r) * 128] = make_float2(y0 + s_b2[c], y1 + s_b2[c + 1]);
        }
      }
      float mean[2], sq[2] = {0.f, 0.f}, rstd[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
        sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
        mean[r] = sum[r] * (1.0f / SMF_C);
      }
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        acc[j] -= mean[(j >> 1) & 1];
        sq[(j >> 1) & 1] += acc[j] * acc[j];
      }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        sq[r] += __shfl_xor_sync(0xffffffffu, sq[r], 1);
        sq[r] += __shfl_xor_sync(0xffffffffu, sq[r], 2);
        rstd[r] = rsqrtf(sq[r] * (1.0f / SMF_C) + SMF_EPS);
      }
      uint32_t ah[8][4], al[8][4];
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        const int c = 8 * (j >> 2) + 2 * q4 + (j & 1);
        acc[j] = acc[j] * rstd[(j >> 1) & 1] * s_lnw[c] + s_lnb[c];
      }
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) split_frag_k16(&acc[8 * ks], ah[ks], al[ks]);
      // ---- M2: h = GELU(LN2(y1) W1^T + b1)
      gemm_rs(ah, al, acc, 8, 0u);
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] = smf_gelu(acc[j] + s_b1[8 * (j >> 2) + 2 * q4 + (j & 1)]);
#pragma unroll
      for (int ks = 0; ks < 8; ++ks) split_frag_k16(&acc[8 * ks], ah[ks], al[ks]);
      // ---- M3: out = (y1 + b2) + h W2^T
#pragma unroll
      for (int nb = 0; nb < 16; ++nb) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float2 y = my_stash[(2 * nb + r) * 128];
          acc[4 * nb + 2 * r] = y.x;
          acc[4 * nb + 2 * r + 1] = y.y;
        }
      }
      gemm_rs(ah, al, acc, 12, 1u);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const long long row = row0 + 8 * r;
        if (row < p.M) {
          float* orow = p.out + row * SMF_C + 2 * q4;
#pragma unroll
          for (int nb = 0; nb < 16; ++nb)
            *reinterpret_cast<float2*>(orow + 8 * nb) = make_float2(acc[4 * nb + 2 * r], acc[4 * nb + 2 * r + 1]);
        }
      }
    }
  }
}

}  // namespace occ

using namespace occ;

// out[M,128] = y1 + W2 gelu(W1 LN(y1) + b1) + b2,  y1 = tok + att Wp^T + bp.   att, Wp, W1, W2 in S32; weights
// (out, in) row-major as in nn.Linear.
extern "C" int occ_swin_proj_ffn(const float* att, const float* tok, const float* wp, const float* bp, const float* ln_w,
                                 const float* ln_b, const float* w1, const float* b1, const float* w2, const float* b2,
                                 float* out, long long M, int C, cudaStream_t stream) {
  OCC_REQUIRE(att && tok && wp && bp && ln_w && ln_b && w1 && b1 && w2 && b2 && out);
  OCC_REQUIRE(M > 0 && M < (1ll << 31) - 128);
  if (C != SMF_C) return OCC_EUNSUPPORTED;
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(att) & 15) == 0 && (reinterpret_cast<uintptr_t>(tok) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (reinterpret_cast<uintptr_t>(wp) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(w1) & 15) == 0 && (reinterpret_cast<uintptr_t>(w2) & 15) == 0);
  CUtensorMap tmA, tmWp, tmW1, tmW2;
  uint32_t box[2] = {32u, 128u};
  uint64_t strides[1] = {(uint64_t)SMF_C * 4};
  {
    uint64_t dims[2] = {(uint64_t)SMF_C, (uint64_t)M};
    int rc = make_tmap_f32(&tmA, att, 2, dims, strides, box, nullptr);
    if (rc) return rc;
  }
  uint64_t wdims[2] = {(uint64_t)SMF_C, (uint64_t)SMF_C};
  int rc = make_tmap_f32(&tmWp, wp, 2, wdims, strides, box, nullptr);
  if (rc) return rc;
  rc = make_tmap_f32(&tmW1, w1, 2, wdims, strides, box, nullptr);
  if (rc) return rc;
  rc = make_tmap_f32(&tmW2, w2, 2, wdims, strides, box, nullptr);
  if (rc) return rc;
  SwinMlpParams p{};
  p.passes = mma_passes();
  p.tok = tok; p.bp = bp; p.lnw = ln_w; p.lnb = ln_b; p.b1 = b1; p.b2 = b2; p.out = out; p.M = M;
  p.n_tiles = (int)((M + 127) / 128);
  const size_t smem = (size_t)SMF_SLOTS * SMF_SLOT + 2 * SMF_STASH + 5 * SMF_C * sizeof(float) + 2 * SMF_SLOTS * 8 +
                      1024 /*align*/;
  int grid = sm_count();
  if (grid > p.n_tiles) grid = p.n_tiles;
  auto launch = [&](auto passes) {
    constexpr int P = decltype(passes)::value;
    OCC_ENSURE_SMEM(swin_mlp_fused_kernel<P>, smem);
    swin_mlp_fused_kernel<P><<<grid, SMF_THREADS, smem, stream>>>(tmA, tmWp, tmW1, tmW2, p);
    OCC_LAUNCH_CHECK();
    return OCC_OK;
  };
  return p.passes == 1 ? launch(std::integral_constant<int, 1>{}) : launch(std::integral_constant<int, 3>{});
}
