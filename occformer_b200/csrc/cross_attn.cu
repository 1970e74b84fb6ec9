// Masked cross-attention of the Mask2Former-3D decoder on the Hopper tensor cores (flash-decoding over key chunks).
//
// Reference: mmcv BaseTransformerLayer 'cross_attn' -> MultiheadAttention -> nn.MultiheadAttention with a bool
// attn_mask (SURVEY.md Appendix C), called from projects/mmdet3d_plugin/occformer/mask2former/mask2former_nusc_occ.py
// :657-667 with attn_mask = (adaptive_max_pool3d(mask_pred) .sigmoid() < 0.5) and the all-blocked-row reset (:652-653).
//
// One CTA = (query tile, key chunk, head, sample); 128 query rows (Q <= 128 real per tile; NQT = 2 tiles for Q <= 256,
// the query tile is the fastest-varying block index so that both tiles of a key chunk run together and the second K/V
// read hits L2), N = 128 keys per tile, head dim 32.
// Split-bf16 operands, three tensor-core passes per contraction (occ_ptx.cuh): Kp / Vp arrive in S32 (one 128-byte chunk
// per (key, head)), the Q tile is split while it is staged, P is split in registers.
//   warp 8     : TMA producer -- K tile (K-major, SWIZZLE_128B) and V tile (MN-major operand, N = 64 = hi | lo of the head
//                dim, SWIZZLE_128B) are plain 2-D boxes of the projected key / value matrices
//   warps 0-7  : two consumer warpgroups, queries 64g .. 64g+63: per key tile S = Q K^T (6 wgmma 64x128x16), online
//                softmax in registers (running max / sum per row, quad shuffles), O' = O' * alpha + [P_hi; P_lo]
//                [V_hi | V_lo] (16 wgmma 64x64x16, P as register A fragments); O = O'[:, :32] + O'[:, 32:] at the end
//   (mask)     : a small pre-pass (mask_bits_kernel) turns the pooled mask logits (ordered ints, blocked <=> negative)
//                into one "blocked" bit per (key, query), 32 keys per word, once per layer instead of once per head; the
//                consumers read their words per tile straight from global (L2-resident, 1 MB at S = 80 000)
// Each CTA writes one partial per (chunk, head, query): (m, l, acc[32]) in the natural-log domain, the format consumed by
// cross_merge_kernel (head_ops.cu).
#include "occ_common.cuh"
#include "occ_ptx.cuh"

namespace occ {

constexpr int XT_HD = 32;
constexpr int XT_KEYS = 128;
constexpr int XT_STAGES = 4;
constexpr int XT_TILE = XT_KEYS * XT_HD * 4;           // 16 KB
constexpr int XT_STAGE_BYTES = 2 * XT_TILE;             // K tile + V tile
constexpr int XT_THREADS = 288;  // warps 0-7 consumers, warp 8 TMA
constexpr int XT_MAX_CHUNKS = 96;

template <int NQT>
__global__ void __launch_bounds__(XT_THREADS, 1)
cross_attn_tc_kernel(const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                     const float* __restrict__ qh, int koff, int voff, const uint32_t* __restrict__ bits /*(B,NW,Q)*/,
                     const int* __restrict__ row_flag, float* __restrict__ part, int S, int Q, int E, int H,
                     int tiles_per_chunk, int nchunk, int passes) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sq = smem + XT_STAGES * XT_STAGE_BYTES;  // Q tile, 16 KB
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sq + XT_TILE);
  uint64_t* empty_bar = full_bar + XT_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x / NQT, h = blockIdx.y, b = blockIdx.z;
  const int q0 = (blockIdx.x % NQT) * 128;  // first query row of this CTA's tile
  const int ntiles_total = (S + XT_KEYS - 1) / XT_KEYS;
  const int tile0 = c * tiles_per_chunk;
  const int n_tiles = min(tiles_per_chunk, ntiles_total - tile0);  // >= 1 by construction of nchunk

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    for (int i = 0; i < XT_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);   // TMA producer (expect_tx)
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp after its P V
    }
    fence_barrier_init();
  }
  // Q tile of this (sample, head): 128 rows x one S32 chunk (32 head-dim values split into hi | lo), K-major
  // SWIZZLE_128B; rows q0 + r >= Q are zero.  Thread (r, ch) converts 4 values: hi pair words -> 16-byte chunk ch >> 1 (half
  // ch & 1), lo pair words -> chunk 4 + (ch >> 1).
  for (int i = threadIdx.x; i < 128 * 8; i += XT_THREADS) {
    const int r = i >> 3, ch = i & 7;
    uint2 hi = make_uint2(0u, 0u), lo = make_uint2(0u, 0u);
    if (q0 + r < Q) {
      const float4 v = *reinterpret_cast<const float4*>(qh + ((size_t)b * Q + q0 + r) * E + h * XT_HD + ch * 4);
      split_pair(v.x, v.y, hi.x, lo.x);
      split_pair(v.z, v.w, hi.y, lo.y);
    }
    uint8_t* row = sq + r * 128;
    *reinterpret_cast<uint2*>(row + ((((ch >> 1)) ^ (r & 7)) << 4) + ((ch & 1) << 3)) = hi;
    *reinterpret_cast<uint2*>(row + (((4 + (ch >> 1)) ^ (r & 7)) << 4) + ((ch & 1) << 3)) = lo;
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == 8) {
    // ===================================================================== TMA producer
    if (lane == 0) {
      for (int t = 0; t < n_tiles; ++t) {
        const int s = t % XT_STAGES;
        mbar_wait(&empty_bar[s], (uint32_t)(((t / XT_STAGES) & 1) ^ 1));
        uint8_t* st = smem + (size_t)s * XT_STAGE_BYTES;
        mbar_expect_tx(&full_bar[s], 2 * XT_TILE);
        const int row0 = b * S + (tile0 + t) * XT_KEYS;
        tma_load_2d(st, &tmK, &full_bar[s], koff + h * XT_HD, row0);
        tma_load_2d(st + XT_TILE, &tmV, &full_bar[s], voff + h * XT_HD, row0);
      }
    }
  } else {
    // ===================================================================== consumer warpgroups: online softmax
    const int cg = warp >> 2, q4 = lane & 3;
    const int qi[2] = {q0 + cg * 64 + (warp & 3) * 16 + (lane >> 2), q0 + cg * 64 + (warp & 3) * 16 + (lane >> 2) + 8};
    bool use_mask[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) use_mask[r] = (qi[r] < Q) && row_flag[b * Q + qi[r]] != 0;
    const int NW = ((S + XT_KEYS - 1) / XT_KEYS) * 4;
    const float L2E = 1.4426950408889634f;
    const uint64_t qdesc = make_sw128_desc(smem_u32(sq) + cg * (64 * 128), 1024, 16);
    float M[2] = {-INFINITY, -INFINITY}, L[2] = {0.f, 0.f}, o[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) o[j] = 0.f;
    for (int t = 0; t < n_tiles; ++t) {
      const int s = t % XT_STAGES;
      uint32_t blk[2][4];
      {
        const int key_base = (tile0 + t) * XT_KEYS;
#pragma unroll
        for (int w = 0; w < 4; ++w) {
          const int nvalid = min(max(S - (key_base + 32 * w), 0), 32);
          const uint32_t tailw = nvalid >= 32 ? 0u : (0xFFFFFFFFu << nvalid);  // keys beyond S are always blocked
#pragma unroll
          for (int r = 0; r < 2; ++r)
            blk[r][w] = use_mask[r] ? __ldg(bits + ((size_t)b * NW + (size_t)(tile0 + t) * 4 + w) * Q + qi[r]) : tailw;
        }
      }
      mbar_wait(&full_bar[s], (uint32_t)((t / XT_STAGES) & 1));
      const uint32_t st = smem_u32(smem + (size_t)s * XT_STAGE_BYTES);
      float sc[64];
#pragma unroll
      for (int j = 0; j < 64; ++j) sc[j] = 0.f;
      wgmma_fence();
      wgmma_bf16x3_ss<XT_KEYS>(sc, qdesc, make_sw128_desc(st, 1024, 16), 0u, passes);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(sc);
      // row maximum over the un-blocked keys of the tile (key 8 nb + 2 q4 + e: word nb / 4, bit 8 (nb % 4) + 2 q4 + e)
      float m[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        const int r = (j >> 1) & 1, nb = j >> 2, bit = 8 * (nb & 3) + 2 * q4 + (j & 1);
        if (!((blk[r][nb >> 2] >> bit) & 1u)) m[r] = fmaxf(m[r], sc[j]);
      }
      float alpha[2], ml2[2], l[2] = {0.f, 0.f};
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 1));
        m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 2));
        const float mn = fmaxf(M[r], m[r]);
        alpha[r] = mn > -INFINITY ? ex2_approx((M[r] - mn) * L2E) : 1.f;
        ml2[r] = mn > -INFINITY ? mn * L2E : 0.f;
        M[r] = mn;
      }
      // P = exp(s - M_new) (zero for blocked keys), split into hi / lo register A fragments of the 8 K = 16 key steps
#pragma unroll
      for (int j = 0; j < 64; ++j) {
        const int r = (j >> 1) & 1, nb = j >> 2, bit = 8 * (nb & 3) + 2 * q4 + (j & 1);
        const float pj = ((blk[r][nb >> 2] >> bit) & 1u) ? 0.f : ex2_approx(fmaf(sc[j], L2E, -ml2[r]));
        l[r] += pj;
        sc[j] = pj;
      }
      uint32_t ph[8][4], pl[8][4];
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) split_frag_k16(&sc[8 * kk], ph[kk], pl[kk]);
#pragma unroll
      for (int j = 0; j < 32; ++j) o[j] *= alpha[(j >> 1) & 1];
#pragma unroll
      for (int r = 0; r < 2; ++r) L[r] = L[r] * alpha[r] + l[r];  // per-lane partial sums, quad-reduced at the end
      const uint64_t vdesc = make_sw128_desc(st + XT_TILE, 1024, 1024);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {  // 16 keys per wgmma = two 8-key (1024 B) atoms of V rows
        wgmma_rs<64, 1>(o, ph[kk], vdesc + (uint64_t)(kk * 128), 1u);                  // P_hi [V_hi | V_lo]
        if (passes == 3) wgmma_rs<64, 1>(o, pl[kk], vdesc + (uint64_t)(kk * 128), 1u);  // P_lo [V_hi | V_lo]
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      L[r] += __shfl_xor_sync(0xffffffffu, L[r], 1);
      L[r] += __shfl_xor_sync(0xffffffffu, L[r], 2);
      if (qi[r] < Q) {
        float* dst = part + ((((size_t)b * H + h) * nchunk + c) * Q + qi[r]) * (XT_HD + 2);
        if (q4 == 0) {
          dst[0] = M[r];
          dst[1] = L[r];
        }
#pragma unroll
        for (int nb = 0; nb < 4; ++nb) {
          const int d = 8 * nb + 2 * q4;
          dst[2 + d] = o[4 * nb + 2 * r] + o[4 * (nb + 4) + 2 * r];
          dst[3 + d] = o[4 * nb + 2 * r + 1] + o[4 * (nb + 4) + 2 * r + 1];
        }
      }
    }
  }
}

// pooled (B,S,Q) ordered ints -> bits (B, NW, Q): bit k of word w = key 32w+k is blocked for query q (negative
// pooled logit, or key >= S).  One thread per (word, query): 32 independent coalesced loads; blockIdx.z = query tile.
__global__ void __launch_bounds__(128)
mask_bits_kernel(const int* __restrict__ pooled, uint32_t* __restrict__ bits, int S, int Q, int NW) {
  const int q = blockIdx.z * 128 + threadIdx.x, w = blockIdx.x, b = blockIdx.y;
  if (q >= Q) return;
  uint32_t word = 0;
  int vals[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    const int key = 32 * w + k;
    vals[k] = key < S ? __ldg(pooled + ((size_t)b * S + key) * Q + q) : -1;
  }
#pragma unroll
  for (int k = 0; k < 32; ++k) word |= (uint32_t)(vals[k] < 0) << k;
  bits[((size_t)b * NW + w) * Q + q] = word;
}

}  // namespace occ

using namespace occ;

extern "C" int occ_mask_bits(const int* pooled, unsigned* bits, int B, int S, int Q, cudaStream_t stream) {
  OCC_REQUIRE(pooled && bits && B > 0 && S > 0 && Q > 0 && Q <= 256 && B <= 65535);
  const int NW = ((S + XT_KEYS - 1) / XT_KEYS) * 4;
  mask_bits_kernel<<<dim3(NW, B, (Q + 127) / 128), 128, 0, stream>>>(pooled, bits, S, Q, NW);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// number of partials per (sample, head) that occ_cross_attn_tc writes for S keys (= key chunks, <= XT_MAX_CHUNKS)
extern "C" int occ_cross_attn_tc_partials(int S) {
  const int tiles = (S + XT_KEYS - 1) / XT_KEYS;
  const int tpc = (tiles + XT_MAX_CHUNKS - 1) / XT_MAX_CHUNKS;
  return (tiles + tpc - 1) / tpc;
}

// qh (B,Q,E) scaled projected queries (fp32); Kp / Vp (B*S, ld) projected keys / values in S32, this layer's slice at
// column koff / voff (ld, koff, voff multiples of 32); bits (B, NW = 4*ceil(S/128), Q) blocked-key words from
// occ_mask_bits; row_flag (B*Q); part (B, H, npart, Q, 34).
extern "C" int occ_cross_attn_tc(const float* qh, const float* Kp, const float* Vp, int ld, int koff, int voff,
                                 const unsigned* bits, const int* row_flag, float* part, int B, int S, int Q, int E,
                                 int H, cudaStream_t stream) {
  OCC_REQUIRE(qh && Kp && Vp && bits && row_flag && part);
  OCC_REQUIRE(B > 0 && S > 0 && Q > 0 && Q <= 256 && Q % 4 == 0 && H > 0 && E == H * XT_HD && B <= 65535 && H <= 65535);
  // one TMA box per (key, head) = one 32-column S32 chunk [hi | lo]: the slices must start on a chunk boundary
  OCC_REQUIRE(ld % 32 == 0 && koff % 32 == 0 && voff % 32 == 0 && koff >= 0 && voff >= 0 && koff + E <= ld &&
              voff + E <= ld);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(qh) & 15) == 0 && (reinterpret_cast<uintptr_t>(Kp) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(Vp) & 15) == 0);
  const int tiles = (S + XT_KEYS - 1) / XT_KEYS;
  const int tpc = (tiles + XT_MAX_CHUNKS - 1) / XT_MAX_CHUNKS;
  const int nchunk = (tiles + tpc - 1) / tpc;
  CUtensorMap tmK, tmV;
  uint64_t dims[2] = {(uint64_t)ld, (uint64_t)B * S};
  uint64_t strides[1] = {(uint64_t)ld * 4};
  uint32_t box[2] = {(uint32_t)XT_HD, (uint32_t)XT_KEYS};
  int rc = make_tmap_f32(&tmK, Kp, 2, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  rc = make_tmap_f32(&tmV, Vp, 2, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;
  const size_t smem = (size_t)XT_STAGES * XT_STAGE_BYTES + XT_TILE + 1024 /*align*/ + 256 /*barriers*/;
  if (Q <= 128) {
    OCC_ENSURE_SMEM(cross_attn_tc_kernel<1>, smem);
    dim3 grid(nchunk, H, B);
    cross_attn_tc_kernel<1><<<grid, XT_THREADS, smem, stream>>>(tmK, tmV, qh, koff, voff, bits, row_flag, part, S, Q, E, H,
                                                                tpc, nchunk, mma_passes());
  } else {
    OCC_ENSURE_SMEM(cross_attn_tc_kernel<2>, smem);
    dim3 grid(2 * nchunk, H, B);
    cross_attn_tc_kernel<2><<<grid, XT_THREADS, smem, stream>>>(tmK, tmV, qh, koff, voff, bits, row_flag, part, S, Q, E, H,
                                                                tpc, nchunk, mma_passes());
  }
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
