// Pixel-decoder encoder layer after the deformable gather, in one kernel: output projection + residual, LayerNorm
// (norms.0), FFN (Linear - ReLU - Linear) + residual, LayerNorm (norms.1), for E = 96 / 192 channels and any FFN width
// F % 32 == 0.  Per 128-token tile the four contractions run on the wgmma tensor cores (split-bf16 operands, three passes
// = fp32-faithful, occ_ptx.cuh); the intermediates never leave the SM.
//
// Reference: BaseTransformerLayer('self_attn', 'norm', 'ffn', 'norm') of the DetrTransformerEncoder in
// projects/mmdet3d_plugin/occformer/necks/multiscale_deformattn_3d.py:203-215, after MultiScaleDeformableAttention3D's core:
//     y  = x + output_proj(att)                      (multi_scale_deform_attn_3d.py:282-286, identity residual)
//     x1 = norms[0](y)
//     y2 = x1 + ffn(x1)                              (FFN: Linear(E, F) -> ReLU -> Linear(F, E), identity residual)
//     x  = norms[1](y2)  -> fp32, S32, and (x + query_pos) S32 for the next layer's projections
// Unfused (three GEMMs, two token-prep passes) every intermediate crosses HBM: 5.95 GB per layer for the 365k tokens of
// four nusc_200 samples at E = 192, F = 768.  Fused: R att, R x, R pos, W the three outputs = 1.47 GB.
//
//   warp 8    : producer -- one ring of k-blocks in the exact order the consumers read them: per tile (att, Wo) x E/32,
//               then (W1 chunk, W2 chunk) x F/32 (att from HBM, the weights from L2).  A W1 chunk is 32 hidden units x
//               E inputs (E/32 K-major tiles of 32 x 128 B), a W2 chunk E outputs x 32 hidden units.
//   warps 0-7 : two consumer warpgroups, rows 64g .. 64g+63 of every tile, acc = 64 x E fp32 in registers:
//               acc = att Wo^T (both operands in shared memory) -> y = acc + bo + x -> LayerNorm with quad shuffles (a
//               row is spread over four lanes) -> x1, parked in shared memory as S32 (the A operand of every W1 chunk)
//               -> acc = x1 + b2; per 32-wide hidden chunk: h = ReLU(x1 W1c^T + b1c) in registers, split into register
//               A fragments, acc += h W2c^T (the residual add is done by the tensor core) -> LayerNorm -> outputs.
#include "occ_common.cuh"
#include "occ_ptx.cuh"
#include "neck_levels.cuh"

namespace occ {

constexpr int NTF_THREADS = 288;
constexpr int NTF_SLOTS = 4;
constexpr int NTF_MAX_F = 4096;
constexpr float NTF_EPS = 1e-5f;

struct NeckTailParams {
  const float* x;  // (M, E) fp32 residual of the output projection
  const float *bo, *ln1w, *ln1b, *b1, *b2, *ln2w, *ln2b;
  const float* pos;  // (Nq, E) fp32, per grid: query_pos of the token (needed by out_pos only)
  float *out_f32, *out_s32, *out_pos;  // any of the three may be null
  NeckLevels g;                        // g.rows = M
  int F;
  int n_tiles;
  int passes;  // tensor-core passes per 32-k block (occ_common.cuh: mma_passes)
};

template <int E>
struct NeckTailShape {
  static_assert(E % 48 == 0, "the output loop stores 48 columns at a time");
  static constexpr int KB = E / 32;                          // 32-k blocks of an E-wide row
  static constexpr int SLOT = (E > 128 ? E : 128) * 128;     // ring slot: att k-block (128 rows) or an E-row weight block
  static constexpr int XS = 64 * E * 4;                      // per warpgroup: x1 of its 64 rows, S32, KB SW128 tiles
  static size_t smem(int F) {
    return (size_t)NTF_SLOTS * SLOT + 2 * XS + (6 * E + F) * sizeof(float) + 2 * NTF_SLOTS * 8 + 1024 /*align*/;
  }
};

// LayerNorm of the two rows a thread holds in an accumulator fragment (acc[4 nb + 2 r + e] = row r0 + 8 r, column
// 8 nb + 2 q4 + e), in place.  The arithmetic of token_prep_kernel (csrc/neck_ops.cu): the row is shifted by its first
// element before the two passes, so a row whose offset dwarfs its spread loses no digits to the offset.
template <int E>
__device__ __forceinline__ void ntf_layernorm(float (&acc)[E / 2], const float* w, const float* b, int lane) {
  const int q4 = lane & 3;
  float shift[2], sum[2] = {0.f, 0.f}, mean[2], sq[2] = {0.f, 0.f}, rstd[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) shift[r] = __shfl_sync(0xffffffffu, acc[2 * r], lane & ~3);  // column 0: q4 == 0
#pragma unroll
  for (int j = 0; j < E / 2; ++j) {
    acc[j] -= shift[(j >> 1) & 1];
    sum[(j >> 1) & 1] += acc[j];
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
    sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
    mean[r] = sum[r] / (float)E;
  }
#pragma unroll
  for (int j = 0; j < E / 2; ++j) {
    const float d = acc[j] - mean[(j >> 1) & 1];
    sq[(j >> 1) & 1] += d * d;
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    sq[r] += __shfl_xor_sync(0xffffffffu, sq[r], 1);
    sq[r] += __shfl_xor_sync(0xffffffffu, sq[r], 2);
    rstd[r] = rsqrtf(sq[r] / (float)E + NTF_EPS);
  }
#pragma unroll
  for (int j = 0; j < E / 2; ++j) {
    const int c = 8 * (j >> 2) + 2 * q4 + (j & 1);
    acc[j] = (acc[j] - mean[(j >> 1) & 1]) * rstd[(j >> 1) & 1] * w[c] + b[c];
  }
}

template <int E, int PASSES>  // PASSES: tensor-core passes per 32-k block, fixed so that each wgmma batch is one straight line
__global__ void __launch_bounds__(NTF_THREADS, 1)
neck_tail_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmWo,
                 const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmW2,
                 const NeckTailParams p) {
  using S = NeckTailShape<E>;
  constexpr int KB = S::KB, SLOT = S::SLOT, XS = S::XS;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* ring = smem;
  uint8_t* xs = ring + NTF_SLOTS * SLOT;
  float* vecs = reinterpret_cast<float*>(xs + 2 * XS);  // bo | ln1w | ln1b | b2 | ln2w | ln2b (E each) | b1 (F)
  uint64_t* full = reinterpret_cast<uint64_t*>(vecs + 6 * E + p.F);
  uint64_t* empty = full + NTF_SLOTS;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_my = (p.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  const int nf = p.F / 32;
  const int per_tile = 2 * KB + 2 * nf;
  const long long M = p.g.rows;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmWo);
    tma_prefetch_desc(&tmW1);
    tma_prefetch_desc(&tmW2);
    for (int i = 0; i < NTF_SLOTS; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < 6 * E + p.F; i += NTF_THREADS) {
    const int which = i < 6 * E ? i / E : 6, c = i < 6 * E ? i % E : i - 6 * E;
    const float* src = which == 0 ? p.bo : which == 1 ? p.ln1w : which == 2 ? p.ln1b : which == 3 ? p.b2
                     : which == 4 ? p.ln2w : which == 5 ? p.ln2b : p.b1;
    vecs[i] = __ldg(src + c);
  }
  __syncthreads();

  if (warp == 8) {
    // ===================================================================== producer (consumption order)
    if (lane == 0) {
      int it = 0;
      for (int i = 0; i < n_my; ++i) {
        const int tile = blockIdx.x + i * gridDim.x;
        for (int k = 0; k < per_tile; ++k, ++it) {
          const int s = it % NTF_SLOTS;
          mbar_wait(&empty[s], (uint32_t)(((it / NTF_SLOTS) & 1) ^ 1));
          uint8_t* dst = ring + (size_t)s * SLOT;
          if (k < 2 * KB) {
            if (k & 1) {
              mbar_expect_tx(&full[s], E * 128);
              tma_load_2d(dst, &tmWo, &full[s], (k >> 1) * 32, 0);
            } else {
              mbar_expect_tx(&full[s], 128 * 128);
              tma_load_2d(dst, &tmA, &full[s], (k >> 1) * 32, tile * 128);
            }
          } else {
            const int j = (k - 2 * KB) >> 1;
            mbar_expect_tx(&full[s], E * 128);
            if ((k - 2 * KB) & 1) {
              tma_load_2d(dst, &tmW2, &full[s], j * 32, 0);
            } else {
              for (int kb = 0; kb < KB; ++kb) tma_load_2d(dst + kb * 4096, &tmW1, &full[s], kb * 32, j * 32);
            }
          }
        }
      }
    }
  } else {
    // ===================================================================== consumer warpgroups
    const int cg = warp >> 2;
    const int q4 = lane & 3;
    const int lr = (warp & 3) * 16 + (lane >> 2);  // my rows of the warpgroup's 64: lr, lr + 8
    const float *s_bo = vecs, *s_ln1w = vecs + E, *s_ln1b = vecs + 2 * E, *s_b2 = vecs + 3 * E, *s_ln2w = vecs + 4 * E,
                *s_ln2b = vecs + 5 * E, *s_b1 = vecs + 6 * E;
    uint8_t* my_xs = xs + cg * XS;
    const uint32_t xs_addr = smem_u32(my_xs);
    int it = 0;
    auto slot_addr = [&](int k) { return smem_u32(ring + (size_t)((it + k) % NTF_SLOTS) * SLOT); };
    auto wait_slot = [&](int k) { mbar_wait(&full[(it + k) % NTF_SLOTS], (uint32_t)(((it + k) / NTF_SLOTS) & 1)); };
    auto free_slot = [&](int k) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[(it + k) % NTF_SLOTS]);
    };
    for (int i = 0; i < n_my; ++i, it += per_tile) {
      const long long row0 = (long long)(blockIdx.x + i * gridDim.x) * 128 + cg * 64 + lr;
      // ---- att Wo^T
      float acc[E / 2];
#pragma unroll
      for (int j = 0; j < E / 2; ++j) acc[j] = 0.f;
#pragma unroll 1
      for (int kb = 0; kb < KB; ++kb) {
        wait_slot(2 * kb);
        wait_slot(2 * kb + 1);
        wgmma_fence();
        wgmma_bf16x3_ss<E, PASSES>(acc, make_sw128_desc(slot_addr(2 * kb) + cg * (64 * 128), 1024, 16),
                                   make_sw128_desc(slot_addr(2 * kb + 1), 1024, 16), kb != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        free_slot(2 * kb);
        free_slot(2 * kb + 1);
      }
      // ---- y = acc + bo + x; x1 = LN1(y)
#pragma unroll
      for (int nb = 0; nb < E / 8; ++nb) {
        const int c = 8 * nb + 2 * q4;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const long long row = row0 + 8 * r;
          const float2 xv = __ldg(reinterpret_cast<const float2*>(p.x + (row < M ? row : 0) * E + c));
          acc[4 * nb + 2 * r] = acc[4 * nb + 2 * r] + s_bo[c] + xv.x;
          acc[4 * nb + 2 * r + 1] = acc[4 * nb + 2 * r + 1] + s_bo[c + 1] + xv.y;
        }
      }
      ntf_layernorm<E>(acc, s_ln1w, s_ln1b, lane);
      // ---- x1 -> shared memory as S32 (K-major SW128 tiles of 64 rows x 32 columns); acc = x1 + b2
      named_bar_sync(1 + cg, 128);  // the previous tile's W1 contractions of all four warps are done with my_xs
#pragma unroll
      for (int nb = 0; nb < E / 8; ++nb) {
        const int c = 8 * nb + 2 * q4, unit = nb & 3;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int row = lr + 8 * r;
          uint8_t* rp = my_xs + (nb >> 2) * (64 * 128) + row * 128 + 4 * q4;
          uint32_t hi, lo;
          split_pair(acc[4 * nb + 2 * r], acc[4 * nb + 2 * r + 1], hi, lo);
          *reinterpret_cast<uint32_t*>(rp + ((unit ^ (row & 7)) << 4)) = hi;
          *reinterpret_cast<uint32_t*>(rp + (((4 + unit) ^ (row & 7)) << 4)) = lo;
          acc[4 * nb + 2 * r] += s_b2[c];
          acc[4 * nb + 2 * r + 1] += s_b2[c + 1];
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1 + cg, 128);
      // ---- FFN, one 32-wide hidden chunk at a time: acc += ReLU(x1 W1c^T + b1c) W2c^T
#pragma unroll 1
      for (int j = 0, k = 2 * KB; j < nf; ++j, k += 2) {
        float h[16];
        wait_slot(k);
        const uint32_t w1 = slot_addr(k);
        wgmma_fence();
#pragma unroll
        for (int kb = 0; kb < KB; ++kb)
          wgmma_bf16x3_ss<32, PASSES>(h, make_sw128_desc(xs_addr + kb * (64 * 128), 1024, 16),
                                      make_sw128_desc(w1 + kb * 4096, 1024, 16), kb != 0);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(h);
        free_slot(k);
#pragma unroll
        for (int e = 0; e < 16; ++e) h[e] = fmaxf(h[e] + s_b1[32 * j + 8 * (e >> 2) + 2 * q4 + (e & 1)], 0.f);
        uint32_t ah[2][4], al[2][4];
        split_frag_k16(&h[0], ah[0], al[0]);
        split_frag_k16(&h[8], ah[1], al[1]);
        wait_slot(k + 1);
        const uint64_t bdesc = make_sw128_desc(slot_addr(k + 1), 1024, 16);
        wgmma_fence();
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          wgmma_rs<E, 0>(acc, ah[hh], bdesc + 2 * hh, 1u);
          if constexpr (PASSES == 3) {
            wgmma_rs<E, 0>(acc, al[hh], bdesc + 2 * hh, 1u);
            wgmma_rs<E, 0>(acc, ah[hh], bdesc + 2 * (2 + hh), 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        free_slot(k + 1);
      }
      // ---- x = LN2(y2) -> fp32 | S32 | (x + pos) S32
      ntf_layernorm<E>(acc, s_ln2w, s_ln2b, lane);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const long long row = row0 + 8 * r;
        if (row >= M) continue;
        // pos values are loaded ahead of the stores, 48 columns at a time: a load after a store to a possibly aliasing
        // output would wait for that store, one memory latency per 8 columns
        const float* prow = nullptr;
        if (p.out_pos) {
          int lvl, b, local;
          nk_locate(p.g, row, lvl, b, local);
          prow = p.pos + ((long long)p.g.start[lvl] + local) * E + 2 * q4;
        }
#pragma unroll
        for (int n0 = 0; n0 < E / 8; n0 += 6) {
          float2 pv[6];
          if (prow) {
#pragma unroll
            for (int u = 0; u < 6; ++u) pv[u] = __ldg(reinterpret_cast<const float2*>(prow + 8 * (n0 + u)));
          }
#pragma unroll
          for (int u = 0; u < 6; ++u) {
            const int nb = n0 + u, c = 8 * nb + 2 * q4;
            const float v0 = acc[4 * nb + 2 * r], v1 = acc[4 * nb + 2 * r + 1];
            uint32_t hi, lo;
            if (p.out_f32) *reinterpret_cast<float2*>(p.out_f32 + row * E + c) = make_float2(v0, v1);
            if (p.out_s32) {
              uint32_t* chunk = reinterpret_cast<uint32_t*>(p.out_s32 + row * E + (c & ~31));
              split_pair(v0, v1, hi, lo);
              chunk[(c & 31) >> 1] = hi;
              chunk[16 + ((c & 31) >> 1)] = lo;
            }
            if (prow) {
              uint32_t* chunk = reinterpret_cast<uint32_t*>(p.out_pos + row * E + (c & ~31));
              split_pair(v0 + pv[u].x, v1 + pv[u].y, hi, lo);
              chunk[(c & 31) >> 1] = hi;
              chunk[16 + ((c & 31) >> 1)] = lo;
            }
          }
        }
      }
    }
  }
}

template <int E>
static int launch_neck_tail(const float* att, const float* wo, const float* w1, const float* w2, NeckTailParams& p,
                            cudaStream_t stream) {
  CUtensorMap tmA, tmWo, tmW1, tmW2;
  uint64_t strides[1] = {(uint64_t)E * 4};
  uint64_t fstrides[1] = {(uint64_t)p.F * 4};
  uint64_t adims[2] = {(uint64_t)E, (uint64_t)p.g.rows}, wodims[2] = {(uint64_t)E, (uint64_t)E},
           w1dims[2] = {(uint64_t)E, (uint64_t)p.F}, w2dims[2] = {(uint64_t)p.F, (uint64_t)E};
  uint32_t abox[2] = {32u, 128u}, ebox[2] = {32u, (uint32_t)E}, w1box[2] = {32u, 32u};
  int rc = make_tmap_f32(&tmA, att, 2, adims, strides, abox, nullptr);
  if (!rc) rc = make_tmap_f32(&tmWo, wo, 2, wodims, strides, ebox, nullptr);
  if (!rc) rc = make_tmap_f32(&tmW1, w1, 2, w1dims, strides, w1box, nullptr);
  if (!rc) rc = make_tmap_f32(&tmW2, w2, 2, w2dims, fstrides, ebox, nullptr);
  if (rc) return rc;
  const size_t smem = NeckTailShape<E>::smem(p.F);
  int grid = sm_count();
  if (grid > p.n_tiles) grid = p.n_tiles;
  auto launch = [&](auto passes) {
    constexpr int P = decltype(passes)::value;
    OCC_ENSURE_SMEM((neck_tail_kernel<E, P>), smem);
    neck_tail_kernel<E, P><<<grid, NTF_THREADS, smem, stream>>>(tmA, tmWo, tmW1, tmW2, p);
    OCC_LAUNCH_CHECK();
    return OCC_OK;
  };
  return p.passes == 1 ? launch(std::integral_constant<int, 1>{}) : launch(std::integral_constant<int, 3>{});
}

}  // namespace occ

using namespace occ;

extern "C" int occ_neck_layer_tail(const float* att, const float* x, const float* wo, const float* bo, const float* ln1_w,
                                   const float* ln1_b, const float* w1, const float* b1, const float* w2, const float* b2,
                                   const float* ln2_w, const float* ln2_b, const float* pos, float* out_f32,
                                   float* out_s32, float* out_pos, int L, int B, const int* grids, int E, int F,
                                   cudaStream_t stream) {
  OCC_REQUIRE(att && x && wo && bo && ln1_w && ln1_b && w1 && b1 && w2 && b2 && ln2_w && ln2_b && grids);
  OCC_REQUIRE((out_f32 || out_s32 || out_pos) && (out_pos == nullptr || pos != nullptr));
  OCC_REQUIRE(F % 32 == 0 && F >= 32 && F <= NTF_MAX_F);
  NeckLevels g;
  OCC_REQUIRE(fill_levels(g, L, B, grids, nullptr) == OCC_OK);
  OCC_REQUIRE(g.rows < (1ll << 31) - 128);
  OCC_REQUIRE(((reinterpret_cast<uintptr_t>(att) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(wo) |
                reinterpret_cast<uintptr_t>(w1) | reinterpret_cast<uintptr_t>(w2) | reinterpret_cast<uintptr_t>(pos) |
                reinterpret_cast<uintptr_t>(out_f32) | reinterpret_cast<uintptr_t>(out_s32) |
                reinterpret_cast<uintptr_t>(out_pos)) & 15) == 0);
  if (E != 96 && E != 192) return OCC_EUNSUPPORTED;
  NeckTailParams p{};
  p.x = x; p.bo = bo; p.ln1w = ln1_w; p.ln1b = ln1_b; p.b1 = b1; p.b2 = b2; p.ln2w = ln2_w; p.ln2b = ln2_b;
  p.pos = pos; p.out_f32 = out_f32; p.out_s32 = out_s32; p.out_pos = out_pos;
  p.g = g; p.F = F;
  p.n_tiles = (int)((g.rows + 127) / 128);
  p.passes = mma_passes();
  return E == 96 ? launch_neck_tail<96>(att, wo, w1, w2, p, stream) : launch_neck_tail<192>(att, wo, w1, w2, p, stream);
}
