// Mask einsum + adaptive max pool of the Mask2Former-3D decoder, "query-stationary" on the Hopper tensor cores.
//
// Reference: projects/mmdet3d_plugin/occformer/mask2former/mask2former_nusc_occ.py:457 (mask_pred = einsum('bqc,bcxyz->
// bqxyz', mask_embed, mask_features)), :463-466 (attn_mask = adaptive_max_pool3d(mask_pred, level size).sigmoid() < .5)
// and :652-653 (rows that block every key attend everywhere).  The (B, Q, X, Y, Z) logits of the intermediate layers
// are only ever consumed through the pooled mask, so this kernel never writes them: the mask features are read once per
// layer and ~1 MB of pooled logits is written.
//
// Both operands arrive in the S32 split format; every 32-k block is three bf16 tensor-core passes (occ_ptx.cuh).
// D[128 queries x 128 voxels] = membed[b] (A, resident in smem, K-major) x mf tile^T (B operand: the voxel rows of a
// (bx, by, bz) box, K-major, TMA 5-D box loads).  Each consumer warpgroup computes 64 queries x 128 voxels (wgmma
// 64x128x16) and stages the tile in shared memory; then two threads per query (one per 64-voxel half of the box) reduce
// their voxels into the pooling cells with compile-time indices, combine with one shuffle, and a cell's Q maxima are
// written by adjacent threads (no atomics when the box holds whole pooling cells).
//   warp 8: TMA producer (ring of 16 KB k-blocks)   warps 0-7: two consumer warpgroups (queries 0-63 / 64-127)
// Q > 128: blockIdx.z = 128-query tile.  Each CTA keeps its tile resident; CTAs of different tiles walk the same
// voxel-tile sequence, so the second read of a mask-feature box is an L2 hit.
#include "occ_common.cuh"
#include "occ_ptx.cuh"

#include <type_traits>

namespace occ {

constexpr int MP_THREADS = 288;
constexpr int MP_KB_BYTES = 128 * 32 * 4;  // one k-block of A or B: 128 rows x 32 floats
constexpr int MP_PITCH = 128 + 8;          // staged accumulator rows (floats)
constexpr int MP_ACC_BYTES = 2 * 64 * MP_PITCH * 4;

struct MaskPoolParams {
  const float* membed;  // (B, Q, E) S32
  int* pooled;          // (B, Xo*Yo*Zo, Q) ordered ints
  int* flag;            // (B, Q)
  int Q, E, KB, stages;
  int tiles_y, tiles_z, n_tiles;  // tiles of one sample
  int Xo, Yo, Zo;
  int passes;  // tensor-core passes per 32-k block (occ_common.cuh: mma_passes)
};

// P: cubic pooling window; (BX, BY, BZ): voxel box of a tile (BX*BY*BZ == 128, z fastest = B-operand row order)
template <int P, int BX, int BY, int BZ>
__global__ void __launch_bounds__(MP_THREADS, 1)
mask_pool_tc_kernel(const __grid_constant__ CUtensorMap tmB, const MaskPoolParams p) {
  static_assert(BX * BY * BZ == 128, "tile = 128 voxels");
  constexpr int CWX = P < BX ? P : BX, CWY = P < BY ? P : BY, CWZ = P < BZ ? P : BZ;  // cell extent inside the box
  constexpr int NCX = BX / CWX, NCY = BY / CWY, NCZ = BZ / CWZ, NC = NCX * NCY * NCZ;
  constexpr bool COMPLETE = CWX == P && CWY == P && CWZ == P;
  static_assert(NC <= 16, "cell maxima live in registers");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint8_t* sa = smem;                                   // A: KB k-blocks
  uint8_t* ring = sa + (size_t)p.KB * MP_KB_BYTES;       // B ring
  float* acc_smem = reinterpret_cast<float*>(ring + (size_t)p.stages * MP_KB_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(acc_smem) + MP_ACC_BYTES);
  uint64_t* empty_bar = full_bar + 8;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.y;
  const int q0 = blockIdx.z * 128;  // first query of the resident tile
  const int n_my = (p.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < p.stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  {  // A = membed[b] rows q0 .. q0+127 (rows >= Q zero) x E, K-major SWIZZLE_128B k-blocks
    const int E4 = p.E >> 2;
    const float* src = p.membed + ((size_t)b * p.Q + q0) * p.E;
    for (int i = threadIdx.x; i < 128 * E4; i += MP_THREADS) {
      const int r = i / E4, c4 = i - r * E4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (q0 + r < p.Q) v = __ldg(reinterpret_cast<const float4*>(src + (size_t)r * p.E) + c4);  // S32 words, copied verbatim
      const int kb = c4 >> 3, ch = c4 & 7;
      *reinterpret_cast<float4*>(sa + (size_t)kb * MP_KB_BYTES + r * 128 + ((ch ^ (r & 7)) << 4)) = v;
    }
  }
  fence_proxy_async_smem();
  __syncthreads();

  if (warp == 8) {
    // ===================================================================== TMA producer
    if (lane == 0) {
      int it = 0;
      for (int i = 0; i < n_my; ++i) {
        const int t = blockIdx.x + i * gridDim.x;
        const int tz = t % p.tiles_z, ty = (t / p.tiles_z) % p.tiles_y, tx = t / (p.tiles_z * p.tiles_y);
        for (int kb = 0; kb < p.KB; ++kb, ++it) {
          const int s = it % p.stages;
          mbar_wait(&empty_bar[s], (uint32_t)(((it / p.stages) & 1) ^ 1));
          mbar_expect_tx(&full_bar[s], MP_KB_BYTES);
          tma_load_5d(ring + (size_t)s * MP_KB_BYTES, &tmB, &full_bar[s], kb * 32, tz * BZ, ty * BY, tx * BX, b);
        }
      }
    }
  } else {
    // ===================================================================== consumer warpgroups
    const int cg = warp >> 2;
    const int wt = threadIdx.x & 127;
    float* acc_wg = acc_smem + cg * 64 * MP_PITCH;
    // reduction phase: query row qr of the warpgroup, voxel half hv of the box
    const int qr = (wt >> 5) * 16 + (wt & 15), hv = (wt >> 4) & 1;
    const int q = q0 + cg * 64 + qr;
    bool anypos = false;
    int* pooled_b = p.pooled + (size_t)b * p.Xo * p.Yo * p.Zo * p.Q;
    int it = 0;
    for (int i = 0; i < n_my; ++i) {
      const int t = blockIdx.x + i * gridDim.x;
      const int tz = t % p.tiles_z, ty = (t / p.tiles_z) % p.tiles_y, tx = t / (p.tiles_z * p.tiles_y);
      {
        float acc[64];
#pragma unroll
        for (int j = 0; j < 64; ++j) acc[j] = 0.f;
        for (int kb = 0; kb < p.KB; ++kb, ++it) {
          const int s = it % p.stages;
          mbar_wait(&full_bar[s], (uint32_t)((it / p.stages) & 1));
          wgmma_fence();
          wgmma_bf16x3_ss<128>(acc, make_sw128_desc(smem_u32(sa + (size_t)kb * MP_KB_BYTES) + cg * (64 * 128), 1024, 16),
                               make_sw128_desc(smem_u32(ring + (size_t)s * MP_KB_BYTES), 1024, 16), kb != 0, p.passes);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_regs(acc);
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[s]);
        }
        const int r0 = (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          *reinterpret_cast<float2*>(acc_wg + r0 * MP_PITCH + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(acc_wg + (r0 + 8) * MP_PITCH + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      named_bar_sync(1 + cg, 128);
      float m[NC];
#pragma unroll
      for (int c = 0; c < NC; ++c) m[c] = -INFINITY;
      auto reduce_half = [&](auto HV) {
        constexpr int h0 = decltype(HV)::value * 64;
        const float* row = acc_wg + qr * MP_PITCH + h0;
#pragma unroll
        for (int j4 = 0; j4 < 16; ++j4) {
          const float4 v4 = *reinterpret_cast<const float4*>(row + 4 * j4);
          const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int n = h0 + 4 * j4 + e;  // voxel of the box, z fastest
            const int x = n / (BY * BZ), y = (n / BZ) % BY, z = n % BZ;
            const int cell = ((x / CWX) * NCY + y / CWY) * NCZ + z / CWZ;
            m[cell] = fmaxf(m[cell], v[e]);
          }
        }
      };
      if (hv) reduce_half(std::integral_constant<int, 1>{});
      else reduce_half(std::integral_constant<int, 0>{});
#pragma unroll
      for (int c = 0; c < NC; ++c) m[c] = fmaxf(m[c], __shfl_xor_sync(0xffffffffu, m[c], 16));
      named_bar_sync(1 + cg, 128);  // the staging block may be overwritten by the next tile
      if (hv == 0 && q < p.Q) {
        const int gx0 = tx * BX / P, gy0 = ty * BY / P, gz0 = tz * BZ / P;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          const int cx = c / (NCY * NCZ), cy = (c / NCZ) % NCY, cz = c % NCZ;
          int* dst = pooled_b + ((size_t)((gx0 + cx) * p.Yo + gy0 + cy) * p.Zo + gz0 + cz) * p.Q + q;
          const int o = ordered_logit(m[c]);
          anypos |= o >= 0;
          if (COMPLETE) *dst = o;
          else atomicMax(dst, o);
        }
      }
    }
    if (hv == 0 && q < p.Q && anypos) p.flag[(size_t)b * p.Q + q] = 1;
  }
}

template <int P, int BX, int BY, int BZ>
static int launch_mask_pool(const float* mf, const MaskPoolParams& p0, int B, int X, int Y, int Z, cudaStream_t stream) {
  MaskPoolParams p = p0;
  p.tiles_y = Y / BY;
  p.tiles_z = Z / BZ;
  p.n_tiles = (X / BX) * p.tiles_y * p.tiles_z;
  CUtensorMap tmB;
  uint64_t dims[5] = {(uint64_t)p.E, (uint64_t)Z, (uint64_t)Y, (uint64_t)X, (uint64_t)B};
  uint64_t strides[4] = {(uint64_t)p.E * 4, (uint64_t)Z * p.E * 4, (uint64_t)Y * Z * p.E * 4, (uint64_t)X * Y * Z * p.E * 4};
  uint32_t box[5] = {32u, (uint32_t)BZ, (uint32_t)BY, (uint32_t)BX, 1u};
  int rc = make_tmap_f32(&tmB, mf, 5, dims, strides, box, nullptr);
  if (rc) return rc;
  const size_t smem = (size_t)(p.KB + p.stages) * MP_KB_BYTES + MP_ACC_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  auto kern = mask_pool_tc_kernel<P, BX, BY, BZ>;
  OCC_ENSURE_SMEM(kern, smem);
  const int nqt = (p.Q + 127) / 128;
  int gx = sm_count() / (B * nqt);
  if (gx < 1) gx = 1;
  if (gx > p.n_tiles) gx = p.n_tiles;
  kern<<<dim3(gx, B, nqt), MP_THREADS, smem, stream>>>(tmB, p);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

}  // namespace occ

using namespace occ;

// Shapes the kernel covers: cubic pooling windows of 2, 4 or 8 voxels that tile the grid, a grid that the window's
// voxel box tiles, E % 32 == 0 with at least three ring stages next to the resident mask embeddings, Q <= 256.  Any
// other shape returns OCC_EUNSUPPORTED before anything is enqueued; the caller then computes the mask logits
// (occ_gemm_bf16x3 per sample) and pools them with occ_mask_pool.
extern "C" int occ_mask_gemm_pool(const float* mf, const float* membed, int* pooled, int* flag, int B, int X, int Y, int Z,
                                  int E, int Q, int Xo, int Yo, int Zo, cudaStream_t stream) {
  OCC_REQUIRE(mf && membed && pooled && flag);
  OCC_REQUIRE(B > 0 && X > 0 && Y > 0 && Z > 0 && E > 0 && Q > 0 && Xo > 0 && Yo > 0 && Zo > 0);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(mf) & 15) == 0 && (reinterpret_cast<uintptr_t>(membed) & 15) == 0);
  const int w = X / Xo;
  if (X != w * Xo || Y != w * Yo || Z != w * Zo || E % 32 != 0 || Q > 256 || B > 65535) return OCC_EUNSUPPORTED;
  MaskPoolParams p{};
  p.passes = mma_passes();
  p.membed = membed; p.pooled = pooled; p.flag = flag;
  p.Q = Q; p.E = E; p.KB = E / 32; p.Xo = Xo; p.Yo = Yo; p.Zo = Zo;
  const int budget = 227 * 1024 - 1024 - 256 - MP_ACC_BYTES - p.KB * MP_KB_BYTES;
  p.stages = budget / MP_KB_BYTES;
  if (p.stages > 8) p.stages = 8;
  if (p.stages < 3) return OCC_EUNSUPPORTED;
  int (*launch)(const float*, const MaskPoolParams&, int, int, int, int, cudaStream_t);
  if (w == 2 && X % 2 == 0 && Y % 4 == 0 && Z % 16 == 0) launch = launch_mask_pool<2, 2, 4, 16>;
  else if (w == 4 && X % 4 == 0 && Y % 4 == 0 && Z % 8 == 0) launch = launch_mask_pool<4, 4, 4, 8>;
  else if (w == 8 && X % 8 == 0 && Y % 8 == 0 && Z % 8 == 0) launch = launch_mask_pool<8, 8, 2, 8>;
  else return OCC_EUNSUPPORTED;
  OCC_MEMSET(flag, 0, (size_t)B * Q * sizeof(int), stream);
  // w = 8: a box holds a quarter of a cell, the partial maxima meet through atomicMax on the ordered ints
  if (w == 8) OCC_MEMSET(pooled, 0x80, (size_t)B * Xo * Yo * Zo * Q * sizeof(int), stream);
  return launch(mf, p, B, X, Y, Z, stream);
}
