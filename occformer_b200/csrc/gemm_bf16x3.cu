// Persistent warp-specialised fp32-faithful GEMM / implicit-GEMM convolution for sm_90a ("bf16x3").
//
//   D[M,N] = epilogue( A[M,K] * W[N,K]^T )          (plain mode: A row-major, W = torch Linear weight)
//   D[vox,Cout] = epilogue( im2col(x)[vox, taps*Cin] * W2[Cout, taps*Cin]^T )   (conv mode)
//
// Operands are fp32 values stored in the S32 split format (occ_ptx.cuh: every 32-column chunk = 32 bf16 hi | 32 bf16
// lo); each 32-k block is contracted by three bf16 tensor-core passes (hi*hi + lo*hi + hi*lo, fp32 accumulate): ~1e-5
// relative error, the bytes, TMA boxes and shared-memory tiles of a plain fp32 operand.
//
// One CTA per SM, 384 threads: warp 8 = TMA producer (cp.async.bulk.tensor, 128B swizzle, STAGES-deep ring; warps 9-11
// only hand their registers to the consumers), warps 0-7 = two consumer warpgroups.  Warpgroup g issues the wgmmas (bf16, M = 64, N = BN, K = 16, fp32 accumulators in registers)
// of rows 64g .. 64g+63 of the 128-row tile, then stages its accumulator in shared memory and runs the epilogue thread =
// row (bias / activation / residual / GroupNorm statistics -> TMA store); the producer fills the ring for the
// next tile meanwhile.  Conv mode never materialises im2col: every filter tap is a 5-D TMA box {32 ch, bz, by, bx, 1}
// with a shifted origin; out-of-bounds = zero fill = the conv padding; stride-2 convs use the tensor map's elementStrides.
//
// Replaces on the reference path: cuDNN Conv3d + cuBLAS Linear calls inside DualpathTransformerBlock
// (projects/mmdet3d_plugin/occformer/backbones/dualpath_block.py:36-48,79), SwinBlock / WindowMSA
// linears (backbones/modules/window_attention.py:65-67,336-344), BottleNeckASPP convs
// (backbones/modules/aspp.py:49-172) and the decoder's K/V projections + mask einsum
// (mask2former/mask2former_nusc_occ.py:446-457).
#include "occ_common.cuh"
#include "occ_ptx.cuh"

namespace occ {

constexpr int BM = 128;
constexpr int BK = 32;  // 32 fp32 = 128 bytes = one swizzle row
constexpr int A_STAGE_BYTES = BM * BK * 4;
constexpr int EPI_BUF_BYTES = 32 * 128;                 // one 32-row x 32-column fp32 chunk, 128-byte swizzled rows
constexpr int EPI_BYTES = 8 /*warps*/ * EPI_BUF_BYTES;
constexpr int CTRL_BYTES = 2048;   // mbarriers + fp64 GroupNorm partial sums of up to 96 groups; a multiple of 1024 so
                                   // that the swizzled epilogue staging buffers behind it stay 1024-byte aligned
constexpr int MAX_STAT_GROUPS = 96;  // 2 * 96 doubles = 1536 B of CTRL_BYTES (barriers < 256 B)
constexpr int GEMM_THREADS = 384;    // two consumer warpgroups + one producer warpgroup (one TMA-issuing lane)
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;  // setmaxnreg: 128 * 40 + 256 * 232 <= 64 K registers
constexpr int MAX_TAPS = 28;

struct GemmParams {
  int M, N, K, num_k_blocks;
  float* out;
  int ldo;
  const float* bias;
  const float* residual;
  int ldr;
  int splits;     // split-K: > 1 => every tile's k-blocks are divided among `splits` CTAs, partial sums meet in `out`
                  // (zero-initialised by the host) through TMA reduce-add; no bias / act / stats in the kernel
  int act;        // 0 none, 1 relu, 2 gelu(erf), 3 swish
  int split_out;  // write the result in the S32 split format (the consumer is another tensor-core contraction)
  int passes;     // tensor-core passes per 32-k block (occ_common.cuh: mma_passes): picks the PASSES instantiation
  // conv mode
  int conv;
  int Cin, KX, KY, KZ, dil, stride;
  int padx, pady, padz;
  int B, Xo, Yo, Zo;
  int bx, by, bz, tiles_x, tiles_y, tiles_z;
  int use_tma_store;  // epilogue writes through a TMA store (output rows 16-byte aligned)
  // conv mode: GroupNorm statistics (sum, sumsq per (batch, group)) of the raw output, accumulated in fp64
  double* gn_stats;
  int cpg;             // channels per group: N % cpg == 0, N / cpg <= MAX_STAT_GROUPS
  int* splitk_sem;     // [SPLITK_SEMS], see above (required when splits > 1)
  // explicit tap table (conv mode, stride 1): tap t reads the input at voxel + (tdx, tdy, tdz)[t] (dilation and padding
  // folded in); 0 = the regular KX x KY x KZ stencil.  Lets several dilated branches share one launch (ASPP).
  int ntaps;
  signed char tdx[MAX_TAPS], tdy[MAX_TAPS], tdz[MAX_TAPS];
};

// Split-K ordering: sem[(m, n) tile] counts the splits that have added their partial sum.  Split s adds after split
// s - 1, so the fp32 reduce-add order -- and with it every bit of the result -- is fixed.  The counters live in a
// caller-provided workspace (occ_conv_workspace_bytes(): 1024 ints, zero before the first call; the last split of
// every tile resets its counter, so one workspace serves every conv of a stream; concurrent streams pass their own).
constexpr int SPLITK_SEMS = 1024;

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
// mmcv Swish (x * sigmoid(x)), the activation of EfficientNet's convs
__device__ __forceinline__ float swish(float x) { return x / (1.0f + expf(-x)); }

template <int CPG>
__device__ __forceinline__ void accum_stats(const float (&v)[32], float (&sv)[32]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    sv[2 * (j / CPG)] += v[j];
    sv[2 * (j / CPG) + 1] += v[j] * v[j];
  }
}

// Sum each of 32 per-lane values over the 32 lanes of the warp with 31 shuffles; afterwards lane L holds
// the total of value index L in v[0].
__device__ __forceinline__ void warp_butterfly32(float (&v)[32], int lane) {
#pragma unroll
  for (int off = 16, n = 32; off >= 1; off >>= 1, n >>= 1) {
    const bool upper = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < n / 2; ++i) {
      const float keep = upper ? v[i + n / 2] : v[i];
      const float send = upper ? v[i] : v[i + n / 2];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
}

// Accumulator staging: after its k-loop every consumer warpgroup writes its 64 x BN fp32 fragment to a row-major
// shared-memory block (pitch BN + 8 floats: conflict-free fragment stores, 2-way conflicted row reads) from which the
// epilogue reads thread = row, 32 consecutive columns per chunk.
template <int BN>
constexpr int acc_pitch() { return BN + 8; }
template <int BN>
constexpr int acc_stage_bytes() { return 2 * 64 * acc_pitch<BN>() * 4; }

// MT = 2: a 256-row tile (two 128-row M tiles sharing every B k-block: a third fewer operand bytes per MAC at BN = 128).
// Warpgroup cg runs two m64 chains over rows 128cg .. 128cg+127; chain h reads the 8-row atoms 16cg + 2i + h (SBO 2048),
// so warp w of the warpgroup holds the 32 consecutive tile rows 128cg + 32w .. +31 (16 of each chain) and stages them
// chunk by chunk through its own TMA-store buffer: no fp32 staging block, which leaves room for a 4-deep ring.
// No split-K.
// PASSES: tensor-core passes per 32-k block (3 = fp32-faithful, 1 = single-pass bf16), fixed at compile time so that a
// k-block's wgmmas form one straight-line batch behind a single wgmma_fence.
template <int BN, int STAGES, bool LEAN, int MT, int PASSES>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16x3_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmC, const __grid_constant__ GemmParams p) {
  // LEAN = plain GEMM, whole 32-column chunks, TMA store, no conv addressing / GroupNorm statistics / split-K: those
  // branches compile away.
  static_assert(MT == 1 || (MT == 2 && !LEAN), "paired M tiles: conv / full-epilogue instantiations only");
  const bool f_conv = !LEAN && p.conv != 0;
  const bool f_stats = f_conv && p.gn_stats != nullptr;
  const int f_splits = (LEAN || MT == 2) ? 1 : p.splits;
  const bool f_tma = LEAN || p.use_tma_store != 0;

  constexpr int TILE_M = MT * BM;
  constexpr int A_BYTES = MT * A_STAGE_BYTES;
  constexpr int B_STAGE_BYTES = BN * BK * 4;
  constexpr int STAGE_BYTES = A_BYTES + B_STAGE_BYTES;
  constexpr int PITCH = acc_pitch<BN>();

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  double* stat_acc = reinterpret_cast<double*>(empty_bar + STAGES);  // (sum, sumsq) per group, <= MAX_STAT_GROUPS groups
  uint8_t* epi_smem = smem + STAGES * STAGE_BYTES + CTRL_BYTES;  // 8 warps x 4 KB, 1024-byte aligned
  float* acc_smem = reinterpret_cast<float*>(epi_smem + EPI_BYTES);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int num_n_tiles = (p.N + BN - 1) / BN;
  const int num_m_tiles = f_conv ? p.B * p.tiles_x * p.tiles_y * p.tiles_z : (p.M + TILE_M - 1) / TILE_M;
  const int num_tiles = num_m_tiles * num_n_tiles * f_splits;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    tma_prefetch_desc(&tmC);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  if (threadIdx.x < 256) {
    for (int i = threadIdx.x; i < 2 * MAX_STAT_GROUPS; i += 256) stat_acc[i] = 0.0;
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------------------------------------- TMA producer
    setmaxnreg_dec<PRODUCER_REGS>();
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int cblocks = f_conv ? (p.Cin / BK) : 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int split = tile % f_splits;
        const int n_tile = (tile / f_splits) % num_n_tiles;
        const int m_tile = tile / (f_splits * num_n_tiles);
        const int kb0 = (int)(((long long)split * p.num_k_blocks) / f_splits);
        const int kb1 = (int)(((long long)(split + 1) * p.num_k_blocks) / f_splits);
        int cb = 0, cx0 = 0, cy0 = 0, cz0 = 0;
        if (f_conv) {
          int t = m_tile;
          const int tz = t % p.tiles_z; t /= p.tiles_z;
          const int ty = t % p.tiles_y; t /= p.tiles_y;
          const int tx = t % p.tiles_x; t /= p.tiles_x;
          cb = t;
          cx0 = tx * p.bx * p.stride - p.padx;
          cy0 = ty * p.by * p.stride - p.pady;
          cz0 = tz * p.bz * p.stride - p.padz;
        }
        int tap = 0, kc = 0, tx_ = 0, ty_ = 0, tz_ = 0;
        if (f_conv && kb0 > 0) {  // split-K: start in the middle of the tap sequence
          tap = kb0 / cblocks;
          kc = kb0 % cblocks;
          tz_ = tap % p.KZ;
          ty_ = (tap / p.KZ) % p.KY;
          tx_ = tap / (p.KZ * p.KY);
        }
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_BYTES;
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          if (f_conv) {
            // input offset of this tap: regular stencil (dilated, padding folded into c?0) or the explicit table
            const int ox = p.ntaps ? p.tdx[tap] : tx_ * p.dil, oy = p.ntaps ? p.tdy[tap] : ty_ * p.dil,
                      oz = p.ntaps ? p.tdz[tap] : tz_ * p.dil;
            tma_load_5d(sa, &tmA, &full_bar[stage], kc * BK, cz0 + oz, cy0 + oy, cx0 + ox, cb);
            if (++kc == cblocks) {
              kc = 0;
              ++tap;
              if (++tz_ == p.KZ) {
                tz_ = 0;
                if (++ty_ == p.KY) { ty_ = 0; ++tx_; }
              }
            }
          } else {
            tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, m_tile * TILE_M);
          }
          tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, n_tile * BN);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        (void)tap;
      }
    }
  } else {
    // ------------------------------------------------------------- consumers: wgmma main loop + epilogue
    setmaxnreg_inc<CONSUMER_REGS>();
    // warpgroup cg = warp >> 2 accumulates rows 64 cg .. 64 cg + 63 of the tile.  In the epilogue warp (cg, w) drains the
    // 32-row slab ew = 2 cg + (w & 1) for the chunks of parity wg = w >> 1 (the four warps of one parity cover the tile's
    // 128 rows).  MT = 2: warp (cg, w) drains its own 32-row slab ew = 4 cg + w, every chunk.
    const int cg = warp >> 2;
    const int ew = MT == 2 ? 4 * cg + (warp & 3) : 2 * cg + (warp & 1);
    const int wg = MT == 2 ? 0 : (warp >> 1) & 1;
    const int row = ew * 32 + lane;
    uint8_t* stage_buf = epi_smem + warp * EPI_BUF_BYTES;
    float* acc_wg = acc_smem + cg * 64 * PITCH;
    const float* acc_row = acc_wg + ((warp & 1) * 32 + lane) * PITCH;
    const bool row_vec = ((reinterpret_cast<uintptr_t>(p.residual) | reinterpret_cast<uintptr_t>(p.out)) & 15) == 0 &&
                         p.ldr % 4 == 0 && p.ldo % 4 == 0;
    int stage = 0;
    uint32_t phase = 0;
    int cur_b = -1;
    // A k-block that never arrives makes the warp leave both loops before any named barrier and trap after them: a trap
    // reachable inside the loops would cap ptxas's register allocation at the launch bound (168), below the
    // accumulators and epilogue of the 256-row tiles (occ_ptx.cuh: mbar_wait).
    bool timed_out = false;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int n_tile = (tile / f_splits) % num_n_tiles;
      const int m_tile = tile / (f_splits * num_n_tiles);
      const int n0 = n_tile * BN;
      float acc[MT][BN / 2];  // MT = 2: held in registers through the epilogue
      {
        const int split = tile % f_splits;
        const int kb0 = (int)(((long long)split * p.num_k_blocks) / f_splits);
        const int kb1 = (int)(((long long)(split + 1) * p.num_k_blocks) / f_splits);
#pragma unroll
        for (int h = 0; h < MT; ++h)
#pragma unroll
          for (int j = 0; j < BN / 2; ++j) acc[h][j] = 0.f;
        int prev_stage = -1;
        for (int kb = kb0; kb < kb1; ++kb) {
          if (!mbar_wait_bounded(&full_bar[stage], phase)) { timed_out = true; break; }
          const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES);
          const uint64_t bdesc = make_sw128_desc(sa + A_BYTES, 1024, 16);
          wgmma_fence();
          // one S32 row block = 32 k values: hi*hi + lo*hi + hi*lo, six K=16 wgmmas stepping 32 bytes inside the row
          if constexpr (MT == 1) {
            wgmma_bf16x3_ss<BN, PASSES>(acc[0], make_sw128_desc(sa + cg * (64 * 128), 1024, 16), bdesc, 1u);
          } else {
            const uint32_t a0 = sa + cg * (128 * 128);
            wgmma_bf16x3_ss2<BN, PASSES>(acc[0], acc[MT - 1], make_sw128_desc(a0, 2048, 16),
                                         make_sw128_desc(a0 + 1024, 2048, 16), bdesc, 1u);
          }
          wgmma_commit();
          wgmma_wait<1>();  // the previous k-block's wgmmas have finished reading their stage
          if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
          prev_stage = stage;
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int h = 0; h < MT; ++h) wgmma_fence_regs(acc[h]);
        if (timed_out) break;
        if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        if constexpr (MT == 1) {
          // fragment -> row-major staging block of this warpgroup (the previous tile's epilogue finished reading it)
          const int r0 = (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            *reinterpret_cast<float2*>(acc_wg + r0 * PITCH + 8 * j + c0) = make_float2(acc[0][4 * j], acc[0][4 * j + 1]);
            *reinterpret_cast<float2*>(acc_wg + (r0 + 8) * PITCH + 8 * j + c0) =
                make_float2(acc[0][4 * j + 2], acc[0][4 * j + 3]);
          }
          named_bar_sync(4 + cg, 128);
        }
      }
      // ---- output row of this thread
      long long m = -1;
      int tile_b = 0, tile_x0 = 0, tile_y0 = 0, tile_z0 = 0;
      if (f_conv) {
        int t = m_tile;
        const int tz = t % p.tiles_z; t /= p.tiles_z;
        const int ty = t % p.tiles_y; t /= p.tiles_y;
        const int tx = t % p.tiles_x; t /= p.tiles_x;
        tile_b = t;
        tile_x0 = tx * p.bx; tile_y0 = ty * p.by; tile_z0 = tz * p.bz;
        const int dz = row % p.bz;
        const int dy = (row / p.bz) % p.by;
        const int dx = row / (p.bz * p.by);
        const int x = tx * p.bx + dx, y = ty * p.by + dy, z = tz * p.bz + dz;
        if (x < p.Xo && y < p.Yo && z < p.Zo)
          m = (((long long)tile_b * p.Xo + x) * p.Yo + y) * p.Zo + z;
      } else {
        const long long mm = (long long)m_tile * TILE_M + row;
        if (mm < p.M) m = mm;
      }
      const bool valid = m >= 0;

      if (f_stats && tile_b != cur_b) {
        // flush the per-CTA fp64 partial sums of the previous batch sample
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (cur_b >= 0) {
          const int ngroups2 = 2 * (p.N / p.cpg);
          for (int i = threadIdx.x; i < ngroups2; i += 256) {
            const double v = stat_acc[i];
            if (v != 0.0) atomicAdd(&p.gn_stats[(size_t)cur_b * ngroups2 + i], v);
            stat_acc[i] = 0.0;
          }
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        cur_b = tile_b;
      }

      if (f_splits > 1) {  // wait until the lower splits of this tile have added their partial sums
        if (threadIdx.x == 0) {
          const int want = tile % f_splits;
          volatile int* sem = p.splitk_sem + ((tile / f_splits) & (SPLITK_SEMS - 1));
          for (int spin = 0; *sem != want && spin < (1 << 16); ++spin) __nanosleep(64);
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
      constexpr int CHUNK_UNROLL = MT == 2 ? BN / 32 : 1;  // MT = 2 indexes the accumulator registers by chunk
#pragma unroll CHUNK_UNROLL
      for (int c = wg; c < BN / 32; c += 3 - MT) {
        const int nc = n0 + c * 32;
        if (nc >= p.N) break;
        float v[32];
        if constexpr (MT == 1) {
#pragma unroll
          for (int j = 0; j < 32; j += 4) {
            const float4 q = *reinterpret_cast<const float4*>(acc_row + c * 32 + j);
            v[j] = q.x; v[j + 1] = q.y; v[j + 2] = q.z; v[j + 3] = q.w;
          }
        } else {
          // the warp's fragment of chunk c -> its 128B-swizzled buffer, row = warp-local tile row (chain h, fragment
          // row r: 8 h + r for r < 8, 16 + 8 h + r - 8 otherwise) -> v = row `lane`
          if (lane == 0) tma_store_wait_read<0>();  // the previous chunk's TMA store has read the buffer
          __syncwarp();
          const int r = lane >> 2;
#pragma unroll
          for (int cc = 0; cc < BN / 32; ++cc) {
            if (cc != c) continue;
#pragma unroll
            for (int h = 0; h < MT; ++h) {
#pragma unroll
              for (int jj = 0; jj < 4; ++jj) {
                const int j = 4 * cc + jj, off = (((2 * jj + ((lane & 3) >> 1)) ^ r) << 4) + (lane & 1) * 8;
                *reinterpret_cast<float2*>(stage_buf + (8 * h + r) * 128 + off) = make_float2(acc[h][4 * j], acc[h][4 * j + 1]);
                *reinterpret_cast<float2*>(stage_buf + (16 + 8 * h + r) * 128 + off) =
                    make_float2(acc[h][4 * j + 2], acc[h][4 * j + 3]);
              }
            }
          }
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 q = *reinterpret_cast<const float4*>(stage_buf + lane * 128 + ((j ^ (lane & 7)) << 4));
            v[4 * j] = q.x; v[4 * j + 1] = q.y; v[4 * j + 2] = q.z; v[4 * j + 3] = q.w;
          }
          __syncwarp();  // every lane has its row before the buffer takes the output chunk
        }
        if (f_stats) {
          // per-group sum / sumsq of the raw conv output, butterfly-reduced over the 32 rows of the warp at sub-groups of
          // `sub` channels (the largest power-of-two divisor of cpg, at most 32; an aligned sub-group lies inside one
          // group), then added into the CTA's fp64 partial sum of its group
          const int cpg = p.cpg;
          const int sub = min(cpg & -cpg, 32);
          if (sub == 1) {
            // one sub-group per channel: 32 sums and 32 sums of squares -> two butterflies
            float ss[32], sq[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) {
              ss[j] = valid ? v[j] : 0.f;
              sq[j] = valid ? v[j] * v[j] : 0.f;
            }
            warp_butterfly32(ss, lane);
            warp_butterfly32(sq, lane);
            if (nc + lane < p.N) {
              atomicAdd(&stat_acc[2 * ((nc + lane) / cpg)], (double)ss[0]);
              atomicAdd(&stat_acc[2 * ((nc + lane) / cpg) + 1], (double)sq[0]);
            }
          } else {
            float sv[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) sv[j] = 0.f;
            if (valid) {
              if (sub == 2) accum_stats<2>(v, sv);
              else if (sub == 4) accum_stats<4>(v, sv);
              else if (sub == 8) accum_stats<8>(v, sv);
              else if (sub == 16) accum_stats<16>(v, sv);
              else accum_stats<32>(v, sv);
            }
            warp_butterfly32(sv, lane);
            // lane L now holds the warp total of value L (value = 2*local_sub_group + {0: sum, 1: sumsq})
            if (lane < 2 * (32 / sub)) atomicAdd(&stat_acc[2 * ((nc + sub * (lane >> 1)) / cpg) + (lane & 1)], (double)sv[0]);
          }
        }
        // ---- epilogue math in the thread = row domain (32 consecutive output columns in registers)
        const bool full_chunk = LEAN || (nc + 32 <= p.N);
        if (p.bias) {
          if (full_chunk && (reinterpret_cast<uintptr_t>(p.bias) & 15) == 0) {
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 bq = __ldg(reinterpret_cast<const float4*>(p.bias + nc + j));
              v[j] += bq.x; v[j + 1] += bq.y; v[j + 2] += bq.z; v[j + 3] += bq.w;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (nc + j < p.N) v[j] += __ldg(p.bias + nc + j);
          }
        }
        if (p.residual && valid) {
          const float* rrow = p.residual + m * p.ldr + nc;
          if (full_chunk && row_vec) {
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 rr = __ldg(reinterpret_cast<const float4*>(rrow + j));
              v[j] += rr.x; v[j + 1] += rr.y; v[j + 2] += rr.z; v[j + 3] += rr.w;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (nc + j < p.N) v[j] += rrow[j];
          }
        }
        if (p.act == 1) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
        } else if (p.act == 2) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = gelu_erf(v[j]);
        } else if (p.act == 3) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = swish(v[j]);
        }
        if (p.split_out) {  // the 32 values of this (row, chunk) become the 32 words of their S32 chunk
          uint32_t w[32];
          split_chunk32(v, w);
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(w[j]);
        }
        if (f_tma) {
          // registers -> 128B-swizzled smem chunk (conflict-free) -> one TMA store per warp and chunk; the TMA unit
          // generates the row addresses and clips rows >= M / columns >= N / voxels outside the grid
          uint8_t* sb = stage_buf;
          if (lane == 0) tma_store_wait_read<0>();  // this warp's previous chunk has been read out of the buffer
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float4*>(sb + lane * 128 + ((j ^ (lane & 7)) << 4)) =
                make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
          fence_proxy_async_smem();
          __syncwarp();
          if (lane == 0) {
            if (f_conv) {
              // rows ew*32 .. ew*32+31 of the tile form a sub-box (ex, ey, ez) of the (bx, by, bz) voxel box
              const int r0 = ew * 32;
              if (f_splits > 1)
                tma_reduce_add_5d(&tmC, sb, nc, tile_z0 + r0 % p.bz, tile_y0 + (r0 / p.bz) % p.by,
                                  tile_x0 + r0 / (p.bz * p.by), tile_b);
              else
                tma_store_5d(&tmC, sb, nc, tile_z0 + r0 % p.bz, tile_y0 + (r0 / p.bz) % p.by,
                             tile_x0 + r0 / (p.bz * p.by), tile_b);
            } else if (f_splits > 1) {
              tma_reduce_add_2d(&tmC, sb, nc, m_tile * TILE_M + ew * 32);
            } else {
              tma_store_2d(&tmC, sb, nc, m_tile * TILE_M + ew * 32);
            }
            tma_store_commit();
          }
        } else if (valid) {
          float* orow = p.out + m * p.ldo + nc;
#pragma unroll
          for (int j = 0; j < 32; ++j)
            if (nc + j < p.N) orow[j] = v[j];
        }
      }
      if constexpr (MT == 1) named_bar_sync(4 + cg, 128);  // the staging block may be overwritten by the next tile
      if (f_splits > 1) {  // publish: this split's reduce-adds are complete
        if (lane == 0) tma_store_wait_all();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (threadIdx.x == 0) {
          __threadfence();
          const int split = tile % f_splits;
          atomicExch(p.splitk_sem + ((tile / f_splits) & (SPLITK_SEMS - 1)), split == f_splits - 1 ? 0 : split + 1);
        }
      }
    }
    if (timed_out) __trap();
    if (f_stats) {
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (cur_b >= 0) {
        const int ngroups2 = 2 * (p.N / p.cpg);
        for (int i = threadIdx.x; i < ngroups2; i += 256) {
          const double v = stat_acc[i];
          if (v != 0.0) atomicAdd(&p.gn_stats[(size_t)cur_b * ngroups2 + i], v);
        }
      }
    }
    if (lane == 0) tma_store_wait_all();  // all bulk stores of this warp have been written
  }
}

}  // namespace occ

// =====================================================================================================
// host side
// =====================================================================================================
namespace occ {

// GroupNorm statistics of a finished (B, rows_per_sample, C) tensor (split-K conv outputs, the neck's input convs):
// stats[b][g] += (sum, sumsq), C % 4 == 0, any cpg with at most MAX_STAT_GROUPS groups.
// One CTA = 32 rows; thread t owns the float4 column t (t + blockDim.x, ...): eight independent row loads in flight, fp64
// sums over the 32 rows, fp64 per group in shared memory, one fp64 global atomic per (CTA, group, moment).  The sums are
// fp64 from the first row on: the consumer takes var = sumsq / n - mean^2, which cancels ~(mean / std)^2 of the digits
// of sumsq, and fp32 column sums lost up to 1e-5 of a group's spread at mean / std = 100 (the kernel is bound by its
// loads).
constexpr int GS_ROWS = 32;
__global__ void __launch_bounds__(256)
conv_gn_stats_kernel(const float* __restrict__ x, double* __restrict__ stats, int rows_per_sample, int C, int cpg) {
  __shared__ double sg[2 * MAX_STAT_GROUPS];
  const int b = blockIdx.y;
  const int r0 = blockIdx.x * GS_ROWS;
  const int nr = min(GS_ROWS, rows_per_sample - r0);
  const int groups = C / cpg;
  const int C4 = C >> 2;
  for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) sg[i] = 0.0;
  __syncthreads();
  const float4* base = reinterpret_cast<const float4*>(x + ((size_t)b * rows_per_sample + r0) * C);
  for (int c4 = threadIdx.x; c4 < C4; c4 += blockDim.x) {
    double s[4] = {0.0, 0.0, 0.0, 0.0}, q[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll 8
    for (int r = 0; r < nr; ++r) {
      const float4 v = __ldg(base + (size_t)r * C4 + c4);
      const double d[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) { s[j] += d[j]; q[j] = fma(d[j], d[j], q[j]); }
    }
    const int c = c4 << 2;
    if (cpg % 4 == 0) {  // the four columns share a group
      atomicAdd(&sg[2 * (c / cpg)], (s[0] + s[1]) + (s[2] + s[3]));
      atomicAdd(&sg[2 * (c / cpg) + 1], (q[0] + q[1]) + (q[2] + q[3]));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        atomicAdd(&sg[2 * ((c + j) / cpg)], s[j]);
        atomicAdd(&sg[2 * ((c + j) / cpg) + 1], q[j]);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * groups; i += blockDim.x) atomicAdd(&stats[(size_t)b * 2 * groups + i], sg[i]);
}

// one thread per float4 column (at most 256): 192 channels -> 64-thread CTAs, several per SM keep enough loads in flight
static int launch_gn_stats(const float* x, double* stats, int B, int rows_per_sample, int C, int cpg, cudaStream_t stream) {
  const int threads = C / 4 >= 256 ? 256 : (C / 4 + 31) / 32 * 32;
  dim3 grid((rows_per_sample + GS_ROWS - 1) / GS_ROWS, B);
  conv_gn_stats_kernel<<<grid, threads, 0, stream>>>(x, stats, rows_per_sample, C, cpg);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// ring depth of an instantiation: as deep as the shared memory allows (MT = 2 has no fp32 staging block)
constexpr int gemm_stages(int bn, int mt) { return mt == 2 ? 4 : bn <= 32 ? 8 : bn <= 64 ? 6 : bn <= 96 ? 4 : 3; }

template <int BN, bool LEAN, int MT, int PASSES>
static int launch_gemm_passes(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmParams& p,
                              int num_tiles, cudaStream_t stream) {
  constexpr int STAGES = gemm_stages(BN, MT);
  constexpr size_t smem = (size_t)STAGES * (MT * A_STAGE_BYTES + BN * BK * 4) + 1024 /*align*/ + CTRL_BYTES + EPI_BYTES +
                          (MT == 1 ? acc_stage_bytes<BN>() : 0);
  static_assert(smem <= 227 * 1024, "shared memory budget");
  OCC_ENSURE_SMEM((gemm_bf16x3_kernel<BN, STAGES, LEAN, MT, PASSES>), smem);
  int grid = num_tiles < sm_count() ? num_tiles : sm_count();
  if (grid < 1) grid = 1;
  gemm_bf16x3_kernel<BN, STAGES, LEAN, MT, PASSES><<<grid, GEMM_THREADS, smem, stream>>>(tmA, tmB, tmC, p);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// p.passes (mma_passes() at the call) selects the three-pass or the single-pass instantiation
template <int BN, bool LEAN = false, int MT = 1>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmParams& p,
                       int num_tiles, cudaStream_t stream) {
  if (p.passes == 1) return launch_gemm_passes<BN, LEAN, MT, 1>(tmA, tmB, tmC, p, num_tiles, stream);
  return launch_gemm_passes<BN, LEAN, MT, 3>(tmA, tmB, tmC, p, num_tiles, stream);
}

// N-tile: 96-wide tiles for the 192-channel neck / head matrices (N = 192, 576: no padded columns), else 32 / 64 / 128
// (a consumer thread holds BN / 2 fp32 accumulators per M chain)
static int gemm_bn(int N) { return N <= 32 ? 32 : N <= 64 ? 64 : (N % 96 == 0 && N % 128 != 0) ? 96 : 128; }

// mt = 2: 256-row tiles (conv mode, BN 96 / 128, no split-K)
static int dispatch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmC, const void* W, GemmParams& p, int num_m_tiles,
                         cudaStream_t stream, int mt = 1) {
  const int BN = gemm_bn(p.N);
  CUtensorMap tmB;
  uint64_t dims[2] = {(uint64_t)p.K, (uint64_t)p.N};
  uint64_t strides[1] = {(uint64_t)p.K * 4};
  uint32_t box[2] = {(uint32_t)BK, (uint32_t)BN};
  int rc = make_tmap_f32(&tmB, W, 2, dims, strides, box, nullptr);
  if (rc) return rc;
  if (p.splits < 1) p.splits = 1;
  const int num_tiles = num_m_tiles * ((p.N + BN - 1) / BN) * p.splits;
  if (mt == 2) {
    OCC_REQUIRE(p.conv && p.splits == 1 && (BN == 96 || BN == 128));
    if (BN == 96) return launch_gemm<96, false, 2>(tmA, tmB, tmC, p, num_tiles, stream);
    return launch_gemm<128, false, 2>(tmA, tmB, tmC, p, num_tiles, stream);
  }
  // plain Linear with whole 32-column chunks through the TMA store: the lean instantiation (shorter epilogue)
  const bool lean = !p.conv && p.splits == 1 && p.use_tma_store && p.N % 32 == 0 &&
                    (reinterpret_cast<uintptr_t>(p.bias) & 15) == 0 &&
                    (p.residual == nullptr || ((reinterpret_cast<uintptr_t>(p.residual) & 15) == 0 && p.ldr % 4 == 0));
  if (lean) {
    switch (BN) {
      case 32: break;
      case 64: return launch_gemm<64, true>(tmA, tmB, tmC, p, num_tiles, stream);
      case 96: return launch_gemm<96, true>(tmA, tmB, tmC, p, num_tiles, stream);
      default: return launch_gemm<128, true>(tmA, tmB, tmC, p, num_tiles, stream);
    }
  }
  switch (BN) {
    case 32: return launch_gemm<32>(tmA, tmB, tmC, p, num_tiles, stream);
    case 64: return launch_gemm<64>(tmA, tmB, tmC, p, num_tiles, stream);
    case 96: return launch_gemm<96>(tmA, tmB, tmC, p, num_tiles, stream);
    default: return launch_gemm<128>(tmA, tmB, tmC, p, num_tiles, stream);
  }
}

// Voxel box of a `rows`-row conv tile: power-of-two sides (so that every warp's 32-row slab is a sub-box for the TMA
// store) with the fewest padded output voxels; ties keep the deepest z, then y extent.  E.g. 100 x 100 x 8 -> 4 x 4 x 8
// (no padding) instead of 1 x 16 x 8 (12 % of the rows past the grid).
static void conv_box(int Xo, int Yo, int Zo, int rows, int stride, int& bx, int& by, int& bz) {
  auto padded = [](int n, int b) { return (long long)((n + b - 1) / b) * b; };
  long long best = -1;
  for (int z = rows; z >= 1; z >>= 1)
    for (int y = rows / z; y >= 1; y >>= 1) {
      const int x = rows / (z * y);
      if (x * stride > 256 || y * stride > 256 || z * stride > 256) continue;
      const long long v = padded(Xo, x) * padded(Yo, y) * padded(Zo, z);
      if (best < 0 || v < best) { best = v; bx = x; by = y; bz = z; }
    }
}

// Tiling of a regular-stencil conv (occ_conv_bf16x3): 256-row tiles (MT = 2) for long-K convs with N <= 128 per tile,
// at least four waves of them and at most 5 % more padded rows than 128-row tiles, else 128-row tiles with split-K for the deep stages (few output tiles, long K = 27 *
// Cin): a 512->512 conv on 50x50x4 voxels has 158 tiles for 132 SMs (second wave 20 % full), a 1024->1024 conv on 25x25x2
// has 40.  Split-K needs `splitk_ok` (no bias / activation / residual / split output, TMA store, a workspace).
struct ConvPlan { int mt, bn, stages, splits, bx, by, bz, tiles_x, tiles_y, tiles_z; };
static ConvPlan conv_plan(int B, int Xo, int Yo, int Zo, int Cout, int stride, int num_k_blocks, bool splitk_ok) {
  ConvPlan c{};
  c.bn = gemm_bn(Cout);
  const int n_tiles = (Cout + c.bn - 1) / c.bn;
  const int sms = sm_count();
  auto tile = [&](int rows) {  // -> number of M tiles
    conv_box(Xo, Yo, Zo, rows, stride, c.bx, c.by, c.bz);
    c.tiles_x = (Xo + c.bx - 1) / c.bx; c.tiles_y = (Yo + c.by - 1) / c.by; c.tiles_z = (Zo + c.bz - 1) / c.bz;
    return (long long)B * c.tiles_x * c.tiles_y * c.tiles_z;
  };
  c.mt = 1;
  c.splits = 1;
  const long long m2 = tile(2 * BM), m1 = tile(BM);
  if ((c.bn == 96 || c.bn == 128) && num_k_blocks >= 64 && m2 * n_tiles >= 4LL * sms && m2 * 2 * 100 <= m1 * 105) {
    c.mt = 2;
    tile(2 * BM);
  } else {
    const long long num_m_tiles = m1;
    const long long tiles = num_m_tiles * n_tiles;
    auto eff = [&](int s) { const long long t = tiles * s; return (double)t / (double)(((t + sms - 1) / sms) * sms); };
    // (not below 8 M-tiles = 1024 output rows: such convs are latency-bound either way, and keeping them on the
    // single-pass path keeps small problems bit-reproducible -- the reduce-add order of the splits is not fixed)
    if (splitk_ok && num_m_tiles >= 8 && tiles < 2 * sms && num_k_blocks >= 64 && eff(1) < 0.85) {
      int best = 1;
      for (int sp = 2; sp <= 8 && sp * 8 <= num_k_blocks; ++sp) {
        if (eff(sp) > eff(best) + 0.02) best = sp;
        if (eff(best) >= 0.85) break;
      }
      c.splits = best;
    }
  }
  c.stages = gemm_stages(c.bn, c.mt);
  return c;
}

}  // namespace occ

using namespace occ;

extern "C" int occ_gemm_bf16x3(const float* A, const float* W, float* out, int M, int N, int K, const float* bias,
                               const float* residual, int act, int split_out, cudaStream_t stream) {
  OCC_REQUIRE(A && W && out);
  OCC_REQUIRE(M > 0 && N > 0 && K > 0);
  OCC_REQUIRE(K % 32 == 0);                 // S32 operand rows: whole 32-k chunks
  OCC_REQUIRE(!split_out || N % 32 == 0);   // S32 output rows
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0);
  OCC_REQUIRE(act >= 0 && act <= 3);
  GemmParams p{};
  p.passes = mma_passes();
  p.M = M; p.N = N; p.K = K; p.num_k_blocks = (K + BK - 1) / BK;
  p.out = out; p.ldo = N; p.bias = bias; p.residual = residual; p.ldr = N; p.act = act; p.split_out = split_out;
  p.conv = 0;
  CUtensorMap tmA;
  uint64_t dims[2] = {(uint64_t)K, (uint64_t)M};
  uint64_t strides[1] = {(uint64_t)K * 4};
  uint32_t box[2] = {(uint32_t)BK, (uint32_t)BM};
  int rc = make_tmap_f32(&tmA, A, 2, dims, strides, box, nullptr);
  if (rc) return rc;
  CUtensorMap tmC = tmA;  // placeholder when the TMA-store path is not usable (N % 4 != 0: scalar row stores)
  p.use_tma_store = (N % 4 == 0) && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  if (p.use_tma_store) {
    uint64_t cd[2] = {(uint64_t)N, (uint64_t)M};
    uint64_t cs[1] = {(uint64_t)N * 4};
    uint32_t cb[2] = {32u, 32u};
    rc = make_tmap_f32(&tmC, out, 2, cd, cs, cb, nullptr);
    if (rc) return rc;
  }
  return dispatch_gemm(tmA, tmC, W, p, (M + BM - 1) / BM, stream);
}

// x: (B, X, Y, Z, Cin) channel-last, S32;  w2: (Cout, KX*KY*KZ*Cin) tap-major repacked weights, S32 per tap;
// out: (B, Xo, Yo, Zo, Cout).  pad = dil*(K-1)/2 per axis ("same" for stride 1), Xo = (X + 2p - dil*(K-1) - 1)/s + 1.
extern "C" size_t occ_conv_workspace_bytes(void) { return SPLITK_SEMS * sizeof(int); }

// occ_conv_bf16x3 / occ_conv_slice_bf16x3: the output rows have pitch ldo floats and the conv writes their columns
// [out_off, out_off + Cout); ldo = Cout, out_off = 0 is the plain contiguous output.
static int conv_bf16x3(const float* x, const float* w2, float* out, int ldo, int out_off, int B, int X, int Y, int Z,
                       int Cin, int Cout, int KX, int KY, int KZ, int stride, int dil, const float* bias,
                       const float* residual, int act, int split_out, double* gn_stats, int cpg, void* workspace,
                       size_t workspace_bytes, cudaStream_t stream) {
  OCC_REQUIRE(x && w2 && out);
  OCC_REQUIRE(!split_out || Cout % 32 == 0);
  OCC_REQUIRE(out_off >= 0 && ldo >= out_off + Cout);
  // an S32 slice is made of whole 32-column chunks; an fp32 slice keeps the TMA store's 16-byte row alignment
  if (ldo != Cout) OCC_REQUIRE(split_out ? (ldo % 32 == 0 && out_off % 32 == 0) : (ldo % 4 == 0 && out_off % 4 == 0));
  OCC_REQUIRE(B > 0 && X > 0 && Y > 0 && Z > 0 && Cin > 0 && Cout > 0);
  OCC_REQUIRE(Cin % BK == 0);
  OCC_REQUIRE((KX == 1 || KX == 3) && (KY == 1 || KY == 3) && (KZ == 1 || KZ == 3));
  OCC_REQUIRE(stride == 1 || stride == 2);
  OCC_REQUIRE(dil >= 1 && act >= 0 && act <= 3);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w2) & 15) == 0);
  if (gn_stats) OCC_REQUIRE(cpg >= 1 && Cout % cpg == 0 && Cout / cpg <= MAX_STAT_GROUPS);
  GemmParams p{};
  p.passes = mma_passes();
  p.conv = 1;
  p.Cin = Cin; p.KX = KX; p.KY = KY; p.KZ = KZ; p.dil = dil; p.stride = stride;
  p.padx = dil * (KX - 1) / 2; p.pady = dil * (KY - 1) / 2; p.padz = dil * (KZ - 1) / 2;
  p.B = B;
  p.Xo = (X + 2 * p.padx - dil * (KX - 1) - 1) / stride + 1;
  p.Yo = (Y + 2 * p.pady - dil * (KY - 1) - 1) / stride + 1;
  p.Zo = (Z + 2 * p.padz - dil * (KZ - 1) - 1) / stride + 1;
  p.N = Cout; p.K = KX * KY * KZ * Cin; p.num_k_blocks = p.K / BK;
  p.M = B * p.Xo * p.Yo * p.Zo;
  out += out_off;
  p.out = out; p.ldo = ldo; p.bias = bias; p.residual = residual; p.ldr = Cout; p.act = act; p.split_out = split_out;
  p.gn_stats = gn_stats; p.cpg = cpg;
  p.use_tma_store = (Cout % 4 == 0) && (ldo % 4 == 0) && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  // split-K: the raw conv output of the encoder has no bias / activation (GroupNorm follows), so the partial sums can
  // meet in `out` through TMA reduce-add; the GroupNorm statistics are then taken from the finished tensor.  Only for a
  // contiguous output: the zero fill and the statistics pass read `out` as (rows, Cout).
  const bool splitk_ok = p.use_tma_store && ldo == Cout && !bias && !residual && act == 0 && !split_out && workspace &&
                         workspace_bytes >= SPLITK_SEMS * sizeof(int) && (reinterpret_cast<uintptr_t>(workspace) & 3) == 0;
  const ConvPlan plan = conv_plan(B, p.Xo, p.Yo, p.Zo, Cout, stride, p.num_k_blocks, splitk_ok);
  p.bx = plan.bx; p.by = plan.by; p.bz = plan.bz;
  p.tiles_x = plan.tiles_x; p.tiles_y = plan.tiles_y; p.tiles_z = plan.tiles_z;
  p.splits = plan.splits;
  CUtensorMap tmA;
  uint64_t dims[5] = {(uint64_t)Cin, (uint64_t)Z, (uint64_t)Y, (uint64_t)X, (uint64_t)B};
  uint64_t strides[4] = {(uint64_t)Cin * 4, (uint64_t)Z * Cin * 4, (uint64_t)Y * Z * Cin * 4,
                         (uint64_t)X * Y * Z * Cin * 4};
  uint32_t box[5] = {(uint32_t)BK, (uint32_t)(p.bz * stride), (uint32_t)(p.by * stride), (uint32_t)(p.bx * stride), 1};
  uint32_t estr[5] = {1, (uint32_t)stride, (uint32_t)stride, (uint32_t)stride, 1};
  int rc = make_tmap_f32(&tmA, x, 5, dims, strides, box, estr);
  if (rc) return rc;
  CUtensorMap tmC = tmA;
  if (p.use_tma_store) {
    // one epilogue warp owns 32 consecutive rows of the (bx, by, bz) box = a sub-box (ex, ey, ez)
    const int ez = p.bz < 32 ? p.bz : 32;
    const int ey = p.by < 32 / ez ? p.by : 32 / ez;
    const int ex = 32 / (ez * ey);
    // columns >= Cout of a slice are clipped by the map (they belong to the rest of the row)
    uint64_t cd[5] = {(uint64_t)Cout, (uint64_t)p.Zo, (uint64_t)p.Yo, (uint64_t)p.Xo, (uint64_t)B};
    uint64_t cs[4] = {(uint64_t)ldo * 4, (uint64_t)p.Zo * ldo * 4, (uint64_t)p.Yo * p.Zo * ldo * 4,
                      (uint64_t)p.Xo * p.Yo * p.Zo * ldo * 4};
    uint32_t cb[5] = {32u, (uint32_t)ez, (uint32_t)ey, (uint32_t)ex, 1u};
    rc = make_tmap_f32(&tmC, out, 5, cd, cs, cb, nullptr);
    if (rc) return rc;
  }
  const int num_m_tiles = B * p.tiles_x * p.tiles_y * p.tiles_z;
  if (p.splits > 1) {
    OCC_MEMSET(out, 0, (size_t)p.M * Cout * sizeof(float), stream);
    p.gn_stats = nullptr;
    p.splitk_sem = static_cast<int*>(workspace);
  }
  rc = dispatch_gemm(tmA, tmC, w2, p, num_m_tiles, stream, plan.mt);
  if (rc) return rc;
  if (p.splits > 1 && gn_stats) return launch_gn_stats(out, gn_stats, B, p.Xo * p.Yo * p.Zo, Cout, cpg, stream);
  return OCC_OK;
}

extern "C" int occ_conv_bf16x3(const float* x, const float* w2, float* out, int B, int X, int Y, int Z, int Cin,
                               int Cout, int KX, int KY, int KZ, int stride, int dil, const float* bias,
                               const float* residual, int act, int split_out, double* gn_stats, int cpg,
                               void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return conv_bf16x3(x, w2, out, Cout, 0, B, X, Y, Z, Cin, Cout, KX, KY, KZ, stride, dil, bias, residual, act, split_out,
                     gn_stats, cpg, workspace, workspace_bytes, stream);
}

extern "C" int occ_conv_slice_bf16x3(const float* x, const float* w2, float* out, int ldo, int out_off, int B, int X,
                                     int Y, int Z, int Cin, int Cout, int KX, int KY, int KZ, int stride, int dil,
                                     const float* bias, const float* residual, int act, int split_out, double* gn_stats,
                                     int cpg, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  return conv_bf16x3(x, w2, out, ldo, out_off, B, X, Y, Z, Cin, Cout, KX, KY, KZ, stride, dil, bias, residual, act,
                     split_out, gn_stats, cpg, workspace, workspace_bytes, stream);
}


// The tiling occ_conv_bf16x3 picks for a conv shape (without a split-K workspace: splits = 1 for a conv that has a bias,
// activation, residual or split output): plan[0..3] = (tile rows, tile columns, ring stages, K splits).
extern "C" int occ_conv_plan(int B, int X, int Y, int Z, int Cin, int Cout, int KX, int KY, int KZ, int stride, int dil,
                             int splitk_ok, int* plan) {
  OCC_REQUIRE(plan && B > 0 && X > 0 && Y > 0 && Z > 0 && Cin > 0 && Cin % BK == 0 && Cout > 0);
  OCC_REQUIRE((stride == 1 || stride == 2) && dil >= 1);
  const int Xo = (X - 1) / stride + 1, Yo = (Y - 1) / stride + 1, Zo = (Z - 1) / stride + 1;  // "same" padding
  const ConvPlan c = conv_plan(B, Xo, Yo, Zo, Cout, stride, KX * KY * KZ * Cin / BK, splitk_ok != 0);
  plan[0] = c.mt * BM; plan[1] = c.bn; plan[2] = c.stages; plan[3] = c.splits;
  return OCC_OK;
}

// Several same-input stride-1 convolutions in one launch: an explicit tap table instead of a regular stencil.
// x (B,X,Y,Z,Cin) S32; taps: ntaps x (dx, dy, dz) input offsets (HOST ints, |offset| <= 127); w2 (Cout, ntaps*Cin) S32,
// tap-major in the table's order (a branch that does not use a tap has zero weights there); out (B,X,Y,Z,Cout) raw fp32;
// gn_stats as occ_conv_bf16x3.  Used for the four ASPP branches (1x1 + three dilated 3x3,
// P/occformer/backbones/modules/aspp.py:107-113): one launch with 25 taps instead of four.
extern "C" int occ_conv_taps_bf16x3(const float* x, const float* w2, float* out, int B, int X, int Y, int Z, int Cin,
                                    int Cout, int ntaps, const int* taps, double* gn_stats, int cpg, cudaStream_t stream) {
  OCC_REQUIRE(x && w2 && out && taps);
  OCC_REQUIRE(B > 0 && X > 0 && Y > 0 && Z > 0 && Cin > 0 && Cout > 0 && Cin % BK == 0 && ntaps >= 1 && ntaps <= MAX_TAPS);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(w2) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(out) & 15) == 0 && Cout % 4 == 0);
  if (gn_stats) OCC_REQUIRE(cpg >= 1 && Cout % cpg == 0 && Cout / cpg <= MAX_STAT_GROUPS);
  GemmParams p{};
  p.passes = mma_passes();
  p.conv = 1;
  p.Cin = Cin; p.KX = p.KY = p.KZ = 1; p.dil = 1; p.stride = 1; p.padx = p.pady = p.padz = 0;
  p.ntaps = ntaps;
  for (int t = 0; t < ntaps; ++t) {
    OCC_REQUIRE(taps[3 * t] >= -127 && taps[3 * t] <= 127 && taps[3 * t + 1] >= -127 && taps[3 * t + 1] <= 127 &&
                taps[3 * t + 2] >= -127 && taps[3 * t + 2] <= 127);
    p.tdx[t] = (signed char)taps[3 * t]; p.tdy[t] = (signed char)taps[3 * t + 1]; p.tdz[t] = (signed char)taps[3 * t + 2];
  }
  p.B = B; p.Xo = X; p.Yo = Y; p.Zo = Z;
  conv_box(X, Y, Z, BM, 1, p.bx, p.by, p.bz);
  p.tiles_x = (X + p.bx - 1) / p.bx; p.tiles_y = (Y + p.by - 1) / p.by; p.tiles_z = (Z + p.bz - 1) / p.bz;
  p.N = Cout; p.K = ntaps * Cin; p.num_k_blocks = p.K / BK; p.M = B * X * Y * Z;
  p.out = out; p.ldo = Cout; p.ldr = Cout; p.act = 0; p.split_out = 0;
  p.gn_stats = gn_stats; p.cpg = cpg; p.splits = 1;
  CUtensorMap tmA;
  uint64_t dims[5] = {(uint64_t)Cin, (uint64_t)Z, (uint64_t)Y, (uint64_t)X, (uint64_t)B};
  uint64_t strides[4] = {(uint64_t)Cin * 4, (uint64_t)Z * Cin * 4, (uint64_t)Y * Z * Cin * 4, (uint64_t)X * Y * Z * Cin * 4};
  uint32_t box[5] = {(uint32_t)BK, (uint32_t)p.bz, (uint32_t)p.by, (uint32_t)p.bx, 1};
  int rc = make_tmap_f32(&tmA, x, 5, dims, strides, box, nullptr);
  if (rc) return rc;
  const int ez = p.bz < 32 ? p.bz : 32;
  const int ey = p.by < 32 / ez ? p.by : 32 / ez;
  const int ex = 32 / (ez * ey);
  CUtensorMap tmC;
  uint64_t cd[5] = {(uint64_t)Cout, (uint64_t)Z, (uint64_t)Y, (uint64_t)X, (uint64_t)B};
  uint64_t cs[4] = {(uint64_t)Cout * 4, (uint64_t)Z * Cout * 4, (uint64_t)Y * Z * Cout * 4, (uint64_t)X * Y * Z * Cout * 4};
  uint32_t cb[5] = {32u, (uint32_t)ez, (uint32_t)ey, (uint32_t)ex, 1u};
  rc = make_tmap_f32(&tmC, out, 5, cd, cs, cb, nullptr);
  if (rc) return rc;
  p.use_tma_store = 1;
  return dispatch_gemm(tmA, tmC, w2, p, B * p.tiles_x * p.tiles_y * p.tiles_z, stream);
}

// stats (B, C/cpg, 2) fp64, zero-initialised by the caller: += (sum, sumsq) of x (B, rows_per_sample, C) per (sample, group)
extern "C" int occ_gn_stats(const float* x, double* stats, int B, int rows_per_sample, int C, int cpg, cudaStream_t stream) {
  OCC_REQUIRE(x && stats && B > 0 && B <= 65535 && rows_per_sample > 0 && C > 0 && C % 4 == 0);
  OCC_REQUIRE(cpg >= 1 && C % cpg == 0 && C / cpg <= MAX_STAT_GROUPS && (reinterpret_cast<uintptr_t>(x) & 15) == 0);
  return launch_gn_stats(x, stats, B, rows_per_sample, C, cpg, stream);
}
