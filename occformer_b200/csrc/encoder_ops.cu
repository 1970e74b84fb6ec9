// Normalisation / layout / fusion kernels of the dual-path encoder block (all HBM-bound, one pass each).
//
// Token layout used by the whole encoder: channel-last rows of C floats.
//   voxel tokens  : row ((b*X + x)*Y + y)*Z + z           (the (B,X,Y,Z,C) tensor itself)
//   BEV tokens    : row B*X*Y*Z + (b*X + x)*Y + y         (mean over Z, appended behind the voxel tokens)
// so the reference's rearrange 'b c x y z -> (b z) c x y', cat, NCHW<->NLC permutes and their inverses
// (projects/mmdet3d_plugin/occformer/backbones/dualpath_block.py:69-76, modules/window_attention.py:350,370)
// disappear: every one of the B*(Z+1) images is addressed in place.
#include "occ_common.cuh"
#include "occ_ptx.cuh"
#include "window_geom.cuh"

namespace occ {

constexpr float kEps = 1e-5f;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// mean / rstd of one GroupNorm group from the fp64 (sum, sumsq) accumulated by the conv epilogue.
__device__ __forceinline__ void gn_mean_rstd(const double* __restrict__ stats, int b, int groups, int g, double count,
                                             float* mean, float* rstd) {
  const double s = stats[((size_t)b * groups + g) * 2 + 0];
  const double q = stats[((size_t)b * groups + g) * 2 + 1];
  const double m = s / count;
  double var = q / count - m * m;
  if (var < 0.0) var = 0.0;
  *mean = (float)m;
  *rstd = (float)(1.0 / sqrt(var + (double)kEps));
}

// LayerNorm of a row held as NV float4 per lane (C = 128*NV).  two-pass in registers, on the row shifted by its first
// element: for a row whose offset dwarfs its spread the shifted values are exact and small, so the fp32 sums lose no
// digits to the offset (an unshifted sum of values near 1e3 puts ~1e-5 of the spread into the mean).
template <int NV>
__device__ __forceinline__ void warp_layernorm(float4 (&v)[NV], int C, const float* __restrict__ gamma,
                                               const float* __restrict__ beta, int lane) {
  const float shift = __shfl_sync(0xffffffffu, v[0].x, 0);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    v[i].x -= shift; v[i].y -= shift; v[i].z -= shift; v[i].w -= shift;
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) s += v[i].x + v[i].y + v[i].z + v[i].w;
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
    q += a * a + b * b + c * c + d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + kEps);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c0 = (i * 32 + lane) * 4;
    const float4 g = *reinterpret_cast<const float4*>(gamma + c0);
    const float4 bb = *reinterpret_cast<const float4*>(beta + c0);
    v[i].x = (v[i].x - mean) * rstd * g.x + bb.x;
    v[i].y = (v[i].y - mean) * rstd * g.y + bb.y;
    v[i].z = (v[i].z - mean) * rstd * g.z + bb.z;
    v[i].w = (v[i].w - mean) * rstd * g.w + bb.w;
  }
}

// ---------------------------------------------------------------------------------------------------------
// input_conv tail: GroupNorm + ReLU of the raw conv output, Z-mean (BEV token), LayerNorm1 of both.
//   y     : (B*X*Y*Z, C) raw Conv3d output                     (dualpath_block.py:43-48)
//   tok   : (B*X*Y*(Z+1), C) <- relu(gn(y)) and its mean over Z (dualpath_block.py:69)
//   tokn  : same rows, LayerNorm1'd, S32 split format (A operand of the QKV GEMM; window_attention.py:355)
// One CTA handles `cols` (b,x,y) columns, one warp per voxel row; the CTA's smem holds the column for the mean.
// R voxel rows (consecutive z of one column) per warp: all R row loads are issued before any of them is consumed, so a
// warp keeps R x 512 B (C = 128) in flight -- with one row per warp the kernel is bound by latency.
template <int NV, int R>
__global__ void __launch_bounds__(512)
gn_relu_zmean_ln_kernel(const float* __restrict__ y, const double* __restrict__ stats, const float* __restrict__ gn_w,
                        const float* __restrict__ gn_b, const float* __restrict__ ln_w,
                        const float* __restrict__ ln_b, float* __restrict__ tok, float* __restrict__ tokn, int B,
                        int XY, int Z, int C, int groups, int cols, const WinGeom wg, int win_layout) {
  extern __shared__ float col_smem[];  // [cols][Z][C]
  __shared__ float s_mean[16][32], s_rstd[16][32];  // GroupNorm mean / rstd per (column of this CTA, group): the fp64
                                                    // division + sqrt runs once per CTA, not once per lane and row
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wpc = Z / R;  // warps per column
  const int col_local = warp / wpc, z0 = (warp % wpc) * R;
  const long long col = (long long)blockIdx.x * cols + col_local;  // (b*XY + xy)
  const long long ncols = (long long)B * XY;
  const bool active = col_local < cols && col < ncols;
  const int cpg = C / groups;
  const double count = (double)XY * Z * cpg;
  for (int i = threadIdx.x; i < cols * groups; i += blockDim.x) {
    const int cl = i / groups, g = i % groups;
    const long long cc = (long long)blockIdx.x * cols + cl;
    if (cc < ncols) gn_mean_rstd(stats, (int)(cc / XY), groups, g, count, &s_mean[cl][g], &s_rstd[cl][g]);
  }
  __syncthreads();
  float4 v[R][NV];
  if (active) {
    const long long row0 = col * Z + z0;
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int i = 0; i < NV; ++i)
        v[r][i] = __ldcs(reinterpret_cast<const float4*>(y + (row0 + r) * C) + i * 32 + lane);
#pragma unroll
    for (int r = 0; r < R; ++r) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c0 = (i * 32 + lane) * 4;
        float4 t = v[r][i];
        const float mean = s_mean[col_local][c0 / cpg], rstd = s_rstd[col_local][c0 / cpg];  // cpg >= 4
        const float4 g = *reinterpret_cast<const float4*>(gn_w + c0);
        const float4 bb = *reinterpret_cast<const float4*>(gn_b + c0);
        t.x = fmaxf((t.x - mean) * rstd * g.x + bb.x, 0.f);
        t.y = fmaxf((t.y - mean) * rstd * g.y + bb.y, 0.f);
        t.z = fmaxf((t.z - mean) * rstd * g.z + bb.z, 0.f);
        t.w = fmaxf((t.w - mean) * rstd * g.w + bb.w, 0.f);
        v[r][i] = t;
        *reinterpret_cast<float4*>(tok + (row0 + r) * C + c0) = t;
        *reinterpret_cast<float4*>(col_smem + ((size_t)col_local * Z + z0 + r) * C + c0) = t;
      }
    }
    // tokn in window layout (operand of the fused QKV + attention kernel): window index = (wx, wy) major, image minor
    // (window_geom.cuh), so the rows of this column's height slices are 64 rows apart -- one 32-bit index computation
    // per warp
    long long wl_row0 = 0;
    if (win_layout) {
      const int ci = (int)col, b = ci / XY, xy = ci - b * XY;
      wl_row0 = window_layout_row(wg, b * Z + z0, xy / wg.Y, xy % wg.Y);
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      warp_layernorm<NV>(v[r], C, ln_w, ln_b, lane);
      long long orow = row0 + r;
      if (win_layout) orow = wl_row0 + (long long)r * 64;  // next height slice = next image of the same window
#pragma unroll
      for (int i = 0; i < NV; ++i) store_split4(tokn + orow * C, (i * 32 + lane) * 4, v[r][i]);
    }
  }
  __syncthreads();
  if (active && z0 == 0) {
    const long long brow = ncols * Z + col;
    const float inv = 1.0f / (float)Z;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c0 = (i * 32 + lane) * 4;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int zz = 0; zz < Z; ++zz) {
        const float4 t = *reinterpret_cast<const float4*>(col_smem + ((size_t)col_local * Z + zz) * C + c0);
        a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
      }
      a.x *= inv; a.y *= inv; a.z *= inv; a.w *= inv;
      v[0][i] = a;
      *reinterpret_cast<float4*>(tok + brow * C + c0) = a;
    }
    warp_layernorm<NV>(v[0], C, ln_w, ln_b, lane);
    long long orow = brow;
    if (win_layout) {
      const int ci = (int)col, b = ci / XY, xy = ci - b * XY;
      orow = window_layout_row(wg, B * Z + b, xy / wg.Y, xy % wg.Y);
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) store_split4(tokn + orow * C, (i * 32 + lane) * 4, v[0][i]);
  }
}

// ---------------------------------------------------------------------------------------------------------
// plain LayerNorm over rows (norm2, window_attention.py:360); warp per row
template <int NV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ b,
                 float* __restrict__ out, long long rows, int C, int split) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = *reinterpret_cast<const float4*>(in + row * C + (i * 32 + lane) * 4);
  warp_layernorm<NV>(v, C, w, b, lane);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (split) store_split4(out + row * C, (i * 32 + lane) * 4, v[i]);
    else *reinterpret_cast<float4*>(out + row * C + (i * 32 + lane) * 4) = v[i];
  }
}

// generic-width LayerNorm (C not a multiple of 128): one warp per row, scalar loop
__global__ void __launch_bounds__(256)
layernorm_generic_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ b,
                         float* __restrict__ out, long long rows, int C, int split) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float* src = in + row * C;
  const float shift = src[0];  // as warp_layernorm: the sums run on the row shifted by its first element
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += src[c] - shift;
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) { const float d = (src[c] - shift) - mean; q += d * d; }
  const float rstd = rsqrtf(warp_sum(q) / (float)C + kEps);
  for (int c = lane; c < C; c += 32) {  // split: C % 32 == 0, lanes (2t, 2t+1) form packed word t of the chunk
    const float o = ((src[c] - shift) - mean) * rstd * w[c] + b[c];
    if (split) {
      const float o2 = __shfl_xor_sync(0xffffffffu, o, 1);
      if (!(lane & 1)) {
        uint32_t hi, lo;
        split_pair(o, o2, hi, lo);
        uint32_t* chunk = reinterpret_cast<uint32_t*>(out + row * C + (c & ~31));
        chunk[lane >> 1] = hi;
        chunk[16 + (lane >> 1)] = lo;
      }
    } else {
      out[row * C + c] = o;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// GroupNorm apply for the small 2-D maps of BottleNeckASPP (aspp.py:49-172) and the strided skip path:
//   o = act(gn(in[row, c])) (+ residual[row, c]);  out[row, c] = o (fp32, optional) and / or
//   out_split[row, out_off + c] = o in the S32 split format (row pitch ldo; operand of the next conv);  rows = B * rows_per_batch.
// grid (row chunks, B): a CTA never straddles two samples, so the per-channel scale / shift of its sample
// (rstd * gamma, beta - mean * rstd * gamma; fp64 division + sqrt once per (CTA, group)) sit in shared memory and an
// element costs one FMA.
// A thread owns ONE float4 column (scale / shift in registers) and walks rows: no per-element index division, and
// GA_UNROLL independent 16-byte loads in flight (a tensor of 5 MB is latency-, not bandwidth-bound).  C/4 > 256: the
// column loop runs more than once.
constexpr int GA_UNROLL = 4;
__global__ void __launch_bounds__(256, 4)
gn_apply_kernel(const float* __restrict__ in, const double* __restrict__ stats, const float* __restrict__ w,
                const float* __restrict__ b, const float* __restrict__ residual, float* __restrict__ out,
                float* __restrict__ out_split, int rows_per_batch, int C, int groups, int ldo, int out_off, int relu,
                int rows_per_cta) {
  extern __shared__ float gsm[];  // scale[C], shift[C]
  float* sc = gsm;
  float* sh = gsm + C;
  const int bidx = blockIdx.y;
  const int cpg = C / groups;
  const double count = (double)rows_per_batch * cpg;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float mean, rstd;
    gn_mean_rstd(stats, bidx, groups, c / cpg, count, &mean, &rstd);
    const float a = rstd * w[c];
    sc[c] = a;
    sh[c] = b[c] - mean * a;
  }
  __syncthreads();
  const int C4 = C >> 2;
  const int cols = C4 < 256 ? C4 : 256;       // float4 columns handled per pass
  const int rstep = 256 / cols;               // rows handled per pass
  const int rl = threadIdx.x / cols, cl = threadIdx.x - rl * cols;
  if (rl >= rstep) return;
  const int r0 = blockIdx.x * rows_per_cta;
  const int r1 = min(r0 + rows_per_cta, rows_per_batch);
  const size_t base = (size_t)bidx * rows_per_batch;
  for (int c4 = cl; c4 < C4; c4 += cols) {
    const int c0 = c4 * 4;
    const float4 a = *reinterpret_cast<const float4*>(sc + c0), d = *reinterpret_cast<const float4*>(sh + c0);
    for (int r = r0 + rl; r < r1; r += GA_UNROLL * rstep) {
      float4 t[GA_UNROLL], rs[GA_UNROLL];
#pragma unroll
      for (int u = 0; u < GA_UNROLL; ++u) {
        const int rr = r + u * rstep;
        if (rr < r1) {
          t[u] = __ldcs(reinterpret_cast<const float4*>(in + (base + rr) * C + c0));
          if (residual) rs[u] = *reinterpret_cast<const float4*>(residual + (base + rr) * C + c0);
        }
      }
#pragma unroll
      for (int u = 0; u < GA_UNROLL; ++u) {
        const int rr = r + u * rstep;
        if (rr < r1) {
          // (v - mean) * rstd * gamma + beta, evaluated as v * (rstd*gamma) + (beta - mean*rstd*gamma)
          float4 o = make_float4(fmaf(t[u].x, a.x, d.x), fmaf(t[u].y, a.y, d.y), fmaf(t[u].z, a.z, d.z), fmaf(t[u].w, a.w, d.w));
          if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
          if (residual) { o.x += rs[u].x; o.y += rs[u].y; o.z += rs[u].z; o.w += rs[u].w; }
          if (out) *reinterpret_cast<float4*>(out + (base + rr) * C + c0) = o;
          if (out_split) store_split4(out_split + (base + rr) * ldo, out_off + c0, o);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// ASPP global-average-pool branch (aspp.py:89-95,113-114): column mean over the rows of each batch sample.
__global__ void __launch_bounds__(256)
colsum_kernel(const float* __restrict__ in, double* __restrict__ sums, int rows_per_batch, int C, int chunk) {
  // grid (chunks, B); block 256 threads = (256/C4) row lanes x C4 float4 columns
  const int b = blockIdx.y;
  const int C4 = C >> 2;
  const int rl = threadIdx.x / C4, c4 = threadIdx.x % C4;
  const int rstep = blockDim.x / C4;
  const int r0 = blockIdx.x * chunk;
  const int r1 = min(r0 + chunk, rows_per_batch);
  __shared__ float4 part[256];  // [rl][c4]
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  if (rl < rstep) {
    for (int r = r0 + rl; r < r1; r += rstep) {
      const float4 t = *reinterpret_cast<const float4*>(in + ((size_t)b * rows_per_batch + r) * C + c4 * 4);
      a.x += t.x; a.y += t.y; a.z += t.z; a.w += t.w;
    }
    part[rl * C4 + c4] = a;
  }
  __syncthreads();
  // one fp64 atomic per (CTA, channel): the row lanes are summed in shared memory first (a per-thread atomic put
  // 256 * chunks adds on C addresses: serialised atomics)
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float* pf = reinterpret_cast<const float*>(part);
    double acc = 0.0;
    for (int l = 0; l < rstep; ++l) acc += (double)pf[(l * C4 + (c >> 2)) * 4 + (c & 3)];
    atomicAdd(&sums[(size_t)b * C + c], acc);
  }
}

// GAP -> 1x1 conv (no bias) -> GN over a 1x1 map -> ReLU -> broadcast into the concat buffer
// (bilinear align_corners=True upsample of a 1x1 map = broadcast, aspp.py:114).  One CTA per batch sample.
__global__ void __launch_bounds__(256)
aspp_gap_branch_kernel(const double* __restrict__ sums, const float* __restrict__ wconv, const float* __restrict__ gw,
                       const float* __restrict__ gb, float* __restrict__ sums_out /*(B, ch) fp32, aliases nothing*/,
                       int rows_per_batch, int ch, int groups) {
  extern __shared__ float sm[];  // mean[ch], conv[ch], outv[ch]
  float* mean = sm;
  float* conv = sm + ch;
  float* outv = sm + 2 * ch;
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < ch; c += blockDim.x) mean[c] = (float)(sums[(size_t)b * ch + c] / (double)rows_per_batch);
  __syncthreads();
  for (int o = threadIdx.x; o < ch; o += blockDim.x) {
    float a = 0.f;
    for (int i = 0; i < ch; ++i) a += wconv[(size_t)o * ch + i] * mean[i];
    conv[o] = a;
  }
  __syncthreads();
  const int cpg = ch / groups;
  for (int o = threadIdx.x; o < ch; o += blockDim.x) {
    const int g = o / cpg;
    float m = 0.f;
    for (int i = 0; i < cpg; ++i) m += conv[g * cpg + i];
    m /= (float)cpg;
    float var = 0.f;
    for (int i = 0; i < cpg; ++i) { const float d = conv[g * cpg + i] - m; var += d * d; }
    var /= (float)cpg;
    outv[o] = fmaxf((conv[o] - m) * rsqrtf(var + kEps) * gw[o] + gb[o], 0.f);
  }
  __syncthreads();
  // the branch output of this sample as one S32 row (ch % 32 == 0; operand of the 1x1 conv that follows); the broadcast
  // over the X*Y rows of the concat buffer is done by gap_broadcast_kernel with a full grid (words copied verbatim)
  for (int t = threadIdx.x; t < ch / 2; t += blockDim.x) {
    uint32_t hi, lo;
    split_pair(outv[2 * t], outv[2 * t + 1], hi, lo);
    uint32_t* chunk = reinterpret_cast<uint32_t*>(sums_out + (size_t)b * ch + ((2 * t) & ~31));
    chunk[t & 15] = hi;
    chunk[16 + (t & 15)] = lo;
  }
}

__global__ void __launch_bounds__(256)
gap_broadcast_kernel(const float* __restrict__ vals /*(B, ch)*/, float* __restrict__ cat, long long rows,
                     int rows_per_batch, int ch, int ldo, int out_off) {
  const int ch4 = ch >> 2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * ch4) return;
  const long long r = i / ch4;
  const int c0 = (int)(i % ch4) * 4;
  const int b = (int)(r / rows_per_batch);
  *reinterpret_cast<float4*>(cat + r * ldo + out_off + c0) = *reinterpret_cast<const float4*>(vals + (size_t)b * ch + c0);
}

// DepthNet's ASPP image-pooling branch (ViewTransformerLSSBEVDepth.py:368-373,388-392): GAP -> 1x1 conv with the eval
// BatchNorm folded into (w, b) -> ReLU -> broadcast.  Both reductions run in a fixed order (no atomics), so the branch is
// bit-reproducible, as every other DepthNet launch.
// Column means: grid (images, ch / 32), CTA = 8 row lanes x 32 columns; lane l sums rows l, l + 8, ... in order, the
// eight partial sums are added in lane order.
__global__ void __launch_bounds__(256)
gap_mean_kernel(const float* __restrict__ in, float* __restrict__ mean, int rows_per_batch, int ch) {
  __shared__ float part[8][33];
  const int img = blockIdx.x, c = blockIdx.y * 32 + (threadIdx.x & 31), rl = threadIdx.x >> 5;
  const float* base = in + (size_t)img * rows_per_batch * ch + c;
  float a = 0.f;
  for (int r = rl; r < rows_per_batch; r += 8) a += __ldg(base + (size_t)r * ch);
  part[rl][threadIdx.x & 31] = a;
  __syncthreads();
  if (threadIdx.x < 32) {
    float s = 0.f;
#pragma unroll
    for (int l = 0; l < 8; ++l) s += part[l][threadIdx.x];
    mean[(size_t)img * ch + c] = s / (float)rows_per_batch;
  }
}

// 1x1 conv + ReLU of the means, one S32 row per image: grid (images, ch / 32), CTA = one 32-channel output chunk, warp w
// = outputs 4w .. 4w + 3 of it (lanes stride over the input channels: coalesced weight rows).
__global__ void __launch_bounds__(256)
gap_fc_relu_kernel(const float* __restrict__ mean, const float* __restrict__ w, const float* __restrict__ b,
                   float* __restrict__ vals /*(images, ch) S32*/, int ch) {
  __shared__ float o32[32];
  const int img = blockIdx.x, chunk = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* m = mean + (size_t)img * ch;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int o = chunk * 32 + warp * 4 + j;
    float a = 0.f;
    for (int i = lane; i < ch; i += 32) a = fmaf(__ldg(w + (size_t)o * ch + i), __ldg(m + i), a);
    a = warp_sum(a);
    if (lane == 0) o32[warp * 4 + j] = fmaxf(a + b[o], 0.f);
  }
  __syncthreads();
  if (threadIdx.x < 16) {
    uint32_t hi, lo;
    split_pair(o32[2 * threadIdx.x], o32[2 * threadIdx.x + 1], hi, lo);
    uint32_t* dst = reinterpret_cast<uint32_t*>(vals + (size_t)img * ch + chunk * 32);
    dst[threadIdx.x] = hi;
    dst[16 + threadIdx.x] = lo;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Dual-path fusion (dualpath_block.py:79-82):
//   coeff = sigmoid(<x, w> + bias);  out = x + coeff * x_bev[col] + identity
// identity = block input (stride 1) or GroupNorm(downsample conv raw output) (stride 2; :36-41).
// R consecutive rows per warp: the x, identity and bev loads of all R rows are issued before the first reduction; MB =
// minimum resident CTAs per SM the register allocation is held to.
template <int NV, int R, int MB = 1>
__global__ void __launch_bounds__(256, MB)
fuse_kernel(const float* __restrict__ x, const float* __restrict__ bev, const float* __restrict__ cw, float cbias,
            const float* __restrict__ identity, int identity_split, const double* __restrict__ id_stats,
            const float* __restrict__ id_w, const float* __restrict__ id_b, int groups, float* __restrict__ out,
            float* __restrict__ out_split, long long rows, int Z, long long rows_per_batch, int C) {
  const int lane = threadIdx.x & 31;
  const long long row0 = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * R;
  if (row0 >= rows) return;
  float4 xv[R][NV], idv[R][NV], bv[R][NV];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const long long row = row0 + r < rows ? row0 + r : rows - 1;  // tail rows are loaded twice, stored once
    const long long col = (int)row / Z;  // 32-bit division (rows < 2^31, checked by the launcher): a 64-bit one is ~100 instructions
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c0 = (i * 32 + lane) * 4;
      xv[r][i] = __ldcs(reinterpret_cast<const float4*>(x + row * C + c0));
      idv[r][i] = identity_split ? load_split4(identity + row * C, c0)
                                 : __ldcs(reinterpret_cast<const float4*>(identity + row * C + c0));
      bv[r][i] = __ldg(reinterpret_cast<const float4*>(bev + col * C + c0));
    }
  }
  const int cpg = C / groups;
  const double count = (double)rows_per_batch * cpg;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const long long row = row0 + r;
    if (row >= rows) break;
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float4 w = *reinterpret_cast<const float4*>(cw + (i * 32 + lane) * 4);
      dot += xv[r][i].x * w.x + xv[r][i].y * w.y + xv[r][i].z * w.z + xv[r][i].w * w.w;
    }
    dot = warp_sum(dot) + cbias;
    const float coeff = 1.0f / (1.0f + expf(-dot));
    const int bidx = (int)row / (int)rows_per_batch;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c0 = (i * 32 + lane) * 4;
      float4 iv = idv[r][i];
      if (id_stats) {
        float mean, rstd;
        gn_mean_rstd(id_stats, bidx, groups, c0 / cpg, count, &mean, &rstd);
        const float4 g = *reinterpret_cast<const float4*>(id_w + c0);
        const float4 bb = *reinterpret_cast<const float4*>(id_b + c0);
        iv.x = (iv.x - mean) * rstd * g.x + bb.x;
        iv.y = (iv.y - mean) * rstd * g.y + bb.y;
        iv.z = (iv.z - mean) * rstd * g.z + bb.z;
        iv.w = (iv.w - mean) * rstd * g.w + bb.w;
      }
      float4 o;
      o.x = xv[r][i].x + coeff * bv[r][i].x + iv.x;
      o.y = xv[r][i].y + coeff * bv[r][i].y + iv.y;
      o.z = xv[r][i].z + coeff * bv[r][i].z + iv.z;
      o.w = xv[r][i].w + coeff * bv[r][i].w + iv.w;
      if (out) *reinterpret_cast<float4*>(out + row * C + c0) = o;
      if (out_split) store_split4(out_split + row * C, c0, o);
    }
  }
}

// fp32 rows -> S32 split rows (C % 32 == 0); for the few operands that are produced in fp32 by a kernel whose other
// consumers need fp32 (BEV tokens entering the ASPP branch, user-supplied module inputs)
__global__ void __launch_bounds__(256)
split_rows_kernel(const float* __restrict__ in, float* __restrict__ out, long long n4, int C) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 >= n4) return;
  const int C4 = C >> 2;
  const long long row = i4 < (1ll << 31) ? (long long)((int)i4 / C4) : i4 / C4;
  const int c0 = (int)(i4 - row * C4) * 4;
  store_split4(out + row * C, c0, __ldg(reinterpret_cast<const float4*>(in + row * C + c0)));
}
__global__ void __launch_bounds__(256)
unsplit_rows_kernel(const float* __restrict__ in, float* __restrict__ out, long long n4, int C) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 >= n4) return;
  const int C4 = C >> 2;
  const long long row = i4 / C4;
  const int c0 = (int)(i4 % C4) * 4;
  *reinterpret_cast<float4*>(out + row * C + c0) = load_split4(in + row * C, c0);
}

}  // namespace occ

using namespace occ;

#define DISPATCH_NV(C, CALL)                     \
  switch ((C) / 128) {                           \
    case 1: { constexpr int NV = 1; CALL; } break; \
    case 2: { constexpr int NV = 2; CALL; } break; \
    case 4: { constexpr int NV = 4; CALL; } break; \
    case 8: { constexpr int NV = 8; CALL; } break; \
    default: return OCC_EUNSUPPORTED;            \
  }

// Static shared memory of gn_relu_zmean_ln_kernel (s_mean, s_rstd).  Without an opt-in, static + dynamic shared memory
// must stay within 48 KiB, so a Z-column buffer above 44 KiB (C = 1024 at Z = 6 or 12) needs the attribute raised.
constexpr size_t kZmeanStaticSmem = 2 * 16 * 32 * sizeof(float);

template <int NV, int R, typename... Args>
static int launch_gn_relu_zmean_ln(int blocks, int threads, size_t smem, cudaStream_t stream, Args... args) {
  auto* kernel = gn_relu_zmean_ln_kernel<NV, R>;
  if (smem + kZmeanStaticSmem > 48 * 1024) OCC_ENSURE_SMEM(kernel, smem);
  kernel<<<blocks, threads, smem, stream>>>(args...);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_gn_relu_zmean_ln(const float* y, const double* stats, const float* gn_w, const float* gn_b,
                                    const float* ln_w, const float* ln_b, float* tok, float* tokn, int B, int XY,
                                    int Z, int C, int groups, int X, int win_shift, cudaStream_t stream) {
  OCC_REQUIRE(y && stats && gn_w && gn_b && ln_w && ln_b && tok && tokn);
  // win_shift < 0: tokn in token order (rows as tok); 0 / 1: tokn in the window layout of the un-shifted / shifted
  // partition (occ_swin_qkv_attention's operand; the buffer must be zero where no token lands: occ_window_layout_rows)
  OCC_REQUIRE(win_shift < 0 || (X > 0 && XY % X == 0));
  OCC_REQUIRE((long long)B * XY < (1ll << 31));
  const WinGeom wg = make_win_geom(B, win_shift < 0 ? 1 : X, win_shift < 0 ? XY : XY / X, Z, C, C / HD, win_shift > 0);
  const int wl = win_shift >= 0;
  OCC_REQUIRE(B > 0 && XY > 0 && Z > 0 && Z <= 16 && C % 128 == 0 && groups > 0 && groups <= 32 && C % groups == 0 &&
              (C / groups) % 4 == 0);
  // rows per warp: 4 for the narrow (C = 128) stage when Z allows it, else 1; 16 warps per CTA where possible
  const int R = (C == 128 && Z % 4 == 0) ? 4 : 1;
  const int wpc = Z / R;
  int cols = 16 / wpc;
  if (cols < 1) cols = 1;
  if (cols > 16) cols = 16;
  while ((size_t)cols * Z * C * 4 > 48 * 1024 && cols > 1) cols >>= 1;
  const size_t smem = (size_t)cols * Z * C * 4;
  OCC_REQUIRE(smem <= 48 * 1024);
  const long long ncols = (long long)B * XY;
  const int blocks = (int)((ncols + cols - 1) / cols);
  const int threads = cols * wpc * 32;
  OCC_REQUIRE(threads <= 512);
  if (R == 4)
    return launch_gn_relu_zmean_ln<1, 4>(blocks, threads, smem, stream, y, stats, gn_w, gn_b, ln_w, ln_b, tok, tokn, B, XY,
                                         Z, C, groups, cols, wg, wl);
  int rc = OCC_OK;
  DISPATCH_NV(C, (rc = launch_gn_relu_zmean_ln<NV, 1>(blocks, threads, smem, stream, y, stats, gn_w, gn_b, ln_w, ln_b, tok,
                                                      tokn, B, XY, Z, C, groups, cols, wg, wl)));
  return rc;
}

extern "C" int occ_layernorm(const float* in, const float* w, const float* b, float* out, long long rows, int C,
                             int split_out, cudaStream_t stream) {
  OCC_REQUIRE(in && w && b && out && rows > 0 && C > 0);
  OCC_REQUIRE(!split_out || C % 32 == 0);
  const int blocks = (int)((rows + 7) / 8);
  if (C % 128 == 0 && (C / 128 == 1 || C / 128 == 2 || C / 128 == 4 || C / 128 == 8)) {
    DISPATCH_NV(C, (layernorm_kernel<NV><<<blocks, 256, 0, stream>>>(in, w, b, out, rows, C, split_out)));
  } else {
    layernorm_generic_kernel<<<blocks, 256, 0, stream>>>(in, w, b, out, rows, C, split_out);
  }
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_gn_apply(const float* in, const double* stats, const float* w, const float* b,
                            const float* residual, float* out, float* out_split, long long rows, int rows_per_batch,
                            int C, int groups, int ldo, int out_off, int relu, cudaStream_t stream) {
  OCC_REQUIRE(in && stats && w && b && (out || out_split) && rows > 0 && rows_per_batch > 0 && rows % rows_per_batch == 0);
  OCC_REQUIRE(C % 4 == 0 && groups > 0 && C % groups == 0);
  if (out_split) OCC_REQUIRE(C % 32 == 0 && ldo % 32 == 0 && out_off % 32 == 0 && out_off + C <= ldo);
  OCC_REQUIRE(C <= 4096 && rows / rows_per_batch <= 65535);
  const int B = (int)(rows / rows_per_batch);
  // rows per CTA: k * GA_UNROLL rows per thread and column pass, k in 1..8 chosen for >= ~4 waves of 3 CTAs per SM
  // (the fp64 scale / shift prologue is per CTA: big tensors amortise it over more rows)
  const int cols = C / 4 < 256 ? C / 4 : 256;
  const int unit = (256 / cols) * GA_UNROLL;
  long long k = rows / ((long long)unit * 12 * sm_count());
  k = k < 1 ? 1 : (k > 8 ? 8 : k);
  int rpc = unit * (int)k;
  dim3 grid((rows_per_batch + rpc - 1) / rpc, B);
  gn_apply_kernel<<<grid, 256, 2 * C * sizeof(float), stream>>>(in, stats, w, b, residual, out, out_split, rows_per_batch, C,
                                                                groups, ldo, out_off, relu, rpc);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_aspp_gap_branch(const float* in, double* sums_ws, const float* wconv, const float* gw,
                                   const float* gb, float* cat, int B, int rows_per_batch, int ch, int groups, int ldo,
                                   int out_off, cudaStream_t stream) {
  OCC_REQUIRE(in && sums_ws && wconv && gw && gb && cat);
  OCC_REQUIRE(B > 0 && B <= 65535 && rows_per_batch > 0 && ch % 32 == 0 && ch <= 1024 && groups > 0 && ch % groups == 0 &&
              256 % (ch / 4) == 0);  // B is the colsum grid's y
  OCC_REQUIRE(ldo % 32 == 0 && out_off % 32 == 0 && out_off + ch <= ldo);  // a slice of the S32 concat buffer
  OCC_MEMSET(sums_ws, 0, (size_t)B * ch * sizeof(double), stream);
  const int chunk = 256;
  dim3 grid((rows_per_batch + chunk - 1) / chunk, B);
  colsum_kernel<<<grid, 256, 0, stream>>>(in, sums_ws, rows_per_batch, ch, chunk);
  OCC_LAUNCH_CHECK();
  // sums_ws holds B*ch doubles; the fp32 branch values are written behind them (caller allocates B*ch*12 bytes)
  float* vals = reinterpret_cast<float*>(sums_ws + (size_t)B * ch);
  aspp_gap_branch_kernel<<<B, 256, 3 * ch * sizeof(float), stream>>>(sums_ws, wconv, gw, gb, vals, rows_per_batch, ch,
                                                                    groups);
  OCC_LAUNCH_CHECK();
  const long long n4 = (long long)B * rows_per_batch * (ch / 4);
  gap_broadcast_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(vals, cat, (long long)B * rows_per_batch,
                                                                        rows_per_batch, ch, ldo, out_off);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_depthnet_gap_branch(const float* in, float* ws, const float* w, const float* b, float* cat, int B,
                                       int rows_per_batch, int ch, int ldo, int out_off, cudaStream_t stream) {
  OCC_REQUIRE(in && ws && w && b && cat);
  OCC_REQUIRE(B > 0 && B <= 65535 && rows_per_batch > 0 && ch % 32 == 0 && ch <= 1024);
  OCC_REQUIRE(ldo % 32 == 0 && out_off % 32 == 0 && out_off + ch <= ldo);  // a slice of the S32 concat buffer
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 15) == 0 && (reinterpret_cast<uintptr_t>(cat) & 15) == 0);
  float* mean = ws;                      // (B, ch) fp32
  float* vals = ws + (size_t)B * ch;     // (B, ch) S32
  gap_mean_kernel<<<dim3(B, ch / 32), 256, 0, stream>>>(in, mean, rows_per_batch, ch);
  OCC_LAUNCH_CHECK();
  gap_fc_relu_kernel<<<dim3(B, ch / 32), 256, 0, stream>>>(mean, w, b, vals, ch);
  OCC_LAUNCH_CHECK();
  const long long n4 = (long long)B * rows_per_batch * (ch / 4);
  gap_broadcast_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(vals, cat, (long long)B * rows_per_batch,
                                                                        rows_per_batch, ch, ldo, out_off);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_dualpath_fuse(const float* x, const float* bev, const float* cw, float cbias, const float* identity,
                                 int identity_split, const double* id_stats, const float* id_w, const float* id_b,
                                 int groups, float* out, float* out_split, int B, int XY, int Z, int C,
                                 cudaStream_t stream) {
  OCC_REQUIRE(x && bev && cw && identity && (out || out_split) && B > 0 && XY > 0 && Z > 0 && C % 128 == 0);
  if (id_stats) OCC_REQUIRE(id_w && id_b && groups > 0 && C % groups == 0 && (C / groups) % 4 == 0);
  const long long rows = (long long)B * XY * Z;
  OCC_REQUIRE(rows < (1ll << 31));
#define FUSE_LAUNCH(NV_, R_, MB_)                                                                                       \
  do {                                                                                                                  \
    const int blocks = (int)((rows + 8 * (R_) - 1) / (8 * (R_)));                                                       \
    fuse_kernel<NV_, R_, MB_><<<blocks, 256, 0, stream>>>(x, bev, cw, cbias, identity, identity_split, id_stats, id_w,  \
                                                          id_b, groups > 0 ? groups : 1, out, out_split, rows, Z,       \
                                                          (long long)XY * Z, C);                                        \
  } while (0)
  if (C == 128) {
    // two rows per warp at <= 40 registers, six resident CTAs per SM rather than four rows per warp at ~110 registers
    // (two resident CTAs): resident warps, not loads per warp, are what keeps HBM busy here
    FUSE_LAUNCH(1, 2, 6);
  } else if (C == 256) {
    FUSE_LAUNCH(2, 2, 1);
  } else if (C == 512) {
    FUSE_LAUNCH(4, 1, 1);
  } else if (C == 1024) {
    FUSE_LAUNCH(8, 1, 1);
  } else {
    return OCC_EUNSUPPORTED;
  }
#undef FUSE_LAUNCH
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// fp32 (rows, C) <-> S32 split format (C % 32 == 0)
extern "C" int occ_split_rows(const float* in, float* out, long long rows, int C, cudaStream_t stream) {
  OCC_REQUIRE(in && out && rows > 0 && C > 0 && C % 32 == 0);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0);
  const long long n4 = rows * (C / 4);
  split_rows_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(in, out, n4, C);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
extern "C" int occ_unsplit_rows(const float* in, float* out, long long rows, int C, cudaStream_t stream) {
  OCC_REQUIRE(in && out && rows > 0 && C > 0 && C % 32 == 0);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0);
  const long long n4 = rows * (C / 4);
  unsplit_rows_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(in, out, n4, C);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// Rows of the window-layout token buffer for a (B, X, Y, Z) grid: one 128-row tile per pair of 7x7 windows over the
// B * (Z + 1) X-Y images (voxel slices, then the BEV image).  The buffer must be zero-initialised once: window pad
// positions and rows 49..63 of every window are never written.
extern "C" long long occ_window_layout_rows(int B, int X, int Y, int Z) {
  if (B <= 0 || X <= 0 || Y <= 0 || Z <= 0) return -1;
  const WinGeom g = make_win_geom(B, X, Y, Z, 128, 4, 0);
  return (g.nwin + 1) / 2 * 128;
}
