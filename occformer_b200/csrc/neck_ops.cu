// MSDeformAttnPixelDecoder3D (the neck between the dual-path encoder and the Mask2Former-3D head; SURVEY.md 8(f)1):
// the kernels that are not GEMMs / convolutions.
//
//   projects/mmdet3d_plugin/occformer/necks/multiscale_deformattn_3d.py:143-248   (MSDeformAttnPixelDecoder3D.forward)
//   projects/mmdet3d_plugin/occformer/necks/multi_scale_deform_attn_3d.py:17-80   (multi_scale_deformable_attn_pytorch)
//                                                                     :185-286  (MultiScaleDeformableAttention3D.forward)
//
// Token layout ("level-major"): the Nq = sum_l X_l*Y_l*Z_l query / value tokens of the B samples are stored level by
// level, row(l, b, x, y, z) = B*start_l + b*n_l + (x*Y_l + y)*Z_l + z, C channels per row (channel-last).  Every level is
// then one contiguous (B, X_l, Y_l, Z_l, C) channel-last tensor: the 1x1x1 input convolutions write their level in place,
// and the encoder output of a level is handed to the FPN / the head without a copy.  (The reference concatenates the
// levels per sample, (Nq, B, C); only the row order differs -- every op of the encoder is per token except the
// deformable gather, which addresses (level, sample, voxel) explicitly.)
#include "occ_common.cuh"
#include "occ_ptx.cuh"
#include "neck_levels.cuh"

namespace occ {

__device__ __forceinline__ float nk_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------------------
// Token preparation: [LayerNorm] of a row, written as up to three tensors
//   out_f32  : x            fp32   (residual of the next sub-layer)
//   out_s32  : x            S32    (operand of value_proj / of the FFN)
//   out_pos  : x + pos[row] S32    (operand of the sampling_offsets | attention_weights projection; pos = sine
//                                   positional encoding + level embedding of the token, a per-grid constant (Nq, C))
// One warp per row, C % 32 == 0, C <= 1024; lane owns element `lane` of every 32-column chunk (coalesced 128-byte loads,
// lanes (2t, 2t+1) form packed word t of a chunk for the S32 stores).
template <int NCH>
__global__ void __launch_bounds__(256)
token_prep_kernel(const float* __restrict__ in, const float* __restrict__ ln_w, const float* __restrict__ ln_b,
                  const float* __restrict__ pos, float* __restrict__ out_f32, float* __restrict__ out_s32,
                  float* __restrict__ out_pos, const NeckLevels g, int C) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= g.rows) return;
  float v[NCH];
#pragma unroll
  for (int c = 0; c < NCH; ++c) v[c] = __ldcs(in + row * C + c * 32 + lane);
  if (ln_w) {
    // two-pass on the row shifted by its first element (lane 0's element 0): for a row whose offset dwarfs its spread
    // the shifted values are exact and small, so the fp32 sums lose no digits to the offset
    const float shift = __shfl_sync(0xffffffffu, v[0], 0);
#pragma unroll
    for (int c = 0; c < NCH; ++c) v[c] -= shift;
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) s += v[c];
    const float mean = nk_warp_sum(s) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int c = 0; c < NCH; ++c) { const float d = v[c] - mean; q += d * d; }
    const float rstd = rsqrtf(nk_warp_sum(q) / (float)C + 1e-5f);
#pragma unroll
    for (int c = 0; c < NCH; ++c) v[c] = (v[c] - mean) * rstd * __ldg(ln_w + c * 32 + lane) + __ldg(ln_b + c * 32 + lane);
  }
  long long prow = 0;
  if (out_pos) {
    int lvl, b, local;
    nk_locate(g, row, lvl, b, local);
    prow = (long long)g.start[lvl] + local;
  }
#pragma unroll
  for (int c = 0; c < NCH; ++c) {
    const float x = v[c];
    if (out_f32) out_f32[row * C + c * 32 + lane] = x;
    const float xp = out_pos ? x + __ldg(pos + prow * C + c * 32 + lane) : 0.f;
    const float x2 = __shfl_xor_sync(0xffffffffu, x, 1), xp2 = __shfl_xor_sync(0xffffffffu, xp, 1);
    if (!(lane & 1)) {
      uint32_t hi, lo;
      if (out_s32) {
        split_pair(x, x2, hi, lo);
        uint32_t* chunk = reinterpret_cast<uint32_t*>(out_s32 + row * C + c * 32);
        chunk[lane >> 1] = hi;
        chunk[16 + (lane >> 1)] = lo;
      }
      if (out_pos) {
        split_pair(xp, xp2, hi, lo);
        uint32_t* chunk = reinterpret_cast<uint32_t*>(out_pos + row * C + c * 32);
        chunk[lane >> 1] = hi;
        chunk[16 + (lane >> 1)] = lo;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Multi-scale deformable attention core, 3-D (multi_scale_deform_attn_3d.py:17-80 + the location arithmetic of :258-272).
//   value (rows, value_ld)     value_proj output, level-major, head h = channels [h*head_ld, h*head_ld + hd): with
//                              head_ld = hd rounded up to 32 floats a head slice is one 128-byte line (the kernel is
//                              bound by the L1 data stage -- LSU wavefronts near peak: a 16-byte load per thread
//                              moves 64 bytes per cycle whatever the alignment)
//   ow    (rows, H*L*P*4)      [ sampling_offsets (h, l, p, 3: z, y, x) | attention logits (h, l, p) ] of the same token
//   out   (rows, E)  S32       sum_{l,p} softmax(logits)[l,p] * trilinear(value level l)(loc), zeros outside,
//                              align_corners=False;  loc = ref + offset / (Z_l, Y_l, X_l),  ref = voxel centre of the
//                              query in its own level, normalised to [0,1] (the same point for every value level)
// One CTA = (patch of NK_PX x NK_PY x Z_l queries of one level, one head), NK_QP queries per pass.  A CTA's value working
// set is then the patch plus the halo its sampling offsets reach, in ONE head's slices (~70 KB at a 2-voxel halo): it
// lives in L1 and L2 / HBM see each slice about once per patch instead of the ~30 times it is sampled.
// A pass has three phases so that the scalar work is done once per sample instead of once per gather thread:
//   0: one thread per query        : softmax of the head's L*P logits                      -> s_w
//   1: one thread per (query, l, p): sampling location -> 8 (value row, softmax * trilinear weight) taps -> s_tap
//   2: hd/4 threads per query      : acc += weight * value[row] over the L*P*8 taps (16-byte loads, 8 in flight)
// Out-of-volume corners keep weight 0 and point at row 0 (zeros padding of grid_sample).
constexpr int NK_QP = 32;
template <int L, int P>
__global__ void __launch_bounds__(256)
ms_deform_attn_kernel(const float* __restrict__ value, const float* __restrict__ ow, float* __restrict__ out,
                      const NeckLevels g, int E, int H, int value_ld, int head_ld) {
  constexpr int LP = L * P, NT = LP * 8, TSTR = NT + 1;  // +1: queries of a warp land in different banks
  extern __shared__ uint2 s_tap[];                       // [NK_QP][TSTR] (value row, weight bits), tap = corner * LP + i
  __shared__ float s_w[NK_QP][LP];
  __shared__ int s_dim[3][L];
  __shared__ long long s_row0[L];
  const int hd = E / H;
  const int T1 = hd >> 2;  // threads per (query, head)
  const int h = blockIdx.y;
  const int T = value_ld >> 2;  // float4 per value row
  // patch -> (level, sample, px, py)
  int lq = 0;
#pragma unroll
  for (int l = 1; l < NK_MAX_LEVELS; ++l)
    if (l < g.L && (int)blockIdx.x >= g.pstart[l]) lq = l;
  const int Zq = g.Z[lq], Yq = g.Y[lq], Xq = g.X[lq];
  int pid = blockIdx.x - g.pstart[lq];
  const int npy = (Yq + NK_PY - 1) / NK_PY, npx = (Xq + NK_PX - 1) / NK_PX;
  const int py = pid % npy; pid /= npy;
  const int px = pid % npx;
  const int b = pid / npx;
  const int nq = NK_PX * NK_PY * Zq;
  if (threadIdx.x < L) {
    const int l = threadIdx.x;
    s_dim[0][l] = g.X[l]; s_dim[1][l] = g.Y[l]; s_dim[2][l] = g.Z[l];
    s_row0[l] = (long long)g.B * g.start[l] + (long long)b * g.n[l];
  }
  const float st = g.stride[lq];
  const long long qrow0 = (long long)g.B * g.start[lq] + (long long)b * g.n[lq];
  // query q of the patch -> voxel (x, y, z); false when outside the volume
  auto locate = [&](int q, int& x, int& y, int& z) {
    z = q % Zq;
    const int iy = (q / Zq) % NK_PY, ix = q / (Zq * NK_PY);
    x = px * NK_PX + ix; y = py * NK_PY + iy;
    return q < nq && x < Xq && y < Yq;
  };
  const int gq = threadIdx.x / T1, gt = threadIdx.x - gq * T1;  // phase 2: query of the pass, float4 of the head slice
  const float4* vbase = reinterpret_cast<const float4*>(value) + h * (head_ld >> 2) + gt;
#pragma unroll 1
  for (int q0 = 0; q0 < nq; q0 += NK_QP) {
    __syncthreads();  // s_dim ready (first pass) / previous pass's taps consumed
    if (threadIdx.x < NK_QP) {
      int x, y, z;
      if (locate(q0 + threadIdx.x, x, y, z)) {
        const long long row = qrow0 + ((long long)x * Yq + y) * Zq + z;
        const float* logit = ow + row * (size_t)(H * LP * 4) + (size_t)H * LP * 3 + (size_t)h * LP;
        float w[LP];
        float m = -INFINITY;
#pragma unroll
        for (int i = 0; i < LP; ++i) { w[i] = __ldg(logit + i); m = fmaxf(m, w[i]); }
        float den = 0.f;
#pragma unroll
        for (int i = 0; i < LP; ++i) { w[i] = expf(w[i] - m); den += w[i]; }
        const float inv = 1.0f / den;
#pragma unroll
        for (int i = 0; i < LP; ++i) s_w[threadIdx.x][i] = w[i] * inv;
      }
    }
    __syncthreads();
    for (int task = threadIdx.x; task < NK_QP * LP; task += blockDim.x) {
      const int ql = task / LP, i = task - ql * LP, l = i / P;
      int x, y, z;
      if (!locate(q0 + ql, x, y, z)) continue;
      const long long row = qrow0 + ((long long)x * Yq + y) * Zq + z;
      const float* offs = ow + row * (size_t)(H * LP * 4) + (size_t)h * LP * 3 + 3 * i;
      const int Xl = s_dim[0][l], Yl = s_dim[1][l], Zl = s_dim[2][l];
      // reference point (normalised voxel centre), computed as the reference does: ((i + 0.5) * stride) / (dim * stride)
      const float rz = ((float)z + 0.5f) * st / ((float)Zq * st);
      const float ry = ((float)y + 0.5f) * st / ((float)Yq * st);
      const float rx = ((float)x + 0.5f) * st / ((float)Xq * st);
      // grid_sample(align_corners=False) un-normalisation, in torch's own form: ((g + 1) * size - 1) / 2 with g = 2 loc - 1
      const float lz = rz + __ldg(offs + 0) / (float)Zl;
      const float ly = ry + __ldg(offs + 1) / (float)Yl;
      const float lx = rx + __ldg(offs + 2) / (float)Xl;
      const float fz = (((2.0f * lz - 1.0f) + 1.0f) * (float)Zl - 1.0f) * 0.5f;
      const float fy = (((2.0f * ly - 1.0f) + 1.0f) * (float)Yl - 1.0f) * 0.5f;
      const float fx = (((2.0f * lx - 1.0f) + 1.0f) * (float)Xl - 1.0f) * 0.5f;
      const float z0f = floorf(fz), y0f = floorf(fy), x0f = floorf(fx);
      // (clamped before the int conversion: a wild offset must not overflow; anything outside is dropped below)
      const int z0 = (int)fminf(fmaxf(z0f, -2.f), (float)Zl), y0 = (int)fminf(fmaxf(y0f, -2.f), (float)Yl),
                x0 = (int)fminf(fmaxf(x0f, -2.f), (float)Xl);
      const float tz = fz - z0f, ty = fy - y0f, tx = fx - x0f;
      const float wa = s_w[ql][i];
      const long long lrow0 = s_row0[l];
      uint2* tp = s_tap + ql * TSTR + i;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int dz = k & 1, dy = (k >> 1) & 1, dx = k >> 2;
        const int zz = z0 + dz, yy = y0 + dy, xx = x0 + dx;
        const bool ok = zz >= 0 && zz < Zl && yy >= 0 && yy < Yl && xx >= 0 && xx < Xl;
        const float cw = (dz ? tz : 1.f - tz) * (dy ? ty : 1.f - ty) * (dx ? tx : 1.f - tx);
        uint2 e;
        e.x = ok ? (uint32_t)(lrow0 + ((long long)xx * Yl + yy) * Zl + zz) : 0u;
        e.y = ok ? __float_as_uint(wa * cw) : 0u;
        tp[k * LP] = e;
      }
    }
    __syncthreads();
    {
      int x, y, z;
      if (gq < NK_QP && locate(q0 + gq, x, y, z)) {
        const uint2* tp = s_tap + gq * TSTR;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 2
        for (int s0 = 0; s0 < NT; s0 += 8) {
          uint2 e[8];
          float4 c[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) e[k] = tp[s0 + k];
#pragma unroll
          for (int k = 0; k < 8; ++k) c[k] = __ldg(vbase + (size_t)e[k].x * T);
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const float w = __uint_as_float(e[k].y);
            acc.x = fmaf(w, c[k].x, acc.x); acc.y = fmaf(w, c[k].y, acc.y);
            acc.z = fmaf(w, c[k].z, acc.z); acc.w = fmaf(w, c[k].w, acc.w);
          }
        }
        const long long row = qrow0 + ((long long)x * Yq + y) * Zq + z;
        store_split4(out + row * E, 4 * (h * T1 + gt), acc);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// FPN step (multiscale_deformattn_3d.py:228-240): y = GroupNorm(lateral conv raw output) + trilinear upsample
// (align_corners=False) of the coarser level; written in S32 (operand of the 3x3x3 output conv).
//   cur (B, X, Y, Z, C) raw lateral conv output + its GN statistics;  coarse (B, Xc, Yc, Zc, C) fp32.
// grid (voxel chunks, B); per-channel GroupNorm scale / shift of the sample in shared memory.
__global__ void __launch_bounds__(256)
gn_upsample_add_kernel(const float* __restrict__ cur, const double* __restrict__ stats, const float* __restrict__ gw,
                       const float* __restrict__ gb, int groups, const float* __restrict__ coarse, float* __restrict__ out_s,
                       int X, int Y, int Z, int Xc, int Yc, int Zc, int C, int vox_per_cta) {
  extern __shared__ float gsm[];  // scale[C], shift[C]
  float* sc = gsm;
  float* sh = gsm + C;
  const int b = blockIdx.y;
  const long long V = (long long)X * Y * Z;
  {
    const int cpg = C / groups;
    const double count = (double)V * cpg;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const int gi = c / cpg;
      const double s = stats[((size_t)b * groups + gi) * 2], q = stats[((size_t)b * groups + gi) * 2 + 1];
      const double mean = s / count;
      double var = q / count - mean * mean;
      if (var < 0.0) var = 0.0;
      const float a = (float)(1.0 / sqrt(var + 1e-5)) * gw[c];
      sc[c] = a;
      sh[c] = gb[c] - (float)mean * a;
    }
  }
  __syncthreads();
  const int C4 = C >> 2;
  const long long v0 = (long long)blockIdx.x * vox_per_cta;
  const long long v1 = v0 + vox_per_cta < V ? v0 + vox_per_cta : V;
  // F.interpolate(trilinear, align_corners=False): src = (dst + 0.5) * (in / out) - 0.5, clamped at 0; the upper
  // neighbour index is clamped to the last element (its weight is then irrelevant: both neighbours coincide)
  auto axis = [](int d, int n_out, int n_in, int& i0, int& i1, float& t) {
    float s = ((float)d + 0.5f) * ((float)n_in / (float)n_out) - 0.5f;
    if (s < 0.f) s = 0.f;
    i0 = (int)s;
    if (i0 > n_in - 1) i0 = n_in - 1;
    i1 = i0 + 1 < n_in ? i0 + 1 : n_in - 1;
    t = s - (float)i0;
  };
  const float4* cb = reinterpret_cast<const float4*>(coarse + (size_t)b * Xc * Yc * Zc * C);
  // a thread owns one float4 column (scale / shift in registers) and walks voxels: 32-bit index arithmetic per voxel,
  // 9 independent 16-byte loads in flight
  const int cols = C4 < 256 ? C4 : 256, rstep = 256 / cols;
  const int rl = threadIdx.x / cols, cl = threadIdx.x - rl * cols;
  if (rl >= rstep) return;
  for (int c4 = cl; c4 < C4; c4 += cols) {
    const float4 a = *reinterpret_cast<const float4*>(sc + 4 * c4), d = *reinterpret_cast<const float4*>(sh + 4 * c4);
#pragma unroll 2
    for (int r = (int)v0 + rl; r < (int)v1; r += rstep) {
      const int z = r % Z, t2 = r / Z;
      const int y = t2 % Y, x = t2 / Y;
      const long long row = (long long)b * V + r;
      const float4 raw = __ldcs(reinterpret_cast<const float4*>(cur + row * C) + c4);
      float4 o = make_float4(fmaf(raw.x, a.x, d.x), fmaf(raw.y, a.y, d.y), fmaf(raw.z, a.z, d.z), fmaf(raw.w, a.w, d.w));
      int x0, x1, y0, y1, z0, z1;
      float tx, ty, tz;
      axis(x, X, Xc, x0, x1, tx);
      axis(y, Y, Yc, y0, y1, ty);
      axis(z, Z, Zc, z0, z1, tz);
      float4 cv[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int dz = k & 1, dy = (k >> 1) & 1, dx = k >> 2;
        cv[k] = __ldg(cb + (((size_t)(dx ? x1 : x0) * Yc + (dy ? y1 : y0)) * Zc + (dz ? z1 : z0)) * C4 + c4);
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int dz = k & 1, dy = (k >> 1) & 1, dx = k >> 2;
        const float wgt = (dx ? tx : 1.f - tx) * (dy ? ty : 1.f - ty) * (dz ? tz : 1.f - tz);
        o.x = fmaf(wgt, cv[k].x, o.x); o.y = fmaf(wgt, cv[k].y, o.y);
        o.z = fmaf(wgt, cv[k].z, o.z); o.w = fmaf(wgt, cv[k].w, o.w);
      }
      store_split4(out_s + row * C, 4 * c4, o);
    }
  }
}

// The same step for exact x2 up-sampling (X = 2 Xc ...), one CTA per (UA_BX x UA_BY x UA_BZ box of fine voxels, 32-channel
// chunk): the box's coarse neighbourhood (<= 6 x 6 x 10 rows of 128 bytes) is staged in shared memory once, so the
// 8 corner reads of a voxel are shared-memory reads -- the first version fetched them from L2 (8 x 16 bytes per 16 bytes
// of input: L2 bandwidth was the kernel's bound).  Arithmetic identical to the kernel
// above (same `axis` expression, same FMA order).
constexpr int UA_BX = 8, UA_BY = 8, UA_BZ = 16;
constexpr int UA_CX = UA_BX / 2 + 2, UA_CY = UA_BY / 2 + 2, UA_CZ = UA_BZ / 2 + 2;
__global__ void __launch_bounds__(256)
gn_upsample_add_x2_kernel(const float* __restrict__ cur, const double* __restrict__ stats, const float* __restrict__ gw,
                          const float* __restrict__ gb, int groups, const float* __restrict__ coarse,
                          float* __restrict__ out_s, int X, int Y, int Z, int Xc, int Yc, int Zc, int C) {
  __shared__ float4 tile[UA_CX * UA_CY * UA_CZ * 8];  // [cx][cy][cz][8 float4 of the 32-channel chunk]
  __shared__ float sc[32], sh[32];
  const int chunk = blockIdx.y, b = blockIdx.z;
  const int nbz = (Z + UA_BZ - 1) / UA_BZ, nby = (Y + UA_BY - 1) / UA_BY;
  int box = blockIdx.x;
  const int bz = box % nbz; box /= nbz;
  const int by = box % nby;
  const int bx = box / nby;
  const int x0 = bx * UA_BX, y0 = by * UA_BY, z0 = bz * UA_BZ;
  const long long V = (long long)X * Y * Z;
  if (threadIdx.x < 32) {
    const int c = chunk * 32 + threadIdx.x;
    const int cpg = C / groups, gi = c / cpg;
    const double count = (double)V * cpg;
    const double s = stats[((size_t)b * groups + gi) * 2], q = stats[((size_t)b * groups + gi) * 2 + 1];
    const double mean = s / count;
    double var = q / count - mean * mean;
    if (var < 0.0) var = 0.0;
    const float a = (float)(1.0 / sqrt(var + 1e-5)) * gw[c];
    sc[threadIdx.x] = a;
    sh[threadIdx.x] = gb[c] - (float)mean * a;
  }
  auto axis = [](int d, int n_out, int n_in, int& i0, int& i1, float& t) {
    float s = ((float)d + 0.5f) * ((float)n_in / (float)n_out) - 0.5f;
    if (s < 0.f) s = 0.f;
    i0 = (int)s;
    if (i0 > n_in - 1) i0 = n_in - 1;
    i1 = i0 + 1 < n_in ? i0 + 1 : n_in - 1;
    t = s - (float)i0;
  };
  // coarse origin of the box: the lower neighbour of its first voxel on every axis
  int cx0, cy0, cz0;
  {
    int i1;
    float t;
    axis(x0, X, Xc, cx0, i1, t);
    axis(y0, Y, Yc, cy0, i1, t);
    axis(z0, Z, Zc, cz0, i1, t);
  }
  const float4* cb = reinterpret_cast<const float4*>(coarse + (size_t)b * Xc * Yc * Zc * C) + chunk * 8;
  const int C4 = C >> 2;
  for (int i = threadIdx.x; i < UA_CX * UA_CY * UA_CZ * 8; i += 256) {
    const int l8 = i & 7, r = i >> 3;
    const int cz = r % UA_CZ, cy = (r / UA_CZ) % UA_CY, cx = r / (UA_CZ * UA_CY);
    const int gx = cx0 + cx, gy = cy0 + cy, gz = cz0 + cz;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gx < Xc && gy < Yc && gz < Zc) v = __ldg(cb + (((size_t)gx * Yc + gy) * Zc + gz) * C4 + l8);
    tile[i] = v;
  }
  __syncthreads();
  // thread = (float4 l8 of the chunk, dz, dy parity): the z-axis terms are per-thread constants, the y-axis terms live in
  // registers for the thread's four dy values, the x-axis terms are computed once per dx
  const int l8 = threadIdx.x & 7;
  const int dz = (threadIdx.x >> 3) & (UA_BZ - 1), yofs = threadIdx.x >> 7;
  static_assert(UA_BZ == 16 && UA_BY == 8, "thread mapping");
  const float4 a = *reinterpret_cast<const float4*>(sc + 4 * l8), d = *reinterpret_cast<const float4*>(sh + 4 * l8);
  const int z = z0 + dz;
  if (z >= Z) return;
  int za, zb;
  float tz;
  axis(z, Z, Zc, za, zb, tz);
  const int oz[2] = {(za - cz0) * 8 + l8, (zb - cz0) * 8 + l8};
  const float wz[2] = {1.f - tz, tz};
  int oy[4][2];
  float wy[4][2];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    int ya, yb;
    float ty;
    const int y = y0 + 2 * j + yofs;
    axis(y < Y ? y : Y - 1, Y, Yc, ya, yb, ty);
    oy[j][0] = (ya - cy0) * UA_CZ * 8; oy[j][1] = (yb - cy0) * UA_CZ * 8;
    wy[j][0] = 1.f - ty; wy[j][1] = ty;
  }
#pragma unroll 1
  for (int dx = 0; dx < UA_BX; ++dx) {
    const int x = x0 + dx;
    if (x >= X) break;
    int xa, xb;
    float tx;
    axis(x, X, Xc, xa, xb, tx);
    const int ox[2] = {(xa - cx0) * UA_CY * UA_CZ * 8, (xb - cx0) * UA_CY * UA_CZ * 8};
    const float wx[2] = {1.f - tx, tx};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int y = y0 + 2 * j + yofs;
      if (y >= Y) continue;
      const long long row = (long long)b * V + ((long long)x * Y + y) * Z + z;
      const float4 raw = __ldcs(reinterpret_cast<const float4*>(cur + row * C) + chunk * 8 + l8);
      float4 o = make_float4(fmaf(raw.x, a.x, d.x), fmaf(raw.y, a.y, d.y), fmaf(raw.z, a.z, d.z), fmaf(raw.w, a.w, d.w));
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int kz = k & 1, ky = (k >> 1) & 1, kx = k >> 2;
        const float4 cv = tile[ox[kx] + oy[j][ky] + oz[kz]];
        const float wgt = wx[kx] * wy[j][ky] * wz[kz];
        o.x = fmaf(wgt, cv.x, o.x); o.y = fmaf(wgt, cv.y, o.y);
        o.z = fmaf(wgt, cv.z, o.z); o.w = fmaf(wgt, cv.w, o.w);
      }
      store_split4(out_s + row * C, chunk * 32 + 4 * l8, o);
    }
  }
}

}  // namespace occ

using namespace occ;

// grids: L x (X, Y, Z) ints on the HOST, levels in token order (coarse -> fine); rows = B * sum X*Y*Z.
extern "C" int occ_neck_token_prep(const float* in, const float* ln_w, const float* ln_b, const float* pos,
                                   float* out_f32, float* out_s32, float* out_pos, int L, int B, const int* grids,
                                   int C, cudaStream_t stream) {
  OCC_REQUIRE(in && grids && (out_f32 || out_s32 || out_pos));
  OCC_REQUIRE((ln_w == nullptr) == (ln_b == nullptr) && (out_pos == nullptr || pos != nullptr));
  OCC_REQUIRE(C % 32 == 0 && C >= 32 && C <= 1024);
  NeckLevels g;
  OCC_REQUIRE(fill_levels(g, L, B, grids, nullptr) == OCC_OK);
  const unsigned blocks = (unsigned)((g.rows + 7) / 8);
  switch (C / 32) {
#define TP_CASE(n) case n: token_prep_kernel<n><<<blocks, 256, 0, stream>>>(in, ln_w, ln_b, pos, out_f32, out_s32, out_pos, g, C); break;
    TP_CASE(1) TP_CASE(2) TP_CASE(3) TP_CASE(4) TP_CASE(6) TP_CASE(8) TP_CASE(12) TP_CASE(16) TP_CASE(24) TP_CASE(32)
#undef TP_CASE
    default: return OCC_EUNSUPPORTED;
  }
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// value (rows, value_ld) with head h at columns [h*head_ld, h*head_ld + E/H), ow (rows, H*L*P*4) = [offsets (h,l,p,3) |
// logits (h,l,p)], out (rows, E) S32.
// strides: the L feature strides of the levels (reference-point arithmetic, multiscale_deformattn_3d.py:166-171).
extern "C" int occ_ms_deform_attn(const float* value, int value_ld, int head_ld, const float* ow, float* out, int L, int B,
                                  const int* grids, const float* strides, int E, int H, int P, cudaStream_t stream) {
  OCC_REQUIRE(value && ow && out && grids && strides);
  OCC_REQUIRE(E % 32 == 0 && H > 0 && E % H == 0 && (E / H) % 4 == 0 && E / 4 <= 256);
  OCC_REQUIRE(head_ld >= E / H && head_ld % 4 == 0 && value_ld >= (H - 1) * head_ld + E / H && value_ld % 4 == 0);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(value) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0);
  NeckLevels g;
  OCC_REQUIRE(fill_levels(g, L, B, grids, strides) == OCC_OK);
  const int T1 = E / H / 4;
  OCC_REQUIRE(H <= 65535 && T1 >= 1 && T1 <= 8 && g.rows < (1ll << 31));
  dim3 grid((unsigned)g.npatches, (unsigned)H);
  const int threads = NK_QP * T1;
  const size_t smem = (size_t)NK_QP * (L * P * 8 + 1) * sizeof(uint2);
#define MSDA_CASE(l)                                                                                    \
  if (L == l && P == 4) {                                                                               \
    OCC_ENSURE_SMEM((ms_deform_attn_kernel<l, 4>), smem);                                               \
    ms_deform_attn_kernel<l, 4><<<grid, threads, smem, stream>>>(value, ow, out, g, E, H, value_ld, head_ld); \
  } else
  MSDA_CASE(3) MSDA_CASE(1) MSDA_CASE(2) MSDA_CASE(4)
#undef MSDA_CASE
    return OCC_EUNSUPPORTED;
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_gn_upsample_add(const float* cur, const double* stats, const float* gw, const float* gb, int groups,
                                   const float* coarse, float* out_s, int B, int X, int Y, int Z, int Xc, int Yc, int Zc,
                                   int C, cudaStream_t stream) {
  OCC_REQUIRE(cur && stats && gw && gb && coarse && out_s);
  OCC_REQUIRE(B > 0 && X > 0 && Y > 0 && Z > 0 && Xc > 0 && Yc > 0 && Zc > 0 && C % 32 == 0 && groups > 0 && C % groups == 0);
  OCC_REQUIRE(B <= 65535 && C <= 4096);
  OCC_REQUIRE(((reinterpret_cast<uintptr_t>(cur) | reinterpret_cast<uintptr_t>(coarse) |
                reinterpret_cast<uintptr_t>(out_s)) & 15) == 0);  // float4 loads and stores
  const long long V = (long long)X * Y * Z;
  OCC_REQUIRE(V < (1ll << 31));
  if (X == 2 * Xc && Y == 2 * Yc && Z == 2 * Zc && B <= 65535 && C / 32 <= 65535) {
    const int nb = ((X + UA_BX - 1) / UA_BX) * ((Y + UA_BY - 1) / UA_BY) * ((Z + UA_BZ - 1) / UA_BZ);
    dim3 grid2((unsigned)nb, (unsigned)(C / 32), (unsigned)B);
    gn_upsample_add_x2_kernel<<<grid2, 256, 0, stream>>>(cur, stats, gw, gb, groups, coarse, out_s, X, Y, Z, Xc, Yc, Zc, C);
    OCC_LAUNCH_CHECK();
    return OCC_OK;
  }
  int vpc = (2048 * 4 + C / 4 - 1) / (C / 4);
  dim3 grid((unsigned)((V + vpc - 1) / vpc), B);
  gn_upsample_add_kernel<<<grid, 256, 2 * C * sizeof(float), stream>>>(cur, stats, gw, gb, groups, coarse, out_s, X, Y, Z, Xc,
                                                                       Yc, Zc, C, vpc);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
