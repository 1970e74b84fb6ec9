// Mask2Former-3D occupancy decoder head kernels for sm_90a (everything except the two tensor-core GEMM families,
// which reuse occ_gemm_bf16x3: the K/V projections of the voxel memories and the mask-embed x voxel-feature einsum).
//
// Reference path replaced (files of the reference checkout, P/ = projects/mmdet3d_plugin/occformer/):
//   P/mask2former/mask2former_nusc_occ.py:589-689  forward (level prep, 1+L forward_head calls, L decoder layers)
//   P/mask2former/mask2former_nusc_occ.py:426-471  forward_head (post_norm LN, cls_embed, mask_embed MLP, einsum,
//                                                  adaptive_max_pool3d, sigmoid < 0.5)
//   P/mask2former/mask2former_nusc_occ.py:691-745  format_results / simple_test (trilinear upsample, sigmoid, class mix)
//   P/mask2former/mask2former_nusc_occ.py:505-542  forward_lidarseg (grid_sample of the class volume at LiDAR points)
//   P/mask2former/positional_encodings/positional_encoding.py:58-108  SinePositionalEncoding3D
//   mmcv 1.4.0 BaseTransformerLayer / MultiheadAttention / FFN (un-vendored; semantics SURVEY.md Appendix C):
//     cross-attn (q = query+query_pos, k = key+key_pos, v = key, bool mask) -> LN -> self-attn -> LN -> FFN -> LN
//
// Layouts: voxel tensors are channel-last rows (B, S, E); query state (B, Q, E); masks / mask logits (B, S, Q)
// ("query-last", so that a voxel's Q logits are one contiguous row).  All arithmetic fp32 (SIMT) -- the query side
// is 100 rows per sample; its cost is launch latency, not FLOPs.
#include "occ_common.cuh"
#include "occ_ptx.cuh"

namespace occ {

constexpr float kLnEps = 1e-5f;

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- query-side building blocks.  CTA = (E, 4) threads: thread (j, g) owns channel j of row row0 + g; the four
// groups also split every reduction dimension four ways (4x fewer dependent iterations per mat-vec: these kernels
// are latency-bound -- 100 rows per sample -- not throughput-bound).
constexpr int QG = 4;  // rows per CTA = k-split groups

// sum over the E threads of group g (E multiple of 32); red = smem [QG][8]
__device__ __forceinline__ float group_sum(float v, int g, int j, int E, float* red) {
  const int lane = j & 31, w = j >> 5, nw = E >> 5;
  v = warp_sum_f(v);
  __syncthreads();
  if (lane == 0) red[g * 8 + w] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < nw; ++i) t += red[g * 8 + i];
  return t;
}

__device__ __forceinline__ float group_layernorm(float x, int g, int j, int E, const float* __restrict__ gamma,
                                                 const float* __restrict__ beta, float* red) {
  const float mean = group_sum(x, g, j, E, red) / (float)E;
  const float d = x - mean;
  const float var = group_sum(d * d, g, j, E, red) / (float)E;
  return d * rsqrtf(var + kLnEps) * gamma[j] + beta[j];
}

// returns out[g][j] = bias[j] + sum_k wT[k*ldw + j] * xs[g*K + k]; all four groups cooperate: group g accumulates
// the k-quarter [g*K/4, (g+1)*K/4) for all four rows, partial sums meet in shared memory.  wT is the K-major
// transposed weight (consecutive threads read consecutive addresses); xs [QG][K] in shared memory (broadcast reads).
__device__ __forceinline__ float matvec4(const float* __restrict__ wT, int ldw, const float* __restrict__ bias,
                                         const float* xs, int K, int j, int g, int E, float* part /*[QG][QG][E]*/) {
  float acc[QG];
#pragma unroll
  for (int r = 0; r < QG; ++r) acc[r] = 0.f;
  const int kq = K / QG;  // multiple of 4 (K is a multiple of 32)
  const int k0 = g * kq;
  // four k per step: 4 independent coalesced weight loads + one LDS.128 per row (xs rows are k-contiguous, 16-byte
  // aligned: K % 4 == 0), unrolled so that 16 weight loads are in flight
#pragma unroll 4
  for (int k = k0; k < k0 + kq; k += 4) {
    const float w0 = __ldg(wT + (size_t)k * ldw + j), w1 = __ldg(wT + (size_t)(k + 1) * ldw + j),
                w2 = __ldg(wT + (size_t)(k + 2) * ldw + j), w3 = __ldg(wT + (size_t)(k + 3) * ldw + j);
#pragma unroll
    for (int r = 0; r < QG; ++r) {
      const float4 x = *reinterpret_cast<const float4*>(xs + r * K + k);
      acc[r] = fmaf(w3, x.w, fmaf(w2, x.z, fmaf(w1, x.y, fmaf(w0, x.x, acc[r]))));
    }
  }
#pragma unroll
  for (int r = 0; r < QG; ++r) part[(g * QG + r) * E + j] = acc[r];
  __syncthreads();
  float o = bias ? __ldg(bias + j) : 0.f;
#pragma unroll
  for (int gg = 0; gg < QG; ++gg) o += part[(gg * QG + g) * E + j];
  __syncthreads();
  return o;
}

// ---------------------------------------------------------------------------------------------------------
// SinePositionalEncoding3D (normalize=True, all-False mask): out (S = X*Y*Z, 3*F) rows in (x,y,z) order.
__global__ void sine_pos3d_kernel(float* __restrict__ out, int X, int Y, int Z, int F, float temperature, float scale,
                                  float eps, float offset) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int E = 3 * F;
  const long long total = (long long)X * Y * Z * E;
  if (i >= total) return;
  const int c = (int)(i % E);
  const long long s = i / E;
  const int z = (int)(s % Z), y = (int)((s / Z) % Y), x = (int)(s / ((long long)Z * Y));
  const int axis = c / F, f = c % F;
  const float idx = axis == 0 ? (float)(x + 1) : axis == 1 ? (float)(y + 1) : (float)(z + 1);
  const float last = axis == 0 ? (float)X : axis == 1 ? (float)Y : (float)Z;
  const float e = (idx + offset) / (last + eps) * scale;
  const float dim_t = powf(temperature, 2.0f * (float)(f / 2) / (float)F);
  const float pe = e / dim_t;
  out[i] = (f & 1) ? cosf(pe) : sinf(pe);
}

// ---------------------------------------------------------------------------------------------------------
// Level / mask-feature preparation: (optional NCDHW -> channel-last transpose) + level embed + positional encoding,
// written in the S32 split format (operands of the projection GEMMs / mask GEMMs; C % 32 == 0).
//   in  : channel-last (B, S, C) when in_cl != 0, else reference layout (B, C, S)
//   mem : (B, S, C) = in + level_embed          (V-projection operand; also the mask-feature operand)
//   kpos: (B, S, C) = in + level_embed + pos    (K-projection operand; optional)
__global__ void head_prep_cl_kernel(const float* __restrict__ in, const float* __restrict__ level_embed,
                                    const float* __restrict__ pos, float* __restrict__ mem, float* __restrict__ kpos,
                                    long long rows, long long S, int C) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int C4 = C >> 2;
  if (i4 >= rows * C4) return;
  const long long row = i4 / C4;
  const int c0 = (int)(i4 % C4) * 4;
  float4 v = __ldcs(reinterpret_cast<const float4*>(in + row * C + c0));
  if (level_embed) {
    const float4 l = *reinterpret_cast<const float4*>(level_embed + c0);
    v.x += l.x; v.y += l.y; v.z += l.z; v.w += l.w;
  }
  store_split4(mem + row * C, c0, v);
  if (kpos) {
    const float4 p = *reinterpret_cast<const float4*>(pos + (row % S) * C + c0);
    store_split4(kpos + row * C, c0, make_float4(v.x + p.x, v.y + p.y, v.z + p.z, v.w + p.w));
  }
}

__global__ void head_prep_ncs_kernel(const float* __restrict__ in, const float* __restrict__ level_embed,
                                     const float* __restrict__ pos, float* __restrict__ mem, float* __restrict__ kpos,
                                     long long S, int C) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int c0 = blockIdx.y * 32;
  const long long s0 = (long long)blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i;
    const long long s = s0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && s < S) ? __ldcs(in + ((size_t)b * C + c) * S + s) : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {  // a warp (threadIdx.x = 0..31) = one S32 chunk of one row
    const long long s = s0 + i;
    const int c = c0 + threadIdx.x;  // C % 32 == 0: c < C for the whole warp
    if (s < S) {
      float v = tile[threadIdx.x][i];
      if (level_embed) v += level_embed[c];
      const float vk = kpos ? v + pos[s * C + c] : 0.f;
      const float v2 = __shfl_xor_sync(0xffffffffu, v, 1), vk2 = __shfl_xor_sync(0xffffffffu, vk, 1);
      if (!(threadIdx.x & 1)) {
        uint32_t hi, lo;
        split_pair(v, v2, hi, lo);
        uint32_t* chunk = reinterpret_cast<uint32_t*>(mem + ((size_t)b * S + s) * C + c0);
        chunk[threadIdx.x >> 1] = hi;
        chunk[16 + (threadIdx.x >> 1)] = lo;
        if (kpos) {
          split_pair(vk, vk2, hi, lo);
          chunk = reinterpret_cast<uint32_t*>(kpos + ((size_t)b * S + s) * C + c0);
          chunk[threadIdx.x >> 1] = hi;
          chunk[16 + (threadIdx.x >> 1)] = lo;
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// forward_head, query side: post_norm LN -> cls_embed, mask_embed MLP (Linear-ReLU-Linear-ReLU-Linear).
//   query (B*Q, E); cls_out (B*Q, NC); membed_out (B*Q, E) in the S32 split format (operand of the mask GEMMs)
__global__ void __launch_bounds__(1024)
query_head_kernel(const float* __restrict__ query_in, const float* __restrict__ n2w, const float* __restrict__ n2b,
                  float* __restrict__ query_state, const float* __restrict__ pn_w, const float* __restrict__ pn_b,
                  const float* __restrict__ clsT, const float* __restrict__ cls_b, int NC,
                  const float* __restrict__ m0T, const float* __restrict__ m0b, const float* __restrict__ m1T,
                  const float* __restrict__ m1b, const float* __restrict__ m2T, const float* __restrict__ m2b,
                  float* __restrict__ cls_out, float* __restrict__ membed_out, const float* __restrict__ query_pos,
                  int Q, const float* __restrict__ wqT, const float* __restrict__ bq, float scale,
                  float* __restrict__ qh_out, const float* __restrict__ ffn_part, int nparts, int rows, int E) {
  extern __shared__ __align__(16) float sm[];  // xs[QG*E], part[QG*QG*E], red[32]
  float* xs = sm;
  float* part = xs + QG * E;
  float* red = part + QG * QG * E;
  const int j = threadIdx.x % E, g = threadIdx.x / E;
  const int row = blockIdx.x * QG + g;  // rows % QG == 0
  float q = query_in[(size_t)row * E + j];
  for (int c = 0; c < nparts; ++c) q += ffn_part[((size_t)c * rows + row) * E + j];  // FFN column blocks, fixed order
  if (n2w) {  // last norm of the decoder layer (norms.2) on the FFN accumulator -> the layer's output query
    q = group_layernorm(q, g, j, E, n2w, n2b, red);
    query_state[(size_t)row * E + j] = q;
  }
  if (wqT) {  // cross-attention query projection of the NEXT layer: ((query + query_pos) Wq^T + bq) * hd^-0.5
    __syncthreads();
    xs[g * E + j] = q + query_pos[(size_t)(row % Q) * E + j];
    __syncthreads();
    qh_out[(size_t)row * E + j] = matvec4(wqT, E, bq, xs, E, j, g, E, part) * scale;
  }
  float x = group_layernorm(q, g, j, E, pn_w, pn_b, red);
  __syncthreads();
  xs[g * E + j] = x;
  __syncthreads();
  {  // class logits: NC <= E outputs; threads j >= NC idle along (all threads must reach the barriers)
    const int jj = j < NC ? j : 0;
    const float c = matvec4(clsT, NC, cls_b, xs, E, jj, g, E, part);
    if (j < NC) cls_out[(size_t)row * NC + j] = c;
  }
  float h = fmaxf(matvec4(m0T, E, m0b, xs, E, j, g, E, part), 0.f);
  xs[g * E + j] = h;
  __syncthreads();
  h = fmaxf(matvec4(m1T, E, m1b, xs, E, j, g, E, part), 0.f);
  xs[g * E + j] = h;
  __syncthreads();
  h = matvec4(m2T, E, m2b, xs, E, j, g, E, part);
  {  // E % 32 == 0: a warp holds one 32-channel chunk of one row; lanes (2t, 2t+1) form packed word t
    const float h2 = __shfl_xor_sync(0xffffffffu, h, 1);
    if (!(j & 1)) {
      uint32_t hi, lo;
      split_pair(h, h2, hi, lo);
      uint32_t* chunk = reinterpret_cast<uint32_t*>(membed_out + (size_t)row * E + (j & ~31));
      chunk[(j & 31) >> 1] = hi;
      chunk[16 + ((j & 31) >> 1)] = lo;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// adaptive_max_pool3d of the mask logits + "has an unmasked key" flag per (b, q).
//   mask (B, X*Y*Z, Q) -> pooled (B, Xo*Yo*Zo, Q); window of output i along an axis: [floor(i*in/out), ceil((i+1)*in/out))
// CTA = (128 q-threads, 4 cells): thread.x <-> query (a voxel's Q logits are one contiguous row -> coalesced 400-byte
// reads), thread.y <-> one pooled cell; all window loads of a thread are independent (no barriers), 32-bit index math.
// blockIdx.y = 128-query tile (Q > 128).
__global__ void __launch_bounds__(512)
mask_pool_kernel(const float* __restrict__ mask, int* __restrict__ pooled, int* __restrict__ row_flag, int B, int X,
                 int Y, int Z, int Xo, int Yo, int Zo, int Q) {
  const int q = blockIdx.y * 128 + threadIdx.x;
  const int So = Xo * Yo * Zo;
  const int ncell = B * So;
  if (q >= Q) return;
  for (int cell = blockIdx.x * 4 + threadIdx.y; cell < ncell; cell += gridDim.x * 4) {
    int t = cell;
    const int zo = t % Zo; t /= Zo;
    const int yo = t % Yo; t /= Yo;
    const int xo = t % Xo;
    const int b = t / Xo;
    const int x0 = (xo * X) / Xo, x1 = ((xo + 1) * X + Xo - 1) / Xo;
    const int y0 = (yo * Y) / Yo, y1 = ((yo + 1) * Y + Yo - 1) / Yo;
    const int z0 = (zo * Z) / Zo, z1 = ((zo + 1) * Z + Zo - 1) / Zo;
    float m = -INFINITY;
    for (int x = x0; x < x1; ++x)
      for (int y = y0; y < y1; ++y) {
        const float* p = mask + ((((size_t)b * X + x) * Y + y) * Z + z0) * Q + q;
#pragma unroll 4
        for (int z = 0; z < z1 - z0; ++z) m = fmaxf(m, __ldg(p + (size_t)z * Q));
      }
    const int code = ordered_logit(m);
    pooled[(size_t)cell * Q + q] = code;
    // attn_mask = sigmoid(m) < 0.5  <=>  code < 0 ; a row that is blocked everywhere is un-blocked (:652-653)
    if (code >= 0) row_flag[b * Q + q] = 1;
  }
}

constexpr int XA_HD = 32;  // head dim of the decoder attentions (embed_dims / num_heads)

// ---------------------------------------------------------------------------------------------------------
// Cross-attention tail + self-attention in-projection (thread (j, g): channel j = head j/32, dim j%32, of row row0+g):
//   merge the key-chunk partials -> out_proj -> + identity -> LN(norms.0) -> query1
//   self-attn in_proj: q = ((query1+pos) Wq^T + bq) * hd^-0.5, k = (query1+pos) Wk^T + bk, v = query1 Wv^T + bv
__global__ void __launch_bounds__(1024)
cross_merge_kernel(const float* __restrict__ part_in, int nchunk, int H, const float* __restrict__ query,
                   const float* __restrict__ query_pos, int Q, const float* __restrict__ woT,
                   const float* __restrict__ bo, const float* __restrict__ n0w, const float* __restrict__ n0b,
                   const float* __restrict__ sa_inT /*(E, 3E) K-major*/, const float* __restrict__ sa_inb, float scale,
                   float* __restrict__ query1, float* __restrict__ sa_qkv /*(rows, 3E)*/, int rows, int E) {
  extern __shared__ __align__(16) float sm[];  // xs[QG*E], ps[QG*E], part[QG*QG*E], red[32]
  float* xs = sm;
  float* ps = xs + QG * E;
  float* part = ps + QG * E;
  float* red = part + QG * QG * E;
  const int j = threadIdx.x % E, g = threadIdx.x / E;
  const int h = j / XA_HD, d = j % XA_HD;
  const int row = blockIdx.x * QG + g;
  {
    const int b = row / Q, t = row % Q;
    const float* p = part_in + (((size_t)b * H + h) * nchunk * Q + t) * (XA_HD + 2);
    const size_t cstride = (size_t)Q * (XA_HD + 2);
    float M = -INFINITY;
    for (int c = 0; c < nchunk; ++c) M = fmaxf(M, __ldg(p + c * cstride));
    float L = 0.f, A = 0.f;
#pragma unroll 4
    for (int c = 0; c < nchunk; ++c) {
      const float mc = __ldg(p + c * cstride);
      const float w = (mc == -INFINITY) ? 0.f : __expf(mc - M);
      L = fmaf(__ldg(p + c * cstride + 1), w, L);
      A = fmaf(__ldg(p + c * cstride + 2 + d), w, A);
    }
    xs[g * E + j] = A / L;
  }
  __syncthreads();
  float x = matvec4(woT, E, bo, xs, E, j, g, E, part) + query[(size_t)row * E + j];
  x = group_layernorm(x, g, j, E, n0w, n0b, red);
  query1[(size_t)row * E + j] = x;
  __syncthreads();
  xs[g * E + j] = x;
  ps[g * E + j] = x + query_pos[(size_t)(row % Q) * E + j];
  __syncthreads();
  float* dst = sa_qkv + (size_t)row * 3 * E;
  dst[j] = matvec4(sa_inT, 3 * E, sa_inb, ps, E, j, g, E, part) * scale;
  dst[E + j] = matvec4(sa_inT + E, 3 * E, sa_inb + E, ps, E, j, g, E, part);
  dst[2 * E + j] = matvec4(sa_inT + 2 * E, 3 * E, sa_inb + 2 * E, xs, E, j, g, E, part);
}

// ---------------------------------------------------------------------------------------------------------
// Self-attention over the Q queries + out_proj + LN(norms.1).  Thread (j, g): row row0+g, warp j/32 of the group <->
// head (hd = 32 = warp size), then channel j.  Writes x1 (LN1 output) and seeds the FFN accumulator ybuf = x1 + b2.
// A sample holds Qs query slots (rows); its first Q are the keys (Q <= Qs <= NKG*32): padded slots never act as keys.
template <int NKG>
__global__ void __launch_bounds__(1024)
self_attn_kernel(const float* __restrict__ sa_qkv, const float* __restrict__ query1, int Q, int Qs,
                 const float* __restrict__ woT, const float* __restrict__ bo, const float* __restrict__ n1w,
                 const float* __restrict__ n1b, const float* __restrict__ f2b, float* __restrict__ x1,
                 float* __restrict__ ybuf, int E) {
  extern __shared__ __align__(16) float sm[];  // xs[QG*E], part[QG*QG*E], red[32]
  float* xs = sm;
  float* part = xs + QG * E;
  float* red = part + QG * QG * E;
  const int j = threadIdx.x % E, g = threadIdx.x / E;
  const int lane = j & 31, h = j >> 5;
  const int row = blockIdx.x * QG + g;
  const int b = row / Qs;
  const float* base = sa_qkv + (size_t)b * Qs * 3 * E;
  // scores of this head: lane handles keys lane, lane+32, ..., lane+32*(NKG-1)
  const float qd = sa_qkv[(size_t)row * 3 * E + j];  // q[h*32 + lane]
  float sc[NKG];
#pragma unroll
  for (int i = 0; i < NKG; ++i) {
    const int key = i * 32 + lane;
    const float* krow = base + (size_t)min(key, Q - 1) * 3 * E + E + h * 32;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < 32; ++d) s = fmaf(__shfl_sync(0xffffffffu, qd, d), krow[d], s);
    sc[i] = key < Q ? s : -INFINITY;
  }
  float m = fmaxf(fmaxf(sc[0], sc[1]), fmaxf(sc[2], sc[3]));
#pragma unroll
  for (int i = 4; i < NKG; i += 4) m = fmaxf(m, fmaxf(fmaxf(sc[i], sc[i + 1]), fmaxf(sc[i + 2], sc[i + 3])));
  m = warp_max_f(m);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NKG; ++i) {
    sc[i] = (i * 32 + lane < Q) ? expf(sc[i] - m) : 0.f;
    sum += sc[i];
  }
  sum = warp_sum_f(sum);
  float o = 0.f;
#pragma unroll
  for (int i = 0; i < NKG; ++i) {
    for (int k = 0; k < 32; ++k) {
      const int key = i * 32 + k;
      const float p = __shfl_sync(0xffffffffu, sc[i], k);
      if (key < Q) o = fmaf(p, base[(size_t)key * 3 * E + 2 * E + j], o);
    }
  }
  xs[g * E + j] = o / sum;
  __syncthreads();
  float x = matvec4(woT, E, bo, xs, E, j, g, E, part) + query1[(size_t)row * E + j];
  x = group_layernorm(x, g, j, E, n1w, n1b, red);
  x1[(size_t)row * E + j] = x;
  ybuf[(size_t)row * E + j] = x + f2b[j];
}

// FFN (mmcv FFN: Linear-ReLU-Linear + identity) as F/E independent column blocks: CTA (blockIdx.y = c) computes the
// hidden units f in [c*E, (c+1)*E) of four rows and writes their contribution to the output as partial c
// (ypart (F/E, rows, E)); query_head_kernel adds the partials to ybuf in the fixed order c = 0, 1, ... -- the decoder
// is bit-reproducible run to run (no floating-point atomics).
__global__ void __launch_bounds__(1024)
ffn_block_kernel(const float* __restrict__ x1, const float* __restrict__ f1T /*(E, F)*/, const float* __restrict__ f1b,
                 const float* __restrict__ f2T /*(F, E)*/, int F, float* __restrict__ ypart, int E) {
  extern __shared__ __align__(16) float sm[];  // xs[QG*E], hs[QG*E], part[QG*QG*E]
  float* xs = sm;
  float* hs = xs + QG * E;
  float* part = hs + QG * E;
  const int j = threadIdx.x % E, g = threadIdx.x / E;
  const int row = blockIdx.x * QG + g;
  const int c = blockIdx.y;
  xs[g * E + j] = x1[(size_t)row * E + j];
  __syncthreads();
  const float hval = fmaxf(matvec4(f1T + (size_t)c * E, F, f1b + (size_t)c * E, xs, E, j, g, E, part), 0.f);
  hs[g * E + j] = hval;
  __syncthreads();
  const float y = matvec4(f2T + (size_t)c * E * E, E, nullptr, hs, E, j, g, E, part);
  ypart[((size_t)c * gridDim.x * QG + row) * E + j] = y;
}

// ---------------------------------------------------------------------------------------------------------
// simple_test tail (mask2former_nusc_occ.py:725-736, 691-696): trilinear upsample (align_corners=True) of the last
// mask logits -> sigmoid -> class mix with softmax(cls)[..., :-1].
//   mask (B, X*Y*Z, Q) with Q query slots per row, cls (B, Qr, NC) of the first Qr <= Q (real) queries
//   -> out (B, NC-1, Xo, Yo, Zo)   (reference layout); padded slots get zero class probabilities
constexpr int CM_THREADS = 128;

template <int KMAX>
__global__ void __launch_bounds__(CM_THREADS)
classmix_kernel(const float* __restrict__ mask, const float* __restrict__ cls, float* __restrict__ out,
                unsigned char* __restrict__ labels, int X, int Y, int Z, int Xo, int Yo, int Zo, int Q, int Qr,
                int NC) {
  extern __shared__ __align__(16) float sm[];  // P[Q][KMAX] (zero padded)
  const int K = NC - 1;
  float* P = sm;
  const int b = blockIdx.y;
  // softmax over the NC class logits of every query, drop the last (no-object) column
  for (int q = threadIdx.x; q < Q; q += blockDim.x) {
    if (q >= Qr) {
      for (int k = 0; k < KMAX; ++k) P[q * KMAX + k] = 0.f;
      continue;
    }
    const float* c = cls + ((size_t)b * Qr + q) * NC;
    float m = -INFINITY;
    for (int k = 0; k < NC; ++k) m = fmaxf(m, c[k]);
    float s = 0.f;
    for (int k = 0; k < NC; ++k) s += expf(c[k] - m);
    for (int k = 0; k < KMAX; ++k) P[q * KMAX + k] = k < K ? expf(c[k] - m) / s : 0.f;
  }
  const long long Vo = (long long)Xo * Yo * Zo;
  const long long v0 = (long long)blockIdx.x * CM_THREADS;
  const long long v = v0 + threadIdx.x;
  const bool identity = (X == Xo && Y == Yo && Z == Zo);
  float acc[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) acc[k] = 0.f;
  if (identity) {
    // thread = voxel: its Q logits are one contiguous run, read straight into registers in 32-byte pieces (no staging,
    // no barrier after the class table: the occupancy hides the latency; every line is consumed completely)
    __syncthreads();
    if (v < Vo) {
      const float4* r4 = reinterpret_cast<const float4*>(mask + ((size_t)b * Vo + v) * Q);
      for (int q8 = 0; q8 < Q; q8 += 8) {
        float lg[8];
        const float4 a = __ldcs(r4 + (q8 >> 2));
        lg[0] = a.x; lg[1] = a.y; lg[2] = a.z; lg[3] = a.w;
        const bool two = q8 + 4 < Q;
        const float4 c = two ? __ldcs(r4 + (q8 >> 2) + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
        lg[4] = c.x; lg[5] = c.y; lg[6] = c.z; lg[7] = c.w;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          if (e >= 4 && !two) break;
          const float s = 1.0f / (1.0f + __expf(-lg[e]));
          const float* pq = P + (q8 + e) * KMAX;
#pragma unroll
          for (int k = 0; k < KMAX; k += 4) {
            const float4 pp = *reinterpret_cast<const float4*>(pq + k);
            acc[k] = fmaf(pp.x, s, acc[k]); acc[k + 1] = fmaf(pp.y, s, acc[k + 1]);
            acc[k + 2] = fmaf(pp.z, s, acc[k + 2]); acc[k + 3] = fmaf(pp.w, s, acc[k + 3]);
          }
        }
      }
    }
  } else {
    __syncthreads();
    if (v < Vo) {
      const int zo = (int)(v % Zo), yo = (int)((v / Zo) % Yo), xo = (int)(v / ((long long)Zo * Yo));
      // torch upsample_trilinear3d, align_corners=True: src = dst * (in-1)/(out-1)
      const float sx = Xo > 1 ? (float)(X - 1) / (float)(Xo - 1) : 0.f;
      const float sy = Yo > 1 ? (float)(Y - 1) / (float)(Yo - 1) : 0.f;
      const float sz = Zo > 1 ? (float)(Z - 1) / (float)(Zo - 1) : 0.f;
      const float fx = sx * xo, fy = sy * yo, fz = sz * zo;
      const int x0 = (int)fx, y0 = (int)fy, z0 = (int)fz;
      const int x1 = x0 + (x0 < X - 1), y1 = y0 + (y0 < Y - 1), z1 = z0 + (z0 < Z - 1);
      const float lx = fx - x0, ly = fy - y0, lz = fz - z0;
      const float hx = 1.f - lx, hy = 1.f - ly, hz = 1.f - lz;
      const float* mb = mask + (size_t)b * X * Y * Z * Q;
      const float* p000 = mb + (((size_t)x0 * Y + y0) * Z + z0) * Q;
      const float* p001 = mb + (((size_t)x0 * Y + y0) * Z + z1) * Q;
      const float* p010 = mb + (((size_t)x0 * Y + y1) * Z + z0) * Q;
      const float* p011 = mb + (((size_t)x0 * Y + y1) * Z + z1) * Q;
      const float* p100 = mb + (((size_t)x1 * Y + y0) * Z + z0) * Q;
      const float* p101 = mb + (((size_t)x1 * Y + y0) * Z + z1) * Q;
      const float* p110 = mb + (((size_t)x1 * Y + y1) * Z + z0) * Q;
      const float* p111 = mb + (((size_t)x1 * Y + y1) * Z + z1) * Q;
      for (int q = 0; q < Q; ++q) {
        const float val = hx * (hy * (hz * __ldg(p000 + q) + lz * __ldg(p001 + q)) +
                                ly * (hz * __ldg(p010 + q) + lz * __ldg(p011 + q))) +
                          lx * (hy * (hz * __ldg(p100 + q) + lz * __ldg(p101 + q)) +
                                ly * (hz * __ldg(p110 + q) + lz * __ldg(p111 + q)));
        const float s = 1.0f / (1.0f + expf(-val));
#pragma unroll
        for (int k = 0; k < KMAX; k += 4) {
          const float4 pp = *reinterpret_cast<const float4*>(P + q * KMAX + k);
          acc[k] = fmaf(pp.x, s, acc[k]); acc[k + 1] = fmaf(pp.y, s, acc[k + 1]);
          acc[k + 2] = fmaf(pp.z, s, acc[k + 2]); acc[k + 3] = fmaf(pp.w, s, acc[k + 3]);
        }
      }
    }
  }
  if (v < Vo) {
    float best = -INFINITY;
    int arg = 0;
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
      if (k < K) {
        __stcs(out + ((size_t)b * K + k) * Vo + v, acc[k]);
        if (acc[k] > best) { best = acc[k]; arg = k; }  // first maximum, like torch.argmax
      }
    if (labels) labels[(size_t)b * Vo + v] = (unsigned char)arg;
  }
}

// (B, S, Q) query-last mask logits -> reference layout (B, Q, S)   (only for API parity of forward())
__global__ void transpose_sq_kernel(const float* __restrict__ in, float* __restrict__ out, long long S, int Q) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const long long s0 = (long long)blockIdx.x * 32;
  const int q0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const long long s = s0 + i;
    const int q = q0 + threadIdx.x;
    tile[i][threadIdx.x] = (s < S && q < Q) ? in[((size_t)b * S + s) * Q + q] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int q = q0 + i;
    const long long s = s0 + threadIdx.x;
    if (q < Q && s < S) out[((size_t)b * Q + q) * S + s] = tile[threadIdx.x][i];
  }
}

// ---------------------------------------------------------------------------------------------------------
// forward_lidarseg (mask2former_nusc_occ.py:505-542, eval): grid_sample(bilinear, align_corners=True, padding_mode
// border | zeros) of the class volume (K, X, Y, Z) at LiDAR points, then softmax over K.
//
// The point -> volume coordinates of forward_lidarseg (:515-530): normalise to [-1, 1] over pc_range, then grid_sample's
// align_corners=True unnormalisation; grid_sample's (x,y,z) = (W,H,D) = (Z,Y,X) axes of the volume after the [2,1,0]
// flip.  Returns the lower corner (x0, y0, z0) and the fractions (lx, ly, lz); corner c = (c>>2, (c>>1)&1, c&1).
struct SamplePos {
  int x0, y0, z0;
  float lx, ly, lz;
};
__device__ __forceinline__ SamplePos grid_sample_pos(const float* __restrict__ p, float x_min, float y_min, float z_min,
                                                     float x_ext, float y_ext, float z_ext, int X, int Y, int Z,
                                                     int border) {
  const float px = p[0], py = p[1], pz = p[2];
  const float gx = ((px - x_min) / x_ext) * 2.f - 1.f;
  const float gy = ((py - y_min) / y_ext) * 2.f - 1.f;
  const float gz = ((pz - z_min) / z_ext) * 2.f - 1.f;
  float ix = (gx + 1.f) / 2.f * (float)(X - 1);
  float iy = (gy + 1.f) / 2.f * (float)(Y - 1);
  float iz = (gz + 1.f) / 2.f * (float)(Z - 1);
  if (border) {
    ix = fminf(fmaxf(ix, 0.f), (float)(X - 1));
    iy = fminf(fmaxf(iy, 0.f), (float)(Y - 1));
    iz = fminf(fmaxf(iz, 0.f), (float)(Z - 1));
  }
  const float fx = floorf(ix), fy = floorf(iy), fz = floorf(iz);
  return SamplePos{(int)fx, (int)fy, (int)fz, ix - fx, iy - fy, iz - fz};
}

__global__ void lidarseg_kernel(const float* __restrict__ vox /*(K,X,Y,Z) of one sample*/,
                                const float* __restrict__ pts, int pts_stride, int n, float x_min, float y_min,
                                float z_min, float x_ext, float y_ext, float z_ext, int X, int Y, int Z, int K,
                                int border, float* __restrict__ out /*(n,K)*/) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const SamplePos sp = grid_sample_pos(pts + (size_t)i * pts_stride, x_min, y_min, z_min, x_ext, y_ext, z_ext, X, Y, Z,
                                       border);
  const int x0 = sp.x0, y0 = sp.y0, z0 = sp.z0;
  const float lx = sp.lx, ly = sp.ly, lz = sp.lz;
  float logit[32];
  float m = -INFINITY;
  for (int k = 0; k < K; ++k) {
    const float* vk = vox + (size_t)k * X * Y * Z;
    float a = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int xx = x0 + (c >> 2), yy = y0 + ((c >> 1) & 1), zz = z0 + (c & 1);
      const float w = ((c >> 2) ? lx : 1.f - lx) * (((c >> 1) & 1) ? ly : 1.f - ly) * ((c & 1) ? lz : 1.f - lz);
      if (xx >= 0 && xx < X && yy >= 0 && yy < Y && zz >= 0 && zz < Z) a += w * __ldg(vk + ((size_t)xx * Y + yy) * Z + zz);
    }
    logit[k] = a;
    m = fmaxf(m, a);
  }
  float s = 0.f;
  for (int k = 0; k < K; ++k) { logit[k] = expf(logit[k] - m); s += logit[k]; }
  for (int k = 0; k < K; ++k) out[(size_t)i * K + k] = logit[k] / s;
}

// ---------------------------------------------------------------------------------------------------------
// Panoptic ids (mask2former_nusc_panoptic_occ.py:715-784): per output voxel / LiDAR point, the winning query
// q(v) = argmax_q logit(v, q) (first maximum); per (sample, query) a (semantic, panoptic) id from the query's label and
// whether it wins anywhere; then id lookup.  The reference's upsampled (B, Q, *occ_size) logits are never formed.
// Logits arrive query-last (B, S, Qs) with Q <= Qs <= 256 real queries (padded slots never win).
//
// pass 1a: thread = output voxel; trilinear upsample (align_corners=True, the class-mix formula) or identity
__global__ void __launch_bounds__(128)
panoptic_vox_argmax_kernel(const float* __restrict__ mask, int Qs, int Q, int X, int Y, int Z, int Xo, int Yo, int Zo,
                           unsigned char* __restrict__ qidx, int* __restrict__ present) {
  const int b = blockIdx.y;
  const long long Vo = (long long)Xo * Yo * Zo;
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= Vo) return;
  const float* mb = mask + (size_t)b * X * Y * Z * Qs;
  float best = -INFINITY;
  int arg = 0;
  if (X == Xo && Y == Yo && Z == Zo) {
    const float4* r4 = reinterpret_cast<const float4*>(mb + (size_t)v * Qs);
    for (int q4 = 0; q4 < Qs; q4 += 4) {
      const float4 a = __ldcs(r4 + (q4 >> 2));
      const float val[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (q4 + e < Q && val[e] > best) { best = val[e]; arg = q4 + e; }
    }
  } else {
    const int zo = (int)(v % Zo), yo = (int)((v / Zo) % Yo), xo = (int)(v / ((long long)Zo * Yo));
    const float sx = Xo > 1 ? (float)(X - 1) / (float)(Xo - 1) : 0.f;
    const float sy = Yo > 1 ? (float)(Y - 1) / (float)(Yo - 1) : 0.f;
    const float sz = Zo > 1 ? (float)(Z - 1) / (float)(Zo - 1) : 0.f;
    const float fx = sx * xo, fy = sy * yo, fz = sz * zo;
    const int x0 = (int)fx, y0 = (int)fy, z0 = (int)fz;
    const int x1 = x0 + (x0 < X - 1), y1 = y0 + (y0 < Y - 1), z1 = z0 + (z0 < Z - 1);
    const float lx = fx - x0, ly = fy - y0, lz = fz - z0;
    const float hx = 1.f - lx, hy = 1.f - ly, hz = 1.f - lz;
    auto row = [&](int x, int y, int z) {
      return reinterpret_cast<const float4*>(mb + (((size_t)x * Y + y) * Z + z) * Qs);
    };
    const float4 *p000 = row(x0, y0, z0), *p001 = row(x0, y0, z1), *p010 = row(x0, y1, z0), *p011 = row(x0, y1, z1),
                 *p100 = row(x1, y0, z0), *p101 = row(x1, y0, z1), *p110 = row(x1, y1, z0), *p111 = row(x1, y1, z1);
    for (int q4 = 0; q4 < Qs; q4 += 4) {
      const int i4 = q4 >> 2;
      const float4 c000 = __ldg(p000 + i4), c001 = __ldg(p001 + i4), c010 = __ldg(p010 + i4), c011 = __ldg(p011 + i4),
                   c100 = __ldg(p100 + i4), c101 = __ldg(p101 + i4), c110 = __ldg(p110 + i4), c111 = __ldg(p111 + i4);
      const float a000[4] = {c000.x, c000.y, c000.z, c000.w}, a001[4] = {c001.x, c001.y, c001.z, c001.w},
                  a010[4] = {c010.x, c010.y, c010.z, c010.w}, a011[4] = {c011.x, c011.y, c011.z, c011.w},
                  a100[4] = {c100.x, c100.y, c100.z, c100.w}, a101[4] = {c101.x, c101.y, c101.z, c101.w},
                  a110[4] = {c110.x, c110.y, c110.z, c110.w}, a111[4] = {c111.x, c111.y, c111.z, c111.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float val = hx * (hy * (hz * a000[e] + lz * a001[e]) + ly * (hz * a010[e] + lz * a011[e])) +
                          lx * (hy * (hz * a100[e] + lz * a101[e]) + ly * (hz * a110[e] + lz * a111[e]));
        if (q4 + e < Q && val > best) { best = val; arg = q4 + e; }
      }
    }
  }
  qidx[(size_t)b * Vo + v] = (unsigned char)arg;
  int* pf = present + (size_t)b * Qs + arg;
  if (__ldcg(pf) == 0) *pf = 1;  // benign race: every writer stores 1
}

// pass 1b: thread = LiDAR point of sample blockIdx.y (n points per sample); grid_sample of the native logits
__global__ void __launch_bounds__(128)
panoptic_pts_argmax_kernel(const float* __restrict__ mask, int Qs, int Q, int X, int Y, int Z,
                           const float* __restrict__ pts, int pts_stride, int n, float x_min, float y_min, float z_min,
                           float x_ext, float y_ext, float z_ext, int border, unsigned char* __restrict__ qidx,
                           int* __restrict__ present) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const SamplePos sp = grid_sample_pos(pts + ((size_t)b * n + i) * pts_stride, x_min, y_min, z_min, x_ext, y_ext, z_ext,
                                       X, Y, Z, border);
  const float* mb = mask + (size_t)b * X * Y * Z * Qs;
  const float4* pc[8];
  float w[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int xx = sp.x0 + (c >> 2), yy = sp.y0 + ((c >> 1) & 1), zz = sp.z0 + (c & 1);
    const bool in = xx >= 0 && xx < X && yy >= 0 && yy < Y && zz >= 0 && zz < Z;
    w[c] = in ? ((c >> 2) ? sp.lx : 1.f - sp.lx) * (((c >> 1) & 1) ? sp.ly : 1.f - sp.ly) * ((c & 1) ? sp.lz : 1.f - sp.lz)
              : 0.f;
    pc[c] = reinterpret_cast<const float4*>(mb + (in ? (((size_t)xx * Y + yy) * Z + zz) * Qs : 0));
  }
  float best = -INFINITY;
  int arg = 0;
  for (int q4 = 0; q4 < Qs; q4 += 4) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float4 t = __ldg(pc[c] + (q4 >> 2));
      a.x += w[c] * t.x; a.y += w[c] * t.y; a.z += w[c] * t.z; a.w += w[c] * t.w;
    }
    const float val[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int e = 0; e < 4; ++e)
      if (q4 + e < Q && val[e] > best) { best = val[e]; arg = q4 + e; }
  }
  qidx[(size_t)b * n + i] = (unsigned char)arg;
  int* pf = present + (size_t)b * Qs + arg;
  if (__ldcg(pf) == 0) *pf = 1;
}

// pass 2: CTA = sample, thread = query.  label(q) = argmax_{k0 <= k < NC-1} softmax(cls[q])[k] (k0 = 0 voxels, 1 points);
// a thing query that wins somewhere is instance 1 + #(winning thing queries ordered before it by (label, query)).
constexpr int PAN_MAXQ = 256;
__global__ void __launch_bounds__(PAN_MAXQ)
panoptic_table_kernel(const float* __restrict__ cls, int Q, int Qs, int NC, int k0, unsigned long long thing,
                      const int* __restrict__ present, long long* __restrict__ table /*(B, Qs, 2)*/) {
  __shared__ int lab[PAN_MAXQ], win[PAN_MAXQ];
  const int b = blockIdx.x, q = threadIdx.x;
  int label = 0;
  if (q < Q) {
    const float* c = cls + ((size_t)b * Q + q) * NC;
    float m = -INFINITY;
    for (int k = 0; k < NC; ++k) m = fmaxf(m, c[k]);
    float s = 0.f;
    for (int k = 0; k < NC; ++k) s += expf(c[k] - m);
    float best = -INFINITY;
    label = k0;
    for (int k = k0; k < NC - 1; ++k) {
      const float p = expf(c[k] - m) / s;
      if (p > best) { best = p; label = k; }
    }
  }
  const bool is_thing = (thing >> label) & 1ull;
  lab[q] = label;
  win[q] = q < Q && is_thing && present[(size_t)b * Qs + q] != 0;
  __syncthreads();
  if (q >= Q) return;
  long long pan = (long long)label * 1000;
  if (is_thing) {
    int id = 1;
    for (int r = 0; r < Q; ++r) id += win[r] && (lab[r] < label || (lab[r] == label && r < q));
    pan += id;
  }
  table[((size_t)b * Qs + q) * 2] = label;
  table[((size_t)b * Qs + q) * 2 + 1] = pan;
}

// pass 3: thread = voxel / point: (semantic, panoptic) of its query
__global__ void panoptic_map_kernel(const unsigned char* __restrict__ qidx, long long n, int Qs,
                                    const long long* __restrict__ table, long long* __restrict__ sem,
                                    long long* __restrict__ pan) {
  const int b = blockIdx.y;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t o = (size_t)b * n + i;
  const longlong2 t = *reinterpret_cast<const longlong2*>(table + ((size_t)b * Qs + qidx[o]) * 2);
  __stcs(sem + o, t.x);
  __stcs(pan + o, t.y);
}

// passes 2 and 3 after a pass 1 that filled qidx (B, n) and present (B, Qs)
static int panoptic_finish(const float* cls, int B, int Q, int Qs, int NC, int k0, unsigned long long thing,
                           const unsigned char* qidx, const int* present, long long* table, long long n,
                           long long* sem, long long* pan, cudaStream_t stream) {
  panoptic_table_kernel<<<B, PAN_MAXQ, 0, stream>>>(cls, Q, Qs, NC, k0, thing, present, table);
  OCC_LAUNCH_CHECK();
  panoptic_map_kernel<<<dim3((unsigned)((n + 255) / 256), B), 256, 0, stream>>>(qidx, n, Qs, table, sem, pan);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

}  // namespace occ

using namespace occ;

extern "C" int occ_sine_pos3d(float* out, int X, int Y, int Z, int num_feats, float temperature, float scale,
                              float eps, float offset, cudaStream_t stream) {
  OCC_REQUIRE(out && X > 0 && Y > 0 && Z > 0 && num_feats > 0);
  const long long total = (long long)X * Y * Z * 3 * num_feats;
  sine_pos3d_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(out, X, Y, Z, num_feats, temperature, scale, eps,
                                                                        offset);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_head_prep(const float* in, int in_channel_last, const float* level_embed, const float* pos,
                             float* mem, float* kpos, int B, long long S, int C, cudaStream_t stream) {
  OCC_REQUIRE(in && mem && B > 0 && S > 0 && C > 0 && C % 32 == 0);  // S32 output rows
  OCC_REQUIRE((kpos == nullptr) == (pos == nullptr));
  if (in_channel_last) {
    const long long n4 = (long long)B * S * (C / 4);
    head_prep_cl_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(in, level_embed, pos, mem, kpos,
                                                                         (long long)B * S, S, C);
  } else {
    OCC_REQUIRE((S + 31) / 32 < (1ll << 31) && B <= 65535 && (C + 31) / 32 <= 65535);
    dim3 grid((unsigned)((S + 31) / 32), (C + 31) / 32, B), block(32, 8);
    head_prep_ncs_kernel<<<grid, block, 0, stream>>>(in, level_embed, pos, mem, kpos, S, C);
  }
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_query_head(const float* query_in, const float* n2w, const float* n2b, float* query_state,
                              const float* pn_w, const float* pn_b, const float* clsT, const float* cls_b, int NC,
                              const float* m0T, const float* m0b, const float* m1T, const float* m1b, const float* m2T,
                              const float* m2b, float* cls_out, float* membed_out, const float* query_pos, int Q,
                              const float* wqT, const float* bq, float scale, float* qh_out, const float* ffn_part,
                              int nparts, int rows, int E, cudaStream_t stream) {
  OCC_REQUIRE(query_in && pn_w && pn_b && clsT && cls_b && m0T && m0b && m1T && m1b && m2T && m2b && cls_out && membed_out);
  OCC_REQUIRE(rows > 0 && rows % QG == 0 && E % 32 == 0 && E <= 256 && NC > 0 && NC <= E);
  OCC_REQUIRE((n2w == nullptr) == (n2b == nullptr) && (n2w == nullptr || query_state != nullptr));
  OCC_REQUIRE(wqT == nullptr || (bq && query_pos && qh_out && Q > 0));
  OCC_REQUIRE(nparts >= 0 && (nparts == 0 || ffn_part != nullptr));
  const size_t smem = ((QG + QG * QG) * E + 32) * sizeof(float);
  query_head_kernel<<<rows / QG, E * QG, smem, stream>>>(query_in, n2w, n2b, query_state, pn_w, pn_b, clsT, cls_b, NC, m0T,
                                                         m0b, m1T, m1b, m2T, m2b, cls_out, membed_out, query_pos, Q, wqT,
                                                         bq, scale, qh_out, ffn_part, nparts, rows, E);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_mask_pool(const float* mask, int* pooled, int* row_flag, int B, int X, int Y, int Z, int Xo,
                             int Yo, int Zo, int Q, cudaStream_t stream) {
  OCC_REQUIRE(mask && pooled && row_flag && B > 0 && X > 0 && Y > 0 && Z > 0 && Xo > 0 && Yo > 0 && Zo > 0 && Q > 0);
  OCC_REQUIRE(Xo <= X && Yo <= Y && Zo <= Z);
  OCC_MEMSET(row_flag, 0, (size_t)B * Q * sizeof(int), stream);
  OCC_REQUIRE(Q <= 256 && (long long)B * Xo * Yo * Zo < (1ll << 31));
  OCC_REQUIRE(X < 32768 && Y < 32768 && Z < 32768);
  long long blocks = ((long long)B * Xo * Yo * Zo + 3) / 4;
  const long long cap = (long long)sm_count() * 16;
  if (blocks > cap) blocks = cap;
  mask_pool_kernel<<<dim3((unsigned)blocks, (Q + 127) / 128), dim3(128, 4), 0, stream>>>(mask, pooled, row_flag, B, X, Y,
                                                                                          Z, Xo, Yo, Zo, Q);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_cross_merge(const float* part, int nchunk, int H, const float* query, const float* query_pos, int Q,
                               const float* woT, const float* bo, const float* n0w, const float* n0b,
                               const float* sa_inT, const float* sa_inb, float scale, float* query1, float* sa_qkv,
                               int rows, int E, cudaStream_t stream) {
  OCC_REQUIRE(part && query && query_pos && woT && bo && n0w && n0b && sa_inT && sa_inb && query1 && sa_qkv);
  OCC_REQUIRE(rows > 0 && rows % QG == 0 && Q > 0 && E == H * XA_HD && E <= 256 && nchunk > 0);
  const size_t smem = ((2 * QG + QG * QG) * E + 32) * sizeof(float);
  cross_merge_kernel<<<rows / QG, E * QG, smem, stream>>>(
      part, nchunk, H, query, query_pos, Q, woT, bo, n0w, n0b, sa_inT, sa_inb, scale, query1, sa_qkv, rows, E);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_self_attn_ffn(const float* sa_qkv, const float* query1, int Q, int nkeys, const float* woT,
                                 const float* bo, const float* n1w, const float* n1b, const float* f1T, const float* f1b,
                                 const float* f2T, const float* f2b, int F, float* x1, float* ybuf, float* ffn_part,
                                 int rows, int E, int H, cudaStream_t stream) {
  OCC_REQUIRE(E == H * XA_HD);
  OCC_REQUIRE(sa_qkv && query1 && woT && bo && n1w && n1b && f1T && f1b && f2T && f2b && x1 && ybuf && ffn_part);
  OCC_REQUIRE(rows > 0 && rows % QG == 0 && Q > 0 && Q <= 256 && nkeys > 0 && nkeys <= Q && E % 32 == 0 && E <= 256 &&
              F > 0 && F % E == 0 && rows % Q == 0 && F / E <= 65535);
  const size_t smem = ((QG + QG * QG) * E + 32) * sizeof(float);
  if (Q <= 128)
    self_attn_kernel<4><<<rows / QG, E * QG, smem, stream>>>(sa_qkv, query1, nkeys, Q, woT, bo, n1w, n1b, f2b, x1, ybuf, E);
  else
    self_attn_kernel<8><<<rows / QG, E * QG, smem, stream>>>(sa_qkv, query1, nkeys, Q, woT, bo, n1w, n1b, f2b, x1, ybuf, E);
  OCC_LAUNCH_CHECK();
  const size_t smem2 = (2 * QG + QG * QG) * E * sizeof(float);
  ffn_block_kernel<<<dim3(rows / QG, F / E), E * QG, smem2, stream>>>(x1, f1T, f1b, f2T, F, ffn_part, E);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_classmix(const float* mask, int Qs, const float* cls, float* out, unsigned char* labels, int B, int X,
                            int Y, int Z, int Xo, int Yo, int Zo, int Q, int NC, cudaStream_t stream) {
  OCC_REQUIRE(mask && cls && out && B > 0 && X > 0 && Y > 0 && Z > 0 && Xo > 0 && Yo > 0 && Zo > 0 && Q > 0);
  OCC_REQUIRE(NC >= 2 && NC - 1 <= 32 && B <= 65535);
  const long long Vo = (long long)Xo * Yo * Zo;
  const int kmax = (NC - 1 <= 20) ? 20 : 32;
  OCC_REQUIRE(Qs % 4 == 0 && Q <= Qs);
  const size_t smem = (size_t)Qs * kmax * sizeof(float);
  OCC_REQUIRE(smem <= 200 * 1024);
  dim3 grid((unsigned)((Vo + CM_THREADS - 1) / CM_THREADS), B);
  if (NC - 1 <= 20) {
    OCC_ENSURE_SMEM(classmix_kernel<20>, 200 * 1024);
    classmix_kernel<20><<<grid, CM_THREADS, smem, stream>>>(mask, cls, out, labels, X, Y, Z, Xo, Yo, Zo, Qs, Q, NC);
  } else {
    OCC_ENSURE_SMEM(classmix_kernel<32>, 200 * 1024);
    classmix_kernel<32><<<grid, CM_THREADS, smem, stream>>>(mask, cls, out, labels, X, Y, Z, Xo, Yo, Zo, Qs, Q, NC);
  }
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_transpose_sq(const float* in, float* out, int B, long long S, int Q, cudaStream_t stream) {
  OCC_REQUIRE(in && out && B > 0 && S > 0 && Q > 0 && B <= 65535);
  dim3 grid((unsigned)((S + 31) / 32), (Q + 31) / 32, B), block(32, 8);
  transpose_sq_kernel<<<grid, block, 0, stream>>>(in, out, S, Q);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_lidarseg_points(const float* vox, const float* pts, int pts_stride, int n, float x_min, float y_min,
                                   float z_min, float x_max, float y_max, float z_max, int X, int Y, int Z, int K,
                                   int border, float* out, cudaStream_t stream) {
  OCC_REQUIRE(vox && out && n >= 0 && X > 0 && Y > 0 && Z > 0 && K > 0 && K <= 32 && pts_stride >= 3);
  if (n == 0) return OCC_OK;
  OCC_REQUIRE(pts != nullptr);
  lidarseg_kernel<<<(n + 127) / 128, 128, 0, stream>>>(vox, pts, pts_stride, n, x_min, y_min, z_min, x_max - x_min,
                                                       y_max - y_min, z_max - z_min, X, Y, Z, K, border, out);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_panoptic_voxels(const float* mask, int Qs, const float* cls, int B, int X, int Y, int Z, int Xo, int Yo,
                                   int Zo, int Q, int NC, unsigned long long thing_mask, int first_label,
                                   unsigned char* qidx, int* present, long long* table, long long* sem, long long* pan,
                                   cudaStream_t stream) {
  OCC_REQUIRE(mask && cls && qidx && present && table && sem && pan);
  OCC_REQUIRE(B > 0 && B <= 65535 && X > 0 && Y > 0 && Z > 0 && Xo > 0 && Yo > 0 && Zo > 0);
  OCC_REQUIRE(Q > 0 && Q <= Qs && Qs <= PAN_MAXQ && Qs % 4 == 0 && NC - 1 <= 63);
  OCC_REQUIRE((first_label == 0 || first_label == 1) && NC - 1 > first_label);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(mask) & 15) == 0 && (reinterpret_cast<uintptr_t>(table) & 15) == 0);
  const long long Vo = (long long)Xo * Yo * Zo;
  OCC_REQUIRE((Vo + 127) / 128 < (1ll << 31));
  OCC_MEMSET(present, 0, (size_t)B * Qs * sizeof(int), stream);
  panoptic_vox_argmax_kernel<<<dim3((unsigned)((Vo + 127) / 128), B), 128, 0, stream>>>(mask, Qs, Q, X, Y, Z, Xo, Yo, Zo,
                                                                                       qidx, present);
  OCC_LAUNCH_CHECK();
  return panoptic_finish(cls, B, Q, Qs, NC, first_label, thing_mask, qidx, present, table, Vo, sem, pan, stream);
}

extern "C" int occ_panoptic_points(const float* mask, int Qs, const float* cls, int B, int X, int Y, int Z, int Q, int NC,
                                   unsigned long long thing_mask, const float* pts, int pts_stride, int n, float x_min,
                                   float y_min, float z_min, float x_max, float y_max, float z_max, int border,
                                   unsigned char* qidx, int* present, long long* table, long long* sem, long long* pan,
                                   cudaStream_t stream) {
  OCC_REQUIRE(mask && cls && qidx && present && table && sem && pan && (n == 0 || pts));
  OCC_REQUIRE(B > 0 && B <= 65535 && X > 0 && Y > 0 && Z > 0 && n >= 0 && pts_stride >= 3);
  OCC_REQUIRE(Q > 0 && Q <= Qs && Qs <= PAN_MAXQ && Qs % 4 == 0 && NC >= 3 && NC - 1 <= 63);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(mask) & 15) == 0 && (reinterpret_cast<uintptr_t>(table) & 15) == 0);
  if (n == 0) return OCC_OK;
  OCC_MEMSET(present, 0, (size_t)B * Qs * sizeof(int), stream);
  panoptic_pts_argmax_kernel<<<dim3((n + 127) / 128, B), 128, 0, stream>>>(
      mask, Qs, Q, X, Y, Z, pts, pts_stride, n, x_min, y_min, z_min, x_max - x_min, y_max - y_min, z_max - z_min, border,
      qidx, present);
  OCC_LAUNCH_CHECK();
  return panoptic_finish(cls, B, Q, Qs, NC, 1, thing_mask, qidx, present, table, n, sem, pan, stream);
}
