// LSS lift-splat voxel pooling for sm_90a (HBM-bound; output-stationary, every grid row written once by its warp).
//
// Reference path replaced (files of the reference checkout):
//   projects/mmdet3d_plugin/occformer/image2bev/ViewTransformerLSSVoxel.py:77-100 (voxel_pooling: index,
//     kept mask, boolean-mask gathers), :110-115 (lift: depth softmax (x) context, 242 MB volume),
//   mmdetection3d/mmdet3d/ops/bev_pool/bev_pool.py:83-97 (rank, argsort, 3 gathers, interval bookkeeping),
//   mmdetection3d/mmdet3d/ops/bev_pool/src/bev_pool_cuda.cu:20-42 (interval-sum kernel) + the
//     (B,Z,X,Y,C)->(B,C,Z,X,Y) transpose copy (bev_pool.py:96).
//
// Pipeline (all on the caller's stream, no allocation, no sync) -- one memset + two kernels:
//   memset  : head[V] = 0 (empty), counts[V] = 0.
//   index   : one thread per frustum point: exact fp32 voxel index ((g - (bx - dx/2)) / dx, trunc toward 0),
//             kept test against float nx, linear voxel id; the point is pushed onto its voxel's list
//             (next[p] = atomicExch(&head[v], p + 1)) and counted (the reference's interval length).  No sort,
//             no scan: the reference's argsort + interval bookkeeping (bev_pool.py:86-93) only groups points by voxel.
//   pool    : a warp owns 32 consecutive voxels.  The rows of the empty ones (most of a nuScenes grid) are streamed
//             out as zeros first.  Then, in rounds of four hops, every lane advances its own voxel's list
//             (lane-parallel pointer chase) and the warp sums depth[p] * feat[pixel(p), :] (fused lift: the volume is
//             never materialised) or rows of a materialised feats[n, C] (drop-in bev_pool), four voxels at a time so
//             that 8-16 row loads are in flight; a voxel with more than four points accumulates into its own row in
//             the following rounds.  (Near-camera voxels hold up to ~60 points and sit next to each other: walking
//             those lists one hop at a time per warp leaves a long tail.)
// Output layout is channel-last (B, X, Y, Z, C); the Python boundary returns permuted views with the
// reference's shapes.
#include "occ_common.cuh"
#include "occ_ptx.cuh"

namespace occ {

// ------------------------------------------------------------------------------------------------ index
// geom: (P,3) fp32 ego coordinates of frustum point p = ((b*N+n)*D+d)*fH*fW + pix.  vox_id[p] = linear voxel
// id ((b*X+x)*Y+y)*Z+z or -1 when dropped.
struct VpGrid {
  float dx0, dx1, dx2, bx0, bx1, bx2, nx0, nx1, nx2;
  int X, Y, Z;
};

// ego point -> linear voxel id of sample b (or -1 when dropped), the reference's index arithmetic bit for bit
__device__ __forceinline__ int vp_voxel_of(float gx, float gy, float gz, int b, const VpGrid& g) {
  // ViewTransformerLSSVoxel.py:84 -- fp32 sub, fp32 div (IEEE, no contraction), .long() truncation
  const float ox = __fsub_rn(g.bx0, __fdiv_rn(g.dx0, 2.0f));
  const float oy = __fsub_rn(g.bx1, __fdiv_rn(g.dx1, 2.0f));
  const float oz = __fsub_rn(g.bx2, __fdiv_rn(g.dx2, 2.0f));
  const long long ix = (long long)__fdiv_rn(__fsub_rn(gx, ox), g.dx0);
  const long long iy = (long long)__fdiv_rn(__fsub_rn(gy, oy), g.dx1);
  const long long iz = (long long)__fdiv_rn(__fsub_rn(gz, oz), g.dx2);
  // :90-92 -- int64 index compared with the *float* nx, upper bound exclusive
  const bool kept = ix >= 0 && (float)ix < g.nx0 && iy >= 0 && (float)iy < g.nx1 && iz >= 0 && (float)iz < g.nx2 &&
                    ix < g.X && iy < g.Y && iz < g.Z;
  return kept ? ((b * g.X + (int)ix) * g.Y + (int)iy) * g.Z + (int)iz : -1;
}

// push point p onto the list of voxel v (1-based ids: 0 = end of list / empty voxel) and count it
__device__ __forceinline__ void vp_push(int p, int v, int* __restrict__ vox_id, int* __restrict__ counts,
                                        int* __restrict__ head, int* __restrict__ next) {
  if (v >= 0) {
    atomicAdd(&counts[v], 1);
    next[p] = atomicExch(&head[v], p + 1);
  }
  vox_id[p] = v;
}

__global__ void vp_index_geom_kernel(const float* __restrict__ geom, int P, int points_per_batch, const VpGrid g,
                                     int* __restrict__ vox_id, int* __restrict__ counts, int* __restrict__ head,
                                     int* __restrict__ next) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int v = vp_voxel_of(geom[3 * (size_t)p + 0], geom[3 * (size_t)p + 1], geom[3 * (size_t)p + 2],
                            p / points_per_batch, g);
  vp_push(p, v, vox_id, counts, head, next);
}

// coords: (n,4) int64 (x,y,z,b) as handed to mmdet3d.ops.bev_pool.bev_pool (already range-filtered by the
// caller in the reference; we re-check and drop out-of-range rows instead of writing out of bounds).
__global__ void vp_index_coords_kernel(const long long* __restrict__ coords, int n, int B, int X, int Y, int Z,
                                       int* __restrict__ vox_id, int* __restrict__ counts, int* __restrict__ head,
                                       int* __restrict__ next) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const long long x = coords[4 * (size_t)p + 0], y = coords[4 * (size_t)p + 1], z = coords[4 * (size_t)p + 2],
                  b = coords[4 * (size_t)p + 3];
  int v = -1;
  if (x >= 0 && x < X && y >= 0 && y < Y && z >= 0 && z < Z && b >= 0 && b < B) {
    v = (((int)b * X + (int)x) * Y + (int)y) * Z + (int)z;
    atomicAdd(&counts[v], 1);
    next[p] = atomicExch(&head[v], p + 1);
  }
  vox_id[p] = v;
}

// ------------------------------------------------------------------------------------------------ pool
// Exact unsigned division of n < 2^31 by a runtime constant: q = (n * mul) >> sh with mul = ceil(2^sh / d),
// sh = 31 + ceil(log2 d) (error term n * (mul*d - 2^sh) < 2^31 * d <= 2^sh).
struct FastDiv {
  uint32_t mul, sh, d;
};
static FastDiv make_fastdiv(uint32_t d) {
  FastDiv f;
  uint32_t s = 0;
  while ((1ull << s) < d) ++s;
  f.sh = 31 + s;
  f.mul = (uint32_t)(((1ull << f.sh) + d - 1) / d);
  f.d = d;
  return f;
}
__device__ __forceinline__ uint32_t fast_div(uint32_t n, const FastDiv& f) {
  return (uint32_t)(((unsigned long long)n * f.mul) >> f.sh);
}

// MODE 0: fused lift  row(p) = depth_prob[p] * feat_cl[pixel(p), :]
// MODE 1: materialised rows feats[p, :]
// One warp owns 32 consecutive voxels (one z-column pair).  Empty voxels get their zero row streamed first; then
// every lane walks the list of its own voxel (independent chains: the hop latencies overlap across lanes), and the
// occupied voxels are reduced four at a time so that 8-16 row loads are in flight per warp.
template <int MODE>
__global__ void __launch_bounds__(256)
vp_pool_kernel(const int* __restrict__ head, const int* __restrict__ next, int V, int C,
               const float* __restrict__ depth_prob, const float* __restrict__ feat, FastDiv div_dhw, FastDiv div_hw,
               float* __restrict__ out, float* __restrict__ out_split /*optional S32 copy of the grid (conv operand)*/) {
  const int lane = threadIdx.x & 31;
  const int C4 = C >> 2;
  const int batch = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int vb = batch << 5;
  if (vb >= V) return;
  const int nv = min(32, V - vb);
  const int h0 = lane < nv ? __ldg(head + vb + lane) : 0;
  const uint32_t valid = nv == 32 ? 0xffffffffu : ((1u << nv) - 1u);
  const uint32_t occupied = __ballot_sync(0xffffffffu, h0 != 0);
  {
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    for (uint32_t e = valid & ~occupied; e != 0u; e &= e - 1u) {
      float4* orow = reinterpret_cast<float4*>(out + (size_t)(vb + __ffs(e) - 1) * C);
      for (int c4 = lane; c4 < C4; c4 += 32) __stcs(orow + c4, z4);
      if (out_split) {  // an all-zero row is its own S32 image
        float4* srow = reinterpret_cast<float4*>(out_split + (size_t)(vb + __ffs(e) - 1) * C);
        for (int c4 = lane; c4 < C4; c4 += 32) __stcs(srow + c4, z4);
      }
    }
  }
  if (occupied == 0u) return;
  // Rounds of four hops: every lane advances the list of its own voxel (independent chains, the hop latencies
  // overlap across lanes), then the warp reduces the voxels that gained points this round, four voxels at a time
  // (8-16 row loads in flight).  Voxels with more than four points continue in the next round and accumulate
  // into their own output row (same lane wrote it: program order makes the partial sum visible).
  int cur = h0;
  bool first = true;
  while (true) {
    int frow[4];
    float wgt[4];
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      frow[j] = 0;
      wgt[j] = 0.f;
      if (cur != 0) {
        const uint32_t p = (uint32_t)cur - 1u;
        // MODE 0: p = ((bn*D + d)*HW + pix) -> feature row bn*HW + pix;  MODE 1: row p
        if (MODE == 0) {
          const uint32_t bn = fast_div(p, div_dhw);
          const uint32_t pix = p - fast_div(p, div_hw) * div_hw.d;
          frow[j] = (int)(bn * div_hw.d + pix);
          wgt[j] = __ldg(depth_prob + p);
        } else {
          frow[j] = (int)p;
          wgt[j] = 1.f;
        }
        cur = __ldg(next + p);
        ++cnt;
      }
    }
    const uint32_t occ_round = __ballot_sync(0xffffffffu, cnt > 0);
    const bool any_gt2 = __any_sync(0xffffffffu, cnt > 2);
    for (int cbase = 0; cbase < C4; cbase += 32) {
      const int c4 = cbase + lane;
      const bool active = c4 < C4;
      const float4* fbase = reinterpret_cast<const float4*>(feat) + c4;
      uint32_t occ = occ_round;
      while (occ) {
        int vi[4];
        bool ok[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          ok[u] = occ != 0u;
          vi[u] = ok[u] ? __ffs(occ) - 1 : 0;
          occ &= occ - 1u;  // 0 stays 0
        }
        float4 acc[4];
        int n[4];
        bool fin[4];  // the voxel's list ended in this round: its sum is final
        {
          int r0[4], r1[4];
          float w0[4], w1[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            n[u] = __shfl_sync(0xffffffffu, cnt, vi[u]);
            fin[u] = __shfl_sync(0xffffffffu, cur, vi[u]) == 0;
            r0[u] = __shfl_sync(0xffffffffu, frow[0], vi[u]);
            w0[u] = __shfl_sync(0xffffffffu, wgt[0], vi[u]);
            r1[u] = __shfl_sync(0xffffffffu, frow[1], vi[u]);
            w1[u] = __shfl_sync(0xffffffffu, wgt[1], vi[u]);
            if (!ok[u]) n[u] = 0;
          }
          float4 f0[4], f1[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            f0[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            f1[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (n[u] > 0 && active) f0[u] = __ldg(fbase + (size_t)r0[u] * C4);
            if (n[u] > 1 && active) f1[u] = __ldg(fbase + (size_t)r1[u] * C4);
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            acc[u].x = w0[u] * f0[u].x + w1[u] * f1[u].x;
            acc[u].y = w0[u] * f0[u].y + w1[u] * f1[u].y;
            acc[u].z = w0[u] * f0[u].z + w1[u] * f1[u].z;
            acc[u].w = w0[u] * f0[u].w + w1[u] * f1[u].w;
          }
        }
        if (any_gt2) {
          int r2[4], r3[4];
          float w2[4], w3[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            r2[u] = __shfl_sync(0xffffffffu, frow[2], vi[u]);
            w2[u] = __shfl_sync(0xffffffffu, wgt[2], vi[u]);
            r3[u] = __shfl_sync(0xffffffffu, frow[3], vi[u]);
            w3[u] = __shfl_sync(0xffffffffu, wgt[3], vi[u]);
          }
          float4 f2[4], f3[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            f2[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            f3[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (n[u] > 2 && active) f2[u] = __ldg(fbase + (size_t)r2[u] * C4);
            if (n[u] > 3 && active) f3[u] = __ldg(fbase + (size_t)r3[u] * C4);
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            acc[u].x += w2[u] * f2[u].x + w3[u] * f3[u].x;
            acc[u].y += w2[u] * f2[u].y + w3[u] * f3[u].y;
            acc[u].z += w2[u] * f2[u].z + w3[u] * f3[u].z;
            acc[u].w += w2[u] * f2[u].w + w3[u] * f3[u].w;
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (ok[u] && active) {
            float4* dst = reinterpret_cast<float4*>(out + (size_t)(vb + vi[u]) * C) + c4;
            if (!first) {
              const float4 o = *dst;
              acc[u].x += o.x; acc[u].y += o.y; acc[u].z += o.z; acc[u].w += o.w;
            }
            *dst = acc[u];
            if (out_split && fin[u]) store_split4(out_split + (size_t)(vb + vi[u]) * C, c4 * 4, acc[u]);
          }
        }
      }
    }
    first = false;
    if (!__any_sync(0xffffffffu, cur != 0)) break;
  }
}

// ------------------------------------------------------------------------------------------------ lift prologue
// depth softmax over D for every (camera, pixel): logits (BN, D, HW) -> prob (BN, D, HW)
__global__ void vp_depth_softmax_kernel(const float* __restrict__ logits, int BN, int D, int HW,
                                        float* __restrict__ prob) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= BN * HW) return;
  const int bn = i / HW, pix = i % HW;
  const float* src = logits + (size_t)bn * D * HW + pix;
  float* dst = prob + (size_t)bn * D * HW + pix;
  float m = -INFINITY;
  for (int d = 0; d < D; ++d) m = fmaxf(m, src[(size_t)d * HW]);
  float s = 0.f;
  for (int d = 0; d < D; ++d) s += expf(src[(size_t)d * HW] - m);
  for (int d = 0; d < D; ++d) dst[(size_t)d * HW] = expf(src[(size_t)d * HW] - m) / s;
}

// (BN, C, HW) -> (BN, HW, C)
__global__ void vp_nchw_to_nhwc_kernel(const float* __restrict__ in, int C, int HW, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int bn = blockIdx.z;
  const int c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, p = p0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < C && p < HW) ? in[((size_t)bn * C + c) * HW + p] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int p = p0 + i, c = c0 + threadIdx.x;
    if (p < HW && c < C) out[((size_t)bn * HW + p) * C + c] = tile[threadIdx.x][i];
  }
}

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Launch grid sizes in 64-bit: n + per - 1 overflows int within per of the 2^31 limit the entry points allow.
static unsigned blocks_for(long long n, long long per) { return (unsigned)((n + per - 1) / per); }
// vp_pool_kernel: one warp per 32 voxels, 8 warps per block
static unsigned pool_blocks(int V) { return blocks_for(blocks_for(V, 32), 8); }

struct VpWorkspace {
  int *head, *counts, *next, *vox_id;  // head and counts are adjacent: one memset clears both
};

static size_t vp_layout(void* base, int P, int V, VpWorkspace* ws) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    void* p = base ? static_cast<char*>(base) + off : nullptr;
    off += align_up(bytes, 256);
    return static_cast<int*>(p);
  };
  ws->head = take((size_t)V * 4);
  ws->counts = take((size_t)V * 4);
  ws->next = take((size_t)P * 4);
  ws->vox_id = take((size_t)P * 4);
  return off;
}

}  // namespace occ

using namespace occ;

extern "C" size_t occ_voxel_pool_workspace_bytes(int n_points, int B, int X, int Y, int Z) {
  VpWorkspace ws;
  return vp_layout(nullptr, n_points, B * X * Y * Z, &ws);
}

// Fused lift-splat.  depth_prob (B*N, D, fH*fW) fp32 (already softmaxed), feat_cl (B*N, fH*fW, C) channel-last,
// geom (B*N*D*fH*fW, 3).  out (B, X, Y, Z, C) fp32; out_split (optional): the same grid in the S32 split format (the
// operand of the encoder's first conv).  Bookkeeping left in the workspace: vox_id[P], counts[V], head[V], next[P].
extern "C" int occ_lift_splat(const float* depth_prob, const float* feat_cl, const float* geom, float* out,
                              float* out_split, int B, int N, int D, int HW, int C, float dx0, float dx1, float dx2,
                              float bx0, float bx1, float bx2, float nx0, float nx1, float nx2, int X, int Y, int Z,
                              void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  OCC_REQUIRE(depth_prob && feat_cl && geom && out && workspace);
  OCC_REQUIRE(!out_split || C % 32 == 0);
  OCC_REQUIRE(B > 0 && N > 0 && D > 0 && HW > 0 && C > 0 && C % 4 == 0 && X > 0 && Y > 0 && Z > 0);
  const long long Pll = (long long)B * N * D * HW, Vll = (long long)B * X * Y * Z;
  OCC_REQUIRE(Pll < (1ll << 31) && Vll < (1ll << 31));
  const int P = (int)Pll, V = (int)Vll;
  VpWorkspace ws;
  OCC_REQUIRE(vp_layout(workspace, P, V, &ws) <= workspace_bytes);
  // head[V] and counts[V] are adjacent in the workspace: one memset
  OCC_MEMSET(ws.head, 0, reinterpret_cast<char*>(ws.counts + V) - reinterpret_cast<char*>(ws.head), stream);
  const VpGrid vg{dx0, dx1, dx2, bx0, bx1, bx2, nx0, nx1, nx2, X, Y, Z};
  vp_index_geom_kernel<<<blocks_for(P, 256), 256, 0, stream>>>(geom, P, N * D * HW, vg, ws.vox_id, ws.counts, ws.head, ws.next);
  OCC_LAUNCH_CHECK();
  vp_pool_kernel<0><<<pool_blocks(V), 256, 0, stream>>>(ws.head, ws.next, V, C, depth_prob, feat_cl,
                                                        make_fastdiv((uint32_t)D * HW), make_fastdiv(HW), out, out_split);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// Drop-in for mmdet3d.ops.bev_pool.bev_pool: feats (n, C), coords (n, 4) int64 (x, y, z, b).
// out (B, X, Y, Z, C)  [reference returns the same values as (B, C, Z, X, Y)].
extern "C" int occ_bev_pool(const float* feats, const long long* coords, float* out, int n, int C, int B, int X,
                            int Y, int Z, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
  OCC_REQUIRE(out && workspace);
  OCC_REQUIRE(n >= 0 && C > 0 && C % 4 == 0 && B > 0 && X > 0 && Y > 0 && Z > 0);
  OCC_REQUIRE(n == 0 || (feats && coords));
  const long long Vll = (long long)B * X * Y * Z;
  OCC_REQUIRE(Vll < (1ll << 31));
  const int V = (int)Vll;
  VpWorkspace ws;
  OCC_REQUIRE(vp_layout(workspace, n, V, &ws) <= workspace_bytes);
  OCC_MEMSET(ws.head, 0, reinterpret_cast<char*>(ws.counts + V) - reinterpret_cast<char*>(ws.head), stream);
  if (n > 0) {
    vp_index_coords_kernel<<<blocks_for(n, 256), 256, 0, stream>>>(coords, n, B, X, Y, Z, ws.vox_id, ws.counts, ws.head,
                                                                  ws.next);
    OCC_LAUNCH_CHECK();
  }
  vp_pool_kernel<1><<<pool_blocks(V), 256, 0, stream>>>(ws.head, ws.next, V, C, nullptr, feats, make_fastdiv(1),
                                                        make_fastdiv(1), out, nullptr);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// Lift prologue: depth softmax + NCHW->NHWC of the context features (ViewTransformerLSSVoxel.py:108-110).
extern "C" int occ_lift_prologue(const float* depth_logits, const float* img_feat, float* depth_prob,
                                 float* feat_cl, int BN, int D, int C, int HW, cudaStream_t stream) {
  OCC_REQUIRE(depth_logits && img_feat && depth_prob && feat_cl && BN > 0 && D > 0 && C > 0 && HW > 0);
  vp_depth_softmax_kernel<<<blocks_for((long long)BN * HW, 128), 128, 0, stream>>>(depth_logits, BN, D, HW, depth_prob);
  OCC_LAUNCH_CHECK();
  dim3 grid(blocks_for(HW, 32), blocks_for(C, 32), BN), block(32, 8);
  vp_nchw_to_nhwc_kernel<<<grid, block, 0, stream>>>(img_feat, C, HW, feat_cl);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// Byte offsets of the bookkeeping arrays inside the workspace (for tests / callers that want them).
extern "C" int occ_voxel_pool_workspace_layout(int n_points, int B, int X, int Y, int Z, size_t* off_counts,
                                               size_t* off_head, size_t* off_next, size_t* off_vox_id) {
  VpWorkspace ws;
  char* base = reinterpret_cast<char*>(0x1000);
  vp_layout(base, n_points, B * X * Y * Z, &ws);
  *off_counts = reinterpret_cast<char*>(ws.counts) - base;
  *off_head = reinterpret_cast<char*>(ws.head) - base;
  *off_next = reinterpret_cast<char*>(ws.next) - base;
  *off_vox_id = reinterpret_cast<char*>(ws.vox_id) - base;
  return OCC_OK;
}

// ViewTransformerLiftSplatShootVoxel.voxel_pooling(geom_feats, x) with a MATERIALISED volume
// (ViewTransformerLSSVoxel.py:77-100): feats (P, C) rows, geom (P, 3).  out (B, X, Y, Z, C).
extern "C" int occ_voxel_pool_geom(const float* feats, const float* geom, float* out, int B, int points_per_batch,
                                   int C, float dx0, float dx1, float dx2, float bx0, float bx1, float bx2, float nx0,
                                   float nx1, float nx2, int X, int Y, int Z, void* workspace, size_t workspace_bytes,
                                   cudaStream_t stream) {
  OCC_REQUIRE(feats && geom && out && workspace);
  OCC_REQUIRE(B > 0 && points_per_batch > 0 && C > 0 && C % 4 == 0 && X > 0 && Y > 0 && Z > 0);
  const long long Pll = (long long)B * points_per_batch, Vll = (long long)B * X * Y * Z;
  OCC_REQUIRE(Pll < (1ll << 31) && Vll < (1ll << 31));
  const int P = (int)Pll, V = (int)Vll;
  VpWorkspace ws;
  OCC_REQUIRE(vp_layout(workspace, P, V, &ws) <= workspace_bytes);
  OCC_MEMSET(ws.head, 0, reinterpret_cast<char*>(ws.counts + V) - reinterpret_cast<char*>(ws.head), stream);
  const VpGrid vg{dx0, dx1, dx2, bx0, bx1, bx2, nx0, nx1, nx2, X, Y, Z};
  vp_index_geom_kernel<<<blocks_for(P, 256), 256, 0, stream>>>(geom, P, points_per_batch, vg, ws.vox_id, ws.counts,
                                                                ws.head, ws.next);
  OCC_LAUNCH_CHECK();
  vp_pool_kernel<1><<<pool_blocks(V), 256, 0, stream>>>(ws.head, ws.next, V, C, nullptr, feats, make_fastdiv(1),
                                                        make_fastdiv(1), out, nullptr);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// ------------------------------------------------------------------------------------------------ frustum geometry
// ViewTransformerLSSBEVDepth.get_geometry (projects/mmdet3d_plugin/occformer/image2bev/ViewTransformerLSSBEVDepth.py:117-150)
// as one kernel: undo the image augmentation (post_trans / post_rots), unproject with depth, camera -> ego
// (rots * inv(intrins), + trans), then the BEV augmentation matrix bda.  The reference issues ~25 batched 3x3
// cuBLAS gemv launches over 473k points for this; the arithmetic is 3 small matvecs per point.
// One CTA column (blockIdx.y) per camera (b, n); thread = frustum point.
namespace occ {

__device__ __forceinline__ void inv3x3(const float* m, float* o) {
  // adjugate / determinant in double, rounded once to fp32
  const double a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
  const double A = e * i - f * h, B = -(d * i - f * g), C = d * h - e * g;
  const double det = a * A + b * B + c * C;
  const double r = 1.0 / det;
  o[0] = (float)(A * r); o[1] = (float)(-(b * i - c * h) * r); o[2] = (float)((b * f - c * e) * r);
  o[3] = (float)(B * r); o[4] = (float)((a * i - c * g) * r);  o[5] = (float)(-(a * f - c * d) * r);
  o[6] = (float)(C * r); o[7] = (float)(-(a * h - b * g) * r); o[8] = (float)((a * e - b * d) * r);
}

__device__ __forceinline__ void mv3(const float* m, float x, float y, float z, float& ox, float& oy, float& oz) {
  ox = fmaf(m[2], z, fmaf(m[1], y, m[0] * x));
  oy = fmaf(m[5], z, fmaf(m[4], y, m[3] * x));
  oz = fmaf(m[8], z, fmaf(m[7], y, m[6] * x));
}

// Per-camera constants of get_geometry in shared memory (36 floats): inverse post-rotation, rots * inverse(K), the
// translations, the KITTI P2 shift column and the BEV augmentation matrix.
struct CamConst {
  float ipr[9], comb[9], vec[9], bda[16];
};

__device__ __forceinline__ void cam_const_build(CamConst* c, int bn, int b, const float* __restrict__ rots,
                                                const float* __restrict__ trans, const float* __restrict__ intrins,
                                                int intrin_rows, int intrin_cols, const float* __restrict__ post_rots,
                                                const float* __restrict__ post_trans, const float* __restrict__ bda,
                                                int bda_dim) {
  inv3x3(post_rots + (size_t)bn * 9, c->ipr);
  float K[9], iK[9];
  const float* I = intrins + (size_t)bn * intrin_rows * intrin_cols;  // (3,3), (3,4) or KITTI's 4x4 P2 per camera
  for (int r = 0; r < 3; ++r)
    for (int cc = 0; cc < 3; ++cc) K[r * 3 + cc] = I[r * intrin_cols + cc];
  inv3x3(K, iK);
  const float* R = rots + (size_t)bn * 9;
  for (int r = 0; r < 3; ++r)
    for (int cc = 0; cc < 3; ++cc)
      c->comb[r * 3 + cc] = fmaf(R[r * 3 + 2], iK[6 + cc], fmaf(R[r * 3 + 1], iK[3 + cc], R[r * 3] * iK[cc]));
  for (int k = 0; k < 3; ++k) {
    c->vec[k] = post_trans[(size_t)bn * 3 + k];
    c->vec[3 + k] = trans[(size_t)bn * 3 + k];
    c->vec[6 + k] = intrin_cols == 4 ? I[k * 4 + 3] : 0.f;  // KITTI P2 shift (:134-137), rows 0..2 of the last column
  }
  for (int k = 0; k < bda_dim * bda_dim; ++k) c->bda[k] = bda[(size_t)b * bda_dim * bda_dim + k];
}

// frustum point (fx, fy, fz) = (u, v, depth) -> ego coordinates (ViewTransformerLSSBEVDepth.py:117-150)
__device__ __forceinline__ void cam_point(const CamConst& c, int bda_dim, float fx, float fy, float fz, float& ox, float& oy,
                                          float& oz) {
  float x = fx - c.vec[0], y = fy - c.vec[1], z = fz - c.vec[2];
  float u, v, w;
  mv3(c.ipr, x, y, z, u, v, w);
  u = u * w - c.vec[6]; v = v * w - c.vec[7]; w = w - c.vec[8];
  mv3(c.comb, u, v, w, x, y, z);
  x += c.vec[3]; y += c.vec[4]; z += c.vec[5];
  if (bda_dim == 4) {
    ox = fmaf(c.bda[2], z, fmaf(c.bda[1], y, c.bda[0] * x)) + c.bda[3];
    oy = fmaf(c.bda[6], z, fmaf(c.bda[5], y, c.bda[4] * x)) + c.bda[7];
    oz = fmaf(c.bda[10], z, fmaf(c.bda[9], y, c.bda[8] * x)) + c.bda[11];
  } else {
    mv3(c.bda, x, y, z, ox, oy, oz);
  }
}

__global__ void __launch_bounds__(256)
lss_geometry_kernel(const float* __restrict__ frustum /*(P,3)*/, int P, const float* __restrict__ rots,
                    const float* __restrict__ trans, const float* __restrict__ intrins, int intrin_rows, int intrin_cols,
                    const float* __restrict__ post_rots, const float* __restrict__ post_trans,
                    const float* __restrict__ bda, int bda_dim, int N, float* __restrict__ geom) {
  __shared__ CamConst cam;
  const int bn = blockIdx.y, b = bn / N;
  if (threadIdx.x == 0) cam_const_build(&cam, bn, b, rots, trans, intrins, intrin_rows, intrin_cols, post_rots, post_trans, bda, bda_dim);
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  float ox, oy, oz;
  cam_point(cam, bda_dim, frustum[3 * (size_t)p], frustum[3 * (size_t)p + 1], frustum[3 * (size_t)p + 2], ox, oy, oz);
  float* o = geom + ((size_t)bn * P + p) * 3;
  o[0] = ox; o[1] = oy; o[2] = oz;
}

// ------------------------------------------------------------------------------------------------ fused lift front end
// One launch for everything in front of the pooling kernel (ViewTransformerLSSVoxel.forward :107-116, voxel_pooling
// :84-95, get_geometry): depth softmax over D, frustum -> ego geometry -> voxel index -> per-voxel point lists, and the
// NCHW -> NHWC transpose of the context features.  The (B,N,D,fH,fW,3) geometry tensor is never written.
//   blocks [0, nb_front): (camera bn, 32-pixel tile): 32 pixels x 8 depth groups; a thread owns D/8 depth bins of one pixel
//   blocks [nb_front, ..): 32x32 tiles of the (C, HW) -> (HW, C) transpose
constexpr int LF_DG = 8;      // depth groups per pixel
constexpr int LF_MAXD = 32;   // depth bins per thread (D <= 256)

__global__ void __launch_bounds__(256)
lift_front_kernel(const float* __restrict__ logits /*(BN, D, HW)*/, const float* __restrict__ img_feat /*(BN, C, HW)*/,
                  const float* __restrict__ frustum /*(D*HW, 3)*/, const float* __restrict__ rots,
                  const float* __restrict__ trans, const float* __restrict__ intrins, int intrin_rows, int intrin_cols,
                  const float* __restrict__ post_rots, const float* __restrict__ post_trans,
                  const float* __restrict__ bda, int bda_dim, int N, int D, int HW, int C, long long lstride,
                  long long fstride, const VpGrid g, float* __restrict__ prob, float* __restrict__ feat_cl, int* __restrict__ vox_id,
                  int* __restrict__ counts, int* __restrict__ head, int* __restrict__ next, int nb_front, int tiles_p,
                  int tiles_c) {
  __shared__ CamConst cam;
  __shared__ float red[LF_DG][32];
  __shared__ float tile[32][33];
  if ((int)blockIdx.x >= nb_front) {  // ---- context features (BN, C, HW) -> (BN, HW, C)
    int t = blockIdx.x - nb_front;
    const int tp = t % tiles_p; t /= tiles_p;
    const int tc = t % tiles_c;
    const int bn = t / tiles_c;
    const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
    const int c0 = tc * 32, p0 = tp * 32;
    for (int i = ly; i < 32; i += 8) {
      const int c = c0 + i, p = p0 + lx;
      tile[i][lx] = (c < C && p < HW) ? img_feat[(size_t)bn * fstride + (size_t)c * HW + p] : 0.f;
    }
    __syncthreads();
    for (int i = ly; i < 32; i += 8) {
      const int p = p0 + i, c = c0 + lx;
      if (p < HW && c < C) feat_cl[((size_t)bn * HW + p) * C + c] = tile[lx][i];
    }
    return;
  }
  const int bn = blockIdx.x / tiles_p, b = bn / N;
  const int lx = threadIdx.x & 31, dg = threadIdx.x >> 5;
  const int pix = (blockIdx.x % tiles_p) * 32 + lx;
  if (threadIdx.x == 0) cam_const_build(&cam, bn, b, rots, trans, intrins, intrin_rows, intrin_cols, post_rots, post_trans, bda, bda_dim);
  const bool live = pix < HW;
  const int dper = (D + LF_DG - 1) / LF_DG;
  const int d0 = dg * dper, d1 = min(d0 + dper, D);
  float l[LF_MAXD];
  float m = -INFINITY;
#pragma unroll
  for (int i = 0; i < LF_MAXD; ++i) {
    l[i] = -INFINITY;
    if (live && d0 + i < d1) l[i] = logits[(size_t)bn * lstride + (size_t)(d0 + i) * HW + pix];
    m = fmaxf(m, l[i]);
  }
  red[dg][lx] = m;
  __syncthreads();
#pragma unroll
  for (int k = 0; k < LF_DG; ++k) m = fmaxf(m, red[k][lx]);
  __syncthreads();
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < LF_MAXD; ++i) {
    l[i] = (live && d0 + i < d1) ? expf(l[i] - m) : 0.f;
    sum += l[i];
  }
  red[dg][lx] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int k = 0; k < LF_DG; ++k) sum += red[k][lx];  // same order for every thread of the pixel
  if (!live) return;
#pragma unroll
  for (int i = 0; i < LF_MAXD; ++i) {
    const int d = d0 + i;
    if (d < d1) {
      const int p = (bn * D + d) * HW + pix;
      prob[p] = l[i] / sum;
      const float* f = frustum + 3 * ((size_t)d * HW + pix);
      float ox, oy, oz;
      cam_point(cam, bda_dim, f[0], f[1], f[2], ox, oy, oz);
      vp_push(p, vp_voxel_of(ox, oy, oz, b, g), vox_id, counts, head, next);
    }
  }
}

}  // namespace occ

extern "C" int occ_lss_geometry(const float* frustum, int P, const float* rots, const float* trans, const float* intrins,
                                int intrin_rows, int intrin_cols, const float* post_rots, const float* post_trans,
                                const float* bda, int bda_dim, int B, int N, float* geom, cudaStream_t stream) {
  OCC_REQUIRE(frustum && rots && trans && intrins && post_rots && post_trans && bda && geom);
  OCC_REQUIRE(P > 0 && B > 0 && N > 0 && (intrin_cols == 3 || intrin_cols == 4) && (bda_dim == 3 || bda_dim == 4));
  OCC_REQUIRE(intrin_rows >= 3 && intrin_rows <= 4 && intrin_rows <= intrin_cols + 1);
  OCC_REQUIRE((long long)B * N <= 65535);
  dim3 grid(blocks_for(P, 256), B * N);
  occ::lss_geometry_kernel<<<grid, 256, 0, stream>>>(frustum, P, rots, trans, intrins, intrin_rows, intrin_cols, post_rots,
                                                     post_trans,
                                                     bda, bda_dim, N, geom);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// (Tried and rejected: zero-filling the grid from spare CTAs of the front kernel and letting the pooling kernel write the
// occupied rows only -- 14 % of the voxels here.  The occupied-only pooling pass is a chain of dependent list hops with
// nothing to hide behind.  Streaming the zero rows from the same warps that
// walk the lists is what hides the hop latency.)
// Fused lift-splat from the view transformer's raw inputs: depth_logits (B*N, D, HW), img_feat (B*N, C, HW) (NCHW, as
// DepthNet returns them), frustum (D*HW, 3) and the camera matrices of occ_lss_geometry.  Three launches: memset of the
// list heads, the front kernel (softmax + geometry + voxel index + lists + NHWC transpose), the pooling kernel.
// depth_prob (B*N, D, HW) and feat_cl (B*N, HW, C) are outputs (depth_prob is the module's second return value).
// logits_stride / feat_stride: floats between consecutive cameras of depth_logits / img_feat (both may be channel
// slices of DepthNet's (B*N, D + C, fH, fW) output: no copy).
extern "C" int occ_lift_splat_fused(const float* depth_logits, long long logits_stride, const float* img_feat,
                                    long long feat_stride, const float* frustum,
                                    const float* rots, const float* trans, const float* intrins, int intrin_rows,
                                    int intrin_cols, const float* post_rots, const float* post_trans, const float* bda,
                                    int bda_dim, float* depth_prob, float* feat_cl, float* out, float* out_split, int B,
                                    int N, int D, int HW, int C, float dx0, float dx1, float dx2, float bx0, float bx1,
                                    float bx2, float nx0, float nx1, float nx2, int X, int Y, int Z, void* workspace,
                                    size_t workspace_bytes, cudaStream_t stream) {
  OCC_REQUIRE(depth_logits && img_feat && frustum && rots && trans && intrins && post_rots && post_trans && bda);
  OCC_REQUIRE(depth_prob && feat_cl && out && workspace);
  OCC_REQUIRE(!out_split || C % 32 == 0);
  OCC_REQUIRE(logits_stride >= (long long)D * HW && feat_stride >= (long long)C * HW);
  OCC_REQUIRE(B > 0 && N > 0 && D > 0 && D <= occ::LF_DG * occ::LF_MAXD && HW > 0 && C > 0 && C % 4 == 0 && X > 0 && Y > 0 && Z > 0);
  OCC_REQUIRE((intrin_cols == 3 || intrin_cols == 4) && intrin_rows >= 3 && intrin_rows <= 4 && (bda_dim == 3 || bda_dim == 4));
  const long long Pll = (long long)B * N * D * HW, Vll = (long long)B * X * Y * Z;
  OCC_REQUIRE(Pll < (1ll << 31) && Vll < (1ll << 31));
  const int P = (int)Pll, V = (int)Vll;
  VpWorkspace ws;
  OCC_REQUIRE(vp_layout(workspace, P, V, &ws) <= workspace_bytes);
  OCC_MEMSET(ws.head, 0, reinterpret_cast<char*>(ws.counts + V) - reinterpret_cast<char*>(ws.head), stream);
  const VpGrid vg{dx0, dx1, dx2, bx0, bx1, bx2, nx0, nx1, nx2, X, Y, Z};
  const int tiles_p = (int)blocks_for(HW, 32), tiles_c = (int)blocks_for(C, 32);
  const int nb_front = B * N * tiles_p;
  const long long nb = (long long)nb_front + (long long)B * N * tiles_p * tiles_c;
  OCC_REQUIRE(nb < (1ll << 31));
  lift_front_kernel<<<(unsigned)nb, 256, 0, stream>>>(depth_logits, img_feat, frustum, rots, trans, intrins, intrin_rows,
                                                      intrin_cols, post_rots, post_trans, bda, bda_dim, N, D, HW, C,
                                                      logits_stride, feat_stride, vg,
                                                      depth_prob, feat_cl, ws.vox_id, ws.counts, ws.head, ws.next, nb_front,
                                                      tiles_p, tiles_c);
  OCC_LAUNCH_CHECK();
  vp_pool_kernel<0><<<pool_blocks(V), 256, 0, stream>>>(ws.head, ws.next, V, C, depth_prob, feat_cl,
                                                        make_fastdiv((uint32_t)D * HW), make_fastdiv(HW), out, out_split);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
