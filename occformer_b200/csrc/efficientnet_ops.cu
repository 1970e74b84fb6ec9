// The kernels of EfficientNet's InvertedResidual block (P/occformer/backbones/efficientnet.py:112-229, the img_backbone of
// the SemanticKITTI model) that are not 1x1 convolutions: the depthwise conv with its folded BatchNorm and Swish, the
// squeeze-and-excitation gate (mmdet 2.14 SELayer) and its application.  The expand / linear 1x1 convs, the stem and
// layers.6 are occ_gemm_bf16x3 launches; activations are channel-last rows (image, y, x) of C floats, C a multiple of 32
// (pad channels carry zero weights, so they stay exactly 0).
#include "occ_common.cuh"
#include "occ_ptx.cuh"

namespace occ {

constexpr int DW_TILE = 256;  // output pixels per CTA of the depthwise conv = per SE partial sum

__device__ __forceinline__ float swish_f(float x) { return x / (1.0f + expf(-x)); }

// One CTA per (DW_TILE output pixels, 32 channels, image): threadIdx.x = 4 channels, threadIdx.y = pixel slot.  The
// CTA's k*k x 32 weights sit in shared memory (a register copy of the 5x5 taps costs 162 registers, one CTA per SM);
// each thread accumulates the taps in (ky, kx) order, the input halo is shared through L1.  The per-channel sums of the Swish outputs run over the thread's pixels in order, then over the 32 pixel
// slots in order: fixed-order partials (no atomics), so the SE mean is bit-reproducible.
template <int K, int S>
__global__ void __launch_bounds__(256)
dwconv_swish_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ bias,
                    float* __restrict__ out, float* __restrict__ partials, int H, int W, int Ho, int Wo, int C, int pad_top,
                    int pad_left, int tiles) {
  __shared__ float4 red[32][8];
  __shared__ float4 wsm[K * K][8];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c0 = blockIdx.y * 32 + tx * 4;
  const long long img = blockIdx.z;
  for (int t = ty; t < K * K; t += 32) wsm[t][tx] = __ldg(reinterpret_cast<const float4*>(w + (size_t)t * C + c0));
  __syncthreads();
  const float4 b = __ldg(reinterpret_cast<const float4*>(bias + c0));
  const float* src = in + img * H * W * C + c0;
  float* dst = out + img * Ho * Wo * C + c0;
  const int npix = Ho * Wo;
  float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int p = (int)blockIdx.x * DW_TILE + ty; p < min(npix, ((int)blockIdx.x + 1) * DW_TILE); p += 32) {
    const int oy = p / Wo, ox = p - (p / Wo) * Wo;
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int ky = 0; ky < K; ++ky) {
      const int iy = oy * S - pad_top + ky;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int kx = 0; kx < K; ++kx) {
        const int ix = ox * S - pad_left + kx;
        if (ix < 0 || ix >= W) continue;
        const float4 v = __ldg(reinterpret_cast<const float4*>(src + ((long long)iy * W + ix) * C));
        const float4 q = wsm[ky * K + kx][tx];
        a.x = fmaf(q.x, v.x, a.x); a.y = fmaf(q.y, v.y, a.y); a.z = fmaf(q.z, v.z, a.z); a.w = fmaf(q.w, v.w, a.w);
      }
    }
    const float4 y = make_float4(swish_f(a.x + b.x), swish_f(a.y + b.y), swish_f(a.z + b.z), swish_f(a.w + b.w));
    *reinterpret_cast<float4*>(dst + (long long)p * C) = y;
    sum.x += y.x; sum.y += y.y; sum.z += y.z; sum.w += y.w;
  }
  red[ty][tx] = sum;
  __syncthreads();
  if (ty == 0) {
    float4 s = red[0][tx];
    for (int j = 1; j < 32; ++j) {
      const float4 r = red[j][tx];
      s.x += r.x; s.y += r.y; s.z += r.z; s.w += r.w;
    }
    *reinterpret_cast<float4*>(partials + (img * tiles + blockIdx.x) * C + c0) = s;
  }
}

// One CTA of 512 threads per image: mean = (partials summed over the tiles in order) / hw; FC1 as G = 512 / S groups of
// S threads, group g summing its slice of the inputs, the slices then added in order after the bias; FC2 one thread per
// output channel.
constexpr int SE_THREADS = 512;

__global__ void __launch_bounds__(SE_THREADS)
se_gate_kernel(const float* __restrict__ partials, int tiles, int hw, const float* __restrict__ w1T,
               const float* __restrict__ b1, const float* __restrict__ w2T, const float* __restrict__ b2,
               float* __restrict__ gate, int C, int S) {
  extern __shared__ float sm[];  // mean[C] | part[G * S] | sq[S]
  float* mean = sm;
  float* part = sm + C;
  const int G = SE_THREADS / S;
  float* sq = part + G * S;
  const long long img = blockIdx.x;
  const int tid = threadIdx.x;
  for (int c = tid; c < C; c += SE_THREADS) {
    const float* p = partials + img * tiles * C + c;
    float s = 0.f;
    for (int t = 0; t < tiles; ++t) s += __ldg(p + (size_t)t * C);
    mean[c] = s / (float)hw;
  }
  __syncthreads();
  const int chunk = (C + G - 1) / G;
  if (tid < G * S) {
    const int o = tid % S, g = tid / S;
    float a = 0.f;
    for (int i = g * chunk; i < min(C, (g + 1) * chunk); ++i) a = fmaf(__ldg(w1T + (size_t)i * S + o), mean[i], a);
    part[g * S + o] = a;
  }
  __syncthreads();
  if (tid < S) {
    float a = __ldg(b1 + tid);
    for (int g = 0; g < G; ++g) a += part[g * S + tid];
    sq[tid] = swish_f(a);
  }
  __syncthreads();
  for (int o = tid; o < C; o += SE_THREADS) {
    float a = __ldg(b2 + o);
    for (int j = 0; j < S; ++j) a = fmaf(__ldg(w2T + (size_t)j * C + o), sq[j], a);
    gate[img * C + o] = 1.f / (1.f + expf(-a));
  }
}

// One thread per 4 columns of a row: out = y * gate[image] in S32
__global__ void __launch_bounds__(256)
se_scale_kernel(const float* __restrict__ y, const float* __restrict__ gate, float* __restrict__ out, long long n4,
                int rows_per_img, int C) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 >= n4) return;
  const int C4 = C >> 2;
  const long long row = i4 / C4;
  const int c0 = (int)(i4 - row * C4) * 4;
  const long long img = row / rows_per_img;
  const float4 v = __ldg(reinterpret_cast<const float4*>(y + row * C + c0));
  const float4 g = __ldg(reinterpret_cast<const float4*>(gate + img * C + c0));
  store_split4(out + row * C, c0, make_float4(v.x * g.x, v.y * g.y, v.z * g.z, v.w * g.w));
}

static bool aligned16_all(std::initializer_list<const void*> ps) {
  for (const void* p : ps)
    if (reinterpret_cast<uintptr_t>(p) & 15) return false;
  return true;
}

template <int K, int S>
static void launch_dw(dim3 grid, const float* in, const float* w, const float* bias, float* out, float* partials, int H,
                      int W, int Ho, int Wo, int C, int pt, int pl, int tiles, cudaStream_t stream) {
  dwconv_swish_kernel<K, S><<<grid, dim3(8, 32), 0, stream>>>(in, w, bias, out, partials, H, W, Ho, Wo, C, pt, pl, tiles);
}

}  // namespace occ

using namespace occ;

extern "C" int occ_dw_tiles(int Ho, int Wo) {
  if (Ho <= 0 || Wo <= 0) return -1;
  return (int)(((long long)Ho * Wo + DW_TILE - 1) / DW_TILE);
}

extern "C" int occ_dwconv_swish(const float* in, const float* w, const float* bias, float* out, float* partials, int n,
                                int H, int W, int C, int k, int stride, int pad_top, int pad_left, int Ho, int Wo,
                                cudaStream_t stream) {
  OCC_REQUIRE(in && w && bias && out && partials && n > 0 && n <= 65535 && H > 0 && W > 0 && C > 0 && C % 32 == 0);
  OCC_REQUIRE((k == 3 || k == 5) && (stride == 1 || stride == 2) && pad_top >= 0 && pad_left >= 0 && pad_top < k &&
              pad_left < k);
  OCC_REQUIRE(Ho > 0 && Wo > 0 && (Ho - 1) * stride - pad_top < H && (Wo - 1) * stride - pad_left < W);
  OCC_REQUIRE(aligned16_all({in, w, bias, out, partials}));
  const int tiles = occ_dw_tiles(Ho, Wo);
  OCC_REQUIRE(tiles > 0 && (long long)tiles * DW_TILE < (1ll << 31));
  const dim3 grid(tiles, C / 32, n);
  if (k == 3 && stride == 1) launch_dw<3, 1>(grid, in, w, bias, out, partials, H, W, Ho, Wo, C, pad_top, pad_left, tiles, stream);
  else if (k == 3) launch_dw<3, 2>(grid, in, w, bias, out, partials, H, W, Ho, Wo, C, pad_top, pad_left, tiles, stream);
  else if (stride == 1) launch_dw<5, 1>(grid, in, w, bias, out, partials, H, W, Ho, Wo, C, pad_top, pad_left, tiles, stream);
  else launch_dw<5, 2>(grid, in, w, bias, out, partials, H, W, Ho, Wo, C, pad_top, pad_left, tiles, stream);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_se_gate(const float* partials, int tiles, int hw, const float* w1T, const float* b1, const float* w2T,
                           const float* b2, float* gate, int n, int C, int S, cudaStream_t stream) {
  OCC_REQUIRE(partials && w1T && b1 && w2T && b2 && gate && n > 0 && n <= 65535 && tiles > 0 && hw > 0);
  OCC_REQUIRE(C > 0 && C <= 8192 && S > 0 && S <= SE_THREADS);
  const size_t smem = (size_t)(C + (SE_THREADS / S) * S + S) * sizeof(float);
  OCC_ENSURE_SMEM(se_gate_kernel, smem);
  se_gate_kernel<<<n, SE_THREADS, smem, stream>>>(partials, tiles, hw, w1T, b1, w2T, b2, gate, C, S);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_se_scale(const float* y, const float* gate, float* out, int n, int rows_per_img, int C,
                            cudaStream_t stream) {
  OCC_REQUIRE(y && gate && out && n > 0 && rows_per_img > 0 && C > 0 && C % 32 == 0);
  OCC_REQUIRE(aligned16_all({y, gate, out}));
  const long long n4 = (long long)n * rows_per_img * (C / 4);
  OCC_REQUIRE((n4 + 255) / 256 < (1ll << 31));
  se_scale_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(y, gate, out, n4, rows_per_img, C);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
