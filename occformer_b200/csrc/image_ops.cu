// The layout kernels of the image encoder (mmdet ResNet-50 + mmdet3d SECONDFPN, the img_backbone / img_neck of the
// nuScenes R50 model; EfficientNet's stem) that the convolutions cannot do themselves: the stem's im2col (Cin = 3, any
// k x k, stride and top / left padding), the stem max-pool,
// and the pixel reshuffles that turn SECONDFPN's stride-f convs and transposed convs into 1x1 convs / GEMMs.  Every
// contraction of the encoder goes through occ_gemm_bf16x3 / occ_conv_bf16x3 / occ_conv_slice_bf16x3; activations are
// channel-last rows (image, y, x).
#include <cuda_bf16.h>

#include "occ_common.cuh"
#include "occ_ptx.cuh"

namespace occ {

// One warp per output pixel; lane l owns column l of each 32-column chunk and writes its hi / lo bf16 halves (every
// chunk is one coalesced 128-byte store).  Column q < 3*k*k: (ky, kx, c) = (q / (3k), q / 3 % k, q % 3), input pixel
// (stride*oy - pad_top + ky, stride*ox - pad_left + kx); columns >= 3*k*k and pixels outside the image are 0.
__global__ void __launch_bounds__(256)
stem_im2col_kernel(const float* __restrict__ img, float* __restrict__ cols, long long rows, int H, int W, int Ho, int Wo,
                   int k, int stride, int pad_top, int pad_left, int ncols) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const long long b = r / ((long long)Ho * Wo);
  const int pix = (int)(r - b * Ho * Wo);
  const int oy = pix / Wo, ox = pix - (pix / Wo) * Wo;
  const int taps3 = 3 * k * k;
  __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(cols + r * ncols);
  for (int q = 0; q < ncols / 32; ++q) {
    const int col = q * 32 + lane;
    float v = 0.f;
    if (col < taps3) {
      const int c = col % 3, t = col / 3;
      const int iy = stride * oy - pad_top + t / k, ix = stride * ox - pad_left + t % k;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(img + ((b * 3 + c) * H + iy) * W + ix);
    }
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    out[q * 64 + lane] = hi;
    out[q * 64 + 32 + lane] = __float2bfloat16_rn(v - __bfloat162float(hi));  // the residual is exact in fp32
  }
}

// One thread per (output pixel, 4 channels).  Window scan in torch's order with torch's rule (a value replaces the
// running maximum when it is larger or NaN); padding positions are skipped, i.e. -inf.
__global__ void __launch_bounds__(256)
maxpool3x3s2_kernel(const float* __restrict__ in, float* __restrict__ out, long long n4, int H, int W, int Ho, int Wo,
                    int C) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 >= n4) return;
  const int C4 = C >> 2;
  const long long row = i4 / C4;
  const int c0 = (int)(i4 - row * C4) * 4;
  const long long b = row / ((long long)Ho * Wo);
  const int pix = (int)(row - b * Ho * Wo);
  const int oy = pix / Wo, ox = pix - (pix / Wo) * Wo;
  float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  auto take = [](float v, float cur) { return (v > cur || isnan(v)) ? v : cur; };
  for (int dy = 0; dy < 3; ++dy) {
    const int iy = 2 * oy - 1 + dy;
    if (iy < 0 || iy >= H) continue;
    for (int dx = 0; dx < 3; ++dx) {
      const int ix = 2 * ox - 1 + dx;
      if (ix < 0 || ix >= W) continue;
      const float4 v = __ldg(reinterpret_cast<const float4*>(in + ((b * H + iy) * W + ix) * C + c0));
      m.x = take(v.x, m.x); m.y = take(v.y, m.y); m.z = take(v.z, m.z); m.w = take(v.w, m.w);
    }
  }
  store_split4(out + row * C, c0, m);
}

// One thread per 16 bytes of the output.  Output float o of a row comes from tap o / C, position o % C of the input row:
// whole 32-float chunks move unchanged, so the copy is bit-exact for S32 and fp32 alike.
__global__ void __launch_bounds__(256)
space_to_depth_kernel(const float* __restrict__ in, float* __restrict__ out, long long n4, int H, int W, int C, int f) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 >= n4) return;
  const int Ho = H / f, Wo = W / f, L4 = f * f * C / 4;
  const long long row = i4 / L4;
  const int o = (int)(i4 - row * L4) * 4;
  const int tap = o / C, c = o - tap * C;
  const long long b = row / ((long long)Ho * Wo);
  const int pix = (int)(row - b * Ho * Wo);
  const int y = pix / Wo * f + tap / f, x = pix % Wo * f + tap % f;
  *reinterpret_cast<float4*>(out + i4 * 4) = __ldg(reinterpret_cast<const float4*>(in + ((b * H + y) * W + x) * C + c));
}

// One thread per 16 bytes of the input: input row (b, y, x), column (i*f + j)*C + c -> output pixel (f*y + i, f*x + j),
// column out_off + c.
__global__ void __launch_bounds__(256)
depth_to_space_kernel(const float* __restrict__ in, float* __restrict__ out, long long n4, int h, int w, int C, int f,
                      int ldo, int out_off) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 >= n4) return;
  const int L4 = f * f * C / 4;
  const long long row = i4 / L4;
  const int o = (int)(i4 - row * L4) * 4;
  const int tap = o / C, c = o - tap * C;
  const long long b = row / ((long long)h * w);
  const int pix = (int)(row - b * h * w);
  const int y = pix / w * f + tap / f, x = pix % w * f + tap % f;
  const long long orow = (b * h * f + y) * (long long)(w * f) + x;
  *reinterpret_cast<float4*>(out + orow * ldo + out_off + c) = __ldg(reinterpret_cast<const float4*>(in + i4 * 4));
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static unsigned blocks_of(long long threads) { return (unsigned)((threads + 255) / 256); }

}  // namespace occ

using namespace occ;

extern "C" int occ_stem_im2col(const float* img, float* cols, int n, int H, int W, int k, int stride, int pad_top,
                               int pad_left, int Ho, int Wo, int ncols, cudaStream_t stream) {
  OCC_REQUIRE(img && cols && n > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && aligned16(cols));
  OCC_REQUIRE(k >= 1 && k <= 7 && stride >= 1 && pad_top >= 0 && pad_left >= 0 && pad_top < k && pad_left < k);
  OCC_REQUIRE(ncols % 32 == 0 && ncols >= 3 * k * k);
  const long long rows = (long long)n * Ho * Wo;
  OCC_REQUIRE((rows + 7) / 8 < (1ll << 31));
  stem_im2col_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(img, cols, rows, H, W, Ho, Wo, k, stride, pad_top,
                                                                      pad_left, ncols);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_maxpool3x3s2(const float* in, float* out, int n, int H, int W, int C, cudaStream_t stream) {
  OCC_REQUIRE(in && out && n > 0 && H > 0 && W > 0 && C > 0 && C % 32 == 0 && aligned16(in) && aligned16(out));
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const long long n4 = (long long)n * Ho * Wo * (C / 4);
  OCC_REQUIRE((n4 + 255) / 256 < (1ll << 31));
  maxpool3x3s2_kernel<<<blocks_of(n4), 256, 0, stream>>>(in, out, n4, H, W, Ho, Wo, C);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_space_to_depth(const float* in, float* out, int n, int H, int W, int C, int f, cudaStream_t stream) {
  OCC_REQUIRE(in && out && n > 0 && H > 0 && W > 0 && C > 0 && C % 32 == 0 && (f == 2 || f == 4));
  OCC_REQUIRE(H % f == 0 && W % f == 0 && aligned16(in) && aligned16(out));
  const long long n4 = (long long)n * H * W * (C / 4);
  OCC_REQUIRE((n4 + 255) / 256 < (1ll << 31));
  space_to_depth_kernel<<<blocks_of(n4), 256, 0, stream>>>(in, out, n4, H, W, C, f);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_depth_to_space(const float* in, float* out, int n, int h, int w, int C, int f, int ldo, int out_off,
                                  cudaStream_t stream) {
  OCC_REQUIRE(in && out && n > 0 && h > 0 && w > 0 && C > 0 && C % 4 == 0 && (f == 2 || f == 4));
  OCC_REQUIRE(ldo % 4 == 0 && out_off % 4 == 0 && out_off >= 0 && ldo >= out_off + C && aligned16(in) && aligned16(out));
  const long long n4 = (long long)n * h * w * f * f * (C / 4);
  OCC_REQUIRE((n4 + 255) / 256 < (1ll << 31));
  depth_to_space_kernel<<<blocks_of(n4), 256, 0, stream>>>(in, out, n4, h, w, C, f, ldo, out_off);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
