// The kernels of DepthNet (P/occformer/image2bev/ViewTransformerLSSBEVDepth.py:435-504) that are not convolutions: the
// camera-aware SE gates, their application to the reduced features, and the deformable im2col of the DCN
// (mmcv-full 1.4.0 DeformConv2dPack, DCNv1), whose modulated instantiation serves the DCNv2 convs of the image encoder's
// ResNetDCN (ModulatedDeformConv2dPack).  Every contraction of DepthNet goes through occ_conv_bf16x3 /
// occ_conv_slice_bf16x3; activations are channel-last rows (image, y, x) of C floats.
#include "occ_common.cuh"
#include "occ_ptx.cuh"

namespace occ {

// out[o] = act(bias[o] + sum_i wT[i * C + o] * in[i]), o < C, for one CTA; wT K-major (in, out): thread o reads a
// coalesced row per i, the input vector comes from shared memory.  act: 0 none, 1 ReLU, 2 sigmoid.
__device__ __forceinline__ void matvec_kmajor(const float* __restrict__ wT, const float* __restrict__ bias,
                                              const float* in, int K, int C, int act, float* out) {
  for (int o = threadIdx.x; o < C; o += blockDim.x) {
    float a = bias[o];
    for (int i = 0; i < K; ++i) a = fmaf(__ldg(wT + (size_t)i * C + o), in[i], a);
    if (act == 1) a = fmaxf(a, 0.f);
    else if (act == 2) a = 1.f / (1.f + expf(-a));
    out[o] = a;
  }
}

// One CTA per (image, chain); chain 0 = depth_mlp / depth_se, 1 = context_mlp / context_se (DepthNet.forward
// :495-504, SELayer :435-448, Mlp :410-432, with the BatchNorm1d of mlp_input folded into fc1):
//   gate = sigmoid(We relu(Wr (W2 relu(W1' m + b1') + b2) + br) + be)
__global__ void __launch_bounds__(256)
cam_gates_kernel(const float* __restrict__ mlp_in, int cam, const float* __restrict__ w1T, const float* __restrict__ b1,
                 const float* __restrict__ w2T, const float* __restrict__ b2, const float* __restrict__ wrT,
                 const float* __restrict__ br, const float* __restrict__ weT, const float* __restrict__ be,
                 float* __restrict__ gates, int n, int C) {
  extern __shared__ float sm[];  // m[cam] | a[C] | b[C]
  float* m = sm;
  float* a = sm + cam;
  float* b = a + C;
  const int img = blockIdx.x, chain = blockIdx.y;
  const size_t cc = (size_t)chain * C * C;
  for (int i = threadIdx.x; i < cam; i += blockDim.x) m[i] = mlp_in[(size_t)img * cam + i];
  __syncthreads();
  matvec_kmajor(w1T + (size_t)chain * cam * C, b1 + chain * C, m, cam, C, 1, a);
  __syncthreads();
  matvec_kmajor(w2T + cc, b2 + chain * C, a, C, C, 0, b);
  __syncthreads();
  matvec_kmajor(wrT + cc, br + chain * C, b, C, C, 1, a);
  __syncthreads();
  matvec_kmajor(weT + cc, be + chain * C, a, C, C, 2, gates + ((size_t)chain * n + img) * C);
}

// x (rows, C) fp32, rows = n * rows_per_img; one thread per 4 columns of a row
__global__ void __launch_bounds__(256)
se_apply_kernel(const float* __restrict__ x, const float* __restrict__ gates, float* __restrict__ xd,
                float* __restrict__ xd_split, float* __restrict__ xc_split, long long n4, int n, int rows_per_img, int C) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 >= n4) return;
  const int C4 = C >> 2;
  const long long row = i4 / C4;
  const int c0 = (int)(i4 - row * C4) * 4;
  const int img = (int)(row / rows_per_img);
  const float4 v = __ldg(reinterpret_cast<const float4*>(x + row * C + c0));
  const float4 gd = __ldg(reinterpret_cast<const float4*>(gates + (size_t)img * C + c0));
  const float4 gc = __ldg(reinterpret_cast<const float4*>(gates + ((size_t)n + img) * C + c0));
  const float4 d = make_float4(v.x * gd.x, v.y * gd.y, v.z * gd.z, v.w * gd.w);
  *reinterpret_cast<float4*>(xd + row * C + c0) = d;
  store_split4(xd_split + row * C, c0, d);
  store_split4(xc_split + row * C, c0, make_float4(v.x * gc.x, v.y * gc.y, v.z * gc.z, v.w * gc.w));
}

// One warp per (pixel, kernel point k): the sample position and corner weights are computed once, the lanes stride over
// the channels in float4 steps.  Sample position, inside test and corner rules of mmcv's deformable_im2col_gpu_kernel /
// deformable_im2col_bilinear (3x3, stride 1, padding 1, dilation 1, one deformable group), in the same fp32 expression
// order.  The input is read in S32 and rebuilt as hi + lo.  cols: (groups, rows, 9 * Cg) S32, column k * Cg + c of
// group g = channel g * Cg + c at kernel point k.
// MOD (DCNv2, mmcv's modulated_deformable_im2col_gpu_kernel / dmcn_im2col_bilinear, same sampling rules): the sample is
// multiplied by mask = sigmoid(off[18 + k]) after the bilinear sum (col = val * mask); groups == 1.
template <bool MOD>
__global__ void __launch_bounds__(256)
deform_im2col_kernel(const float* __restrict__ x, const float* __restrict__ off, int off_ld, float* __restrict__ cols,
                     long long rows, int H, int W, int C, int Cg) {
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (wid >= rows * 9) return;
  const long long p = wid / 9;
  const int k = (int)(wid - p * 9);
  const int HW = H * W;
  const long long img = p / HW;
  const int pix = (int)(p - img * HW);
  const int py = pix / W, px = pix - (pix / W) * W;
  const float h = (float)(py - 1 + k / 3) + __ldg(off + p * off_ld + 2 * k);
  const float w = (float)(px - 1 + k % 3) + __ldg(off + p * off_ld + 2 * k + 1);
  float mask = 1.f;
  if constexpr (MOD) mask = 1.f / (1.f + expf(-__ldg(off + p * off_ld + 18 + k)));
  const bool inside = h > -1.f && w > -1.f && h < (float)H && w < (float)W;
  const int h_low = (int)floorf(h), w_low = (int)floorf(w);
  const int h_high = h_low + 1, w_high = w_low + 1;
  const float lh = h - (float)h_low, lw = w - (float)w_low;
  const float hh = 1.f - lh, hw = 1.f - lw;
  const float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
  const bool c1 = inside && h_low >= 0 && w_low >= 0, c2 = inside && h_low >= 0 && w_high <= W - 1;
  const bool c3 = inside && h_high <= H - 1 && w_low >= 0, c4 = inside && h_high <= H - 1 && w_high <= W - 1;
  const float* base = x + (size_t)img * HW * C;
  const float* r1 = base + ((long long)h_low * W + w_low) * C;
  const float* r2 = base + ((long long)h_low * W + w_high) * C;
  const float* r3 = base + ((long long)h_high * W + w_low) * C;
  const float* r4 = base + ((long long)h_high * W + w_high) * C;
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int c0 = lane * 4; c0 < C; c0 += 128) {
    const float4 v1 = c1 ? load_split4(r1, c0) : z, v2 = c2 ? load_split4(r2, c0) : z;
    const float4 v3 = c3 ? load_split4(r3, c0) : z, v4 = c4 ? load_split4(r4, c0) : z;
    float4 o;
    o.x = w1 * v1.x + w2 * v2.x + w3 * v3.x + w4 * v4.x;
    o.y = w1 * v1.y + w2 * v2.y + w3 * v3.y + w4 * v4.y;
    o.z = w1 * v1.z + w2 * v2.z + w3 * v3.z + w4 * v4.z;
    o.w = w1 * v1.w + w2 * v2.w + w3 * v3.w + w4 * v4.w;
    if constexpr (MOD) o = make_float4(o.x * mask, o.y * mask, o.z * mask, o.w * mask);
    const int g = c0 / Cg, cl = c0 - g * Cg;
    store_split4(cols + ((size_t)g * rows + p) * (9 * Cg), k * Cg + cl, o);
  }
}

}  // namespace occ

using namespace occ;

extern "C" int occ_depthnet_cam_gates(const float* mlp_in, int cam, const float* w1T, const float* b1, const float* w2T,
                                      const float* b2, const float* wrT, const float* br, const float* weT,
                                      const float* be, float* gates, int n, int C, cudaStream_t stream) {
  OCC_REQUIRE(mlp_in && w1T && b1 && w2T && b2 && wrT && br && weT && be && gates);
  OCC_REQUIRE(n > 0 && n <= 65535 && cam > 0 && cam <= 256 && C > 0 && C <= 4096);
  cam_gates_kernel<<<dim3(n, 2), 256, (cam + 2 * C) * sizeof(float), stream>>>(mlp_in, cam, w1T, b1, w2T, b2, wrT, br,
                                                                               weT, be, gates, n, C);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_se_apply(const float* x, const float* gates, float* xd, float* xd_split, float* xc_split, int n,
                            int rows_per_img, int C, cudaStream_t stream) {
  OCC_REQUIRE(x && gates && xd && xd_split && xc_split && n > 0 && rows_per_img > 0 && C > 0 && C % 32 == 0);
  OCC_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(gates) | reinterpret_cast<uintptr_t>(xd) |
                reinterpret_cast<uintptr_t>(xd_split) | reinterpret_cast<uintptr_t>(xc_split)) & 15) == 0);
  const long long n4 = (long long)n * rows_per_img * (C / 4);
  se_apply_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(x, gates, xd, xd_split, xc_split, n4, n, rows_per_img,
                                                                    C);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_deform_im2col(const float* x, const float* off, int off_ld, float* cols, int n, int H, int W, int C,
                                 int groups, cudaStream_t stream) {
  OCC_REQUIRE(x && off && cols && n > 0 && H > 0 && W > 0 && groups > 0 && C % groups == 0);
  OCC_REQUIRE((C / groups) % 32 == 0 && off_ld >= 18);  // whole S32 chunks per group
  OCC_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(cols)) & 15) == 0);
  const long long rows = (long long)n * H * W;
  const long long warps = rows * 9;
  OCC_REQUIRE((warps + 7) / 8 < (1ll << 31));
  deform_im2col_kernel<false><<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(x, off, off_ld, cols, rows, H, W, C,
                                                                              C / groups);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

extern "C" int occ_modulated_deform_im2col(const float* x, const float* off, int off_ld, float* cols, int n, int H, int W,
                                           int C, cudaStream_t stream) {
  OCC_REQUIRE(x && off && cols && n > 0 && H > 0 && W > 0 && C > 0 && C % 32 == 0 && off_ld >= 27);
  OCC_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(cols)) & 15) == 0);
  const long long rows = (long long)n * H * W;
  const long long warps = rows * 9;
  OCC_REQUIRE((warps + 7) / 8 < (1ll << 31));
  deform_im2col_kernel<true><<<(unsigned)((warps + 7) / 8), 256, 0, stream>>>(x, off, off_ld, cols, rows, H, W, C, C);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
