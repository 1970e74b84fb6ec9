/* occ_b200.h -- C ABI of libocc_b200.so: the H100 (sm_90a) hot path of OccFormer.
 *
 * The reference has no C FFI on this path; its boundary is Python (mmcv Registry names, nn.Module forward
 * signatures, one pybind11 torch extension).  This header is what the reference-side Python binds with ctypes
 * (see INTEGRATION.md).  Each entry point cites the reference interface it replaces (paths relative to the
 * reference checkout; P/ = projects/mmdet3d_plugin/, M/ = mmdetection3d/mmdet3d/).
 *
 * Conventions (all functions):
 *   - pointers are DEVICE pointers to contiguous fp32 buffers unless stated; no torch types cross the ABI;
 *   - return 0 on success, <0 for an argument error (-1 invalid, -2 unsupported shape, -3 driver entry point
 *     missing), >0 = cudaError_t of a failed runtime call / launch;
 *   - never allocate, never synchronise, never exit; all work is enqueued on `stream`;
 *   - the current device must already be set by the caller (torch does this).
 *
 * Numerics: every tensor-core contraction is an fp32 problem computed as three bf16 tensor-core passes on hi/lo split
 * operands (a ~= hi + lo, hi = bf16(a), lo = bf16(a - hi); a*b ~= hi*hi' + lo*hi' + hi*lo', fp32 accumulate): ~1e-5
 * relative error.  Operands of such contractions are exchanged in the "S32" split format: an fp32-container tensor
 * (rows, C), C % 32 == 0, whose every aligned 32-column chunk (128 bytes) holds [32 bf16 hi | 32 bf16 lo] of its 32
 * values (same bytes and row pitch as the fp32 tensor).  occ_split_rows / occ_unsplit_rows convert.  Arguments
 * documented "S32" are in this format; everything else is plain fp32.
 */
#ifndef OCC_B200_H_
#define OCC_B200_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* occ_stream_t; /* = cudaStream_t */

int occ_version(void);
/* Kernel launches and cudaMemsetAsync calls the library has enqueued in this process so far (host-side counter over
 * all threads, devices and streams; a call captured into a CUDA graph counts once, at capture). */
long long occ_launch_count(void);

/* ---------------------------------------------------------------------------------------------------------
 * LSS voxel pooling.
 * Replaces: mmdet3d.ops.bev_pool.bev_pool(feats, coords, B, D, H, W)      M/ops/bev_pool/bev_pool.py:83-97
 *           bev_pool_ext.bev_pool_forward                                  M/ops/bev_pool/src/bev_pool.cpp:22-47
 *           ViewTransformerLiftSplatShootVoxel.voxel_pooling / lift        P/occformer/image2bev/ViewTransformerLSSVoxel.py:77-100,110-115
 * Output layout is channel-last (B, X, Y, Z, C); the Python wrapper returns permuted views carrying the
 * reference's shapes ((B,C,Z,X,Y) for bev_pool, (B,C,X,Y,Z) for voxel_pooling).
 * Bookkeeping left in the workspace after a call (byte offsets from occ_voxel_pool_workspace_layout):
 *   vox_id[n_points] int32 (linear voxel id ((b*X+x)*Y+y)*Z+z, -1 = dropped), counts[B*X*Y*Z] int32 (points per
 *   voxel = the reference's interval lengths), head[B*X*Y*Z] / next[n_points] int32 (per-voxel point lists, ids are
 *   1-based, 0 terminates).
 */
size_t occ_voxel_pool_workspace_bytes(int n_points, int B, int X, int Y, int Z);
int occ_voxel_pool_workspace_layout(int n_points, int B, int X, int Y, int Z, size_t* off_counts,
                                    size_t* off_head, size_t* off_next, size_t* off_vox_id);
/* get_geometry (ViewTransformerLSSBEVDepth.py:117-150): frustum (P = D*fH*fW, 3) + camera matrices -> geom
 * (B, N, P, 3) ego-frame points.  intrins (B,N,intrin_rows,intrin_cols): 3x3 (nuScenes), 3x4 or 4x4 (KITTI P2,
 * semantic_kitti_lss_dataset.py:62-64 builds a 4x4); bda (B,d,d), d 3|4. */
int occ_lss_geometry(const float* frustum, int P, const float* rots, const float* trans, const float* intrins,
                     int intrin_rows, int intrin_cols, const float* post_rots, const float* post_trans,
                     const float* bda, int bda_dim, int B, int N, float* geom, occ_stream_t stream);
/* depth softmax over D + NCHW->NHWC of the context features (ViewTransformerLSSVoxel.py:108-110):
 * depth_logits (BN, D, HW), img_feat (BN, C, HW) -> depth_prob (BN, D, HW), feat_cl (BN, HW, C) */
int occ_lift_prologue(const float* depth_logits, const float* img_feat, float* depth_prob, float* feat_cl, int BN,
                      int D, int C, int HW, occ_stream_t stream);
/* fused lift-splat: out[b,x,y,z,:] = sum_{p in voxel} depth_prob[p] * feat_cl[pixel(p), :]; geom (B*N*D*HW, 3);
 * dx/bx/nx = the view transformer's float parameters (ViewTransformerLSSBEVDepth.py:21-25,81-83).
 * out_split (optional, C % 32 == 0): the same grid in S32 (operand of the encoder's first conv). */
int occ_lift_splat(const float* depth_prob, const float* feat_cl, const float* geom, float* out, float* out_split,
                   int B, int N, int D, int HW, int C, float dx0, float dx1, float dx2, float bx0, float bx1, float bx2,
                   float nx0, float nx1, float nx2, int X, int Y, int Z, void* workspace, size_t workspace_bytes,
                   occ_stream_t stream);
/* The whole ViewTransformerLiftSplatShootVoxel.forward after DepthNet (ViewTransformerLSSVoxel.py:107-119) in three
 * launches: depth softmax + get_geometry + voxel index + per-voxel lists + NCHW->NHWC of the context features in one
 * front kernel (the (B,N,D,fH,fW,3) geometry tensor is never written), then the pooling kernel.  depth_logits
 * (B*N, D, HW) and img_feat (B*N, C, HW) with logits_stride / feat_stride floats between cameras (channel slices of
 * DepthNet's (B*N, D + C, fH, fW) output are passed without a copy), frustum (D*HW, 3), camera matrices as
 * occ_lss_geometry; outputs: depth_prob (B*N, D, HW), feat_cl (B*N, HW, C), out (B,X,Y,Z,C) fp32, out_split (optional) S32. */
int occ_lift_splat_fused(const float* depth_logits, long long logits_stride, const float* img_feat,
                         long long feat_stride, const float* frustum, const float* rots,
                         const float* trans, const float* intrins, int intrin_rows, int intrin_cols,
                         const float* post_rots, const float* post_trans, const float* bda, int bda_dim,
                         float* depth_prob, float* feat_cl, float* out, float* out_split, int B, int N, int D, int HW,
                         int C, float dx0, float dx1, float dx2, float bx0, float bx1, float bx2, float nx0, float nx1,
                         float nx2, int X, int Y, int Z, void* workspace, size_t workspace_bytes, occ_stream_t stream);
/* voxel_pooling(geom, volume) with a materialised volume: feats (B*points_per_batch, C), geom (same rows, 3)
 * (ViewTransformerLSSVoxel.py:77-100) */
int occ_voxel_pool_geom(const float* feats, const float* geom, float* out, int B, int points_per_batch, int C,
                        float dx0, float dx1, float dx2, float bx0, float bx1, float bx2, float nx0, float nx1,
                        float nx2, int X, int Y, int Z, void* workspace, size_t workspace_bytes, occ_stream_t stream);
/* drop-in bev_pool: feats (n, C), coords (n, 4) int64 (x, y, z, b) -> out (B, X, Y, Z, C) */
int occ_bev_pool(const float* feats, const long long* coords, float* out, int n, int C, int B, int X, int Y, int Z,
                 void* workspace, size_t workspace_bytes, occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * fp32-faithful tensor-core GEMM / implicit-GEMM convolution (wgmma bf16 x 3 passes + TMA), fused epilogues.
 * Replaces the cuBLAS / cuDNN calls issued by nn.Linear / nn.Conv3d / nn.Conv2d inside
 *   DualpathTransformerBlock  P/occformer/backbones/dualpath_block.py:36-48,79
 *   SwinBlock / WindowMSA     P/occformer/backbones/modules/window_attention.py:65-67,336-344
 *   BottleNeckASPP / ASPP     P/occformer/backbones/modules/aspp.py:49-172
 *   MSDeformAttnPixelDecoder3D  P/occformer/necks/multiscale_deformattn_3d.py:60-141 (input/lateral/output convs, Linears)
 *   Mask2Former*OccHead       P/occformer/mask2former/mask2former_nusc_occ.py:446-457 (mask einsum), decoder K/V proj
 * out[M,N] = act(A[M,K] W[N,K]^T + bias + residual): the residual is added BEFORE the activation (ResNet's
 * relu(bn2(conv2) + identity)); A, W in S32 (K % 32 == 0); act: 0 none, 1 ReLU, 2 GELU(erf), 3 Swish x*sigmoid(x)
 * (mmcv Swish); split_out: write out in
 * S32 (N % 32 == 0) instead of fp32; bias / residual fp32. */
int occ_gemm_bf16x3(const float* A, const float* W, float* out, int M, int N, int K, const float* bias,
                    const float* residual, int act, int split_out, occ_stream_t stream);
/* x (B,X,Y,Z,Cin) channel-last S32, w2 (Cout, KX*KY*KZ*Cin) tap-major S32, out (B,Xo,Yo,Zo,Cout); K in {1,3}, stride in
 * {1,2}, "same" padding dil*(K-1)/2.  2-D convs: Z = KZ = 1.  workspace (optional): occ_conv_workspace_bytes() bytes,
 * zero before its first use, one per stream -- the split-K ordering counters of the deep stages (without it the conv
 * runs single-pass).
 * gn_stats (optional, zero-initialised by the caller): (B, Cout/cpg, 2) fp64 += (sum, sumsq) per (sample, group) of the
 * raw conv output (before bias / residual / activation); cpg >= 1 channels per group, Cout % cpg == 0, at most 96
 * groups. */
size_t occ_conv_workspace_bytes(void);
int occ_conv_bf16x3(const float* x, const float* w2, float* out, int B, int X, int Y, int Z, int Cin, int Cout, int KX,
                    int KY, int KZ, int stride, int dil, const float* bias, const float* residual, int act,
                    int split_out, double* gn_stats, int cpg, void* workspace, size_t workspace_bytes,
                    occ_stream_t stream);
/* occ_conv_bf16x3 into a column slice of a wider output: out has rows of ldo floats and the conv writes columns
 * [out_off, out_off + Cout) of each row; the other columns are left untouched.  S32 output (split_out): ldo and out_off
 * multiples of 32; fp32 output: multiples of 4 (ldo == Cout, out_off == 0 is occ_conv_bf16x3).  residual stays
 * (rows, Cout) contiguous; a slice narrower than its row never runs split-K. */
int occ_conv_slice_bf16x3(const float* x, const float* w2, float* out, int ldo, int out_off, int B, int X, int Y, int Z,
                          int Cin, int Cout, int KX, int KY, int KZ, int stride, int dil, const float* bias,
                          const float* residual, int act, int split_out, double* gn_stats, int cpg, void* workspace,
                          size_t workspace_bytes, occ_stream_t stream);
/* The tiling occ_conv_bf16x3 uses for a conv shape ("same" padding): plan[0..3] = (tile rows 128 | 256, tile columns,
 * ring stages, K splits).  splitk_ok = 0 answers for a conv with bias / residual / activation / split output or without a
 * workspace (never split). */
int occ_conv_plan(int B, int X, int Y, int Z, int Cin, int Cout, int KX, int KY, int KZ, int stride, int dil,
                  int splitk_ok, int* plan);
/* Several same-input stride-1 convolutions in ONE launch via an explicit tap table: taps = ntaps x (dx, dy, dz) input offsets
 * (HOST ints), w2 (Cout, ntaps*Cin) S32 tap-major in the table's order (zero where a branch does not use a tap).  The four
 * ASPP branches (1x1 + three dilated 3x3, P/occformer/backbones/modules/aspp.py:107-113) become one 25-tap launch.
 * gn_stats / cpg as occ_conv_bf16x3. */
int occ_conv_taps_bf16x3(const float* x, const float* w2, float* out, int B, int X, int Y, int Z, int Cin, int Cout,
                         int ntaps, const int* taps, double* gn_stats, int cpg, occ_stream_t stream);
/* Tensor-core passes per 32-k operand block, library-wide launch-time setting (host side; every launcher reads it when it
 * is called).  3 (default) = fp32-faithful: hi*hi + lo*hi + hi*lo, the mode of every parity claim against the reference.
 * 1 = single-pass bf16 operands (hi halves only): BASELINE config 5's "bf16" -- a third of the tensor work, ~3e-3
 * relative error per contraction; the reference has no twin of it (SURVEY 0.7), it is validated against the fp32 oracle at
 * its own tolerance.  occ_set_mma_passes returns the previous value, or -1 for an unsupported count. */
int occ_set_mma_passes(int passes);
int occ_get_mma_passes(void);
/* fp32 rows (rows, C) <-> S32 (C % 32 == 0) */
int occ_split_rows(const float* in, float* out, long long rows, int C, occ_stream_t stream);
int occ_unsplit_rows(const float* in, float* out, long long rows, int C, occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * DepthNet of the LSS view transformer (P/occformer/image2bev/ViewTransformerLSSBEVDepth.py:435-504), inference with
 * eval-mode BatchNorms folded into the convolutions before them.  Its convolutions (reduce_conv, the BasicBlocks, the
 * ASPP branches and projection, conv_offset, the DCN's group contractions and the 1x1 heads) are occ_conv_bf16x3 /
 * occ_conv_slice_bf16x3 launches; activations are channel-last rows (image, y, x) of C floats.
 * Camera-aware SE gates (DepthNet.forward :495-504, Mlp :410-432, SELayer :435-448), fp32: for chain 0 (depth_mlp /
 * depth_se) and 1 (context_mlp / context_se) of image i, gates[chain, i] = sigmoid(We relu(Wr (W2 relu(W1' m + b1') +
 * b2) + br) + be) with m = mlp_in (n, cam) and W1', b1' = fc1 with the BatchNorm1d of mlp_input folded in.  Weights
 * K-major (in, out), both chains stacked: w1T (2, cam, C), w2T / wrT / weT (2, C, C), biases (2, C); gates (2, n, C). */
int occ_depthnet_cam_gates(const float* mlp_in, int cam, const float* w1T, const float* b1, const float* w2T,
                           const float* b2, const float* wrT, const float* br, const float* weT, const float* be,
                           float* gates, int n, int C, occ_stream_t stream);
/* x (n*rows_per_img, C) fp32 (reduce_conv output), gates (2, n, C): xd = x * gates[0] (fp32 and S32), xc_split =
 * x * gates[1] (S32); C % 32 == 0, all pointers 16-byte aligned. */
int occ_se_apply(const float* x, const float* gates, float* xd, float* xd_split, float* xc_split, int n, int rows_per_img,
                 int C, occ_stream_t stream);
/* ASPP image-pooling branch of DepthNet (:368-373,388-392): per image mean of in (B*rows_per_batch, ch) fp32 -> 1x1 conv
 * w (ch, ch) row-major + b (its BatchNorm folded in) -> ReLU -> broadcast into columns [out_off, out_off + ch) of the
 * S32 concat buffer cat (rows of ldo floats; ldo, out_off multiples of 32); ch % 32 == 0, ch <= 1024.  ws: 2*B*ch floats,
 * 16-byte aligned.  Fixed-order sums: bit-reproducible. */
int occ_depthnet_gap_branch(const float* in, float* ws, const float* w, const float* b, float* cat, int B,
                            int rows_per_batch, int ch, int ldo, int out_off, occ_stream_t stream);
/* Deformable im2col of mmcv DeformConv2dPack (DCNv1, 3x3, stride 1, padding 1, one deformable group;
 * deform_conv_cuda_kernel.cuh deformable_im2col_gpu_kernel): x (n, H, W, C) S32, off (n*H*W, off_ld) fp32 whose columns
 * 2k / 2k+1 are the (dy, dx) offset of kernel point k.  Sample point h = y - 1 + k/3 + dy, w = x - 1 + k%3 + dx (fp32);
 * it contributes only when h > -1 && w > -1 && h < H && w < W, bilinear with corners outside the map = 0.  cols (groups,
 * n*H*W, 9*C/groups) S32: column k*Cg + c of group g = channel g*Cg + c at point k, Cg = C/groups a multiple of 32. */
int occ_deform_im2col(const float* x, const float* off, int off_ld, float* cols, int n, int H, int W, int C, int groups,
                      occ_stream_t stream);
/* Modulated deformable im2col of mmcv ModulatedDeformConv2dPack (DCNv2, 3x3, stride 1, padding 1, dilation 1, one
 * deformable group; mmcv-full 1.4.0 mmcv/ops/modulated_deform_conv.py forward, modulated_deform_conv_cuda_kernel.cuh
 * modulated_deformable_im2col_gpu_kernel / dmcn_im2col_bilinear), the 3x3 conv2 of ResNetDCN's DCN Bottlenecks:
 * x (n, H, W, C) S32, C % 32 == 0; off (n*H*W, off_ld) fp32, off_ld >= 27, the conv_offset output rows: column 2k / 2k+1
 * is the (dy, dx) offset of kernel point k = ky*3 + kx, column 18 + k its mask logit (chunk(out, 3) -> o1, o2, mask;
 * offset = cat(o1, o2); mask = sigmoid(mask), applied here); columns 27.. are not read.  Sampling as occ_deform_im2col
 * (h = y - 1 + ky + dy, inside test h > -1 && w > -1 && h < H && w < W, corners outside the map = 0), then col = val *
 * sigmoid(logit).  cols (n*H*W, 9*C) S32: column k*C + c = channel c at point k.  x and cols 16-byte aligned. */
int occ_modulated_deform_im2col(const float* x, const float* off, int off_ld, float* cols, int n, int H, int W, int C,
                                occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Image encoder of the nuScenes R50 model (projects/configs/occformer_nusc/occformer_nusc_r50_256x704.py:65-79):
 * img_backbone = mmdet 2.14.0 ResNet(depth=50) (mmdet/models/backbones/resnet.py), img_neck = SECONDFPN
 * (M/models/necks/second_fpn.py:11-91), inference with eval-mode BatchNorms folded into the convolutions.  Every
 * convolution is an occ_gemm_bf16x3 / occ_conv_bf16x3 / occ_conv_slice_bf16x3 launch; the entry points below are the
 * layout steps those cannot do.  Activations are channel-last rows (image, y, x) of C floats. */
/* A stem conv on Cin = 3 as im2col: img (n, 3, H, W) NCHW fp32 -> cols (n*Ho*Wo, ncols) S32.  Column (ky*k + kx)*3 + c
 * holds img[c, stride*oy - pad_top + ky, stride*ox - pad_left + kx] (0 outside the image); columns 3*k*k .. ncols-1 are
 * 0 (ncols % 32 == 0).  The caller gives the output size, so the bottom / right padding is whatever Ho, Wo imply.
 * occ_gemm_bf16x3 with the weight repacked in the same column order then computes the conv.
 *   ResNet conv1 (ResNet._make_stem_layer): k 7, stride 2, pads 3 / 3, Ho = (H - 1)/2 + 1, ncols 160.
 *   CustomEfficientNet layers.0 (P/occformer/backbones/efficientnet.py:418-427, mmcv Conv2dAdaptivePadding): k 3,
 *   stride 2, Ho = ceil(H/2), top / left pad = pad // 2 of pad = max((Ho - 1)*2 + 3 - H, 0), ncols 32. */
int occ_stem_im2col(const float* img, float* cols, int n, int H, int W, int k, int stride, int pad_top, int pad_left,
                    int Ho, int Wo, int ncols, occ_stream_t stream);
/* ResNet.maxpool = nn.MaxPool2d(3, stride 2, padding 1): in (n, H, W, C) fp32 -> out (n, Ho, Wo, C) S32 with
 * Ho = (H - 1)/2 + 1, Wo = (W - 1)/2 + 1; padding counts as -inf, a NaN wins as in torch.  C % 32 == 0. */
int occ_maxpool3x3s2(const float* in, float* out, int n, int H, int W, int C, occ_stream_t stream);
/* (n, H, W, C) -> (n, H/f, W/f, f*f*C) with column (i*f + j)*C + c = in[f*y + i, f*x + j, c]; f in {2, 4}, H and W
 * multiples of f, C % 32 == 0.  Whole 32-column chunks are copied unchanged, so S32 stays S32.  With a (Cout, C, f, f)
 * weight repacked tap-major (occ_conv_bf16x3's layout), a kernel-f stride-f conv becomes a 1x1 conv of the result
 * (SECONDFPN's deblocks with upsample stride 1/f, second_fpn.py:52-60). */
int occ_space_to_depth(const float* in, float* out, int n, int H, int W, int C, int f, occ_stream_t stream);
/* ConvTranspose2d(kernel f, stride f) scatter (SECONDFPN's deblocks with upsample stride f, second_fpn.py:44-51):
 * in (n*h*w, f*f*C) fp32 = the GEMM of the input rows with the (f*f*C, Cin) matrix whose row (i*f + j)*C + o is
 * weight[:, o, i, j]; row (b, y, x) column (i*f + j)*C + o goes to pixel (f*y + i, f*x + j), column out_off + o of out
 * (n*(f*h)*(f*w) rows of ldo floats); the other columns are left untouched.  f in {2, 4}; C, ldo, out_off multiples of 4. */
int occ_depth_to_space(const float* in, float* out, int n, int h, int w, int C, int f, int ldo, int out_off,
                       occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * EfficientNet image encoder of the SemanticKITTI model (projects/configs/occformer_kitti/occformer_kitti.py:66-80,
 * img_backbone = CustomEfficientNet(arch='b7'), P/occformer/backbones/efficientnet.py).  Per InvertedResidual block
 * (:204-222): expand conv = occ_gemm_bf16x3 act 3 (Swish), the depthwise conv below, occ_se_gate, occ_se_scale, linear
 * conv = occ_gemm_bf16x3 with the residual.  Activations are channel-last rows (image, y, x) of C floats with C a multiple
 * of 32; a narrower layer is zero-padded (zero weights, biases and BatchNorm entries), so its pad channels stay 0. */
/* Number of per-CTA SE partial sums occ_dwconv_swish writes per image and channel for an Ho x Wo output. */
int occ_dw_tiles(int Ho, int Wo);
/* Depthwise conv + folded BatchNorm + Swish (the depthwise_conv ConvModule, :180-189, groups = C, mmcv
 * Conv2dAdaptivePadding): in (n, H, W, C) fp32 -> out (n, Ho, Wo, C) fp32,
 *   out[o, c] = swish(bias[c] + sum over (ky, kx) in order of w[ky*k + kx, c] * in[stride*oy - pad_top + ky,
 *                                                                              stride*ox - pad_left + kx, c])
 * with taps outside the input skipped (zero padding; the bottom / right padding is what Ho, Wo imply).  w tap-major
 * (k*k, C), bias (C); k in {3, 5}, stride in {1, 2}, C % 32 == 0, n <= 65535, all pointers 16-byte aligned.
 * The same launch writes partials (n, occ_dw_tiles(Ho, Wo), C): per-CTA sums of out over its pixels, in a fixed order
 * (bit-reproducible; occ_se_gate reduces them). */
int occ_dwconv_swish(const float* in, const float* w, const float* bias, float* out, float* partials, int n, int H, int W,
                     int C, int k, int stride, int pad_top, int pad_left, int Ho, int Wo, occ_stream_t stream);
/* mmdet 2.14 SELayer(C, ratio, act_cfg=(Swish, Sigmoid)) gate, fp32, one CTA per image: mean[c] = (sum over the tiles in
 * order of partials[img, t, c]) / hw, s = swish(W1 mean + b1), gate[img] = sigmoid(W2 s + b2).  Weights K-major:
 * w1T (C, S), b1 (S), w2T (S, C), b2 (C); gate (n, C).  C <= 8192, S <= 512. */
int occ_se_gate(const float* partials, int tiles, int hw, const float* w1T, const float* b1, const float* w2T,
                const float* b2, float* gate, int n, int C, int S, occ_stream_t stream);
/* SELayer output x * gate (:214-215) as the linear conv's operand: y (n*rows_per_img, C) fp32, gate (n, C) -> out S32;
 * C % 32 == 0, pointers 16-byte aligned. */
int occ_se_scale(const float* y, const float* gate, float* out, int n, int rows_per_img, int C, occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Dual-path encoder block glue (P/occformer/backbones/dualpath_block.py:65-82).
 * Token rows: voxel tokens ((b*X+x)*Y+y)*Z+z, then BEV tokens B*X*Y*Z + (b*X+x)*Y+y. */
/* GroupNorm+ReLU of the raw conv output, Z-mean, LayerNorm1 (dualpath_block.py:43-48,69; window_attention.py:355):
 * tok fp32 (residual), tokn S32 (operand of the QKV GEMM).
 * win_shift < 0: tokn rows in token order;  win_shift = 0 / 1 (needs X, XY % X == 0): tokn in the WINDOW LAYOUT of the
 * un-shifted / shifted 7x7 partition -- token (img, x, y) at row window*64 + t with window = (wx*nWy + wy)*n_images + img,
 * occ_window_layout_rows() rows in total,
 * zero-initialised once by the caller (pad positions are never written) -- the operand of occ_swin_qkv_attention.
 * Limits: C in {128, 256, 512, 1024}, Z <= 16, groups <= 32 with C / groups a multiple of 4, and the Z-column buffer
 * Z * C * 4 bytes of one (b, x, y) column within 48 KiB (C = 1024 needs Z <= 12); -1 / -2 otherwise, nothing enqueued. */
int occ_gn_relu_zmean_ln(const float* y, const double* stats, const float* gn_w, const float* gn_b,
                         const float* ln_w, const float* ln_b, float* tok, float* tokn, int B, int XY, int Z, int C,
                         int groups, int X, int win_shift, occ_stream_t stream);
long long occ_window_layout_rows(int B, int X, int Y, int Z);
int occ_layernorm(const float* in, const float* w, const float* b, float* out, long long rows, int C, int split_out,
                  occ_stream_t stream);
/* o = act(gn(in[row, c])) (+ residual[row, c]) -- ASPP / neck norms (aspp.py:42-46,117-120,166-172): out[row, c] = o
 * (fp32, optional) and / or out_split[row, out_off + c] = o in S32 with row pitch ldo (optional) */
int occ_gn_apply(const float* in, const double* stats, const float* w, const float* b, const float* residual,
                 float* out, float* out_split, long long rows, int rows_per_batch, int C, int groups, int ldo,
                 int out_off, int relu, occ_stream_t stream);
/* ASPP image-pooling branch: GAP -> 1x1 conv -> GN -> ReLU -> broadcast (aspp.py:89-95,113-114) into columns
 * [out_off, out_off + ch) of the S32 concat buffer cat (rows of ldo floats; ldo, out_off multiples of 32,
 * out_off + ch <= ldo); ch % 32 == 0, ch <= 1024, 256 % (ch / 4) == 0, B <= 65535.
 * sums_ws: workspace of B*ch doubles followed by B*ch floats.  The column sums are fp64 atomics: not bit-reproducible. */
int occ_aspp_gap_branch(const float* in, double* sums_ws, const float* wconv, const float* gw, const float* gb,
                        float* cat, int B, int rows_per_batch, int ch, int groups, int ldo, int out_off,
                        occ_stream_t stream);
/* coeff = sigmoid(<x,w>+b); out = x + coeff * bev + identity (identity optionally GroupNorm'd: strided skip path)
 * dualpath_block.py:36-41,79-82.  x / identity / out rows are voxel tokens, bev (B*XY, C) one row per (b, x, y) column.
 * C in {128, 256, 512, 1024} (-2 otherwise, nothing enqueued); with id_stats, C / groups a multiple of 4. */
int occ_dualpath_fuse(const float* x, const float* bev, const float* cw, float cbias, const float* identity,
                      int identity_split /*identity is S32*/, const double* id_stats, const float* id_w,
                      const float* id_b, int groups, float* out /*fp32, optional*/, float* out_split /*S32, optional*/,
                      int B, int XY, int Z, int C, occ_stream_t stream);
/* Swin block tail for C == 128 in one tensor-core kernel (csrc/swin_mlp_fused.cu): y1 = tok + att Wp^T + bp (WindowMSA.proj
 * + the ShiftWindowMSA residual, window_attention.py:105-107 / swin.py SwinBlock.forward), out = y1 + W2 GELU(W1 LN2(y1)
 * + b1) + b2 (norm2 + FFN + residual).  att and the weights ((out, in) row-major) in S32; tok / out fp32.  Returns -2 for
 * C != 128 (the caller then uses occ_gemm_bf16x3 / occ_layernorm). */
int occ_swin_proj_ffn(const float* att, const float* tok, const float* wp, const float* bp, const float* ln_w,
                      const float* ln_b, const float* w1, const float* b1, const float* w2, const float* b2, float* out,
                      long long M, int C, occ_stream_t stream);
/* (shifted) 7x7 window attention core over B*(Z+1) images: ShiftWindowMSA.forward + WindowMSA.forward
 * (window_attention.py:168-242, 69-107) minus the qkv / proj linears, on the wgmma tensor cores.
 * bias_pad = relative_position_bias_table[relative_position_index] as (heads, 49*49 padded to 2404 floats).
 * qkv_head_major = 0: qkv / qkv_bias columns in the reference order [q|k|v][head][32] (WindowMSA.qkv);  1: [head][q|k|v][32]
 * (the caller permuted the rows of the qkv weight: one contiguous 384-byte run per (token, head)). */
int occ_window_attention(const float* qkv /*S32*/, const float* qkv_bias /*S32 row*/, const float* bias_pad,
                         float* out /*S32*/, int B, int X, int Y, int Z, int C, int heads, int shift,
                         int qkv_head_major, occ_stream_t stream);

/* The same attention with the QKV projection fused in (C == 128; csrc/swin_attn_fused.cu): tokn
 * (occ_window_layout_rows(B,X,Y,Z), 128) S32 = LayerNorm1'ed tokens in the window layout of THIS shift (see
 * occ_gn_relu_zmean_ln), out (B*X*Y*(Z+1), 128) S32 in token order; wqkv (384, 128) S32 / bqkv (384) fp32 = WindowMSA.qkv with HEAD-MAJOR rows [head][q|k|v][32]; the
 * q/k/v tensor never exists in HBM.  Returns -2 for C != 128 (use occ_gemm_bf16x3 + occ_window_attention). */
int occ_swin_qkv_attention(const float* tokn, const float* wqkv, const float* bqkv, const float* bias_pad, float* out,
                           int B, int X, int Y, int Z, int C, int heads, int shift, occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * MSDeformAttnPixelDecoder3D, the neck between encoder and head (P/occformer/necks/multiscale_deformattn_3d.py:143-248,
 * P/occformer/necks/multi_scale_deform_attn_3d.py:17-80,185-286).  Token rows are "level-major":
 * row(l, b, x, y, z) = B*start_l + b*n_l + (x*Y_l + y)*Z_l + z with the L levels ordered coarse -> fine (start_l = tokens
 * of the coarser levels of one sample), so every level is a contiguous channel-last (B, X_l, Y_l, Z_l, C) tensor.
 * `grids` = L x (X, Y, Z) ints in HOST memory.  The Linears / 1x1x1 / 3x3x3 convolutions go through occ_gemm_bf16x3 /
 * occ_conv_bf16x3. */
/* [LayerNorm (norms.k of the encoder layer) of each row ->] out_f32 = x (fp32), out_s32 = x (S32), out_pos = x + pos[token]
 * (S32; pos (Nq, C) = SinePositionalEncoding3D + level_encoding of the token's level: query_pos of the reference); any of
 * the three outputs may be NULL (not all three); ln_w / ln_b NULL = no normalisation, both or neither; out_pos needs pos.
 * C % 32 == 0, 32 <= C <= 1024, C / 32 in {1, 2, 3, 4, 6, 8, 12, 16, 24, 32} (else -2); 1 <= L <= 4.  LayerNorm eps 1e-5,
 * biased variance. */
int occ_neck_token_prep(const float* in, const float* ln_w, const float* ln_b, const float* pos, float* out_f32,
                        float* out_s32, float* out_pos, int L, int B, const int* grids, int C, occ_stream_t stream);
/* One encoder layer after the deformable gather, in one tensor-core kernel (csrc/neck_tail_fused.cu):
 * y = x + att Wo^T + bo (output_proj + identity), x1 = LayerNorm(y; ln1), y2 = x1 + W2 ReLU(W1 x1 + b1) + b2 (FFN + identity),
 * out = LayerNorm(y2; ln2) written as out_f32 (fp32), out_s32 (S32) and out_pos = out + pos[token] (S32), each optional as
 * in occ_neck_token_prep (not all three; out_pos needs pos).  att (rows, E) S32, x (rows, E) fp32, rows = B * sum X*Y*Z
 * of the L level grids (HOST ints); wo (E, E), w1 (F, E), w2 (E, F) S32, (out, in) row-major as in nn.Linear.
 * E in {96, 192} (else -2, nothing enqueued), F % 32 == 0, F <= 4096; every matrix 16-byte aligned.  LayerNorm eps 1e-5,
 * biased variance. */
int occ_neck_layer_tail(const float* att, const float* x, const float* wo, const float* bo, const float* ln1_w,
                        const float* ln1_b, const float* w1, const float* b1, const float* w2, const float* b2,
                        const float* ln2_w, const float* ln2_b, const float* pos, float* out_f32, float* out_s32,
                        float* out_pos, int L, int B, const int* grids, int E, int F, occ_stream_t stream);
/* multi_scale_deformable_attn_pytorch + the sampling-location arithmetic of MultiScaleDeformableAttention3D.forward:
 * value (rows, value_ld) = value_proj output, head h at columns [h*head_ld, h*head_ld + E/H) (head_ld = E/H, or E/H
 * rounded up to 32 floats so that a head slice is one 128-byte line); ow (rows, H*L*P*4) = [sampling_offsets (h,l,p,(z,y,x)) | attention logits (h,l,p)];
 * out (rows, E) S32 = sum_{l,p} softmax(logits) * trilinear(value level l)(ref + offset / (Z_l,Y_l,X_l)), zeros outside,
 * align_corners=False; strides = the L feature strides (HOST floats; reference-point arithmetic).  Softmax over all L*P
 * points of a head.  P == 4 (else -2); 1 <= L <= 4, E % 32 == 0, E / H % 4 == 0, E / H <= 32, head_ld % 4 == 0,
 * value_ld >= (H - 1) * head_ld + E / H and % 4 == 0, value and out 16-byte aligned; B * sum X*Y*Z < 2^31. */
int occ_ms_deform_attn(const float* value, int value_ld, int head_ld, const float* ow, float* out, int L, int B,
                       const int* grids, const float* strides, int E, int H, int P, occ_stream_t stream);
/* FPN step (:228-240): out_s (S32) = GroupNorm(cur raw lateral-conv output, stats) + trilinear upsample
 * (align_corners=False) of coarse (B, Xc, Yc, Zc, C) fp32, any size ratio (exact x2 on every axis takes a tiled kernel).
 * C % 32 == 0, C <= 4096, groups divides C; cur, coarse and out_s 16-byte aligned; GroupNorm eps 1e-5. */
int occ_gn_upsample_add(const float* cur, const double* stats, const float* gw, const float* gb, int groups,
                        const float* coarse, float* out_s, int B, int X, int Y, int Z, int Xc, int Yc, int Zc, int C,
                        occ_stream_t stream);
/* GroupNorm statistics of a finished tensor x (B, rows_per_sample, C), 16-byte aligned, C % 4 == 0: stats (B, C/cpg, 2)
 * fp64 += (sum, sumsq); any cpg with at most 96 groups.  For a conv whose bias precedes the GroupNorm (the neck's input
 * convs): the statistics of occ_conv_bf16x3 are those of the raw output. */
int occ_gn_stats(const float* x, double* stats, int B, int rows_per_sample, int C, int cpg, occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Mask2Former-3D occupancy decoder head (P/occformer/mask2former/mask2former_nusc_occ.py, mask2former_occ.py).
 * Layouts: voxel memories channel-last (B, S, E); queries (B, Q, E); mask logits "query-last" (B, S, Q).
 * The voxel-side GEMMs (K/V projections :657-667 via nn.MultiheadAttention in_proj; mask einsum :457) go through
 * occ_gemm_bf16x3; the entry points below are the fused query-side / reduction kernels. */
/* SinePositionalEncoding3D.forward, normalize=True, all-False mask (positional_encoding.py:58-108): out (X*Y*Z, 3F) */
int occ_sine_pos3d(float* out, int X, int Y, int Z, int num_feats, float temperature, float scale, float eps,
                   float offset, occ_stream_t stream);
/* level prep (mask2former_nusc_occ.py:614-630): mem = in + level_embed, kpos = in + level_embed + pos, both S32;
 * in is channel-last (B,S,C) or the reference layout (B,C,S); level_embed / pos+kpos optional. */
int occ_head_prep(const float* in, int in_channel_last, const float* level_embed, const float* pos, float* mem,
                  float* kpos, int B, long long S, int C, occ_stream_t stream);
/* Query counts.  The decoder runs Qs = round_up(Q, 4) query slots per sample (rows 16-byte aligned for TMA / float4);
 * slots >= Q hold zero query_feat / query_embed and never act as self-attention keys.  Every per-query buffer below
 * ((B, S, Q) masks / pooled / bits, (B, Q) flags, (B*Q, E) rows) uses the slot count as its Q, Q <= 256; the kernels
 * tile queries by 128 above 128. */
/* forward_head query side (:446-455): [optional: query = LN(norms.2)(query_in) -> query_state] -> post_norm LN ->
 * cls_embed -> cls_out (rows, NC); mask_embed MLP -> membed_out (rows, E) S32; [optional: the NEXT layer's
 * cross-attention query projection qh_out = ((query + query_pos) Wq^T + bq) * scale].  Weights K-major (in, out). */
int occ_query_head(const float* query_in, const float* n2w, const float* n2b, float* query_state, const float* pn_w,
                   const float* pn_b, const float* clsT, const float* cls_b, int NC, const float* m0T, const float* m0b,
                   const float* m1T, const float* m1b, const float* m2T, const float* m2b, float* cls_out,
                   float* membed_out, const float* query_pos, int Q, const float* wqT, const float* bq, float scale,
                   float* qh_out, const float* ffn_part /*(nparts, rows, E) FFN column-block partials, added to query_in
                   in the order 0..nparts-1; may be NULL with nparts = 0*/, int nparts, int rows, int E, occ_stream_t stream);
/* adaptive_max_pool3d of the mask logits (:463), general windows -> pooled (B, Xo*Yo*Zo, Q) as order-preserving ints
 * (see occ_mask_gemm_pool; a -0.0 maximum encodes as +0.0); row_flag[b*Q+q] = 1 iff some key of the row is un-blocked
 * (code >= 0), else the row attends everywhere (:652-653).  attn_mask == code < 0. */
int occ_mask_pool(const float* mask, int* pooled, int* row_flag, int B, int X, int Y, int Z, int Xo, int Yo, int Zo,
                  int Q, occ_stream_t stream);
/* mask einsum fused with the attention-mask pooling (:457-466) of the intermediate decoder layers, the (B,V,Q) logits
 * never written: pooled[b,cell,q] = max over the cell of <mf[b,v,:], membed[b,q,:]> as an order-preserving int
 * (i >= 0 ? i : i ^ 0x7FFFFFFF of the float bits i, except that -0.0 encodes as +0.0, i.e. 0: sigmoid(-0.0) = 0.5 is not
 * blocked; blocked <=> code < 0), flag[b,q] as occ_mask_pool.  Covers cubic
 * windows of 2, 4 or 8 voxels (box-divisible grids, E % 32 == 0, Q <= 256); returns -2 with nothing enqueued for any other
 * shape (the caller then uses occ_gemm_bf16x3 per sample + occ_mask_pool). */
int occ_mask_gemm_pool(const float* mf /*S32*/, const float* membed /*S32*/, int* pooled, int* flag, int B, int X, int Y,
                       int Z, int E, int Q, int Xo, int Yo, int Zo, occ_stream_t stream);
/* masked cross attention (mmcv MultiheadAttention -> nn.MultiheadAttention, bool attn_mask) on the wgmma tensor cores
 * (128-key tiles, TMA operand loads, P in registers); qh fp32, Kp / Vp S32 (one chunk per (key, head)) with row pitch
 * ld and this layer's columns at koff / voff, all three multiples of 32 (a head's slice is one aligned chunk); writes
 * occ_cross_attn_tc_partials(S) partials per (sample, head): part (B, H, npart, Q, 34) = running max, running sum, 32
 * value accumulators */
int occ_cross_attn_tc_partials(int S);
/* pooled (B,S,Q) ordered-int mask logits -> bits (B, 4*ceil(S/128), Q): one "blocked" bit per (key, query) */
int occ_mask_bits(const int* pooled, unsigned* bits, int B, int S, int Q, occ_stream_t stream);
int occ_cross_attn_tc(const float* qh, const float* Kp, const float* Vp, int ld, int koff, int voff, const unsigned* bits,
                      const int* row_flag, float* part, int B, int S, int Q, int E, int H, occ_stream_t stream);
/* merge partials -> out_proj -> +identity -> LN(norms.0) -> query1; self-attention in_proj -> sa_qkv (rows, 3E) */
int occ_cross_merge(const float* part, int nchunk, int H, const float* query, const float* query_pos, int Q,
                    const float* woT, const float* bo, const float* n0w, const float* n0b, const float* sa_inT,
                    const float* sa_inb, float scale, float* query1, float* sa_qkv, int rows, int E,
                    occ_stream_t stream);
/* self attention of the Q query slots of a sample over its first nkeys (real) queries -> out_proj -> +identity -> LN(norms.1) -> x1; FFN(ReLU) + identity accumulated
 * as F/E column blocks: ybuf = x1 + b2, ffn_part (F/E, rows, E) = the blocks' contributions; occ_query_head adds them in
 * a fixed order (bit-reproducible, no floating-point atomics) and applies the closing LN(norms.2). */
int occ_self_attn_ffn(const float* sa_qkv, const float* query1, int Q, int nkeys, const float* woT, const float* bo,
                      const float* n1w, const float* n1b, const float* f1T, const float* f1b, const float* f2T,
                      const float* f2b, int F, float* x1, float* ybuf, float* ffn_part, int rows, int E, int H,
                      occ_stream_t stream);
/* simple_test tail (:725-736, format_results :691-696): trilinear upsample (align_corners=True) -> sigmoid ->
 * einsum with softmax(cls)[..., :-1]; mask (B, X*Y*Z, Qs) (Qs % 4 == 0 slots per row), cls (B, Q, NC) of the first
 * Q <= Qs slots (the others contribute nothing) -> out (B, NC-1, Xo, Yo, Zo); labels (optional, (B, Xo, Yo, Zo) uint8) =
 * argmax over the class axis (post_process_semantic, occupancyformer.py:238-243) */
int occ_classmix(const float* mask, int Qs, const float* cls, float* out, unsigned char* labels, int B, int X, int Y,
                 int Z, int Xo, int Yo, int Zo, int Q, int NC, occ_stream_t stream);
/* (B, S, Q) -> (B, Q, S): the reference's mask_pred layout, for forward()'s return value */
int occ_transpose_sq(const float* in, float* out, int B, long long S, int Q, occ_stream_t stream);
/* forward_lidarseg eval branch (:505-542): grid_sample of one sample's class volume (K,X,Y,Z) at n points
 * (rows of pts_stride floats, xyz first) + softmax -> out (n, K) */
int occ_lidarseg_points(const float* vox, const float* pts, int pts_stride, int n, float x_min, float y_min,
                        float z_min, float x_max, float y_max, float z_max, int X, int Y, int Z, int K, int border,
                        float* out, occ_stream_t stream);
/* Panoptic ids, P/mask2former/mask2former_nusc_panoptic_occ.py:715-784.  mask (B, X*Y*Z, Qs) query-last logits
 * (Qs % 4 == 0, Qs <= 256) of Q real queries, cls (B, Q, NC).  Per output voxel (trilinear upsample to (Xo,Yo,Zo),
 * align_corners=True; identity when equal) q(v) = first argmax over the Q queries; label(q) = argmax of
 * softmax(cls[q])[:NC-1]; sem = label(q(v)); pan = label * 1000 for stuff labels, label * 1000 + i for thing labels
 * (bit k of thing_mask), where i numbers the (label, query) pairs that win a voxel in ascending (label, query) order
 * from 1, per sample (format_panoptic_occupancy_results :749-784).  sem / pan int64 (B, Xo, Yo, Zo).  Workspaces: qidx
 * (B*Xo*Yo*Zo bytes), present (B*Qs ints), table (B*Qs*2 int64, 16-byte aligned).  No host synchronisation.
 * first_label = 1 applies the LiDAR point rule instead (label(q) = 1 + argmax of softmax(cls[q])[1:NC-1],
 * format_panoptic_lidar_results :715-747) to logits already sampled at the points (grid (n, 1, 1)). */
int occ_panoptic_voxels(const float* mask, int Qs, const float* cls, int B, int X, int Y, int Z, int Xo, int Yo, int Zo,
                        int Q, int NC, unsigned long long thing_mask, int first_label, unsigned char* qidx, int* present,
                        long long* table, long long* sem, long long* pan, occ_stream_t stream);
/* The same for n LiDAR points per sample (pts (B, n, pts_stride), xyz first; forward_lidar_panopticseg :515-563,
 * format_panoptic_lidar_results :715-747): the Q logits are grid-sampled (bilinear, align_corners=True, border | zeros
 * padding) as in occ_lidarseg_points, label(q) = 1 + argmax of softmax(cls[q])[1:NC-1], presence over the points.
 * sem / pan int64 (B, n); workspaces as above with qidx (B*n bytes). */
int occ_panoptic_points(const float* mask, int Qs, const float* cls, int B, int X, int Y, int Z, int Q, int NC,
                        unsigned long long thing_mask, const float* pts, int pts_stride, int n, float x_min, float y_min,
                        float z_min, float x_max, float y_max, float z_max, int border, unsigned char* qidx,
                        int* present, long long* table, long long* sem, long long* pan, occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Evaluation tail (SURVEY.md 8(f)4): the integer counts behind the path's single collective
 * (P/occformer/apis/test.py:195-212 sums them over ranks). */
/* SSCMetrics.get_score_completion + get_score_semantic_and_completion (P/utils/ssc_metric.py:104-168), masked by
 * target != ignore: pred / target n uint8 voxel labels -> out[0..2] = completion tp, fp, fn; out[3 + c], out[3 + K + c],
 * out[3 + 2K + c] = semantic tp, fp, fn of class c (3 + 3K int64).  conf_ws: K*K int64 scratch. */
int occ_ssc_counts(const unsigned char* pred, const unsigned char* target, long long n, int K, int ignore,
                   long long* conf_ws, long long* out, occ_stream_t stream);
/* OccupancyFormer.simple_evaluation_semantic (P/occformer/detectors/occupancyformer.py:219-224,246-254) + fast_hist_crop
 * (P/utils/metric_util.py:8-23): scores (n, K) point class scores, labels (n) int64 -> hist[(gt-1)*(K-1) + (pred-1)] += 1
 * for gt in 1..K-1, pred = 1 + argmax(scores[:, 1:]); hist ((K-1)^2 int64) is accumulated. */
int occ_lidarseg_hist(const float* scores, const long long* labels, int n, int K, long long* hist, occ_stream_t stream);
/* PanopticEval.addBatch (P/utils/panoptic_eval.py:11-246) on one flat scan of n elements (n <= 2^29): x = prediction,
 * y = target; semantic labels in [0, K), K <= 32; bit c of ignore_mask = class c is ignored.  parts: 1 = confusion
 * matrix only (addBatchSemIoU; x_inst / y_inst may be NULL), 2 = panoptic counts only (addBatchPanoptic), 3 = both.
 * state (int64, ACCUMULATED): conf K*K [pred][target] | tp K | fp K | fn K | iou K x 3 | invalid, where the iou sum of
 * class c is (l0 + l1 * 2^31 + l2 * 2^62) * 2^-53 over its limbs -- exact integers, so states of several calls or ranks
 * add element by element.  An element with a label outside [0, K) or an id >= 2^31 - 1 only increments invalid.
 * Segments are (class, id >= 0) pairs of non-ignored classes, after dropping elements whose target class is ignored;
 * a pair of the same class with 2 * intersection > union is a match.  ws: occ_panoptic_eval_workspace_bytes(n) bytes,
 * 16-byte aligned, zeroed by the call.  No host synchronisation. */
size_t occ_panoptic_eval_workspace_bytes(long long n);
int occ_panoptic_eval(const long long* x_sem, const long long* x_inst, const long long* y_sem, const long long* y_inst,
                      long long n, int K, unsigned int ignore_mask, int min_points, int parts, void* ws,
                      size_t ws_bytes, long long* state, occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Occupancy ground truth from the labelled LiDAR points (csrc/occ_targets.cu): the gt_occ of
 *   LoadNuscOccupancyAnnotations          P/datasets/pipelines/loading_nusc_occ.py:95-138 (nb_process_label :122-138)
 *   LoadNuscPanopticOccupancyAnnotations  P/datasets/pipelines/loading_nusc_panoptic_occ.py:120-166 (nb_process_label :147-166)
 * built from the points_occ the test loop already hands to the model.  pts (n, ld >= 4) fp32 rows [x, y, z, label, ...]
 * of B samples, sample b at rows [offsets[b], offsets[b+1]); offsets = B + 1 HOST int64, offsets[0] = 0, non-decreasing,
 * 1 <= B <= 256.  Voxel index floor((clip(p, lo, hi - 1e-5) - lo) / voxel_size) in float64, voxel_size = (hi - lo) / grid
 * computed on the host as numpy does.  Each occupied voxel takes its majority id (ties: the smallest id, np.argmax), then
 * 0 -> ignore and empty_id -> 0; unoccupied voxels are 0.  panoptic = 0: ids < 256, every id votes.  panoptic = 1: ids
 * < 65536, id 0 does not vote (a voxel holding only id 0 becomes ignore) except in the voxel that comes last in
 * np.lexsort((x, y, z)) order (largest z, then y, then x) of its sample, where the reference's counter keeps it.
 * out (B, X, Y, Z) int64, overwritten.  Points with a label that is negative, not an integer or >= the mode's limit, or
 * with a non-finite coordinate, and (voxel, id) pairs of more than 65535 points (the reference's uint16 counter wraps)
 * add to *invalid (one device int, ACCUMULATED) and are never written out of bounds.  n = 0 gives an all-zero volume.
 * ws: occ_lidarseg_occupancy_workspace_bytes(n, B) bytes, 16-byte aligned, zeroed by the call.  Five enqueued launches /
 * memsets per call, deterministic (integer atomics only), no host synchronisation. */
size_t occ_lidarseg_occupancy_workspace_bytes(long long n, int B);
int occ_lidarseg_occupancy(const float* pts, int ld, const long long* offsets /*HOST*/, int B, double x_min,
                           double y_min, double z_min, double x_max, double y_max, double z_max, int X, int Y, int Z,
                           int panoptic, long long empty_id, long long ignore, int* invalid, void* ws, size_t ws_bytes,
                           long long* out, occ_stream_t stream);

/* SemanticKITTI occupancy ground truth from the dataset's voxel files (csrc/semkitti_labels.cu), replacing the offline
 *   semantic_kitti_preprocess.main _1_1 volume    P/tools/kitti_process/semantic_kitti_preprocess.py:117-142
 * and LoadSemKittiAnnotation's torch.tensor(np.load(...)).long() (P/datasets/pipelines/loading_kitti_occ.py:34-53).
 * label: B samples of nvox uint16 little-endian values (the .label files' bytes, sample b at b * 2 * nvox), 16-byte
 * aligned; invalid: B samples of nvox / 8 bytes (the .invalid files, bit-packed, most significant bit first,
 * io_data.unpack); nvox % 8 == 0, 1 <= B <= 65536.  lut: lut_size int32 values, the remap LUT as io_data.get_remap_lut
 * builds it.  out (B, nvox) int64, 16-byte aligned, overwritten: lut[label], then 255 where the invalid bit is set.  A
 * label >= lut_size (the reference's numpy IndexError) adds to bad[b] (B device ints, ACCUMULATED) and is written as
 * 255; nothing is read or written out of bounds.  One launch per call, no host synchronisation. */
int occ_semkitti_labels(const unsigned char* label, const unsigned char* invalid, int B, long long nvox,
                        const int* lut, int lut_size, int* bad, long long* out, occ_stream_t stream);

/* The training-mode SemanticKITTI ground truth (csrc/semkitti_labels.cu): occ_semkitti_labels' volume through
 *   LoadSemKittiAnnotation(is_train=True) / voxel_transform   P/datasets/pipelines/loading_kitti_occ.py:34-53,55-117
 *   custom_rotate_3d                                          P/datasets/pipelines/loading_nusc_occ.py:206-225
 * bit for bit: .astype(np.uint8), then, when the sample's rotate flag is set, Image.rotate(angle, NEAREST,
 * fillcolor=255) of every z slice (a 256 x 256 mode-"L" image, rows = x, columns = y), then [:, :, ::-1] when flip_dz,
 * [:, ::-1] when flip_dy, [::-1] when flip_dx, then .long().  The volume is SemanticKITTI's 256 x 256 x 32.
 *   label, invalid  as occ_semkitti_labels with nvox = 2^21; label 16-byte aligned, invalid 4-byte aligned
 *   aug             device int32 (B, 10), 4-byte aligned: flip_dx, flip_dy, flip_dz, rotate (each 0 / nonzero), then
 *                   a0..a5, the 16.16 coefficients of occ_prepare_images_aug (occformer_b200.image_prep.rotate_coeffs of
 *                   (angle, 256, 256), Pillow's copy and transposes included): output slice pixel (y, x) reads
 *                   (x', y') = ((a5 + x a4 + y a3) >> 16, (a2 + x a1 + y a0) >> 16), 255 outside the slice; the host
 *                   sets rotate only when not np.isclose(angle, 0), as the reference decides; ignored when rotate = 0
 *   lut             as occ_semkitti_labels; its values must lie in [0, 255] (the reference's uint8 cast)
 *   out             (B, 256, 256, 32) int64, 16-byte aligned, overwritten
 * A label >= lut_size adds to bad[b] (B device ints, ACCUMULATED) once per voxel of the source volume, whether or not
 * the rotation reads it, and is written as 255.  1 <= B <= 65536.  One launch per call, no host synchronisation. */
int occ_semkitti_labels_aug(const unsigned char* label, const unsigned char* invalid, int B, const int* aug,
                            const int* lut, int lut_size, int* bad, long long* out, occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Camera images from the decoded frames (csrc/image_prep.cu): steps 2-4 of the test loaders' image side,
 *   LoadMultiViewImageFromFiles_OccFormer     P/datasets/pipelines/loading_nusc_imgs.py:34-62,181-195
 *   LoadMultiViewImageFromFiles_SemanticKitti P/datasets/pipelines/loading_kitti_imgs.py:35-65
 * bit for bit: Pillow 9.4's Image.resize((rW, rH)) (BICUBIC, a = -0.5, no reducing_gap) of the uint8 BGR frame, then
 * Image.crop((x0, y0, x0 + fW, y0 + fH)) (0 outside the resized image), then mmcv's imnormalize as a table lookup.
 * Resize: separable, horizontal pass first; each pass accumulates (1 << 21) + sum w * p in int32 over Pillow's
 * precompute_coeffs taps (weights normalised in float64, then int32 with 22 fractional bits, rounded away from zero) and
 * clips >> 22 to [0, 255]; the horizontal result is uint8.  An unchanged axis gives identity weights, i.e. Pillow's copy.
 * Only the source rows and resized columns the crop needs are computed.
 *   frames     uint8, frame_bytes bytes; image m is HWC BGR at byte offsets[m] (HOST int64), H x W x 3 bytes
 *   geom       HOST int32 (M, 6): H, W, rW, rH, x0, y0 per image
 *   tables     HOST int64 (M, 2): device addresses of image m's horizontal (W -> rW) and vertical (H -> rH) tables,
 *              each int32 [2 * n] (first tap, tap count) per output index, then [ksize * n] weights tap-major
 *              (w[k * n + i]), n = rW | rH, ksize = 2 * ceil(2 * max(in / n, 1)) + 1 (Pillow's; unused taps 0)
 *   norm       device float (3, 256): output channel c of source value v = norm[c * 256 + v]; swap_rb = 1 reads output
 *              channel c from source channel 2 - c (BGR -> RGB), swap_rb = 0 from channel c
 *   out        float (M, 3, fH, fW), overwritten
 *   ws         occ_prepare_images_workspace_bytes(geom, M, fH, fW) bytes (the uint8 horizontal-pass rows), 16-byte
 *              aligned; 0 bytes when no crop overlaps its resized image
 * 1 <= M <= 256.  Two kernel launches per call whatever M and the geometries, no memset, no host synchronisation.
 * Returns -1 for: M out of range, a non-positive size, a frame past frame_bytes, a crop origin with |x0|, |y0| >= 2^30,
 * a null table, a short or misaligned workspace, swap_rb not 0 / 1.  Returns -2 when an axis needs more than 129 taps
 * (a downscale by more than 32), the bound of the kernels' shared-memory row span.  Nothing is enqueued on an error. */
size_t occ_prepare_images_workspace_bytes(const int* geom /*HOST*/, int M, int fH, int fW);
int occ_prepare_images(const unsigned char* frames, long long frame_bytes, const long long* offsets /*HOST*/,
                       const int* geom /*HOST*/, int M, int fH, int fW, const long long* tables /*HOST*/,
                       const float* norm, int swap_rb, void* ws, size_t ws_bytes, float* out, occ_stream_t stream);

/* The training loaders' camera images (csrc/image_prep.cu): occ_prepare_images with the flip and rotation of
 *   LoadMultiViewImageFromFiles_OccFormer(is_train=True).img_transform_core      P/datasets/pipelines/loading_nusc_imgs.py:55-62
 *   LoadMultiViewImageFromFiles_SemanticKitti(is_train=True).img_transform_core  P/datasets/pipelines/loading_kitti_imgs.py:57-65
 * bit for bit: resize and crop as above, then Image.transpose(FLIP_LEFT_RIGHT) when flipped, then Pillow's
 * Image.rotate(angle) (NEAREST, no expand, black fill) of the fW x fH crop, then the normalisation table.
 *   aug        HOST int32 (M, 7): flip (0 / 1), then a0..a5, the 16.16 fixed-point coefficients of Pillow's affine_fixed:
 *              output pixel (x, y) reads crop pixel ((a2 + y a1 + x a0) >> 16, (a5 + y a4 + x a3) >> 16) of the
 *              (mirrored) crop and takes 0 outside it.  occformer_b200.image_prep.rotate_coeffs computes them, also for
 *              the angles where Pillow copies or transposes instead (0, 180, and 90 / 270 of a square crop).  At the
 *              crop's corners a2 + y a1 + x a0 and a5 + y a4 + x a3 must fit in int32.
 * Every other argument, the workspace (occ_prepare_images_workspace_bytes) and the errors are occ_prepare_images';
 * a flip other than 0 / 1 or coefficients past int32 also return -1.  Two kernel launches per call whatever M, no
 * memset, no host synchronisation; nothing is enqueued on an error. */
int occ_prepare_images_aug(const unsigned char* frames, long long frame_bytes, const long long* offsets /*HOST*/,
                           const int* geom /*HOST*/, const int* aug /*HOST*/, int M, int fH, int fW,
                           const long long* tables /*HOST*/, const float* norm, int swap_rb, void* ws, size_t ws_bytes,
                           float* out, occ_stream_t stream);

/* Depth maps from the LiDAR scan (csrc/lidar_depth.cu): the gt_depths of
 *   CreateDepthFromLiDAR   P/datasets/pipelines/lidar2depth.py:15-82
 * bit for bit as the reference computes them with one torch thread (a DataLoader worker).  For each point p of sample
 * b and camera n, in fp32, each dot product summed left to right without fused multiply-adds:
 *   c = inv_rot (p - trans);  (x, y, d) = rows 0..2 of K c (K 4 x 4: of K (c, 1));  u = x / d, v = y / d;
 *   (u', v') = post_rot[:2, :2] (u, v) + post_tran[:2];
 * a point with u' >= 0, v' >= 0, u' <= fW - 1, v' <= fH - 1 and d > 0 (false for NaN) lands on pixel
 * (rint(v'), rint(u')), round half to even.  Each pixel holds the smallest d that lands on it, else 0 (the reference's
 * descending sort and last write win with one thread; with several its index_put_ picks any).
 *   pts         float (n, 3), sample b's points at rows [offsets[b], offsets[b + 1]); NULL allowed when n = 0
 *   offsets     HOST int64 (B + 1): offsets[0] = 0, non-decreasing, 1 <= B <= 256
 *   inv_rots    float (B, N, 3, 3): rots.inverse() computed on the host in CPU fp32, as the reference does
 *   trans       float (B, N, 3);  intrins float (B, N, k, k), k = intrin_dim = 3 or 4
 *   post_rots   float (B, N, 3, 3);  post_trans float (B, N, 3)
 *   out         float (B, N, fH, fW), overwritten
 * 1 <= N <= 65535, fH, fW >= 1, fH * fW <= 2^31.  Three enqueued launches and memsets per call whatever the scans,
 * deterministic, no host synchronisation (capturable in a CUDA graph).  Returns -1 for a bad count, size or offset,
 * with nothing enqueued. */
int occ_lidar_depth(const float* pts, const long long* offsets /*HOST*/, int B, int N, const float* inv_rots,
                    const float* trans, const float* intrins, int intrin_dim, const float* post_rots,
                    const float* post_trans, int fH, int fW, float* out, occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Camera frames from their JPEG files (csrc/jpeg_decode.cu): step 1 of the test loaders' image side,
 *   LoadMultiViewImageFromFiles_OccFormer     P/datasets/pipelines/loading_nusc_imgs.py:181-195 (mmcv.imread, cv2)
 * bit for bit as cv2.imdecode(buf, IMREAD_UNCHANGED) with libjpeg-turbo: Huffman-coded sequential DCT, 8-bit samples,
 * three components (YCbCr) in one interleaved scan, luma sampling 1x1 / 2x1 / 2x2 with chroma 1x1, any restart interval;
 * libjpeg's islow IDCT with the output + 128 clamped to [0, 255] (libjpeg-turbo's SIMD IDCT, not its wrapping C table),
 * fancy (triangle) chroma upsampling with edges replicated at the component's real size, libjpeg's YCbCr -> RGB tables.
 * occformer_b200/jpeg.py parses the headers and refuses everything else on the host.
 *   data         uint8, data_bytes bytes, holding the files
 *   scan         HOST int64 (M, 2): byte offset in data and length of image m's entropy-coded segment (from the end of
 *                the SOS header to the EOI marker); offset + length <= data_bytes, length < 2^28
 *   geom         HOST int32 (M, 5): H, W (1..16384), luma sampling hs, vs ((1,1), (2,1) or (2,2)), restart interval in
 *                MCUs (0: none, up to 65535)
 *   tables       HOST int64 (M, 9): device addresses (4-byte aligned) of the quantisation tables of components 0..2
 *                (64 int32, natural order; used as 16-bit multipliers, as libjpeg does), their DC Huffman tables and
 *                their AC Huffman tables (occformer_b200.jpeg.huff_table's flat int32 form)
 *   out_offsets  HOST int64 (M): byte offset of image m's (H, W, 3) uint8 B, G, R frame in out (out_bytes bytes); only
 *                those bytes of out are written
 *   seq_bits     S, 32 .. 2^20: bits per subsequence of the parallel Huffman decode; sync_rounds R, 0 .. 64:
 *                self-synchronisation rounds before the serial fix-up.  Neither changes the result.
 *   status       (M, 2) int32, overwritten: status[m, 0] = 0 for a decoded image, else the OR of 1 (a marker other than
 *                RSTn inside the segment), 2 (RSTn markers missing, surplus or out of order), 4 (an invalid Huffman
 *                code or a coefficient run past 63), 8 (the data of a restart interval, or of the scan, ends before
 *                its last MCU); status[m, 1] = subsequences the fix-up decoded again serially.  libjpeg would warn and
 *                fill in grey instead of failing; the frame of a failed image is undefined, but nothing is written
 *                outside it.
 *   ws           occ_decode_jpeg_workspace_bytes(scan, geom, M, seq_bits) bytes, 16-byte aligned
 * 1 <= M <= 96.  11 + R enqueued launches and memsets per call whatever M and the data, no host synchronisation
 * (capturable in a CUDA graph).  Returns -1 for a bad M, S, R, geometry, segment, table address, output range or a
 * short or misaligned workspace, with nothing enqueued. */
size_t occ_decode_jpeg_workspace_bytes(const long long* scan /*HOST*/, const int* geom /*HOST*/, int M, int seq_bits);
int occ_decode_jpeg(const unsigned char* data, long long data_bytes, const long long* scan /*HOST*/,
                    const int* geom /*HOST*/, const long long* tables /*HOST*/, const long long* out_offsets /*HOST*/,
                    int M, int seq_bits, int sync_rounds, void* ws, size_t ws_bytes, unsigned char* out,
                    long long out_bytes, int* status, occ_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Camera frames from their PNG files (csrc/png_decode.cu): step 1 of the SemanticKITTI test loader's image side,
 *   LoadMultiViewImageFromFiles_SemanticKitti  P/datasets/pipelines/loading_kitti_imgs.py:103 (mmcv.imread, cv2)
 * bit for bit as cv2.imdecode(buf, IMREAD_UNCHANGED) with libpng and zlib: 8-bit RGB, non-interlaced, DEFLATE with
 * stored, fixed and dynamic Huffman blocks, the five PNG filter types.  occformer_b200/png.py walks the chunks and
 * refuses everything else on the host.
 *   data         uint8, data_bytes bytes, holding the zlib streams (each image's IDAT payloads back to back)
 *   streams      HOST int64 (M): byte offset in data of image m's zlib stream (from its 2-byte header)
 *   geom         HOST int32 (M, 4): H, W (1..16384), stream bytes (7 .. 2^27 - 1; offset + bytes <= data_bytes),
 *                CINFO of the zlib header (0..7)
 *   idat_counts  HOST int32 (M): IDAT chunks of image m (1 .. stream bytes)
 *   idat         int32, idat_len entries: per image in order, the stream offset at which each IDAT chunk's payload
 *                starts (the first is 0).  libpng hands zlib each chunk in reads of 8192 bytes, which decides whether a
 *                wrong Adler-32 fails the image (status 4)
 *   out_offsets  HOST int64 (M): byte offset of image m's (H, W, 3) uint8 B, G, R frame in out (out_bytes bytes); only
 *                those bytes of out are written
 *   status       (M, 2) int32, overwritten: status[m, 0] = 0 where cv2 decodes the image, else the OR of 1 (invalid
 *                DEFLATE data that zlib meets while libpng reads the rows: before the rows are complete, or an
 *                invalid code or block header right after the last row's byte in the same read), 2 (the stream ends
 *                early, or inflates to fewer than H (1 + 3W) bytes), 4 (an Adler-32 mismatch libpng meets while
 *                reading the rows), 8 (a filter type above 4); status[m, 1] = blocks decoded serially while linking.
 *                Errors zlib meets only after the rows (libpng's benign "too much image data" and later checks) and
 *                bytes after the end of the stream are ignored, as libpng ignores them.  The frame of a failed image
 *                is undefined, but nothing is written outside it.
 *   ws           occ_decode_png_workspace_bytes(streams, geom, idat_counts, M) bytes, 16-byte aligned
 * 1 <= M <= 96.  37 enqueued launches and memsets per call (7 + 30 pointer-jumping rounds) whatever M and the data, no
 * host synchronisation (capturable in a CUDA graph).  Returns -1 for a bad M, geometry, stream, IDAT count, output
 * range, a short idat array or a short or misaligned workspace, with nothing enqueued. */
size_t occ_decode_png_workspace_bytes(const long long* streams /*HOST*/, const int* geom /*HOST*/,
                                      const int* idat_counts /*HOST*/, int M);
int occ_decode_png(const unsigned char* data, long long data_bytes, const long long* streams /*HOST*/,
                   const int* geom /*HOST*/, const int* idat_counts /*HOST*/, const int* idat, long long idat_len,
                   const long long* out_offsets /*HOST*/, int M, void* ws, size_t ws_bytes, unsigned char* out,
                   long long out_bytes, int* status, occ_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* OCC_B200_H_ */
