// Shared helpers of libocc_b200.so: error codes, driver entry point for TMA descriptors, the pooled-logit encoding.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>

#include "../../include/occ_b200.h"  // every extern "C" definition is compiled against its declaration

// C-ABI return convention (include/occ_b200.h): 0 = ok, negative = argument error,
// positive = cudaError_t of the failed runtime call / launch.
#define OCC_OK 0
#define OCC_EINVAL (-1)
#define OCC_EUNSUPPORTED (-2)
#define OCC_EDRIVER (-3)

#define OCC_REQUIRE(cond)                                                        \
  do {                                                                           \
    if (!(cond)) {                                                               \
      fprintf(stderr, "occ_b200: argument check failed: %s (%s:%d)\n", #cond, __FILE__, __LINE__); \
      return OCC_EINVAL;                                                         \
    }                                                                            \
  } while (0)

#define OCC_CUDA(call)                                  \
  do {                                                  \
    cudaError_t e__ = (call);                           \
    if (e__ != cudaSuccess) return static_cast<int>(e__); \
  } while (0)

// Follows every kernel launch (exactly one per executed launch): returns the launch error, else counts the launch.
#define OCC_LAUNCH_CHECK()                              \
  do {                                                  \
    cudaError_t e__ = cudaGetLastError();               \
    if (e__ != cudaSuccess) return static_cast<int>(e__); \
    occ::count_launch();                                \
  } while (0)

// cudaMemsetAsync, checked and counted like a launch
#define OCC_MEMSET(ptr, value, bytes, stream)                          \
  do {                                                                 \
    OCC_CUDA(cudaMemsetAsync((ptr), (value), (bytes), (stream)));      \
    occ::count_launch();                                               \
  } while (0)

namespace occ {

// Adds one to the process-wide count of enqueued launches and memsets (occ_launch_count, csrc/config.cu).
void count_launch();

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled resolved at run time so that the library loads (and exports its symbols) on a
// machine without libcuda.so.1.
inline PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(p);
  return fn;
}

constexpr int OCC_MAX_DEVICES = 64;

// SM count of the CURRENT device (cached per device: one process may drive several GPUs).
inline int sm_count() {
  static int n[OCC_MAX_DEVICES] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= OCC_MAX_DEVICES) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    return v > 0 ? v : 132;
  }
  if (n[dev]) return n[dev];
  cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
  if (n[dev] <= 0) n[dev] = 132;
  return n[dev];
}

// Opt a kernel into `bytes` of dynamic shared memory on the current device (cudaFuncSetAttribute applies per device;
// the largest request seen so far is remembered per device, so the call is made once per kernel and device).
#define OCC_ENSURE_SMEM(kernel, bytes)                                                                            \
  do {                                                                                                            \
    static size_t cfg__[occ::OCC_MAX_DEVICES] = {};                                                               \
    int dev__ = 0;                                                                                                \
    cudaGetDevice(&dev__);                                                                                        \
    const bool known__ = dev__ >= 0 && dev__ < occ::OCC_MAX_DEVICES;                                              \
    if (!known__ || cfg__[dev__] < (size_t)(bytes)) {                                                             \
      OCC_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)));          \
      if (known__) cfg__[dev__] = (size_t)(bytes);                                                                \
    }                                                                                                             \
  } while (0)

// Pooled attention-mask logit -> order-preserving int (occ_mask_pool / occ_mask_gemm_pool): the float bits for x >= +0,
// bits ^ 0x7FFFFFFF for x < 0, so that int order is float order and "blocked" (sigmoid(x) < 0.5, i.e. x < 0) is code < 0.
// -0.0 encodes as +0.0 (code 0): sigmoid(-0.0) = 0.5 is not blocked.  ops.decode_ordered inverts it.
__device__ __forceinline__ int ordered_logit(float x) {
  const int i = __float_as_int(x);
  return i >= 0 ? i : (i == (int)0x80000000 ? 0 : i ^ 0x7FFFFFFF);
}

// Tensor-core passes per 32-k operand block: 3 = fp32-faithful (hi*hi + lo*hi + hi*lo, the default and the only mode the
// parity gate covers), 1 = single-pass bf16 (hi*hi only; occ_set_mma_passes, csrc/config.cu).  Host-side setting, read by
// every launcher at launch time and handed to the kernel as an argument (the GEMM / conv launcher picks the kernel
// instantiation compiled for that pass count).
int mma_passes();

// fp32 tensor map, rank <= 5, 128-byte swizzle, zero OOB fill.  dims/box/estr innermost first;
// strides_bytes[i] = byte stride of dim i+1.
inline int make_tmap_f32(CUtensorMap* m, const void* base, int rank, const uint64_t* dims,
                         const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* estr,
                         CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return OCC_EDRIVER;
  cuuint64_t d[5], s[4];
  cuuint32_t b[5], e[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; b[i] = box[i]; e[i] = estr ? estr[i] : 1; }
  for (int i = 0; i + 1 < rank; ++i) s[i] = strides_bytes[i];
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<void*>(base), d, s, b, e,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "occ_b200: cuTensorMapEncodeTiled failed (%d) rank=%d\n", (int)r, rank);
    return OCC_EDRIVER;
  }
  return OCC_OK;
}

}  // namespace occ
