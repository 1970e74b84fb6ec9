// SemanticKITTI occupancy ground truth from the dataset's own voxel files, on the device:
//
//   semantic_kitti_preprocess.main, one frame's _1_1 volume    P/tools/kitti_process/semantic_kitti_preprocess.py:117-142
//   io_data._read_label_SemKITTI / _read_invalid_SemKITTI / unpack    P/tools/kitti_process/io_data.py:10-22,113-127
//   LoadSemKittiAnnotation, test mode: torch.tensor(gt_occ).long()  P/datasets/pipelines/loading_kitti_occ.py:34-53
//
// The reference writes remap_lut[label] (float32) per voxel, then 255 wherever the bit-packed .invalid mask is set, to a
// .npy that the loader turns into int64.  Every value is a small integer, exact in float32, so the volume is the int64
// lut value directly.  One thread per invalid byte: eight uint16 labels in one 16-byte load, eight int64 in four
// 16-byte stores.  A label at or past the LUT (numpy's IndexError) is counted per sample and written as 255.
#include "occ_common.cuh"

namespace occ {

constexpr long long SK_MAX_B = 1 << 16;

__global__ void __launch_bounds__(256)
sk_labels_kernel(const uint4* __restrict__ label, const unsigned char* __restrict__ invalid, long long groups,
                 long long groups_per_sample, const int* __restrict__ lut, int lut_size, int* __restrict__ bad,
                 longlong2* __restrict__ out) {
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (long long)gridDim.x * blockDim.x) {
    const uint4 l = label[g];
    const unsigned int inv = invalid[g];
    const unsigned int w[4] = {l.x, l.y, l.z, l.w};
    int n_bad = 0;
    long long v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int lab = (int)((w[j >> 1] >> ((j & 1) * 16)) & 0xffffu);  // little-endian uint16 pairs
      long long x = 255;
      if (lab < lut_size) x = __ldg(lut + lab);
      else ++n_bad;
      v[j] = (inv >> (7 - j)) & 1u ? 255 : x;  // most significant bit first (io_data.unpack)
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) out[g * 4 + j] = make_longlong2(v[2 * j], v[2 * j + 1]);
    if (n_bad) atomicAdd(bad + g / groups_per_sample, n_bad);
  }
}

}  // namespace occ

using namespace occ;

extern "C" int occ_semkitti_labels(const unsigned char* label, const unsigned char* invalid, int B, long long nvox,
                                   const int* lut, int lut_size, int* bad, long long* out, cudaStream_t stream) {
  OCC_REQUIRE(label && invalid && lut && bad && out && B >= 1 && B <= SK_MAX_B);
  OCC_REQUIRE(nvox >= 8 && nvox % 8 == 0 && nvox <= (1LL << 31) && lut_size >= 1 && lut_size <= 65536);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(label) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0);
  const long long groups = (long long)B * (nvox / 8);
  const long long lim = (long long)sm_count() * 16;
  long long blocks = (groups + 255) / 256;
  blocks = blocks > lim ? lim : blocks;
  sk_labels_kernel<<<(unsigned)blocks, 256, 0, stream>>>(reinterpret_cast<const uint4*>(label), invalid, groups,
                                                        nvox / 8, lut, lut_size, bad,
                                                        reinterpret_cast<longlong2*>(out));
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
