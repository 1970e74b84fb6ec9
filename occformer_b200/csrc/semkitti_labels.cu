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

// The training-mode volume (occ_semkitti_labels_aug): voxel_transform's Pillow rotation of every z slice, then its
//   flips, of the same volume          P/datasets/pipelines/loading_kitti_occ.py:34-53 (is_train), loading_nusc_occ.py:140-225
// One thread per output (x, y) column of one sample.  Every z slice is rotated by the same gather, so the column's 32
// values come from one source column (or are all 255 outside the slice): four 16-byte label loads and one 4-byte
// invalid load, the z reversal a register permutation, sixteen 16-byte stores.
constexpr int SK_X = 256, SK_Y = 256, SK_Z = 32;
constexpr int SK_AUG = 10;  // flip_dx, flip_dy, flip_dz, rotate, a0..a5

__device__ __forceinline__ int sk_column(const uint4* __restrict__ label, const unsigned int* __restrict__ invalid,
                                         long long col, const int* __restrict__ lut, int lut_size, int* v) {
  unsigned int w[16];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const uint4 l = label[col * 4 + q];
    w[4 * q] = l.x; w[4 * q + 1] = l.y; w[4 * q + 2] = l.z; w[4 * q + 3] = l.w;
  }
  const unsigned int inv = invalid[col];  // z = 8 k + j at bit 8 k + 7 - j (bytes little-endian, bits MSB first)
  int n_bad = 0;
#pragma unroll
  for (int z = 0; z < SK_Z; ++z) {
    const int lab = (int)((w[z >> 1] >> ((z & 1) * 16)) & 0xffffu);
    int x = 255;
    if (lab < lut_size) x = __ldg(lut + lab);
    else ++n_bad;
    v[z] = (inv >> (8 * (z >> 3) + 7 - (z & 7))) & 1u ? 255 : x;
  }
  return n_bad;
}

__global__ void __launch_bounds__(256)
sk_labels_aug_kernel(const uint4* __restrict__ label, const unsigned int* __restrict__ invalid,
                     const int* __restrict__ aug, const int* __restrict__ lut, int lut_size, int* __restrict__ bad,
                     longlong2* __restrict__ out) {
  constexpr long long COLS = (long long)SK_X * SK_Y;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // the grid is exactly B * COLS threads
  const int b = (int)(t / COLS);
  const int i = (int)((t / SK_Y) % SK_X), j = (int)(t % SK_Y);
  const int* a = aug + b * SK_AUG;
  // the flips come last in voxel_transform: output (i, j, z) is the rotated volume's (i', j', z')
  const int ir = a[0] ? SK_X - 1 - i : i, jr = a[1] ? SK_Y - 1 - j : j;
  const bool flip_z = a[2] != 0, rotate = a[3] != 0;
  long long src = (long long)b * COLS + (long long)ir * SK_Y + jr;
  bool inside = true;
  if (rotate) {  // slice pixel (column jr, row ir) reads column ys = Y index, row xs = X index (Pillow's affine_fixed)
    const long long ys = ((long long)a[6] + (long long)ir * a[5] + (long long)jr * a[4]) >> 16;
    const long long xs = ((long long)a[9] + (long long)ir * a[8] + (long long)jr * a[7]) >> 16;
    inside = ys >= 0 && ys < SK_Y && xs >= 0 && xs < SK_X;
    src = (long long)b * COLS + xs * SK_Y + ys;
  }
  int v[SK_Z];  // lut values, widened at the store
  int n_bad = 0;
  if (inside) {
    n_bad = sk_column(label, invalid, src, lut, lut_size, v);
  } else {
#pragma unroll
    for (int z = 0; z < SK_Z; ++z) v[z] = 255;  // fillcolor=255
  }
  // every voxel of the source volume is counted once, as the preprocessing's table lookup meets it: flips alone are a
  // permutation of the columns, a rotation gathers some columns twice and others never, so it counts the own column
  if (rotate) {
    int own[SK_Z];
    n_bad = sk_column(label, invalid, t, lut, lut_size, own);
  }
  longlong2* o = out + t * (SK_Z / 2);
#pragma unroll
  for (int k = 0; k < SK_Z / 2; ++k) {
    const int lo = flip_z ? v[SK_Z - 1 - 2 * k] : v[2 * k];
    const int hi = flip_z ? v[SK_Z - 2 - 2 * k] : v[2 * k + 1];
    o[k] = make_longlong2(lo, hi);
  }
  if (n_bad) atomicAdd(bad + b, n_bad);
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

extern "C" int occ_semkitti_labels_aug(const unsigned char* label, const unsigned char* invalid, int B, const int* aug,
                                       const int* lut, int lut_size, int* bad, long long* out, cudaStream_t stream) {
  OCC_REQUIRE(label && invalid && aug && lut && bad && out && B >= 1 && B <= SK_MAX_B);
  OCC_REQUIRE(lut_size >= 1 && lut_size <= 65536);
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(label) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 &&
              (reinterpret_cast<uintptr_t>(invalid) & 3) == 0 && (reinterpret_cast<uintptr_t>(aug) & 3) == 0);
  const long long blocks = (long long)B * SK_X * SK_Y / 256;
  sk_labels_aug_kernel<<<(unsigned)blocks, 256, 0, stream>>>(
      reinterpret_cast<const uint4*>(label), reinterpret_cast<const unsigned int*>(invalid), aug, lut, lut_size, bad,
      reinterpret_cast<longlong2*>(out));
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
