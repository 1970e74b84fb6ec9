// Occupancy ground truth of nuScenes from the labelled LiDAR points, on the device:
//
//   LoadNuscOccupancyAnnotations.__call__ + nb_process_label                P/datasets/pipelines/loading_nusc_occ.py:95-138
//   LoadNuscPanopticOccupancyAnnotations.__call__ + nb_process_label        P/datasets/pipelines/loading_nusc_panoptic_occ.py:120-166
//
// The reference voxelises each point in float64, lexsorts the (voxel, id) pairs and walks them with a fresh 256-entry
// (semantic) or 65 536-entry (panoptic) counter per occupied voxel, whose argmax (first maximum: the smallest id of a
// tie) is the voxel's id.  Here no sort is needed, and nothing depends on the order of the points:
//   memset  the output volume and the workspace
//   scan    per point: fp64 voxel index (as numpy), one slot per (voxel, id) pair in an open-addressing hash table
//           (64-bit key, linear probing, capacity a power of two >= 2n) with a warp-aggregated count; in panoptic mode
//           a per-sample atomicMax of the lexsort key (z, y, x) finds the voxel the reference writes last
//   vote    per pair slot: atomicMax of OCC | count << 16 | (65535 - id) into the voxel's int64 word.  The largest
//           word has the largest count and, among equal counts, the smallest id: np.argmax.  A panoptic id-0 pair votes
//           with count 0 (counter[0] = 0 before every write but the last, loading_nusc_panoptic_occ.py:157,164), so it
//           still marks its voxel occupied and wins only a voxel that holds nothing else
//   decode  per voxel: unoccupied -> 0, else id -> (0 -> ignore, empty -> 0, other ids unchanged)
// Five enqueued operations per call whatever n and the mode, all integer: the volume is bit-reproducible.
#include "occ_common.cuh"

namespace occ {

constexpr unsigned long long OT_OCC = 1ull << 32;  // above any count << 16 | id: every occupied word beats 0
constexpr unsigned int OT_MAX_COUNT = 65535;       // the reference's uint16 counter wraps above it
constexpr int OT_MAX_B = 256;                      // per-sample row offsets travel in the kernel parameters

struct OtOffsets {
  long long off[OT_MAX_B + 1];
};

struct OtGrid {
  double lo[3], hi_eps[3], vs[3];  // point_cloud_range[:3], point_cloud_range[3:] - 1e-5, voxel_size
  int X, Y, Z;
};

__device__ __forceinline__ int ot_insert(unsigned long long* keys, unsigned long long key, unsigned int mask) {
  unsigned int h = (unsigned int)((key * 0x9E3779B97F4A7C15ull) >> 32) & mask;
  while (true) {
    const unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(keys + h);
    if (k == key) return (int)h;
    if (k == 0ull) {
      const unsigned long long prev = atomicCAS(keys + h, 0ull, key);
      if (prev == 0ull || prev == key) return (int)h;
    }
    h = (h + 1) & mask;
  }
}

// voxel index of one coordinate exactly as numpy computes it in float64:
// floor((clip(p, lo, hi - 1e-5) - lo) / voxel_size), every operation rounded on its own
__device__ __forceinline__ int ot_index(float p, double lo, double hi_eps, double vs) {
  double c = (double)p;
  c = c < lo ? lo : c;
  c = c > hi_eps ? hi_eps : c;
  return (int)floor(__ddiv_rn(__dsub_rn(c, lo), vs));
}

// grid (blocks, B): sample b = blockIdx.y walks its rows [off[b], off[b+1]) with a block-uniform trip count, so every
// lane reaches the warp-collective count
__global__ void __launch_bounds__(256)
ot_scan_kernel(const float* __restrict__ pts, int ld, OtOffsets offs, OtGrid g, int limit, int panoptic,
               unsigned long long* __restrict__ keys, unsigned int* __restrict__ cnt, unsigned int mask,
               int* __restrict__ last, int* __restrict__ invalid) {
  const int b = blockIdx.y;
  const long long s = offs.off[b], e = offs.off[b + 1];
  unsigned int bad = 0;
  for (long long base = s + (long long)blockIdx.x * blockDim.x; base < e; base += (long long)gridDim.x * blockDim.x) {
    const long long i = base + threadIdx.x;
    int slot = -1;
    if (i < e) {
      const float* r = pts + i * (long long)ld;
      const float px = r[0], py = r[1], pz = r[2], fl = r[3];
      const bool label_ok = fl >= 0.f && fl < (float)limit && floorf(fl) == fl;  // NaN fails every comparison
      if (!label_ok || !isfinite(px) || !isfinite(py) || !isfinite(pz)) {
        ++bad;
      } else {
        const int x = ot_index(px, g.lo[0], g.hi_eps[0], g.vs[0]);
        const int y = ot_index(py, g.lo[1], g.hi_eps[1], g.vs[1]);
        const int z = ot_index(pz, g.lo[2], g.hi_eps[2], g.vs[2]);
        if (x < 0 || x >= g.X || y < 0 || y >= g.Y || z < 0 || z >= g.Z) {
          ++bad;  // cannot happen for a range whose voxels are wider than 1e-5; never written out of bounds
        } else {
          const long long v = (((long long)b * g.X + x) * g.Y + y) * g.Z + z;
          slot = ot_insert(keys, (((unsigned long long)v << 16) | (unsigned long long)(int)fl) + 1ull, mask);
          if (panoptic) atomicMax(last + b, (z * g.Y + y) * g.X + x + 1);  // np.lexsort((x, y, z)): z, then y, then x
        }
      }
    }
    const unsigned int peers = __match_any_sync(0xffffffffu, slot);
    if (slot >= 0 && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(cnt + slot, (unsigned)__popc(peers));
  }
  if (bad) atomicAdd(invalid, (int)bad);
}

__global__ void __launch_bounds__(256)
ot_vote_kernel(const unsigned long long* __restrict__ keys, const unsigned int* __restrict__ cnt, long long cap,
               OtGrid g, int panoptic, const int* __restrict__ last, unsigned long long* __restrict__ vol,
               int* __restrict__ invalid) {
  unsigned int bad = 0;
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[s];
    if (!k) continue;
    const long long v = (long long)((k - 1ull) >> 16);
    const unsigned int id = (unsigned int)((k - 1ull) & 0xffffull);
    unsigned int c = cnt[s];
    if (c > OT_MAX_COUNT) {
      c = OT_MAX_COUNT;
      ++bad;
    }
    if (panoptic && id == 0) {
      const int z = (int)(v % g.Z), y = (int)((v / g.Z) % g.Y), x = (int)((v / ((long long)g.Z * g.Y)) % g.X);
      const int b = (int)(v / ((long long)g.Z * g.Y * g.X));
      if ((z * g.Y + y) * g.X + x + 1 != last[b]) c = 0;
    }
    atomicMax(vol + v, OT_OCC | ((unsigned long long)c << 16) | (unsigned long long)(65535u - id));
  }
  if (bad) atomicAdd(invalid, (int)bad);
}

__global__ void __launch_bounds__(256)
ot_decode_kernel(long long* __restrict__ vol, long long nvox, long long empty_id, long long ignore) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvox; i += (long long)gridDim.x * blockDim.x) {
    const long long w = vol[i];
    if (!w) continue;
    const long long id = 65535 - (w & 0xffff);
    vol[i] = id == 0 ? ignore : (id == empty_id ? 0 : id);
  }
}

inline long long ot_capacity(long long n) {
  long long cap = 64;
  while (cap < 2 * n) cap <<= 1;
  return cap;
}

inline size_t ot_align(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace occ

using namespace occ;

extern "C" size_t occ_lidarseg_occupancy_workspace_bytes(long long n, int B) {
  if (n < 0 || n > (1LL << 30) || B < 1 || B > OT_MAX_B) return 0;
  const long long cap = ot_capacity(n);
  return ot_align((size_t)cap * 8) + ot_align((size_t)cap * 4) + ot_align((size_t)B * 4);
}

extern "C" int occ_lidarseg_occupancy(const float* pts, int ld, const long long* offsets, int B, double x_min,
                                      double y_min, double z_min, double x_max, double y_max, double z_max, int X, int Y,
                                      int Z, int panoptic, long long empty_id, long long ignore, int* invalid, void* ws,
                                      size_t ws_bytes, long long* out, cudaStream_t stream) {
  OCC_REQUIRE(offsets && invalid && out && ws && B >= 1 && B <= OT_MAX_B && ld >= 4);
  OCC_REQUIRE(X >= 1 && Y >= 1 && Z >= 1 && (long long)X * Y * Z < (1LL << 31) && (long long)B * X * Y * Z < (1LL << 40));
  OCC_REQUIRE(panoptic == 0 || panoptic == 1);
  OtOffsets offs;
  for (int b = 0; b <= B; ++b) {
    offs.off[b] = offsets[b];
    OCC_REQUIRE(offs.off[b] >= 0 && (b == 0 ? offs.off[0] == 0 : offs.off[b] >= offs.off[b - 1]));
  }
  const long long n = offs.off[B];
  long long max_rows = 0;
  for (int b = 0; b < B; ++b) max_rows = max_rows > offs.off[b + 1] - offs.off[b] ? max_rows : offs.off[b + 1] - offs.off[b];
  OCC_REQUIRE(n <= (1LL << 30) && (n == 0 || pts) && ws_bytes >= occ_lidarseg_occupancy_workspace_bytes(n, B));
  OCC_REQUIRE((reinterpret_cast<uintptr_t>(ws) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0);
  OtGrid g;
  const double lo[3] = {x_min, y_min, z_min}, hi[3] = {x_max, y_max, z_max};
  const int dims[3] = {X, Y, Z};
  for (int a = 0; a < 3; ++a) {
    // numpy's (hi - lo) / grid_size and point_cloud_range[3:] - eps, each rounded once in float64 (host IEEE doubles)
    g.lo[a] = lo[a];
    g.vs[a] = (hi[a] - lo[a]) / (double)dims[a];
    g.hi_eps[a] = hi[a] - 1e-5;
    OCC_REQUIRE(g.vs[a] > 0.0);
  }
  g.X = X; g.Y = Y; g.Z = Z;
  const long long cap = ot_capacity(n);
  unsigned char* p = static_cast<unsigned char*>(ws);
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(p);
  unsigned int* cnt = reinterpret_cast<unsigned int*>(p + ot_align((size_t)cap * 8));
  int* last = reinterpret_cast<int*>(p + ot_align((size_t)cap * 8) + ot_align((size_t)cap * 4));
  const long long nvox = (long long)B * X * Y * Z;
  OCC_MEMSET(out, 0, (size_t)nvox * 8, stream);
  OCC_MEMSET(ws, 0, occ_lidarseg_occupancy_workspace_bytes(n, B), stream);
  const long long lim = (long long)sm_count() * 8;
  long long bx = (max_rows + 255) / 256;
  bx = bx < 1 ? 1 : (bx > lim ? lim : bx);
  ot_scan_kernel<<<dim3((unsigned)bx, (unsigned)B), 256, 0, stream>>>(pts, ld, offs, g, panoptic ? 65536 : 256, panoptic,
                                                                       keys, cnt, (unsigned int)(cap - 1), last, invalid);
  OCC_LAUNCH_CHECK();
  long long sb = (cap + 255) / 256;
  sb = sb > lim ? lim : sb;
  ot_vote_kernel<<<(unsigned)sb, 256, 0, stream>>>(keys, cnt, cap, g, panoptic, last,
                                                   reinterpret_cast<unsigned long long*>(out), invalid);
  OCC_LAUNCH_CHECK();
  long long db = (nvox + 255) / 256;
  db = db > lim ? lim : db;
  ot_decode_kernel<<<(unsigned)db, 256, 0, stream>>>(out, nvox, empty_id, ignore);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
