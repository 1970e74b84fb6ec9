// Evaluation tail on the device (SURVEY.md 8(f)4): the integer counts that feed the path's single collective.
//
//   SSCMetrics.get_score_completion / get_score_semantic_and_completion   projects/mmdet3d_plugin/utils/ssc_metric.py:104-168
//   OccupancyFormer.simple_evaluation_semantic + fast_hist_crop           occformer/detectors/occupancyformer.py:219-224,246-254
//                                                                         utils/metric_util.py:8-23
//   summed over ranks by one all-reduce / gather                          occformer/apis/test.py:195-212
//
// Both are confusion matrices: conf[target][pred] over the voxels (target != ignore) resp. hist[gt-1][pred-1] over the
// LiDAR points (gt in 1..K-1, pred = 1 + argmax of the class scores without the 'empty' column).  One pass over the
// labels, per-CTA histogram in shared memory, 64-bit global atomics once per CTA and bin -- exact integers in any order.
#include "occ_common.cuh"

namespace occ {

constexpr int EV_MAXK = 32;

__global__ void __launch_bounds__(256)
confusion_kernel(const unsigned char* __restrict__ pred, const unsigned char* __restrict__ target, long long n, int K,
                 int ignore, unsigned long long* __restrict__ conf) {
  __shared__ unsigned int sh[EV_MAXK * EV_MAXK];
  for (int i = threadIdx.x; i < K * K; i += blockDim.x) sh[i] = 0u;
  __syncthreads();
  const long long stride = (long long)gridDim.x * blockDim.x * 16;
  for (long long base = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 16; base < n; base += stride) {
    if (base + 16 <= n && ((reinterpret_cast<uintptr_t>(pred + base) | reinterpret_cast<uintptr_t>(target + base)) & 15) == 0) {
      const uint4 p4 = __ldg(reinterpret_cast<const uint4*>(pred + base));
      const uint4 t4 = __ldg(reinterpret_cast<const uint4*>(target + base));
      const unsigned int pw[4] = {p4.x, p4.y, p4.z, p4.w}, tw[4] = {t4.x, t4.y, t4.z, t4.w};
#pragma unroll
      for (int w = 0; w < 4; ++w)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int t = (tw[w] >> (8 * k)) & 255, p = (pw[w] >> (8 * k)) & 255;
          if (t != ignore && t < K && p < K) atomicAdd(&sh[t * K + p], 1u);
        }
    } else {
      for (long long i = base; i < n && i < base + 16; ++i) {
        const int t = target[i], p = pred[i];
        if (t != ignore && t < K && p < K) atomicAdd(&sh[t * K + p], 1u);
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < K * K; i += blockDim.x)
    if (sh[i]) atomicAdd(&conf[i], (unsigned long long)sh[i]);
}

// conf (K,K) [target][pred] -> out[0..2] = completion tp, fp, fn (occupied = class > 0); out[3 + c], out[3 + K + c],
// out[3 + 2K + c] = semantic tp, fp, fn of class c  (ssc_metric.py:104-168: masked by target != 255, no nonempty mask)
__global__ void ssc_pack_kernel(const unsigned long long* __restrict__ conf, int K, long long* __restrict__ out) {
  const int c = threadIdx.x;
  if (c < K) {
    unsigned long long row = 0, col = 0;
    for (int j = 0; j < K; ++j) { row += conf[c * K + j]; col += conf[j * K + c]; }
    const unsigned long long tp = conf[c * K + c];
    out[3 + c] = (long long)tp;
    out[3 + K + c] = (long long)(col - tp);
    out[3 + 2 * K + c] = (long long)(row - tp);
  }
  if (c == 0) {
    unsigned long long ctp = 0, cfp = 0, cfn = 0;
    for (int t = 0; t < K; ++t)
      for (int p = 0; p < K; ++p) {
        const unsigned long long v = conf[t * K + p];
        if (t > 0 && p > 0) ctp += v;
        else if (t == 0 && p > 0) cfp += v;
        else if (t > 0 && p == 0) cfn += v;
      }
    out[0] = (long long)ctp; out[1] = (long long)cfp; out[2] = (long long)cfn;
  }
}

// scores (n, K) fp32 point class scores (column 0 = 'empty'), labels (n) int64 in 0..K-1 (0 = unlabelled, skipped):
// hist[(gt-1)*(K-1) + (pred-1)] += 1 with pred = 1 + argmax(scores[:, 1:]) (first maximum, as torch.argmax)
__global__ void __launch_bounds__(256)
lidarseg_hist_kernel(const float* __restrict__ scores, const long long* __restrict__ labels, int n, int K,
                     unsigned long long* __restrict__ hist) {
  __shared__ unsigned int sh[EV_MAXK * EV_MAXK];
  const int M = K - 1;
  for (int i = threadIdx.x; i < M * M; i += blockDim.x) sh[i] = 0u;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const long long g = labels[i];
    if (g < 1 || g >= K) continue;
    const float* s = scores + (size_t)i * K;
    int best = 1;
    float bv = s[1];
    for (int c = 2; c < K; ++c)
      if (s[c] > bv) { bv = s[c]; best = c; }
    atomicAdd(&sh[((int)g - 1) * M + best - 1], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < M * M; i += blockDim.x)
    if (sh[i]) atomicAdd(&hist[i], (unsigned long long)sh[i]);
}

// ------------------------------------------------------------------------------------------------- panoptic evaluation
// PanopticEval.addBatch (P/utils/panoptic_eval.py:11-246) on one flat scan.  The reference loops over the include
// classes with three np.unique calls each; here every (class, id) segment is a slot of an open-addressing hash table
// (64-bit key (id + 1) << 5 | class, 0 = empty, linear probing, capacity a power of two >= 2n, so the load stays <= 1/2):
//   pass 1  per element: confusion matrix (per-CTA shared histogram), prediction / GT segment areas, and the intersection
//           of every (pred slot, GT slot) pair of the same class -- a third table keyed by (pred slot + 1) << 32 | GT slot
//   pass 2  per pair slot: IoU > 1/2 (exactly: 2 * inter > union) -> tp, iou units, matched flags.  A segment has at most
//           one partner above 1/2, so the flags need no arbitration
//   pass 3  per segment slot: unmatched with area >= min_points -> fp (prediction) / fn (GT)
//   fold    one CTA adds the call's scratch into the state vector
// Every IoU in (1/2, 1] is a double that is an integer multiple of 2^-53, so the iou sum is kept as an exact count of
// 2^-53 units (__ddiv_rn(inter, union) * 2^53, at most 2^53 per match): independent of atomic order, launch shape and
// rank split.  Counts are integers throughout, so the whole state is bit-reproducible.
constexpr long long PE_ID_LIMIT = 2147483647LL;  // ids >= 2^31 - 1 overflow the reference's pred + 2^32 * gt key
constexpr int PE_LIMB_BITS = 31;
constexpr unsigned long long PE_LIMB_MASK = (1ull << PE_LIMB_BITS) - 1;
constexpr long long PE_MAX_N = 1LL << 29;         // slots (< 2^30) fit an int and the 32-bit halves of a pair key
// scratch (unsigned long long): conf K*K | tp K | fp K | fn K | units lo K | units hi K | invalid
constexpr int PE_SC_WORDS = 1280;                 // >= EV_MAXK^2 + 5 * EV_MAXK + 1, padded to 128-byte lines
static_assert(PE_SC_WORDS >= EV_MAXK * EV_MAXK + 5 * EV_MAXK + 1, "scratch too small");

struct PanTables {
  unsigned long long *pkey, *gkey, *xkey;  // prediction segments, GT segments, (pred, GT) pairs
  unsigned int *pcnt, *gcnt, *xcnt;        // areas / intersections
  unsigned char *pmatch, *gmatch;
  int shift;                               // 64 - log2(capacity)
  unsigned int mask;                       // capacity - 1
};

__device__ __forceinline__ int pe_insert(unsigned long long* keys, unsigned long long key, int shift, unsigned int mask) {
  unsigned int h = (unsigned int)((key * 0x9E3779B97F4A7C15ull) >> shift) & mask;
  while (true) {
    // a published key never changes: a plain read that already shows `key` spares the CAS on a hot segment's slot
    const unsigned long long k = *reinterpret_cast<volatile unsigned long long*>(keys + h);
    if (k == key) return (int)h;
    if (k == 0ull) {
      const unsigned long long prev = atomicCAS(keys + h, 0ull, key);
      if (prev == 0ull || prev == key) return (int)h;
    }
    h = (h + 1) & mask;
  }
}

// warp-aggregated cnt[slot] += 1 (slot < 0: no-op); every lane of the warp must call it
__device__ __forceinline__ void pe_count(unsigned int* cnt, int slot) {
  const unsigned int peers = __match_any_sync(0xffffffffu, slot);
  if (slot >= 0 && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(cnt + slot, (unsigned)__popc(peers));
}

__global__ void __launch_bounds__(256)
pan_scan_kernel(const long long* __restrict__ xs, const long long* __restrict__ xi, const long long* __restrict__ ys,
                const long long* __restrict__ yi, long long n, int K, unsigned int ignore, int parts, PanTables t,
                unsigned long long* __restrict__ sc) {
  __shared__ unsigned int sh[EV_MAXK * EV_MAXK];
  __shared__ unsigned int sh_bad;
  for (int i = threadIdx.x; i < K * K; i += blockDim.x) sh[i] = 0u;
  if (threadIdx.x == 0) sh_bad = 0u;
  __syncthreads();
  const bool pan = parts & 2;
  // block-uniform trip count: every lane reaches the warp-collective pe_count
  for (long long b = (long long)blockIdx.x * blockDim.x; b < n; b += (long long)gridDim.x * blockDim.x) {
    const long long i = b + threadIdx.x;
    int sp = -1, sg = -1, sx = -1;
    if (i < n) {
      const long long ps = xs[i], gs = ys[i];
      const long long pid = pan ? xi[i] : 0, gid = pan ? yi[i] : 0;
      if (ps < 0 || ps >= K || gs < 0 || gs >= K || pid >= PE_ID_LIMIT || gid >= PE_ID_LIMIT) {
        atomicAdd(&sh_bad, 1u);
      } else {
        if (parts & 1) atomicAdd(&sh[ps * K + gs], 1u);
        if (pan && !((ignore >> gs) & 1u)) {
          if (pid >= 0 && !((ignore >> ps) & 1u))
            sp = pe_insert(t.pkey, ((unsigned long long)(pid + 1) << 5) | (unsigned long long)ps, t.shift, t.mask);
          if (gid >= 0)
            sg = pe_insert(t.gkey, ((unsigned long long)(gid + 1) << 5) | (unsigned long long)gs, t.shift, t.mask);
          if (sp >= 0 && sg >= 0 && ps == gs)
            sx = pe_insert(t.xkey, ((unsigned long long)(sp + 1) << 32) | (unsigned long long)sg, t.shift, t.mask);
        }
      }
    }
    if (pan) {
      pe_count(t.pcnt, sp);
      pe_count(t.gcnt, sg);
      pe_count(t.xcnt, sx);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < K * K; i += blockDim.x)
    if (sh[i]) atomicAdd(&sc[i], (unsigned long long)sh[i]);
  if (threadIdx.x == 0 && sh_bad) atomicAdd(&sc[K * K + 5 * K], (unsigned long long)sh_bad);
}

__global__ void __launch_bounds__(256)
pan_pair_kernel(PanTables t, long long cap, int K, unsigned long long* __restrict__ sc) {
  __shared__ unsigned long long s_tp[EV_MAXK], s_lo[EV_MAXK], s_hi[EV_MAXK];
  for (int c = threadIdx.x; c < K; c += blockDim.x) s_tp[c] = s_lo[c] = s_hi[c] = 0ull;
  __syncthreads();
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < cap; s += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = t.xkey[s];
    if (!k) continue;
    const int sp = (int)(k >> 32) - 1, sg = (int)(k & 0xffffffffull);
    const long long inter = t.xcnt[s];
    const long long uni = (long long)t.pcnt[sp] + (long long)t.gcnt[sg] - inter;
    if (2 * inter <= uni) continue;
    const int cl = (int)(t.pkey[sp] & 31ull);
    const unsigned long long units =
        (unsigned long long)(__ddiv_rn((double)inter, (double)uni) * 9007199254740992.0);  // exact: * 2^53
    atomicAdd(&s_tp[cl], 1ull);
    atomicAdd(&s_lo[cl], units & PE_LIMB_MASK);
    atomicAdd(&s_hi[cl], units >> PE_LIMB_BITS);
    t.pmatch[sp] = 1;
    t.gmatch[sg] = 1;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < K; c += blockDim.x) {
    unsigned long long* tp = sc + K * K;
    if (s_tp[c]) {
      atomicAdd(&tp[c], s_tp[c]);
      atomicAdd(&tp[3 * K + c], s_lo[c]);
      atomicAdd(&tp[4 * K + c], s_hi[c]);
    }
  }
}

__global__ void __launch_bounds__(256)
pan_segment_kernel(PanTables t, long long cap, int K, int min_points, unsigned long long* __restrict__ sc) {
  __shared__ unsigned int s_fp[EV_MAXK], s_fn[EV_MAXK];
  for (int c = threadIdx.x; c < K; c += blockDim.x) s_fp[c] = s_fn[c] = 0u;
  __syncthreads();
  for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < 2 * cap; s += (long long)gridDim.x * blockDim.x) {
    const bool gt = s >= cap;
    const long long j = gt ? s - cap : s;
    const unsigned long long k = gt ? t.gkey[j] : t.pkey[j];
    if (!k || (gt ? t.gmatch[j] : t.pmatch[j])) continue;
    if ((long long)(gt ? t.gcnt[j] : t.pcnt[j]) < min_points) continue;
    atomicAdd(gt ? &s_fn[k & 31ull] : &s_fp[k & 31ull], 1u);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < K; c += blockDim.x) {
    if (s_fp[c]) atomicAdd(&sc[K * K + K + c], (unsigned long long)s_fp[c]);
    if (s_fn[c]) atomicAdd(&sc[K * K + 2 * K + c], (unsigned long long)s_fn[c]);
  }
}

// state (int64): conf K*K | tp K | fp K | fn K | iou units K x 3 base-2^31 limbs | invalid.  Adds the scratch and
// carries the limbs, so limbs stay below 2^31 (they may exceed it in a vector summed over ranks; the carry absorbs that)
__global__ void pan_fold_kernel(const unsigned long long* __restrict__ sc, int K, long long* __restrict__ state) {
  for (int i = threadIdx.x; i < K * K + 3 * K; i += blockDim.x) state[i] += (long long)sc[i];
  for (int c = threadIdx.x; c < K; c += blockDim.x) {
    unsigned long long* l = reinterpret_cast<unsigned long long*>(state + K * K + 3 * K + 3 * c);
    const unsigned long long lo = sc[K * K + 3 * K + c], hi = sc[K * K + 4 * K + c];
    const unsigned long long t0 = l[0] + (lo & PE_LIMB_MASK);
    const unsigned long long t1 = l[1] + (t0 >> PE_LIMB_BITS) + (lo >> PE_LIMB_BITS) + hi;
    l[0] = t0 & PE_LIMB_MASK;
    l[1] = t1 & PE_LIMB_MASK;
    l[2] += t1 >> PE_LIMB_BITS;
  }
  if (threadIdx.x == 0) state[K * K + 6 * K] += (long long)sc[K * K + 5 * K];
}

inline long long pe_capacity(long long n) {
  long long cap = 64;
  while (cap < 2 * n) cap <<= 1;
  return cap;
}

}  // namespace occ

using namespace occ;

extern "C" size_t occ_panoptic_eval_workspace_bytes(long long n) {
  if (n < 0 || n > PE_MAX_N) return 0;
  return (size_t)PE_SC_WORDS * 8 + (size_t)pe_capacity(n) * (3 * 8 + 3 * 4 + 2);
}

extern "C" int occ_panoptic_eval(const long long* x_sem, const long long* x_inst, const long long* y_sem,
                                 const long long* y_inst, long long n, int K, unsigned int ignore_mask, int min_points,
                                 int parts, void* ws, size_t ws_bytes, long long* state, cudaStream_t stream) {
  OCC_REQUIRE(state && n >= 0 && n <= PE_MAX_N && K >= 1 && K <= EV_MAXK && parts >= 1 && parts <= 3);
  if (n == 0) return OCC_OK;
  OCC_REQUIRE(x_sem && y_sem && ws && (!(parts & 2) || (x_inst && y_inst)));
  OCC_REQUIRE(ws_bytes >= occ_panoptic_eval_workspace_bytes(n) && (reinterpret_cast<uintptr_t>(ws) & 15) == 0);
  const long long cap = pe_capacity(n);
  unsigned char* p = static_cast<unsigned char*>(ws);
  unsigned long long* sc = reinterpret_cast<unsigned long long*>(p);
  p += (size_t)PE_SC_WORDS * 8;
  PanTables t;
  t.pkey = reinterpret_cast<unsigned long long*>(p);
  t.gkey = t.pkey + cap;
  t.xkey = t.gkey + cap;
  t.pcnt = reinterpret_cast<unsigned int*>(t.xkey + cap);
  t.gcnt = t.pcnt + cap;
  t.xcnt = t.gcnt + cap;
  t.pmatch = reinterpret_cast<unsigned char*>(t.xcnt + cap);
  t.gmatch = t.pmatch + cap;
  t.mask = (unsigned int)(cap - 1);
  t.shift = 64 - (63 - __builtin_clzll((unsigned long long)cap));
  const bool pan = parts & 2;
  OCC_MEMSET(ws, 0, pan ? occ_panoptic_eval_workspace_bytes(n) : (size_t)PE_SC_WORDS * 8, stream);
  long long blocks = (n + 255) / 256;
  if (blocks > (long long)sm_count() * 8) blocks = (long long)sm_count() * 8;
  pan_scan_kernel<<<(unsigned)blocks, 256, 0, stream>>>(x_sem, x_inst, y_sem, y_inst, n, K, ignore_mask, parts, t, sc);
  OCC_LAUNCH_CHECK();
  if (pan) {
    long long sblocks = (cap + 255) / 256;
    if (sblocks > (long long)sm_count() * 8) sblocks = (long long)sm_count() * 8;
    pan_pair_kernel<<<(unsigned)sblocks, 256, 0, stream>>>(t, cap, K, sc);
    OCC_LAUNCH_CHECK();
    pan_segment_kernel<<<(unsigned)sblocks, 256, 0, stream>>>(t, cap, K, min_points, sc);
    OCC_LAUNCH_CHECK();
  }
  pan_fold_kernel<<<1, 256, 0, stream>>>(sc, K, state);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// pred, target: n uint8 labels; conf_ws: K*K int64 scratch (overwritten); out: 3 + 3K int64 (overwritten)
extern "C" int occ_ssc_counts(const unsigned char* pred, const unsigned char* target, long long n, int K, int ignore,
                              long long* conf_ws, long long* out, cudaStream_t stream) {
  OCC_REQUIRE(pred && target && conf_ws && out && n >= 0 && K >= 2 && K <= EV_MAXK);
  OCC_MEMSET(conf_ws, 0, (size_t)K * K * sizeof(long long), stream);
  if (n > 0) {
    long long blocks = (n + 256 * 16 - 1) / (256 * 16);
    const long long cap = (long long)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    confusion_kernel<<<(unsigned)blocks, 256, 0, stream>>>(pred, target, n, K, ignore,
                                                           reinterpret_cast<unsigned long long*>(conf_ws));
    OCC_LAUNCH_CHECK();
  }
  ssc_pack_kernel<<<1, 32, 0, stream>>>(reinterpret_cast<const unsigned long long*>(conf_ws), K, out);
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}

// hist ((K-1)*(K-1) int64) is ACCUMULATED (+=): zero it once per evaluation run
extern "C" int occ_lidarseg_hist(const float* scores, const long long* labels, int n, int K, long long* hist,
                                 cudaStream_t stream) {
  OCC_REQUIRE(hist && n >= 0 && K >= 2 && K <= EV_MAXK);
  if (n == 0) return OCC_OK;
  OCC_REQUIRE(scores && labels);
  int blocks = (n + 255) / 256;
  if (blocks > sm_count() * 4) blocks = sm_count() * 4;
  lidarseg_hist_kernel<<<blocks, 256, 0, stream>>>(scores, labels, n, K, reinterpret_cast<unsigned long long*>(hist));
  OCC_LAUNCH_CHECK();
  return OCC_OK;
}
