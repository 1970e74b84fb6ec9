// Library-wide host state (no device state): the launch-time configuration and the launch counter.
#include <atomic>

#include "occ_common.cuh"

namespace occ {
static int g_mma_passes = 3;
static std::atomic<long long> g_launches{0};
int mma_passes() { return g_mma_passes; }
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
}  // namespace occ

// passes = 3: every contraction is an fp32 problem in three bf16 tensor-core passes (default; the mode of every parity
// claim).  passes = 1: single-pass bf16 operands (the hi halves of the S32 operands only) -- BASELINE config 5's "bf16":
// ~3e-3 relative error per contraction, a third of the tensor work; the reference has no twin of this mode, it is
// validated against the fp32 oracle at its own tolerance (tests/test_gpu_bf16_mode.py).  Returns the previous value.
extern "C" int occ_set_mma_passes(int passes) {
  if (passes != 1 && passes != 3) return -1;
  const int prev = occ::g_mma_passes;
  occ::g_mma_passes = passes;
  return prev;
}
extern "C" int occ_get_mma_passes(void) { return occ::g_mma_passes; }

extern "C" long long occ_launch_count(void) { return occ::g_launches.load(std::memory_order_relaxed); }
