// Shared by the thresholded-pair joins of gemm_tc.cu (dense, tensor cores) and similarity_sparse.cu (CSR): the warp-aggregated
// reservation of output slots and the capacity rule (see dae_similarity_pairs_bf16x3 in dae_sm100.h).
#pragma once
#include <cmath>
#include "common.cuh"

namespace dae {

// The first output slot of this lane's `hits` pairs.  One atomicAdd on the 64-bit counter reserves the warp's total; the lanes take
// consecutive runs in lane order (exclusive prefix of the counts by shuffles).  Every lane of the warp must call it, converged.
__device__ __forceinline__ unsigned long long pair_slots(unsigned long long* count, int hits) {
  const int lane = threadIdx.x & 31;
  int incl = hits;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  unsigned long long base = 0;
  if (lane == 31) base = atomicAdd(count, (unsigned long long)incl);
  base = __shfl_sync(0xffffffffu, base, 31);
  return base + (unsigned long long)(incl - hits);
}

// one pair into slot `slot` if it lies below the capacity; the counter has already counted it either way
__device__ __forceinline__ void pair_put(unsigned long long slot, unsigned long long capacity, int i, int j, float s, int32_t* i_out,
                                         int32_t* j_out, float* s_out) {
  if (slot < capacity) { i_out[slot] = i; j_out[slot] = j; s_out[slot] = s; }
}

inline bool pair_threshold_ok(float tau) { return std::isfinite(tau); }

}  // namespace dae
