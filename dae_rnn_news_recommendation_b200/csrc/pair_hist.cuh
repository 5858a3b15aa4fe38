// Shared by the related / unrelated pair histograms of gemm_tc.cu (dense, tensor cores) and similarity_sparse.cu (CSR): the bin
// of a score, the uint64 histogram add and the argument checks of the grid (see dae_similarity_pair_hist_bf16x3 in dae_sm100.h).
#pragma once
#include <cmath>
#include "common.cuh"

namespace dae {

constexpr int kHistMinLog2Bins = 10, kHistMaxLog2Bins = 24;

// b = clamp(floor(fl32(s + M) * bins / (2M)), 0, bins - 1).  scale = bins / (2M) is a power of two, so the product is exact and the
// only rounding is the fp32 add: monotone non-decreasing in s, and numpy's float32 (s + M) * scale gives the same bin.  The clamp
// comes before the conversion (its bounds are integers, so the order does not change the result) and sends NaN to bin 0.
__device__ __forceinline__ uint32_t pair_bin(float s, float M, float scale, uint32_t bins) {
  const float u = fminf(fmaxf(__fmul_rn(__fadd_rn(s, M), scale), 0.0f), (float)(bins - 1));
  return (uint32_t)__float2uint_rd(u);
}

__device__ __forceinline__ void red_add_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

inline bool is_pow2_i(int v) { return v > 0 && (v & (v - 1)) == 0; }
inline bool hist_bins_ok(int bins) { return is_pow2_i(bins) && bins >= (1 << kHistMinLog2Bins) && bins <= (1 << kHistMaxLog2Bins); }
// M a power of two in [2^-64, 2^64]: bins / (2M) stays a normal fp32 power of two
inline bool hist_range_ok(float M) {
  if (!(M > 0.0f) || !std::isfinite(M)) return false;
  int e = 0;
  const float m = std::frexp(M, &e);
  return m == 0.5f && e >= -63 && e <= 65;
}

}  // namespace dae
