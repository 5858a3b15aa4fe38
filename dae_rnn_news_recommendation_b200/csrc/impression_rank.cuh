// The per-impression ranking metrics (DESIGN 4.13, 4.20), shared by dae_impression_metrics (dense query rows) and
// dae_csr_impression_metrics (CSR query rows and articles): both kernels score an impression's shown articles into scores[] and
// then call impression_rank_metrics, so the rank rule, the integer AUC and the NaN rule are one piece of device code.
#pragma once
#include "common.cuh"

namespace dae {

constexpr int kImpChunk = 256;   // scores staged per warp in shared memory

__device__ __forceinline__ int warp_sum_int(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Clicked count of one impression's flags [0, m).
__device__ __forceinline__ int count_clicked(const uint8_t* __restrict__ c, int64_t m, int lane) {
  int n = 0;
  for (int64_t k = lane; k < m; k += 32) n += c[k] != 0;
  return warp_sum_int(n);
}

// One warp: out[0..3] = (AUC, MRR, nDCG@5, nDCG@10) of the fp32 scores [b0, b0 + m) with click flags clicked[b0, b0 + m), the
// scores written by the warp before a __syncwarp.  rank_j = #{k: s_k > s_j} + #{k < j: s_k = s_j}.  The clicked candidates are
// taken 32 at a time, one per lane, against the whole list staged kImpChunk scores at a time in s_s / s_f (the warp's shared
// staging): O(|C| m) comparisons, the AUC counted in integers.  No click or no non-click: NaN x 4.
__device__ __forceinline__ void impression_rank_metrics(const float* scores, const uint8_t* __restrict__ clicked, int64_t b0, int64_t m,
                                                        float* s_s, uint8_t* s_f, double* out, int lane) {
  const int nc = count_clicked(clicked + b0, m, lane);
  const int64_t nn = m - nc;
  if (nc == 0 || nn == 0) {
    if (lane < 4) out[lane] = __longlong_as_double(0x7ff8000000000000LL);
    return;
  }
  long long auc2 = 0;
  double rr = 0.0, g5 = 0.0, g10 = 0.0;
  for (int64_t j0 = 0; j0 < m; j0 += 32) {
    const int64_t j = j0 + lane;
    const bool mine = j < m && clicked[b0 + j] != 0;
    if (!__any_sync(0xffffffffu, mine)) continue;
    const float sj = mine ? scores[b0 + j] : 0.0f;
    long long gt = 0, tie_before = 0, below_n = 0, tie_n = 0;
    for (int64_t k0 = 0; k0 < m; k0 += kImpChunk) {
      const int nk = (int)min((int64_t)kImpChunk, m - k0);
      __syncwarp();
      for (int t = lane; t < nk; t += 32) {
        s_s[t] = scores[b0 + k0 + t];
        s_f[t] = clicked[b0 + k0 + t] != 0;
      }
      __syncwarp();
      if (mine) {
        for (int t = 0; t < nk; ++t) {
          const float sk = s_s[t];
          gt += sk > sj;
          tie_before += (sk == sj) && (k0 + t < j);
          if (!s_f[t]) {
            below_n += sk < sj;
            tie_n += sk == sj;
          }
        }
      }
    }
    if (mine) {
      const long long rank = gt + tie_before;
      auc2 += 2 * below_n + tie_n;
      rr += 1.0 / (double)(rank + 1);
      if (rank < 10) {
        const double g = 1.0 / log2((double)(rank + 2));
        g10 += g;
        if (rank < 5) g5 += g;
      }
    }
  }
  auc2 = warp_sum_ll(auc2);
  rr = warp_sum(rr);
  g5 = warp_sum(g5);
  g10 = warp_sum(g10);
  if (lane == 0) {
    double i5 = 0.0, i10 = 0.0;
    for (int r = 0; r < 10 && r < nc; ++r) {
      const double g = 1.0 / log2((double)(r + 2));
      i10 += g;
      if (r < 5) i5 += g;
    }
    out[0] = (double)auc2 / (2.0 * (double)nc * (double)nn);
    out[1] = rr / (double)nc;
    out[2] = g5 / i5;
    out[3] = g10 / i10;
  }
}

}  // namespace dae
