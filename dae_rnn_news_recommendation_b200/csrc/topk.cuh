// k-best selection pieces shared by the dense (gemm_tc.cu) and the sparse (similarity_sparse.cu) similarity top-k.
#pragma once
#include "common.cuh"

namespace dae {

__device__ __forceinline__ float neg_inf() { return __int_as_float(0xff800000); }

// (v1, i1) ranks before (v2, i2): higher score first, lower index among equal scores; index -1 (no entry) ranks last
__device__ __forceinline__ bool topk_before(float v1, int i1, float v2, int i2) {
  return i1 >= 0 && (i2 < 0 || v1 > v2 || (v1 == v2 && i1 < i2));
}

// one warp per query row: n_lists sorted partial lists of k (lane l owns lists l and l + 32) -> the row's k best, padded with -1 / -inf
static __global__ void __launch_bounds__(256) topk_merge_kernel(const float* __restrict__ ws_val, const int32_t* __restrict__ ws_idx,
                                                                int rows, int n_lists, int k, int32_t* __restrict__ idx_out,
                                                                float* __restrict__ val_out) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int64_t base = (int64_t)r * n_lists * k;
  const int la = lane, lb = lane + 32;
  int ha = 0, hb = 0;                          // heads of the two lists
  for (int j = 0; j < k; ++j) {
    float va = neg_inf(), vb = neg_inf();
    int ia = -1, ib = -1;
    if (la < n_lists && ha < k) { va = ws_val[base + (int64_t)la * k + ha]; ia = ws_idx[base + (int64_t)la * k + ha]; }
    if (lb < n_lists && hb < k) { vb = ws_val[base + (int64_t)lb * k + hb]; ib = ws_idx[base + (int64_t)lb * k + hb]; }
    float bv = va;
    int bi = ia;
    if (topk_before(vb, ib, bv, bi)) { bv = vb; bi = ib; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (topk_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (bi >= 0) {                             // corpus indices are unique across the lists: exactly one head moves
      if (ia == bi) ++ha;
      else if (ib == bi) ++hb;
    }
    if (lane == 0) { idx_out[(int64_t)r * k + j] = bi; val_out[(int64_t)r * k + j] = (bi >= 0) ? bv : neg_inf(); }
  }
}

// topk_merge_kernel for partial lists of group representatives (groups[c] is corpus row c's label): the row's k best entries of
// distinct groups.  Entries are popped in (score desc, index asc) order and an entry whose group is already taken is skipped --
// it ranks below that group's taken entry, and every entry that is not an answer ranks below all answers, so the first k distinct
// groups popped are the answer.  Lane t < n_out holds the t-th taken group; one ballot tests a popped entry.  Up to n_lists * k
// pops; padded with -1 / -inf when the lists run out first.
static __global__ void __launch_bounds__(256) topk_merge_groups_kernel(const float* __restrict__ ws_val, const int32_t* __restrict__ ws_idx,
                                                                       const int32_t* __restrict__ groups, int rows, int n_lists, int k,
                                                                       int32_t* __restrict__ idx_out, float* __restrict__ val_out) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int64_t base = (int64_t)r * n_lists * k;
  const int la = lane, lb = lane + 32;
  int ha = 0, hb = 0;                          // heads of the two lists
  int taken = -1;                              // lane t < n_out: the group of output entry t
  int n_out = 0;
  while (n_out < k) {
    float va = neg_inf(), vb = neg_inf();
    int ia = -1, ib = -1;
    if (la < n_lists && ha < k) { va = ws_val[base + (int64_t)la * k + ha]; ia = ws_idx[base + (int64_t)la * k + ha]; }
    if (lb < n_lists && hb < k) { vb = ws_val[base + (int64_t)lb * k + hb]; ib = ws_idx[base + (int64_t)lb * k + hb]; }
    float bv = va;
    int bi = ia;
    if (topk_before(vb, ib, bv, bi)) { bv = vb; bi = ib; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (topk_before(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    if (bi < 0) break;                         // every list is exhausted
    if (ia == bi) ++ha;                        // corpus indices are unique across the lists: exactly one head moves
    else if (ib == bi) ++hb;
    const int g = groups[bi];
    if (__ballot_sync(0xffffffffu, lane < n_out && taken == g)) continue;
    if (lane == n_out) taken = g;
    if (lane == 0) { idx_out[(int64_t)r * k + n_out] = bi; val_out[(int64_t)r * k + n_out] = bv; }
    ++n_out;
  }
  for (int j = n_out + lane; j < k; j += 32) { idx_out[(int64_t)r * k + j] = -1; val_out[(int64_t)r * k + j] = neg_inf(); }
}

}  // namespace dae
