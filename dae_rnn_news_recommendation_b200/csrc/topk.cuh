// k-best selection pieces shared by the dense (gemm_tc.cu) and the sparse (similarity_sparse.cu) similarity top-k.
#pragma once
#include <cfloat>
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

// ---------------------------------------------------------------------------------------------------------------------
// Long lists (k up to kTopkLongMaxK): one CTA per query row ranks a row's entries in shared memory.  An entry is its position
// pos in the row's source (a partial-list slice or a candidate segment); its 64-bit rank key sorts ascending in
// (score desc, pos asc) order, and positions are in increasing corpus index, so that is (score desc, index asc).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kTopkLongMaxK = 1024;
constexpr int kRankThreads = 256;
constexpr unsigned long long kNoEntry = ~0ull;   // ranks after every entry

// -0.0 ranks as +0.0 (equal under the kernels' >); a larger score gives a smaller high word
__device__ __forceinline__ unsigned long long rank_key(float s, uint32_t pos) {
  uint32_t u = __float_as_uint(s);
  if (u == 0x80000000u) u = 0u;
  const uint32_t d = (u & 0x80000000u) ? u : (~u & 0x7fffffffu);
  return ((unsigned long long)d << 32) | pos;
}

// ascending bitonic sort of a[0, n), n a power of two, by all threads of the block; synchronised on entry and exit
__device__ __forceinline__ void block_bitonic_sort(unsigned long long* a, int n) {
  for (int size = 2; size <= n; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < (n >> 1); t += blockDim.x) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        const bool up = (lo & size) == 0;
        const unsigned long long x = a[lo], y = a[hi];
        if ((x > y) == up) { a[lo] = y; a[hi] = x; }
      }
    }
  }
  __syncthreads();
}

// The k best entries of one row, any number n of them, in chunks of L (a power of two >= k): key[0, L) holds the best so far and
// key[L, 2L) the next chunk; one sort of the 2L keys keeps the best.  GROUPS: after that sort, every entry whose group (groups of
// the entry's corpus index src.col(pos)) already appears at a better rank is dropped -- a sort of (group, rank) pairs in aux finds
// them -- and a second sort moves the drops to the end, so key[0, kept) holds distinct groups, each its best entry seen.  Returns
// kept = min(k, entries left); key[0, kept) sorted best first.  Src: key(pos) (kNoEntry for a slot without an entry), col(pos).
template <bool GROUPS, class Src>
__device__ int rank_best(unsigned long long* key, unsigned long long* aux, int L, int k, int64_t n, const Src& src,
                         const int32_t* __restrict__ groups) {
  int kept = 0;
  for (int64_t c0 = 0; c0 < n; c0 += L) {
    for (int t = threadIdx.x; t < 2 * L; t += blockDim.x) {
      if (t < kept) continue;
      const int64_t pos = c0 + t - L;
      key[t] = (t >= L && pos < n) ? src.key(pos) : kNoEntry;
    }
    block_bitonic_sort(key, 2 * L);
    if constexpr (GROUPS) {
      for (int t = threadIdx.x; t < 2 * L; t += blockDim.x) {
        const unsigned long long e = key[t];
        aux[t] = e == kNoEntry ? kNoEntry : ((unsigned long long)(uint32_t)groups[src.col((int64_t)(uint32_t)e)] << 32) | (uint32_t)t;
      }
      block_bitonic_sort(aux, 2 * L);
      for (int t = threadIdx.x + 1; t < 2 * L; t += blockDim.x)
        if (aux[t] != kNoEntry && (aux[t] >> 32) == (aux[t - 1] >> 32)) key[(uint32_t)aux[t]] = kNoEntry;
      block_bitonic_sort(key, 2 * L);
    }
    int valid = 0;   // 2L is a multiple of the block size
    for (int t0 = 0; t0 < 2 * L; t0 += blockDim.x) valid += __syncthreads_count(key[t0 + threadIdx.x] != kNoEntry);
    kept = min(k, valid);
  }
  return kept;
}

// partial lists of topk_kernel<32> (2 * splits lists of 32 per row) as a rank source
struct ListSrc {
  const float* val; const int32_t* idx;
  __device__ __forceinline__ unsigned long long key(int64_t pos) const {
    return idx[pos] >= 0 ? rank_key(val[pos], (uint32_t)pos) : kNoEntry;
  }
  __device__ __forceinline__ int col(int64_t pos) const { return idx[pos]; }
};

// one row's candidates, in increasing corpus index (a segment of dae_pairs_sort's output)
struct SegSrc {
  const int32_t* j; const float* s;
  __device__ __forceinline__ unsigned long long key(int64_t pos) const { return rank_key(s[pos], (uint32_t)pos); }
  __device__ __forceinline__ int col(int64_t pos) const { return j[pos]; }
};

// Bound: tau[r] = the k-th best score among row r's partial lists (the k-th best distinct group's best with GROUPS), a lower bound
// on the row's true k-th score: the lists hold a subset of the row's candidates.  -FLT_MAX when the lists hold fewer than k (groups),
// so that every finite score qualifies.  One CTA per row; dynamic shared memory: 2L keys (4L with GROUPS).
template <bool GROUPS>
static __global__ void __launch_bounds__(kRankThreads) topk_bound_kernel(const float* __restrict__ ws_val, const int32_t* __restrict__ ws_idx,
                                                                        int n_lists, int list_len, int k, int L,
                                                                        const int32_t* __restrict__ groups, float* __restrict__ tau) {
  extern __shared__ unsigned long long rank_smem[];
  const int r = blockIdx.x;
  const int64_t n = (int64_t)n_lists * list_len, base = (int64_t)r * n;
  const ListSrc src{ws_val + base, ws_idx + base};
  const int kept = rank_best<GROUPS>(rank_smem, rank_smem + 2 * L, L, k, n, src, groups);
  if (threadIdx.x == 0) tau[r] = kept == k ? src.val[(uint32_t)rank_smem[k - 1]] : -FLT_MAX;
}

// Select: row r's k best candidates among the pairs (i sorted, then j ascending within a row), padded with -1 / -inf.  The row's
// segment is found by binary search on i.  One CTA per row; dynamic shared memory as topk_bound_kernel.
template <bool GROUPS>
static __global__ void __launch_bounds__(kRankThreads) topk_select_kernel(const int32_t* __restrict__ pi, const int32_t* __restrict__ pj,
                                                                         const float* __restrict__ ps, int64_t n_pairs, int k, int L,
                                                                         const int32_t* __restrict__ groups, int32_t* __restrict__ idx_out,
                                                                         float* __restrict__ val_out) {
  extern __shared__ unsigned long long rank_smem[];
  __shared__ int64_t seg[2];
  const int r = blockIdx.x;
  if (threadIdx.x < 2) {   // first pair of row r + threadIdx.x
    int64_t lo = 0, hi = n_pairs;
    const int want = r + (int)threadIdx.x;
    while (lo < hi) {
      const int64_t mid = lo + ((hi - lo) >> 1);
      if (pi[mid] < want) lo = mid + 1; else hi = mid;
    }
    seg[threadIdx.x] = lo;
  }
  __syncthreads();
  const int64_t b = seg[0];
  const SegSrc src{pj + b, ps + b};
  const int kept = rank_best<GROUPS>(rank_smem, rank_smem + 2 * L, L, k, seg[1] - b, src, groups);
  for (int t = threadIdx.x; t < k; t += blockDim.x) {
    const int64_t o = (int64_t)r * k + t;
    if (t < kept) {
      const uint32_t pos = (uint32_t)rank_smem[t];
      idx_out[o] = src.j[pos]; val_out[o] = src.s[pos];
    } else {
      idx_out[o] = -1; val_out[o] = neg_inf();
    }
  }
}

}  // namespace dae
