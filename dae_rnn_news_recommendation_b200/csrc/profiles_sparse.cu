// Bag-of-words user profiles (DESIGN 4.20): P = W.X for a history CSR W [U x N] and the articles' CSR X [N x F], with a sparse
// result and never O(U F) memory, and the impression metrics of CSR query rows against the articles' CSR.
//   profiles : one warp per user, F cut into slabs of kPfSlab columns.  For each slab the warp takes the user's reads in
//              increasing article order, 32 at a time (lane j binary-searches read j's row for the slab's entries), then walks
//              each read's entries in the slab, lanes over entries: a row's columns are distinct, so no two lanes touch one
//              accumulator, and a __syncwarp between reads keeps each column's term order.  A bitmap in shared memory marks the
//              touched columns (explicit zeros included).  At the end of the slab the warp compacts the bitmap with popc prefixes:
//              count mode adds the popcounts, fill mode writes the columns (increasing) and their sums, and both re-zero what they
//              read.  Slabs that no read touches are skipped: the next slab is the smallest column a read has past the current one.
//   numerics : P[u, f] accumulates in fp32 from +0, one term __fmul_rn(w, x) per history entry in increasing article order, added
//              with __fadd_rn (no FMA): the result does not depend on the launch shape, and a float32 host loop reproduces it.
//              normalise: n^2 = the fp32 sum of the rounded squares in increasing column order (lane 0, sequential), then
//              v = __fdiv_rn(v, __fsqrt_rn(n^2)); a row with n^2 = 0 is left as it is.
//   metrics  : one warp per impression.  For each shown article the lanes take its entries, 32 at a time, and binary-search their
//              columns in the query row; lane 0 adds the rounded products (and, for cosine, the rounded squares) of the round in
//              column order, so the dot product is the sparse top-k's score of the same pair, bit for bit.  The metrics of the
//              scores come from impression_rank_metrics, the code dae_impression_metrics runs.
#include "common.cuh"
#include "impression_rank.cuh"

namespace dae {
namespace {

constexpr int kPfSlab = 2048;              // columns per slab: 8 KB of accumulators and 256 B of bitmap per warp
constexpr int kPfWords = kPfSlab / 32;
constexpr int kPfWarps = 4;                // 33 KB of static shared memory per CTA in fill mode
constexpr int kPfMaxFeatures = 1 << 24;
constexpr int kCsrImpWarps = 4;
constexpr unsigned kFull = 0xffffffffu;

// first position p in [lo, hi) with idx[p] >= c (hi when none)
__device__ __forceinline__ int64_t lower_bound_col(const int32_t* __restrict__ idx, int64_t lo, int64_t hi, int c) {
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (idx[mid] < c) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ int warp_min_int(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(kFull, v, o));
  return v;
}

struct PfParams {
  const int64_t* w_indptr; const int32_t* w_indices; const float* w_values;
  const int64_t* x_indptr; const int32_t* x_indices; const float* x_values;
  int F, first_user, n_users;
  int64_t* p_count;                          // count mode: p_count[u + 1] = row u's column count
  const int64_t* p_indptr;                   // fill mode
  int32_t* p_indices; float* p_values;       // fill mode: entry t of row u at p_indptr[u] - p_indptr[first_user] + t
  int normalise;
};

// FILL = false: dae_csr_profiles_count's per-user counts; FILL = true: dae_csr_profiles' rows
template <bool FILL>
__global__ void __launch_bounds__(kPfWarps * 32) profiles_kernel(const PfParams p) {
  __shared__ float s_acc[kPfWarps][FILL ? kPfSlab : 1];
  __shared__ unsigned s_bits[kPfWarps][kPfWords];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t item = (int64_t)blockIdx.x * kPfWarps + w;
  if (item >= p.n_users) return;                       // whole warps only: no block-wide barrier below
  const int u = p.first_user + (int)item;
  float* acc = s_acc[w];
  unsigned* bits = s_bits[w];
  for (int j = lane; j < kPfWords; j += 32) bits[j] = 0u;
  if constexpr (FILL)
    for (int j = lane; j < kPfSlab; j += 32) acc[j] = 0.0f;
  const int64_t rb = p.w_indptr[u], re = p.w_indptr[u + 1];
  const int n_slabs = (p.F + kPfSlab - 1) / kPfSlab;
  int64_t out = 0, count = 0;
  if constexpr (FILL) out = p.p_indptr[u] - p.p_indptr[p.first_user];
  const int64_t row0 = out;
  __syncwarp();
  for (int slab = 0; slab < n_slabs;) {
    const int base = slab * kPfSlab, end = base + kPfSlab;
    int next = INT_MAX;                                // the smallest column >= end of any read
    for (int64_t c0 = rb; c0 < re; c0 += 32) {
      const int nc = (int)(re - c0 < 32 ? re - c0 : 32);
      int64_t lo = 0, hi = 0;
      float wv = 0.0f;
      if (lane < nc) {
        const int a = p.w_indices[c0 + lane];
        if constexpr (FILL) wv = p.w_values[c0 + lane];
        const int64_t xb = p.x_indptr[a], xe = p.x_indptr[a + 1];
        lo = n_slabs == 1 ? xb : lower_bound_col(p.x_indices, xb, xe, base);
        hi = n_slabs == 1 ? xe : lower_bound_col(p.x_indices, lo, xe, end);
        if (hi < xe) next = min(next, p.x_indices[hi]);
      }
      for (int j = 0; j < nc; ++j) {
        const int64_t a0 = __shfl_sync(kFull, lo, j), a1 = __shfl_sync(kFull, hi, j);
        const float wj = __shfl_sync(kFull, wv, j);
        for (int64_t t = a0 + lane; t < a1; t += 32) {
          const int c = p.x_indices[t] - base;
          atomicOr(bits + (c >> 5), 1u << (c & 31));
          if constexpr (FILL) acc[c] = __fadd_rn(acc[c], __fmul_rn(wj, p.x_values[t]));
        }
        if constexpr (FILL) __syncwarp();              // a column's next term (next read) may come from another lane
      }
    }
    __syncwarp();
    // compact: lane l owns bitmap words 2l and 2l + 1 (columns base + 64 l .. base + 64 l + 63, increasing with the lane)
    const unsigned b0 = bits[2 * lane], b1 = bits[2 * lane + 1];
    bits[2 * lane] = 0u;
    bits[2 * lane + 1] = 0u;
    const int n = __popc(b0) + __popc(b1);
    int incl = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(kFull, incl, o); if (lane >= o) incl += t; }
    if constexpr (FILL) {
      int64_t pos = out + incl - n;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        for (unsigned m = h ? b1 : b0; m; m &= m - 1u) {
          const int c = 64 * lane + 32 * h + __ffs(m) - 1;
          p.p_indices[pos] = base + c;
          p.p_values[pos] = acc[c];
          acc[c] = 0.0f;
          ++pos;
        }
      }
    }
    const int total = __shfl_sync(kFull, incl, 31);
    out += total;
    count += total;
    __syncwarp();
    next = warp_min_int(next);
    slab = next == INT_MAX ? n_slabs : next / kPfSlab;
  }
  if constexpr (!FILL) {
    if (lane == 0) p.p_count[u + 1] = count;
  } else {
    if (!p.normalise || count == 0) return;
    float n2 = 0.0f;
    if (lane == 0) {
#pragma unroll 4
      for (int64_t t = row0; t < out; ++t) {
        const float v = p.p_values[t];
        n2 = __fadd_rn(n2, __fmul_rn(v, v));
      }
    }
    n2 = __shfl_sync(kFull, n2, 0);
    if (n2 == 0.0f) return;
    const float nrm = __fsqrt_rn(n2);
    for (int64_t t = row0 + lane; t < out; t += 32) p.p_values[t] = __fdiv_rn(p.p_values[t], nrm);
  }
}

// p[1 .. n] = inclusive prefix sums of p[1 .. n] in place, p[0] = 0: one CTA, 8 elements per thread and piece
constexpr int kPfScanThreads = 1024, kPfScanPer = 8;
__global__ void __launch_bounds__(kPfScanThreads) profiles_scan_kernel(int64_t* __restrict__ p, int64_t n) {
  __shared__ long long s_warp[32];
  __shared__ long long s_carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) { s_carry = 0; p[0] = 0; }
  __syncthreads();
  for (int64_t b = 1; b <= n; b += (int64_t)kPfScanThreads * kPfScanPer) {
    long long v[kPfScanPer], sum = 0;
#pragma unroll
    for (int j = 0; j < kPfScanPer; ++j) {
      const int64_t i = b + (int64_t)tid * kPfScanPer + j;
      v[j] = i <= n ? p[i] : 0;
      sum += v[j];
    }
    long long incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(kFull, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      const long long x = s_warp[lane];
      long long xi = x;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(kFull, xi, o); if (lane >= o) xi += t; }
      s_warp[lane] = xi - x;
    }
    __syncthreads();
    long long run = s_carry + s_warp[wid] + incl - sum;
#pragma unroll
    for (int j = 0; j < kPfScanPer; ++j) {
      const int64_t i = b + (int64_t)tid * kPfScanPer + j;
      run += v[j];
      if (i <= n) p[i] = run;
    }
    __syncthreads();
    if (tid == kPfScanThreads - 1) s_carry = run;
    __syncthreads();
  }
}

// One warp per impression i: scores[k] = q_i . x(items[k]) (cosine: over sqrt(qq) sqrt(ee), 0 when either is 0), then
// impression_rank_metrics.  Query row q_i = rows [q_indptr[i], q_indptr[i + 1]) of the query CSR.
__global__ void __launch_bounds__(kCsrImpWarps * 32) csr_impression_metrics_kernel(
    const int64_t* __restrict__ q_indptr, const int32_t* __restrict__ q_indices, const float* __restrict__ q_values,
    const int64_t* __restrict__ x_indptr, const int32_t* __restrict__ x_indices, const float* __restrict__ x_values, int cosine,
    const int64_t* __restrict__ indptr, const int32_t* __restrict__ items, const uint8_t* __restrict__ clicked, int64_t n_imp,
    float* scores, double* __restrict__ metrics) {
  __shared__ float s_s[kCsrImpWarps][kImpChunk];
  __shared__ uint8_t s_f[kCsrImpWarps][kImpChunk];
  __shared__ float s_p[kCsrImpWarps][32], s_e[kCsrImpWarps][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int64_t i = (int64_t)blockIdx.x * kCsrImpWarps + w; i < n_imp; i += (int64_t)gridDim.x * kCsrImpWarps) {
    const int64_t b0 = indptr[i], m = indptr[i + 1] - b0;
    const int64_t qb = q_indptr[i], qe = q_indptr[i + 1];
    float qq = 0.0f;
    if (cosine && lane == 0)
      for (int64_t t = qb; t < qe; ++t) qq = __fadd_rn(qq, __fmul_rn(q_values[t], q_values[t]));
    for (int64_t k = 0; k < m; ++k) {
      const int a = items[b0 + k];
      const int64_t xb = x_indptr[a], xe = x_indptr[a + 1];
      float dot = 0.0f, ee = 0.0f;
      for (int64_t t0 = xb; t0 < xe; t0 += 32) {
        const int n = (int)(xe - t0 < 32 ? xe - t0 : 32);
        float prod = 0.0f, sq = 0.0f;
        if (lane < n) {
          const int c = x_indices[t0 + lane];
          const float x = x_values[t0 + lane];
          sq = __fmul_rn(x, x);
          const int64_t pos = lower_bound_col(q_indices, qb, qe, c);
          if (pos < qe && q_indices[pos] == c) prod = __fmul_rn(q_values[pos], x);
        }
        s_p[w][lane] = prod;
        s_e[w][lane] = sq;
        __syncwarp();
        if (lane == 0) {
          // + 0 for a column q lacks leaves the sum's bits as they are (it is never -0: it starts at +0 and x + (-x) = +0)
          for (int j = 0; j < n; ++j) dot = __fadd_rn(dot, s_p[w][j]);
          if (cosine)
            for (int j = 0; j < n; ++j) ee = __fadd_rn(ee, s_e[w][j]);
        }
        __syncwarp();
      }
      if (lane == 0) {
        float s = dot;
        if (cosine) s = (qq > 0.0f && ee > 0.0f) ? __fdiv_rn(dot, __fmul_rn(__fsqrt_rn(qq), __fsqrt_rn(ee))) : 0.0f;
        scores[b0 + k] = s;
      }
    }
    __syncwarp();   // the scores written by lane 0 are read by every lane below
    impression_rank_metrics(scores, clicked, b0, m, s_s[w], s_f[w], metrics + i * 4, lane);
  }
}

int pf_grid(int64_t rows, int warps) {
  const int64_t b = (rows + warps - 1) / warps, cap = (int64_t)sm_count() * 16;
  return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

}  // namespace
}  // namespace dae

using namespace dae;

extern "C" int dae_csr_profiles_count(const int64_t* w_indptr, const int32_t* w_indices, int32_t n_users, int32_t n_articles,
                                      const int64_t* x_indptr, const int32_t* x_indices, int32_t n_features, int64_t* p_indptr,
                                      void* stream) {
  DAE_REQUIRE(w_indptr && x_indptr && p_indptr, "dae_csr_profiles_count: null pointer");
  DAE_REQUIRE(n_users > 0 && n_articles > 0 && n_features > 0 && n_features <= kPfMaxFeatures,
              "dae_csr_profiles_count: bad sizes (%d users, %d articles, %d features: every count > 0, features <= 2^24)", n_users,
              n_articles, n_features);
  DAE_REQUIRE(((uintptr_t)w_indptr | (uintptr_t)x_indptr | (uintptr_t)p_indptr) % 8 == 0 &&
              ((uintptr_t)w_indices | (uintptr_t)x_indices) % 4 == 0,
              "dae_csr_profiles_count: indptr arrays must be 8-byte, index arrays 4-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  PfParams p{};
  p.w_indptr = w_indptr; p.w_indices = w_indices; p.x_indptr = x_indptr; p.x_indices = x_indices;
  p.F = n_features; p.first_user = 0; p.n_users = n_users; p.p_count = p_indptr;
  profiles_kernel<false><<<(unsigned)((n_users + kPfWarps - 1) / kPfWarps), kPfWarps * 32, 0, st>>>(p);
  DAE_CHECK_LAUNCH("dae_csr_profiles_count");
  profiles_scan_kernel<<<1, kPfScanThreads, 0, st>>>(p_indptr, n_users);
  DAE_CHECK_LAUNCH("dae_csr_profiles_count (scan)");
  return DAE_OK;
}

extern "C" int dae_csr_profiles(const int64_t* w_indptr, const int32_t* w_indices, const float* w_values, int32_t n_users,
                                int32_t n_articles, const int64_t* x_indptr, const int32_t* x_indices, const float* x_values,
                                int32_t n_features, const int64_t* p_indptr, int32_t first_user, int32_t n_fill, int32_t normalise,
                                int32_t* p_indices, float* p_values, void* stream) {
  DAE_REQUIRE(w_indptr && x_indptr && p_indptr, "dae_csr_profiles: null pointer");
  DAE_REQUIRE(n_users > 0 && n_articles > 0 && n_features > 0 && n_features <= kPfMaxFeatures,
              "dae_csr_profiles: bad sizes (%d users, %d articles, %d features: every count > 0, features <= 2^24)", n_users,
              n_articles, n_features);
  DAE_REQUIRE(first_user >= 0 && n_fill > 0 && first_user <= n_users - n_fill,
              "dae_csr_profiles: users [%d, %d + %d) are not a non-empty range of [0, %d)", first_user, first_user, n_fill, n_users);
  DAE_REQUIRE(normalise == 0 || normalise == 1, "dae_csr_profiles: normalise = %d: 0 or 1", normalise);
  DAE_REQUIRE(((uintptr_t)w_indptr | (uintptr_t)x_indptr | (uintptr_t)p_indptr) % 8 == 0 &&
              ((uintptr_t)w_indices | (uintptr_t)w_values | (uintptr_t)x_indices | (uintptr_t)x_values | (uintptr_t)p_indices |
               (uintptr_t)p_values) % 4 == 0,
              "dae_csr_profiles: indptr arrays must be 8-byte, the other arrays 4-byte aligned");
  PfParams p{};
  p.w_indptr = w_indptr; p.w_indices = w_indices; p.w_values = w_values;
  p.x_indptr = x_indptr; p.x_indices = x_indices; p.x_values = x_values;
  p.F = n_features; p.first_user = first_user; p.n_users = n_fill;
  p.p_indptr = p_indptr; p.p_indices = p_indices; p.p_values = p_values; p.normalise = normalise;
  profiles_kernel<true><<<(unsigned)((n_fill + kPfWarps - 1) / kPfWarps), kPfWarps * 32, 0, (cudaStream_t)stream>>>(p);
  DAE_CHECK_LAUNCH("dae_csr_profiles");
  return DAE_OK;
}

extern "C" int dae_csr_impression_metrics(const int64_t* q_indptr, const int32_t* q_indices, const float* q_values,
                                          const int64_t* x_indptr, const int32_t* x_indices, const float* x_values, int32_t n_articles,
                                          int32_t n_features, int32_t cosine, const int64_t* indptr, const int32_t* items,
                                          const uint8_t* clicked, int64_t n_imp, float* scores, double* metrics, void* stream) {
  DAE_REQUIRE(q_indptr && x_indptr && indptr && items && clicked && scores && metrics, "dae_csr_impression_metrics: null pointer");
  DAE_REQUIRE(n_articles > 0 && n_features > 0 && n_imp > 0 && (cosine == 0 || cosine == 1),
              "dae_csr_impression_metrics: bad arguments (%d articles, %d features, %lld impressions, cosine = %d)", n_articles,
              n_features, (long long)n_imp, cosine);
  DAE_REQUIRE(((uintptr_t)q_indptr | (uintptr_t)x_indptr | (uintptr_t)indptr | (uintptr_t)metrics) % 8 == 0 &&
              ((uintptr_t)q_indices | (uintptr_t)q_values | (uintptr_t)x_indices | (uintptr_t)x_values | (uintptr_t)items |
               (uintptr_t)scores) % 4 == 0,
              "dae_csr_impression_metrics: indptr arrays and metrics must be 8-byte, the other arrays 4-byte aligned");
  csr_impression_metrics_kernel<<<pf_grid(n_imp, kCsrImpWarps), kCsrImpWarps * 32, 0, (cudaStream_t)stream>>>(
      q_indptr, q_indices, q_values, x_indptr, x_indices, x_values, cosine, indptr, items, clicked, n_imp, scores, metrics);
  DAE_CHECK_LAUNCH("dae_csr_impression_metrics");
  return DAE_OK;
}
