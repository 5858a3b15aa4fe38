// Salt-and-pepper corruption of a CSR matrix on the device (dae_salt_pepper_csr): utils.salt_and_pepper_noise without the host loop.
//
// One CTA per row.  The row's v draws (column m_j, coin b_j) are resolved in a shared-memory slab of int32 slots, one per column of a
// window of at most kWin columns: every slot starts at -1, draw j does atomicMax(slot[m_j], 2j + b_j), so the slot ends up holding the
// LAST draw of its column (later draws overwrite earlier ones in the reference's loop).  The clean row's entries then claim the slots no
// draw touched, as -2 - e (e = the entry's offset in the row).  A walk over the window's columns in order emits, per slot s:
//   s >= 0   : the draw's value (hi if s & 1, else lo), stored only when it is non-zero (assigning 0 into a lil_matrix deletes)
//   s <= -2  : the clean entry e, stored as it is (explicit zeros included)
//   s == -1  : nothing
// A row wider than kWin columns is processed window by window, each rescanning the draws.  The count pass writes the per-row entry
// counts, one CTA scans them (so the workspace size needs no CUDA call), and the fill
// pass recomputes the resolve and writes the rows at their scanned offsets.
#include "common.cuh"

namespace dae {
namespace {

constexpr int kSpThreads = 512;
constexpr int kWin = 16384;   // slab columns per window: 64 KB of shared memory (three CTAs per SM)

// Draw j of global row r: column and coin (1 = hi).  Philox4x32-10, key (seed lo, seed hi), counter (j / 2, r, epoch lo, epoch hi);
// an even j takes the words (c0, c1), an odd j (c2, c3): column = c_a * F >> 32, coin = c_b >> 31.
__device__ __forceinline__ void philox_pair(uint64_t seed, uint64_t epoch, int64_t r, int64_t pair, uint32_t (&c)[4]) {
  c[0] = (uint32_t)pair; c[1] = (uint32_t)r; c[2] = (uint32_t)epoch; c[3] = (uint32_t)(epoch >> 32);
  uint32_t k[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
#pragma unroll
  for (int i = 0; i < 10; ++i) philox_round(c, k);
}

// Resolve the draws and the clean entries of row r into the slab for the window [w0, w0 + wn).  Ends with a barrier.
__device__ __forceinline__ void sp_resolve(int32_t* slab, int32_t w0, int32_t wn, const int32_t* __restrict__ idx, int64_t nnz_r,
                                           int32_t F, int64_t v, const uint32_t* __restrict__ draws_row, uint64_t seed, uint64_t epoch,
                                           int64_t r) {
  for (int32_t c = threadIdx.x; c < wn; c += blockDim.x) slab[c] = -1;
  __syncthreads();
  if (draws_row) {
    for (int64_t j = threadIdx.x; j < v; j += blockDim.x) {
      const uint32_t d = draws_row[j];
      const int32_t m = (int32_t)(d & 0x7fffffffu) - w0;
      if ((uint32_t)m < (uint32_t)wn) atomicMax(&slab[m], (int32_t)(2 * j + (d >> 31)));
    }
  } else {
    for (int64_t p = threadIdx.x; 2 * p < v; p += blockDim.x) {
      uint32_t c[4];
      philox_pair(seed, epoch, r, p, c);
      const int32_t m0 = (int32_t)(((uint64_t)c[0] * (uint32_t)F) >> 32) - w0;
      if ((uint32_t)m0 < (uint32_t)wn) atomicMax(&slab[m0], (int32_t)(4 * p + (c[1] >> 31)));
      if (2 * p + 1 < v) {
        const int32_t m1 = (int32_t)(((uint64_t)c[2] * (uint32_t)F) >> 32) - w0;
        if ((uint32_t)m1 < (uint32_t)wn) atomicMax(&slab[m1], (int32_t)(4 * p + 2 + (c[3] >> 31)));
      }
    }
  }
  __syncthreads();
  for (int64_t e = threadIdx.x; e < nnz_r; e += blockDim.x) {   // columns are unique within a canonical row: no two entries race
    const int32_t m = idx[e] - w0;
    if ((uint32_t)m < (uint32_t)wn && slab[m] == -1) slab[m] = (int32_t)(-2 - e);
  }
  __syncthreads();
}

__device__ __forceinline__ bool sp_keep(int32_t s, float lo, float hi) {
  return s >= 0 ? (((s & 1) ? hi : lo) != 0.0f) : s <= -2;
}

// pass 1: entries of each corrupted row -> counts[i]
__global__ void __launch_bounds__(kSpThreads) sp_count_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                                               int64_t row0, int32_t F, int64_t v, float lo, float hi,
                                                               const uint32_t* __restrict__ draws, uint64_t seed, uint64_t epoch,
                                                               int64_t* __restrict__ counts) {
  extern __shared__ int32_t slab[];
  __shared__ int64_t red[kSpThreads / 32];
  const int64_t i = blockIdx.x, r = row0 + i;
  const int64_t a = indptr[r], nnz_r = indptr[r + 1] - a;
  const uint32_t* dr = draws ? draws + i * v : nullptr;
  int64_t cnt = 0;
  for (int32_t w0 = 0; w0 < F; w0 += kWin) {
    const int32_t wn = min(kWin, F - w0);
    sp_resolve(slab, w0, wn, indices + a, nnz_r, F, v, dr, seed, epoch, r);
    for (int32_t c = threadIdx.x; c < wn; c += blockDim.x) cnt += sp_keep(slab[c], lo, hi);
    __syncthreads();   // the next window re-initialises the slab
  }
  cnt = __reduce_add_sync(0xffffffffu, (unsigned)cnt);   // a warp's count is at most F < 2^30
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int64_t t = 0;
    for (int w = 0; w < kSpThreads / 32; ++w) t += red[w];
    counts[i] = t;
  }
}

// inclusive sum of counts[0, n) -> incl, on one CTA: each thread sums a contiguous chunk, the chunk sums are scanned through the warps
constexpr int kScanThreads = 1024;
__global__ void __launch_bounds__(kScanThreads) sp_scan_kernel(const int64_t* __restrict__ counts, int64_t n, int64_t* __restrict__ incl) {
  __shared__ int64_t warp_tot[kScanThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t chunk = (n + kScanThreads - 1) / kScanThreads;
  const int64_t b = min(n, (int64_t)threadIdx.x * chunk), e = min(n, b + chunk);
  int64_t s = 0;
  for (int64_t q = b; q < e; ++q) s += counts[q];
  int64_t x = s;   // inclusive scan of the chunk sums within the warp
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_tot[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int64_t t = warp_tot[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    warp_tot[lane] = t;
  }
  __syncthreads();
  int64_t run = x - s + (wid ? warp_tot[wid - 1] : 0);   // exclusive prefix of this thread's chunk
  for (int64_t q = b; q < e; ++q) {
    run += counts[q];
    incl[q] = run;
  }
}

// pass 2: row i lands at base + incl[i] - counts[i], base = indptr_out[row0] (0, or where the previous call on the stream ended).  A total
// beyond cap writes no entries: every row of the call stays empty and *overflow is set.
__global__ void __launch_bounds__(kSpThreads) sp_fill_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                                              const float* __restrict__ values, int64_t row0, int64_t n, int32_t F, int64_t v,
                                                              float lo, float hi, const uint32_t* __restrict__ draws, uint64_t seed,
                                                              uint64_t epoch, const int64_t* __restrict__ counts,
                                                              const int64_t* __restrict__ incl, int64_t* __restrict__ indptr_out,
                                                              int32_t* __restrict__ indices_out, float* __restrict__ values_out, int64_t cap,
                                                              int32_t* __restrict__ overflow) {
  extern __shared__ int32_t slab[];
  __shared__ int32_t warp_cnt[2][kSpThreads / 32];
  const int64_t i = blockIdx.x, r = row0 + i;
  const int64_t base = indptr_out[row0];
  if (base + incl[n - 1] > cap) {
    if (threadIdx.x == 0) {
      indptr_out[r + 1] = base;
      if (i == 0) *overflow = 1;
    }
    return;
  }
  int64_t pos = base + incl[i] - counts[i];
  if (threadIdx.x == 0) indptr_out[r + 1] = base + incl[i];
  const int64_t a = indptr[r], nnz_r = indptr[r + 1] - a;
  const uint32_t* dr = draws ? draws + i * v : nullptr;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int buf = 0;
  for (int32_t w0 = 0; w0 < F; w0 += kWin) {
    const int32_t wn = min(kWin, F - w0);
    sp_resolve(slab, w0, wn, indices + a, nnz_r, F, v, dr, seed, epoch, r);
    // columns in tiles of blockDim, in order: ballot within the warp, the warps' counts through shared memory (double-buffered, so one
    // barrier per tile)
    for (int32_t t0 = 0; t0 < wn; t0 += blockDim.x) {
      const int32_t c = t0 + threadIdx.x;
      const int32_t s = c < wn ? slab[c] : -1;
      const bool keep = sp_keep(s, lo, hi);
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) warp_cnt[buf][wid] = __popc(bal);
      __syncthreads();
      int32_t before = 0, total = 0;
#pragma unroll
      for (int w = 0; w < kSpThreads / 32; ++w) {
        const int32_t x = warp_cnt[buf][w];
        before += w < wid ? x : 0;
        total += x;
      }
      if (keep) {
        const int64_t o = pos + before + __popc(bal & ((1u << lane) - 1u));
        indices_out[o] = w0 + c;
        values_out[o] = s >= 0 ? ((s & 1) ? hi : lo) : values[a + (-2 - s)];
      }
      pos += total;
      buf ^= 1;
    }
    __syncthreads();
  }
}

}  // namespace
}  // namespace dae

using namespace dae;

namespace {
// workspace: the per-row counts and their inclusive sum, int64 each
size_t sp_ws_half(int64_t n) { return ((size_t)(n > 0 ? n : 1) * 8 + 255) & ~(size_t)255; }
}  // namespace

extern "C" int dae_salt_pepper_workspace(int64_t n, size_t* bytes) {
  DAE_REQUIRE(bytes && n >= 0 && n <= INT32_MAX, "dae_salt_pepper_workspace: bad arguments");
  *bytes = 2 * sp_ws_half(n);
  return DAE_OK;
}

extern "C" int dae_salt_pepper_csr(const int64_t* indptr, const int32_t* indices, const float* values, int64_t row0, int64_t n, int32_t F,
                                   int64_t v, float lo, float hi, const uint32_t* draws, uint64_t seed, uint64_t epoch, int64_t* indptr_out,
                                   int32_t* indices_out, float* values_out, int64_t cap, int32_t* overflow, void* ws, size_t ws_bytes,
                                   void* stream) {
  DAE_REQUIRE(indptr && indices && values && indptr_out && indices_out && values_out && overflow,
              "dae_salt_pepper_csr: null pointer");
  DAE_REQUIRE(row0 >= 0 && n >= 0 && n <= INT32_MAX, "dae_salt_pepper_csr: bad rows (row0 %lld, n %lld)", (long long)row0,
              (long long)n);
  DAE_REQUIRE(F >= 1 && F < (1 << 30), "dae_salt_pepper_csr: F = %d outside [1, 2^30)", (int)F);
  DAE_REQUIRE(v >= 0 && v < (1 << 30), "dae_salt_pepper_csr: v = %lld outside [0, 2^30)", (long long)v);
  DAE_REQUIRE(cap >= 0, "dae_salt_pepper_csr: negative cap");
  const size_t cb = sp_ws_half(n);
  DAE_REQUIRE(ws && ws_bytes >= 2 * cb, "dae_salt_pepper_csr: workspace of %zu bytes, %zu needed (dae_salt_pepper_workspace)", ws_bytes,
              2 * cb);
  if (n == 0) return DAE_OK;
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* counts = (int64_t*)ws;
  int64_t* incl = (int64_t*)((char*)ws + cb);
  const int smem = (int)(sizeof(int32_t) * (F < kWin ? F : kWin));
  if (smem > 48 * 1024) {   // (per call: the attribute is per device)
    DAE_CUDA(cudaFuncSetAttribute(sp_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    DAE_CUDA(cudaFuncSetAttribute(sp_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  }
  sp_count_kernel<<<(unsigned)n, kSpThreads, smem, st>>>(indptr, indices, row0, F, v, lo, hi, draws, seed, epoch, counts);
  DAE_CHECK_LAUNCH("dae_salt_pepper_csr (count)");
  sp_scan_kernel<<<1, kScanThreads, 0, st>>>(counts, n, incl);
  DAE_CHECK_LAUNCH("dae_salt_pepper_csr (scan)");
  sp_fill_kernel<<<(unsigned)n, kSpThreads, smem, st>>>(indptr, indices, values, row0, n, F, v, lo, hi, draws, seed, epoch, counts, incl,
                                                         indptr_out, indices_out, values_out, cap, overflow);
  DAE_CHECK_LAUNCH("dae_salt_pepper_csr (fill)");
  return DAE_OK;
}
