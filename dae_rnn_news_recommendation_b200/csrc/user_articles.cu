// Fine-tuning the article encoder through the user encoders' losses (DESIGN 4.19): the per-batch compact table of the articles a
// training batch touches, and the scatter of per-position gradients into it.
//
// A joint batch encodes only the articles it touches (its reads, next reads, negatives and shown articles), T of them, into a
// compact table E_t [T, H]; every user-encoder kernel then runs on E_t with slot ids in place of article ids.  dae_touch_compact
// builds that table's row list and remaps the ids; dae_rows_scatter_add adds the input projection's gradient dX [P, H] into dE_t.
#include "common.cuh"

namespace dae {

constexpr int kTouchThreads = 256, kTouchPer = 4, kTouchTile = kTouchThreads * kTouchPer;

// The key of occurrence i in a call with stamp s: larger for a later call, and within one call larger for an earlier occurrence, so
// that atomicMax leaves in tag[id] the first occurrence of id in this call whatever tag held from earlier calls.
__device__ __forceinline__ unsigned long long touch_key(uint32_t stamp, int64_t i) {
  return ((unsigned long long)stamp << 32) | (unsigned long long)(0xffffffffu - (uint32_t)i);
}

__global__ void touch_mark_kernel(const int32_t* __restrict__ ids, int64_t n, uint32_t stamp, unsigned long long* __restrict__ tag) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t a = ids[i];
    if (a >= 0) atomicMax(tag + a, touch_key(stamp, i));
  }
}

// Flags of this thread's kTouchPer consecutive occurrences of the tile: 1 where the occurrence is its article's first in the call.
__device__ __forceinline__ int touch_firsts(const int32_t* __restrict__ ids, int64_t n, uint32_t stamp,
                                            const unsigned long long* __restrict__ tag, int64_t i0, int (&f)[kTouchPer]) {
  int c = 0;
#pragma unroll
  for (int k = 0; k < kTouchPer; ++k) {
    const int64_t i = i0 + k;
    const int32_t a = i < n ? ids[i] : -1;
    f[k] = a >= 0 && tag[a] == touch_key(stamp, i);
    c += f[k];
  }
  return c;
}

// Exclusive prefix of v over the CTA's threads (kTouchThreads) and the CTA total.
__device__ __forceinline__ int block_exclusive_scan(int v, int& total) {
  __shared__ int s_warp[kTouchThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
  if (lane == 31) s_warp[w] = incl;
  __syncthreads();
  int before = 0;
  total = 0;
#pragma unroll
  for (int k = 0; k < kTouchThreads / 32; ++k) {
    const int x = s_warp[k];
    if (k < w) before += x;
    total += x;
  }
  __syncthreads();
  return before + incl - v;
}

__global__ void __launch_bounds__(kTouchThreads) touch_count_kernel(const int32_t* __restrict__ ids, int64_t n, uint32_t stamp,
                                                                    const unsigned long long* __restrict__ tag, int32_t* __restrict__ ws) {
  int f[kTouchPer];
  const int c = touch_firsts(ids, n, stamp, tag, (int64_t)blockIdx.x * kTouchTile + threadIdx.x * kTouchPer, f);
  int total;
  block_exclusive_scan(c, total);
  if (threadIdx.x == 0) ws[1 + blockIdx.x] = total;
}

// Tile b's first occurrences take slots [sum of the earlier tiles' counts, ...) in occurrence order; the last tile writes T.
__global__ void __launch_bounds__(kTouchThreads) touch_place_kernel(const int32_t* __restrict__ ids, int64_t n, uint32_t stamp,
                                                                    const unsigned long long* __restrict__ tag, int32_t* __restrict__ ws,
                                                                    int32_t* __restrict__ slot_of, int32_t* __restrict__ rows) {
  int part = 0;
  for (int b = threadIdx.x; b < (int)blockIdx.x; b += kTouchThreads) part += ws[1 + b];
  int base;
  block_exclusive_scan(part, base);   // base: the sum of every earlier tile's count
  int f[kTouchPer];
  const int64_t i0 = (int64_t)blockIdx.x * kTouchTile + threadIdx.x * kTouchPer;
  const int c = touch_firsts(ids, n, stamp, tag, i0, f);
  int total;
  int s = base + block_exclusive_scan(c, total);
#pragma unroll
  for (int k = 0; k < kTouchPer; ++k) {
    if (f[k]) {
      const int32_t a = ids[i0 + k];
      rows[s] = a;
      slot_of[a] = s;
      ++s;
    }
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) ws[0] = base + total;
}

__global__ void touch_remap_kernel(const int32_t* __restrict__ ids, int64_t n, const int32_t* __restrict__ slot_of,
                                   int32_t* __restrict__ slots) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t a = ids[i];
    slots[i] = a >= 0 ? slot_of[a] : -1;
  }
}

__global__ void rows_scatter_add_kernel(const float* __restrict__ src, int64_t ld_src, const int32_t* __restrict__ idx, int64_t n,
                                        int cols, float* __restrict__ dst, int64_t ld_dst) {
  const int64_t total = n * cols;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = e / cols;
    const int c = (int)(e - p * cols);
    const int32_t r = idx[p];
    if (r >= 0) atomicAdd(dst + (int64_t)r * ld_dst + c, src[p * ld_src + c]);
  }
}

static int grid_cap(int64_t work, int per_block) {
  const int64_t b = (work + per_block - 1) / per_block, cap = (int64_t)sm_count() * 16;
  return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

}  // namespace dae

using namespace dae;

extern "C" int dae_touch_compact_workspace(int64_t n, int64_t* count) {
  DAE_REQUIRE(count && n >= 0, "dae_touch_compact_workspace: bad arguments");
  *count = 1 + (n + kTouchTile - 1) / kTouchTile;
  return DAE_OK;
}

extern "C" int dae_touch_compact(const int32_t* ids, int64_t n, uint32_t stamp, void* tag, int32_t* slot_of, int32_t* rows,
                                 int32_t* slots, int32_t* ws, void* stream) {
  DAE_REQUIRE(ids && tag && slot_of && rows && slots && ws, "dae_touch_compact: null pointer");
  DAE_REQUIRE(n > 0 && n < 0x7fffffffLL && stamp > 0, "dae_touch_compact: bad arguments (n = %lld, stamp = %u)", (long long)n, stamp);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* t = (unsigned long long*)tag;
  const int tiles = (int)((n + kTouchTile - 1) / kTouchTile);
  touch_mark_kernel<<<grid_cap(n, 256), 256, 0, st>>>(ids, n, stamp, t);
  touch_count_kernel<<<tiles, kTouchThreads, 0, st>>>(ids, n, stamp, t, ws);
  touch_place_kernel<<<tiles, kTouchThreads, 0, st>>>(ids, n, stamp, t, ws, slot_of, rows);
  touch_remap_kernel<<<grid_cap(n, 256), 256, 0, st>>>(ids, n, slot_of, slots);
  DAE_CHECK_LAUNCH("dae_touch_compact");
  return DAE_OK;
}

extern "C" int dae_rows_scatter_add(const float* src, int64_t ld_src, const int32_t* idx, int64_t n, int32_t cols, float* dst,
                                    int64_t ld_dst, void* stream) {
  DAE_REQUIRE(src && idx && dst && n > 0 && cols > 0 && ld_src >= cols && ld_dst >= cols, "dae_rows_scatter_add: bad arguments");
  rows_scatter_add_kernel<<<grid_cap(n * cols, 256), 256, 0, (cudaStream_t)stream>>>(src, ld_src, idx, n, cols, dst, ld_dst);
  DAE_CHECK_LAUNCH("dae_rows_scatter_add");
  return DAE_OK;
}
