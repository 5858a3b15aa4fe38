// Fine-tuning the article encoder through the user encoders' losses (DESIGN 4.19): the per-batch compact table of the articles a
// training batch touches, and the scatter of per-position gradients into it.
//
// A joint batch encodes only the articles it touches (its reads, next reads, negatives and shown articles), T of them, into a
// compact table E_t [T, H]; every user-encoder kernel then runs on E_t with slot ids in place of article ids.  dae_touch_compact
// builds that table's row list and remaps the ids; dae_rows_scatter_add adds the input projection's gradient dX [P, H] into dE_t.
// In the deterministic mode (DESIGN 4.21) dae_ordered_rows replaces both the loss kernels' atomics and that scatter: it groups the
// article-gradient triples by slot with a stable radix sort and sums each slot's terms in triple order.
#include <cub/device/device_radix_sort.cuh>
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

// ---- ordered article gradient (DESIGN 4.21) ------------------------------------------------------------------------------------
// Term i < n_a is the triple (a_slot[i], a_row[i], a_coef[i]) over src_a; term n_a + p is (b_slot[p], p, 1) over src_b.  key = the
// term's slot, n_slots for none (slot < 0), so the sort leaves those last; val = i.
__global__ void ordered_keys_kernel(const int32_t* __restrict__ a_slot, int64_t n_a, const int32_t* __restrict__ b_slot, int64_t n,
                                    int32_t n_slots, uint32_t* __restrict__ key, int32_t* __restrict__ val) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t s = i < n_a ? a_slot[i] : b_slot[i - n_a];
    key[i] = s < 0 ? (uint32_t)n_slots : (uint32_t)s;
    val[i] = (int32_t)i;
  }
}

__device__ __forceinline__ int64_t lower_bound_u32(const uint32_t* __restrict__ k, int64_t n, uint32_t v) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (k[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

constexpr int kOrdWarps = 4, kOrdCols = 4;   // warps per CTA; columns per lane per pass (a pass covers 128 columns)

// One warp per slot t: its terms are [lower_bound(t), lower_bound(t + 1)) of the sorted keys, in increasing term index (the sort is
// stable).  dst[t, j] = (((+0 + c_0 src_0[j]) + c_1 src_1[j]) + ...), each product and sum rounded on its own, stored.
__global__ void __launch_bounds__(kOrdWarps * 32) ordered_rows_kernel(
    const uint32_t* __restrict__ key, const int32_t* __restrict__ val, int64_t n, const int32_t* __restrict__ a_row,
    const float* __restrict__ a_coef, int64_t n_a, const float* __restrict__ src_a, int64_t ld_a, const float* __restrict__ src_b,
    int64_t ld_b, int32_t n_slots, int cols, float* __restrict__ dst, int64_t ld_dst) {
  const int lane = threadIdx.x & 31;
  for (int64_t t = (int64_t)blockIdx.x * kOrdWarps + (threadIdx.x >> 5); t < n_slots; t += (int64_t)gridDim.x * kOrdWarps) {
    const int64_t lo = lower_bound_u32(key, n, (uint32_t)t), hi = lower_bound_u32(key, n, (uint32_t)t + 1u);
    float* d = dst + t * ld_dst;
    for (int j0 = 0; j0 < cols; j0 += 32 * kOrdCols) {
      float acc[kOrdCols];
#pragma unroll
      for (int r = 0; r < kOrdCols; ++r) acc[r] = 0.0f;
      for (int64_t e = lo; e < hi; ++e) {
        const int64_t i = val[e];
        const float* src;
        float c;
        if (i < n_a) { src = src_a + (int64_t)a_row[i] * ld_a; c = a_coef[i]; }
        else { src = src_b + (i - n_a) * ld_b; c = 1.0f; }
#pragma unroll
        for (int r = 0; r < kOrdCols; ++r) {
          const int j = j0 + lane + 32 * r;
          if (j < cols) acc[r] = __fadd_rn(acc[r], __fmul_rn(c, src[j]));
        }
      }
#pragma unroll
      for (int r = 0; r < kOrdCols; ++r) {
        const int j = j0 + lane + 32 * r;
        if (j < cols) d[j] = acc[r];
      }
    }
  }
}

static int key_bits_for(int32_t n_slots) {   // bits of the largest key, n_slots
  int b = 1;
  while (b < 32 && ((uint32_t)n_slots >> b) != 0u) ++b;
  return b;
}

struct OrderedLayout {
  int64_t off_key_alt, off_val, off_val_alt, off_temp, temp_bytes, bytes;
};

static int64_t align256(int64_t x) { return (x + 255) / 256 * 256; }

static int ordered_layout(int64_t n, int32_t n_slots, OrderedLayout& L) {
  size_t tb = 0;
  if (n > 0) {
    cub::DoubleBuffer<uint32_t> k(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> v(nullptr, nullptr);
    DAE_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, k, v, (int)n, 0, key_bits_for(n_slots)));
  }
  const int64_t a = align256(4 * n);
  L.off_key_alt = a;
  L.off_val = 2 * a;
  L.off_val_alt = 3 * a;
  L.off_temp = 4 * a;
  L.temp_bytes = (int64_t)tb;
  L.bytes = 4 * a + align256((int64_t)tb);
  return DAE_OK;
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

extern "C" int dae_ordered_rows_workspace(int64_t n_a, int64_t n_b, int32_t n_slots, int64_t* bytes) {
  DAE_REQUIRE(bytes && n_a >= 0 && n_b >= 0 && n_a + n_b < 0x7fffffffLL && n_slots >= 1, "dae_ordered_rows_workspace: bad arguments");
  OrderedLayout L;
  const int rc = ordered_layout(n_a + n_b, n_slots, L);
  if (rc) return rc;
  *bytes = L.bytes;
  return DAE_OK;
}

extern "C" int dae_ordered_rows(const int32_t* a_slot, const int32_t* a_row, const float* a_coef, int64_t n_a, const float* src_a,
                                int64_t ld_a, const int32_t* b_slot, int64_t n_b, const float* src_b, int64_t ld_b, int32_t n_slots,
                                int32_t cols, float* dst, int64_t ld_dst, void* workspace, int64_t workspace_bytes, void* stream) {
  DAE_REQUIRE(dst && workspace && (n_a == 0 || (a_slot && a_row && a_coef && src_a)) && (n_b == 0 || (b_slot && src_b)),
              "dae_ordered_rows: null pointer");
  DAE_REQUIRE(n_a >= 0 && n_b >= 0 && n_a + n_b < 0x7fffffffLL && n_slots >= 1 && cols > 0 && ld_dst >= cols &&
              (n_a == 0 || ld_a >= cols) && (n_b == 0 || ld_b >= cols), "dae_ordered_rows: bad shape");
  DAE_REQUIRE((((uintptr_t)a_slot | (uintptr_t)a_row | (uintptr_t)a_coef | (uintptr_t)src_a | (uintptr_t)b_slot | (uintptr_t)src_b |
                (uintptr_t)dst) & 3) == 0 && ((uintptr_t)workspace & 255) == 0,
              "dae_ordered_rows: arrays must be 4-byte and the workspace 256-byte aligned");
  const int64_t n = n_a + n_b;
  OrderedLayout L;
  int rc = ordered_layout(n, n_slots, L);
  if (rc) return rc;
  DAE_REQUIRE(workspace_bytes >= L.bytes, "dae_ordered_rows: workspace of %lld bytes, need %lld", (long long)workspace_bytes,
              (long long)L.bytes);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = (uint8_t*)workspace;
  cub::DoubleBuffer<uint32_t> k((uint32_t*)w, (uint32_t*)(w + L.off_key_alt));
  cub::DoubleBuffer<int32_t> v((int32_t*)(w + L.off_val), (int32_t*)(w + L.off_val_alt));
  if (n > 0) {
    ordered_keys_kernel<<<grid_cap(n, 256), 256, 0, st>>>(a_slot, n_a, b_slot, n, n_slots, k.Current(), v.Current());
    size_t tb = (size_t)L.temp_bytes;
    DAE_CUDA(cub::DeviceRadixSort::SortPairs(w + L.off_temp, tb, k, v, (int)n, 0, key_bits_for(n_slots), st));
  }
  const int64_t blocks = ((int64_t)n_slots + kOrdWarps - 1) / kOrdWarps, cap = (int64_t)sm_count() * 16;
  ordered_rows_kernel<<<(int)(blocks < cap ? blocks : cap), kOrdWarps * 32, 0, st>>>(
      k.Current(), v.Current(), n, a_row, a_coef, n_a, src_a, ld_a, src_b, ld_b, n_slots, cols, dst, ld_dst);
  DAE_CHECK_LAUNCH("dae_ordered_rows");
  return DAE_OK;
}
