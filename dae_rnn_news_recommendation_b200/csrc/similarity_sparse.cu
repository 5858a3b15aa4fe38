// Sparse similarity + k-best selection (dae_csr_similarity_topk): for every row q of a CSR matrix Q the k rows c of a CSR matrix C
// with the largest S[q, c] = sum_f Q[q, f] C[c, f], without forming S.  The bag-of-words (binary / tf-idf) counterpart of
// dae_similarity_topk_bf16x3: a pair only costs the columns the two rows share, sum_f df_q(f) df_c(f) multiply-adds in all.
//   postings : C's entries bucketed by (range of kSpW corpus rows, column) in the workspace -- a count, an exclusive scan and an
//              atomic-cursor scatter.  A corpus row appears at most once per bucket, so the order inside a bucket is irrelevant.
//   main     : one warp per (query, split).  The warp owns a slab of kSpW fp32 accumulators in shared memory.  For each range of
//              its split it walks the query's columns in increasing order and adds v_q * v_c into slab[c - range start] for every
//              posting of the (range, column) bucket, lanes over postings (distinct rows, so no two lanes touch one slot); a
//              __syncwarp between columns keeps the per-slot order.  Then it scans the slab into its k-best list and zeroes it.
//   numerics : every pair accumulates in fp32 from 0, one term per shared column in increasing column order, each term rounded
//              (__fmul_rn, then __fadd_rn: no FMA contraction).  The scores therefore do not depend on the launch shape, and a
//              float32 host loop over the columns reproduces them bit for bit.
//   k-best   : lane j < k holds entry j of the list, ordered (score desc, index asc).  Candidates arrive in increasing corpus
//              index and only a strict > inserts, so the first of equal scores wins -- the rule of dae_similarity_topk_bf16x3.
//   splits   : with too few queries to fill the SMs the ranges are cut into `splits` groups, one warp each, and topk_merge_kernel
//              merges the partial lists.  The extra memory is the buckets ((Nc / kSpW + 1) F int32), the postings (8 B per corpus
//              entry) and, with splits > 1, the partial lists (8 B per entry): never Nq x Nc or Nq x F.
//   histogram: sp_topk_kernel<kSpHist> (dae_csr_similarity_pair_hist) bins the same scores of the strict lower triangle of Q.Q^T
//              into related / unrelated histograms instead of k-best lists.
//   pairs    : sp_topk_kernel<kSpPairs> (dae_csr_similarity_pairs) emits every slot with a score >= tau as an (i, j, s) triple, of
//              Q.C^T or of the strict lower triangle of Q.Q^T.
#include "common.cuh"
#include "pair_hist.cuh"
#include "pairs.cuh"
#include "topk.cuh"

namespace dae {
namespace {

constexpr int kSpW = 2048;                 // corpus rows per range = accumulator slab of one warp (8 KB)
constexpr int kSpWarps = 8;                // warps (queries) per CTA: 64 KB of slabs, three CTAs per SM
constexpr int kSpMaxK = 32;
constexpr int kSpMaxSplits = 32;
constexpr int kSpWarpsPerSm = 24;          // automatic splits: enough (query, split) warps for every resident warp slot
constexpr int kScanThreads = 1024, kScanPer = 8, kScanPiece = kScanThreads * kScanPer;
constexpr int64_t kScanTile = kScanPiece;  // elements per CTA of the first scan pass
constexpr unsigned kFull = 0xffffffffu;

struct SpLayout {
  int ranges, splits;
  int64_t n_bucket, n_tiles;
  int64_t off_tiles, off_post, off_val, off_idx, total;
};

int sp_splits(int n_query, int ranges, int requested) {
  int s = requested;
  if (s <= 0) s = (sm_count() * kSpWarpsPerSm + n_query - 1) / n_query;
  if (s > ranges) s = ranges;
  if (s > kSpMaxSplits) s = kSpMaxSplits;
  return s < 1 ? 1 : s;
}

int64_t align16(int64_t b) { return (b + 15) / 16 * 16; }

SpLayout sp_layout(int n_query, int n_corpus, int64_t corpus_nnz, int F, int k, int splits) {
  SpLayout L{};
  L.ranges = (n_corpus + kSpW - 1) / kSpW;
  L.splits = sp_splits(n_query, L.ranges, splits);
  L.n_bucket = (int64_t)L.ranges * F + 1;                      // + 1: the end of the last bucket (= corpus nnz)
  L.n_tiles = (L.n_bucket + kScanTile - 1) / kScanTile;
  L.off_tiles = align16(L.n_bucket * 4);
  L.off_post = L.off_tiles + align16(L.n_tiles * 4);
  L.off_val = L.off_post + align16(corpus_nnz * 8);
  const int64_t lists = L.splits > 1 ? (int64_t)n_query * L.splits * k : 0;
  L.off_idx = L.off_val + align16(lists * 4);
  L.total = L.off_idx + align16(lists * 4);
  return L;
}

// bucket[(r / kSpW) F + f] += 1 for every corpus entry (r, f): one warp per row
__global__ void sp_count_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, int rows, int F,
                                int32_t* __restrict__ bucket) {
  const int lane = threadIdx.x & 31;
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += (gridDim.x * blockDim.x) >> 5) {
    int32_t* b = bucket + (int64_t)(r / kSpW) * F;
    for (int64_t p = indptr[r] + lane; p < indptr[r + 1]; p += 32) atomicAdd(&b[indices[p]], 1);
  }
}

// inclusive scan of data[tile b] in place, one CTA per tile (8 elements per thread, warp-shuffle scans, running carry between
// pieces of 8192); tile_total[b] = the tile's sum
__global__ void __launch_bounds__(kScanThreads) sp_scan_tiles_kernel(int32_t* __restrict__ data, int64_t n, int64_t tile,
                                                                     int32_t* __restrict__ tile_total) {
  __shared__ int s[kScanPiece];
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int64_t lo = (int64_t)blockIdx.x * tile, hi = lo + tile < n ? lo + tile : n;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (int64_t base = lo; base < hi; base += kScanPiece) {
    const int m = (int)(hi - base < kScanPiece ? hi - base : kScanPiece);
    for (int i = tid; i < kScanPiece; i += kScanThreads) s[i] = (i < m) ? data[base + i] : 0;
    __syncthreads();
    int v[kScanPer], sum = 0;
#pragma unroll
    for (int j = 0; j < kScanPer; ++j) { v[j] = s[tid * kScanPer + j]; sum += v[j]; }
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(kFull, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      const int w = s_warp[lane];
      int wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(kFull, wi, o); if (lane >= o) wi += t; }
      s_warp[lane] = wi - w;   // exclusive prefix of the warp totals
    }
    __syncthreads();
    int run = s_carry + s_warp[wid] + incl - sum;
#pragma unroll
    for (int j = 0; j < kScanPer; ++j) { run += v[j]; s[tid * kScanPer + j] = run; }
    __syncthreads();
    for (int i = tid; i < m; i += kScanThreads) data[base + i] = s[i];
    if (tid == kScanThreads - 1) s_carry = run;
    __syncthreads();
  }
  if (tid == 0 && tile_total) tile_total[blockIdx.x] = s_carry;
}

// data[i] += inclusive sum of the tiles before i's tile
__global__ void sp_add_tile_offsets_kernel(int32_t* __restrict__ data, int64_t n, int64_t tile, const int32_t* __restrict__ tile_incl) {
  for (int64_t i = tile + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    data[i] += tile_incl[i / tile - 1];
}

// bucket holds inclusive ends; each entry takes the slot below its bucket's end and moves the end down, so afterwards bucket[b] is
// the start of bucket b.  post = (row - range start, value bits).
__global__ void sp_scatter_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const float* __restrict__ values,
                                  int rows, int F, int32_t* __restrict__ bucket, int2* __restrict__ post) {
  const int lane = threadIdx.x & 31;
  for (int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < rows; r += (gridDim.x * blockDim.x) >> 5) {
    const int range = r / kSpW;
    int32_t* b = bucket + (int64_t)range * F;
    for (int64_t p = indptr[r] + lane; p < indptr[r + 1]; p += 32) {
      const int pos = atomicSub(&b[indices[p]], 1) - 1;
      post[pos] = make_int2(r - range * kSpW, __float_as_int(values[p]));
    }
  }
}

struct SpParams {
  const int64_t* q_indptr;
  const int32_t* q_indices;
  const float* q_values;
  const int32_t* bucket;           // [ranges x F + 1] bucket starts
  const int2* post;
  int n_query, n_corpus, F, k, splits, ranges, exclude;
  int64_t diag_offset;
  int32_t* idx_out; float* val_out;   // splits == 1: the result
  float* ws_val; int32_t* ws_idx;     // splits > 1: [n_query x splits x k] partial lists
  // histogram mode (Q = C): labels [n_corpus] (-1 = none), grid M / bins / (2M) / bins, hist [2 x bins], sums [2]
  const int32_t* labels;
  float range, scale;
  uint32_t bins;
  unsigned long long* hist;
  double* sums;
  // pairs mode: self (Q = C: ranges below q, slots c < q), threshold, caller-zeroed counter, output slots
  int self;
  float tau;
  unsigned long long* count;
  unsigned long long capacity;
  int32_t* pair_i; int32_t* pair_j; float* pair_s;
  // kSpTopkExcl: per-query exclusion lists (CSR structure, rows sorted, no duplicates, indices in [0, n_corpus)).  Last, so the
  // fields above keep their parameter offsets in the other modes.
  const int64_t* ex_indptr; const int32_t* ex_indices;
  // kSpTopkGroups: groups[c] >= 0 is corpus row c's group label; only one row per group enters a list
  const int32_t* groups;
};

enum SpMode { kSpTopk, kSpHist, kSpPairs, kSpTopkExcl, kSpTopkGroups };

// offer (v, col) to the warp's list (lane j < k holds entry j); warp-uniform arguments
__device__ __forceinline__ void sp_offer(float v, int col, int n_corpus, int excl, int k, int lane, float& lv, int& li, float& thr) {
  if (!(v > thr) || col >= n_corpus || col == excl) return;
  const int pos = __popc(__ballot_sync(kFull, lane < k && lv >= v));   // equal scores already listed have lower indices
  const float uv = __shfl_up_sync(kFull, lv, 1);
  const int ui = __shfl_up_sync(kFull, li, 1);
  if (lane == pos) { lv = v; li = col; }
  else if (lane > pos && lane < k) { lv = uv; li = ui; }
  thr = __shfl_sync(kFull, lv, k - 1);
}

// sp_offer for a list of group representatives (lane j < k also holds entry j's group lg; the groups are distinct).  If entry
// `last` holds g, v replaces it only if it beats it, and the entries from v's position to `last` move down one lane; otherwise
// (v, col) goes through the ordinary insert.
__device__ __forceinline__ void sp_offer_group(float v, int col, const int32_t* __restrict__ groups, int n_corpus, int excl, int k,
                                               int lane, float& lv, int& li, int& lg, float& thr) {
  if (!(v > thr) || col >= n_corpus || col == excl) return;
  const int g = __ldg(groups + col);
  const unsigned same = __ballot_sync(kFull, lane < k && lg == g);
  int last = k - 1;                       // the last entry that may move
  if (same) {
    last = __ffs(same) - 1;
    if (!(v > __shfl_sync(kFull, lv, last))) return;
  }
  const int pos = __popc(__ballot_sync(kFull, lane < k && lv >= v));   // <= last: the list is sorted and lv[last] < v
  const float uv = __shfl_up_sync(kFull, lv, 1);
  const int ui = __shfl_up_sync(kFull, li, 1);
  const int ug = __shfl_up_sync(kFull, lg, 1);
  if (lane == pos) { lv = v; li = col; lg = g; }
  else if (lane > pos && lane <= last) { lv = uv; li = ui; lg = ug; }
  thr = __shfl_sync(kFull, lv, k - 1);
}

// kSpTopk: k-best lists (dae_csr_similarity_topk).  kSpHist: the related / unrelated pair histogram of Q against itself
// (dae_csr_similarity_pair_hist): the same postings, accumulation and scores, but only the ranges that start below q are
// accumulated and only slots c < q are counted -- the strict lower triangle.  The scan bins every non-zero slot (runs of equal
// (group, bin) in one red.global.add.u64); the zero slots, most of them, are only counted per group in registers and added with
// one atomic per group when the warp is done.  kSpPairs: the scan emits the slots with s >= tau (c < q in self mode, whose ranges
// stop below q as in kSpHist); a warp with any hit in a 128-slot chunk reserves its slots with one atomicAdd (pair_slots).
// kSpTopkExcl: kSpTopk, but the corpus rows in q's exclusion list are never candidates.  Before each slab scan the warp writes -inf
// into the listed slots of the range, 32 list entries per load from a cursor that only moves forward (placed by binary search at
// the split's first row); -inf never beats thr, and the scan zeroes those slots as it does the others.
// kSpTopkGroups: kSpTopkExcl (ex_indptr may be null: no lists) whose list holds the k best group representatives of the slots
// scanned (sp_offer_group); the duplicate test is one ballot over the lanes' groups.
template <SpMode MODE>
__global__ void __launch_bounds__(kSpWarps * 32, 3) sp_topk_kernel(const SpParams p) {
  constexpr bool HIST = MODE == kSpHist;
  constexpr bool EXCL = MODE == kSpTopkExcl || MODE == kSpTopkGroups;
  extern __shared__ float4 sp_smem4[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t item = (int64_t)blockIdx.x * kSpWarps + warp;
  if (item >= (int64_t)p.n_query * p.splits) return;   // whole warps only: the kernel has no block-wide barrier
  float4* slab4 = sp_smem4 + warp * (kSpW / 4);
  float* slab = reinterpret_cast<float*>(slab4);
  const int q = (int)(item / p.splits), split = (int)(item - (int64_t)q * p.splits);
  const int r0 = (int)((int64_t)split * p.ranges / p.splits);
  int r1 = (int)((int64_t)(split + 1) * p.ranges / p.splits);
  int lq = 0;
  if constexpr (HIST) {
    lq = p.labels[q];
    if (lq < 0) return;                                 // warp-uniform: a row without a label has no pairs
    r1 = min(r1, (q + kSpW - 1) / kSpW);                // ranges that start below q
  }
  if constexpr (MODE == kSpPairs) {
    if (p.self) r1 = min(r1, (q + kSpW - 1) / kSpW);
  }
  double sum_rel = 0.0, sum_unrel = 0.0;
  uint32_t zero_rel = 0, zero_unrel = 0, run_key = 0, run_n = 0;
  const int64_t qb = p.q_indptr[q], qe = p.q_indptr[q + 1];
  const int64_t e = (int64_t)q + p.diag_offset;
  const int excl = (p.exclude && e >= 0 && e < p.n_corpus) ? (int)e : -1;
  const int k = p.k;
  for (int j = lane; j < kSpW / 4; j += 32) slab4[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  float lv = neg_inf(), thr = neg_inf();
  int li = -1;
  [[maybe_unused]] int lg = -1;                      // kSpTopkGroups: the group of entry `lane`
  [[maybe_unused]] int64_t ex_cur = 0, ex_end = 0;   // EXCL: cursor into q's list and its end (warp-uniform)
  if constexpr (EXCL) if (MODE == kSpTopkExcl || p.ex_indptr) {
    int64_t lo = p.ex_indptr[q], hi = p.ex_indptr[q + 1];
    ex_end = hi;
    const int c_first = r0 * kSpW;
    while (lo < hi) {
      const int64_t mid = lo + ((hi - lo) >> 1);
      if (p.ex_indices[mid] < c_first) lo = mid + 1; else hi = mid;
    }
    ex_cur = lo;
  }
  __syncwarp();
  for (int r = r0; r < r1; ++r) {
    const int32_t* brow = p.bucket + (int64_t)r * p.F;
    // accumulate: the query's columns in increasing order, 32 at a time; lane j fetches column j's value and bucket bounds
    for (int64_t c0 = qb; c0 < qe; c0 += 32) {
      const int nc = (int)(qe - c0 < 32 ? qe - c0 : 32);
      float v = 0.f;
      int s0 = 0, s1 = 0;
      if (lane < nc) {
        const int f = p.q_indices[c0 + lane];
        v = p.q_values[c0 + lane];
        s0 = brow[f];
        s1 = brow[f + 1];                 // the next bucket's start (the last one's is the corpus nnz)
      }
      for (int j = 0; j < nc; ++j) {
        const float vj = __shfl_sync(kFull, v, j);
        const int a = __shfl_sync(kFull, s0, j), b = __shfl_sync(kFull, s1, j);
        for (int t = a + lane; t < b; t += 32) {
          const int2 pe = __ldg(p.post + t);
          slab[pe.x] = __fadd_rn(slab[pe.x], __fmul_rn(vj, __int_as_float(pe.y)));
        }
        __syncwarp();                     // a slot's next term (next column) may come from another lane
      }
    }
    const int base = r * kSpW;
    const int width = p.n_corpus - base < kSpW ? p.n_corpus - base : kSpW;
    if constexpr (HIST) {
      // bin the slots c < q, zero the whole slab for the next range
      auto count = [&](float s, int c) {
        if (c >= q) return;
        const int lc = p.labels[c];
        if (lc < 0) return;
        const bool rel = (lc == lq);
        if (s == 0.0f) { zero_rel += rel; zero_unrel += !rel; return; }
        const uint32_t key = (rel ? 0u : p.bins) + pair_bin(s, p.range, p.scale, p.bins);
        if (rel) sum_rel += (double)s; else sum_unrel += (double)s;
        if (key != run_key && run_n) { red_add_u64(p.hist + run_key, run_n); run_n = 0; }
        run_key = key;
        ++run_n;
      };
      for (int j0 = 0; j0 < width; j0 += 128) {
        const float4 x = slab4[j0 / 4 + lane];
        slab4[j0 / 4 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
        const int c = base + j0 + 4 * lane;
        count(x.x, c); count(x.y, c + 1); count(x.z, c + 2); count(x.w, c + 3);
      }
    } else if constexpr (MODE == kSpPairs) {
      // emit the slots c < lim with s >= tau (tau > 0: the slots past width, never written, stay 0), zero the slab
      const int lim = p.self ? q : p.n_corpus;
      const float tau = p.tau;
      for (int j0 = 0; j0 < width; j0 += 128) {
        const float4 x = slab4[j0 / 4 + lane];
        slab4[j0 / 4 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
        const int c = base + j0 + 4 * lane;
        const bool h0 = x.x >= tau && c < lim, h1 = x.y >= tau && c + 1 < lim;
        const bool h2 = x.z >= tau && c + 2 < lim, h3 = x.w >= tau && c + 3 < lim;
        const int hits = h0 + h1 + h2 + h3;
        if (__any_sync(kFull, hits != 0)) {
          unsigned long long slot = pair_slots(p.count, hits);
          if (h0) pair_put(slot++, p.capacity, q, c, x.x, p.pair_i, p.pair_j, p.pair_s);
          if (h1) pair_put(slot++, p.capacity, q, c + 1, x.y, p.pair_i, p.pair_j, p.pair_s);
          if (h2) pair_put(slot++, p.capacity, q, c + 2, x.z, p.pair_i, p.pair_j, p.pair_s);
          if (h3) pair_put(slot, p.capacity, q, c + 3, x.w, p.pair_i, p.pair_j, p.pair_s);
        }
      }
    } else {
      if constexpr (EXCL) {
        // -inf into the listed slots of this range; the list is sorted, so the lanes below the range's end form a prefix
        while (ex_cur < ex_end) {
          const int c = (ex_cur + lane < ex_end) ? p.ex_indices[ex_cur + lane] : INT_MAX;
          const bool in = c < base + kSpW;
          if (in) slab[c - base] = neg_inf();
          const int n_in = __popc(__ballot_sync(kFull, in));
          ex_cur += n_in;
          if (n_in < 32) break;
        }
        __syncwarp();
      }
      // scan the slab in increasing corpus index (lane-major float4s), offer what beats the k-th score, zero it for the next range
      for (int j0 = 0; j0 < width; j0 += 128) {
        const float4 x = slab4[j0 / 4 + lane];
        slab4[j0 / 4 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
        unsigned mask = __ballot_sync(kFull, fmaxf(fmaxf(x.x, x.y), fmaxf(x.z, x.w)) > thr);
        while (mask) {
          const int l = __ffs(mask) - 1;
          mask &= mask - 1;
          const float y0 = __shfl_sync(kFull, x.x, l), y1 = __shfl_sync(kFull, x.y, l);
          const float y2 = __shfl_sync(kFull, x.z, l), y3 = __shfl_sync(kFull, x.w, l);
          const int c = base + j0 + 4 * l;
          if constexpr (MODE == kSpTopkGroups) {
            sp_offer_group(y0, c, p.groups, p.n_corpus, excl, k, lane, lv, li, lg, thr);
            sp_offer_group(y1, c + 1, p.groups, p.n_corpus, excl, k, lane, lv, li, lg, thr);
            sp_offer_group(y2, c + 2, p.groups, p.n_corpus, excl, k, lane, lv, li, lg, thr);
            sp_offer_group(y3, c + 3, p.groups, p.n_corpus, excl, k, lane, lv, li, lg, thr);
          } else {
            sp_offer(y0, c, p.n_corpus, excl, k, lane, lv, li, thr);
            sp_offer(y1, c + 1, p.n_corpus, excl, k, lane, lv, li, thr);
            sp_offer(y2, c + 2, p.n_corpus, excl, k, lane, lv, li, thr);
            sp_offer(y3, c + 3, p.n_corpus, excl, k, lane, lv, li, thr);
          }
        }
      }
    }
    __syncwarp();
  }
  if constexpr (HIST) {
    if (run_n) red_add_u64(p.hist + run_key, run_n);
    zero_rel = __reduce_add_sync(kFull, zero_rel);
    zero_unrel = __reduce_add_sync(kFull, zero_unrel);
    sum_rel = warp_sum(sum_rel);
    sum_unrel = warp_sum(sum_unrel);
    if (lane == 0) {
      const uint32_t zb = pair_bin(0.0f, p.range, p.scale, p.bins);
      if (zero_rel) red_add_u64(p.hist + zb, zero_rel);
      if (zero_unrel) red_add_u64(p.hist + p.bins + zb, zero_unrel);
      if (sum_rel != 0.0) atomicAdd(p.sums, sum_rel);
      if (sum_unrel != 0.0) atomicAdd(p.sums + 1, sum_unrel);
    }
    return;
  }
  if constexpr (MODE == kSpPairs) return;
  if (lane < k) {
    if (p.splits == 1) {
      p.idx_out[(int64_t)q * k + lane] = li;
      p.val_out[(int64_t)q * k + lane] = lv;
    } else {
      const int64_t o = ((int64_t)q * p.splits + split) * k + lane;
      p.ws_val[o] = lv;
      p.ws_idx[o] = li;
    }
  }
}

}  // namespace

// corpus postings bucketed by (range, column) into the workspace (layout L)
static int sp_postings(const SpLayout& L, const int64_t* c_indptr, const int32_t* c_indices, const float* c_values, int n_corpus,
                       int F, uint8_t* ws, cudaStream_t st) {
  int32_t* bucket = reinterpret_cast<int32_t*>(ws);
  int32_t* tiles = reinterpret_cast<int32_t*>(ws + L.off_tiles);
  int2* post = reinterpret_cast<int2*>(ws + L.off_post);
  DAE_CUDA(cudaMemsetAsync(bucket, 0, (size_t)L.n_bucket * 4, st));
  const int row_blocks = (int)((n_corpus + 7) / 8 < sm_count() * 16 ? (n_corpus + 7) / 8 : sm_count() * 16);
  sp_count_kernel<<<row_blocks, 256, 0, st>>>(c_indptr, c_indices, n_corpus, F, bucket);
  sp_scan_tiles_kernel<<<(unsigned)L.n_tiles, kScanThreads, 0, st>>>(bucket, L.n_bucket, kScanTile, tiles);
  if (L.n_tiles > 1) {
    sp_scan_tiles_kernel<<<1, kScanThreads, 0, st>>>(tiles, L.n_tiles, L.n_tiles, nullptr);
    const int64_t rest = L.n_bucket - kScanTile;
    const int blocks = (int)((rest + 255) / 256 < sm_count() * 16 ? (rest + 255) / 256 : sm_count() * 16);
    sp_add_tile_offsets_kernel<<<blocks, 256, 0, st>>>(bucket, L.n_bucket, kScanTile, tiles);
  }
  sp_scatter_kernel<<<row_blocks, 256, 0, st>>>(c_indptr, c_indices, c_values, n_corpus, F, bucket, post);
  DAE_CHECK_LAUNCH("sparse similarity (postings)");
  return DAE_OK;
}

template <SpMode MODE>
static int sp_launch(const SpParams& sp, cudaStream_t st) {
  constexpr int smem = kSpWarps * kSpW * 4;
  static bool attr_done[64] = {false};
  int dev = 0;
  DAE_CUDA(cudaGetDevice(&dev));
  if (dev >= 0 && dev < 64 && !attr_done[dev]) {
    DAE_CUDA(cudaFuncSetAttribute(sp_topk_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_done[dev] = true;
  }
  const int64_t warps = (int64_t)sp.n_query * sp.splits;
  sp_topk_kernel<MODE><<<(unsigned)((warps + kSpWarps - 1) / kSpWarps), kSpWarps * 32, smem, st>>>(sp);
  return DAE_OK;
}

}  // namespace dae

using namespace dae;

extern "C" int dae_csr_similarity_topk_workspace(int32_t n_query, int32_t n_corpus, int64_t corpus_nnz, int32_t n_features, int32_t k,
                                                 int32_t splits, int64_t* bytes) {
  DAE_REQUIRE(bytes && n_query > 0 && n_corpus > 0 && n_features > 0 && corpus_nnz >= 0 && corpus_nnz < INT32_MAX,
              "dae_csr_similarity_topk_workspace: bad arguments");
  DAE_REQUIRE(k >= 1 && k <= kSpMaxK, "dae_csr_similarity_topk_workspace: k = %d is outside the supported range 1 <= k <= %d", k, kSpMaxK);
  *bytes = sp_layout(n_query, n_corpus, corpus_nnz, n_features, k, splits).total;
  return DAE_OK;
}

// dae_csr_similarity_topk (excl false), dae_csr_similarity_topk_excl (excl true, the lists ex_indptr / ex_indices) and
// dae_csr_similarity_topk_groups (excl true, groups non-null; ex_indptr may be null when ex_nnz = 0: no lists)
static int csr_topk(const char* fn, const int64_t* q_indptr, const int32_t* q_indices, const float* q_values, int32_t n_query,
                    int64_t q_nnz, int32_t q_features, const int64_t* c_indptr, const int32_t* c_indices, const float* c_values,
                    int32_t n_corpus, int64_t c_nnz, int32_t c_features, int32_t k, int64_t diag_offset, int32_t exclude,
                    int32_t splits, void* workspace, int64_t workspace_bytes, int32_t* idx_out, float* val_out, bool excl,
                    const int64_t* ex_indptr, const int32_t* ex_indices, int64_t ex_nnz, const int32_t* groups, bool grouped,
                    void* stream) {
  DAE_REQUIRE(q_indptr && c_indptr && workspace && idx_out && val_out && (q_nnz == 0 || (q_indices && q_values)) &&
              (c_nnz == 0 || (c_indices && c_values)) &&
              (!excl || (grouped ? (groups && (ex_nnz == 0 || (ex_indptr && ex_indices))) : (ex_indptr && (ex_nnz == 0 || ex_indices)))),
              "%s: null pointer", fn);
  DAE_REQUIRE(n_query > 0 && n_corpus > 0 && q_features > 0 && c_features > 0 && q_nnz >= 0 && c_nnz >= 0 && c_nnz < INT32_MAX &&
              (!excl || ex_nnz >= 0), "%s: bad sizes", fn);
  DAE_REQUIRE(k >= 1 && k <= kSpMaxK, "%s: k = %d is outside the supported range 1 <= k <= %d", fn, k, kSpMaxK);
  DAE_REQUIRE(q_features == c_features, "%s: queries have %d features, the corpus %d", fn, q_features, c_features);
  DAE_REQUIRE((uintptr_t)workspace % 16 == 0, "%s: workspace must be 16-byte aligned", fn);
  DAE_REQUIRE(!excl || ((uintptr_t)ex_indptr % 8 == 0 && (uintptr_t)ex_indices % 4 == 0),
              "%s: ex_indptr must be 8-byte, ex_indices 4-byte aligned", fn);
  DAE_REQUIRE((uintptr_t)groups % 4 == 0, "%s: groups must be 4-byte aligned", fn);
  const SpLayout L = sp_layout(n_query, n_corpus, c_nnz, c_features, k, splits);
  DAE_REQUIRE(workspace_bytes >= L.total, "%s: workspace of %lld bytes, %lld needed (dae_csr_similarity_topk_workspace)", fn,
              (long long)workspace_bytes, (long long)L.total);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  int32_t* bucket = reinterpret_cast<int32_t*>(ws);
  int2* post = reinterpret_cast<int2*>(ws + L.off_post);
  const int F = c_features;
  int rc = sp_postings(L, c_indptr, c_indices, c_values, n_corpus, F, ws, st);
  if (rc) return rc;

  SpParams sp{};
  sp.q_indptr = q_indptr; sp.q_indices = q_indices; sp.q_values = q_values; sp.bucket = bucket; sp.post = post;
  sp.n_query = n_query; sp.n_corpus = n_corpus; sp.F = F; sp.k = k; sp.splits = L.splits; sp.ranges = L.ranges;
  sp.exclude = exclude ? 1 : 0; sp.diag_offset = diag_offset;
  sp.idx_out = idx_out; sp.val_out = val_out;
  sp.ws_val = reinterpret_cast<float*>(ws + L.off_val);
  sp.ws_idx = reinterpret_cast<int32_t*>(ws + L.off_idx);
  sp.ex_indptr = ex_indptr; sp.ex_indices = ex_indices; sp.groups = groups;
  if ((rc = grouped ? sp_launch<kSpTopkGroups>(sp, st) : excl ? sp_launch<kSpTopkExcl>(sp, st) : sp_launch<kSpTopk>(sp, st))) return rc;
  DAE_CHECK_LAUNCH(fn);
  if (L.splits > 1) {
    if (grouped)
      topk_merge_groups_kernel<<<(n_query + 7) / 8, 256, 0, st>>>(sp.ws_val, sp.ws_idx, groups, n_query, L.splits, k, idx_out, val_out);
    else
      topk_merge_kernel<<<(n_query + 7) / 8, 256, 0, st>>>(sp.ws_val, sp.ws_idx, n_query, L.splits, k, idx_out, val_out);
    DAE_CHECK_LAUNCH("sparse similarity top-k (merge)");
  }
  return DAE_OK;
}

extern "C" int dae_csr_similarity_topk(const int64_t* q_indptr, const int32_t* q_indices, const float* q_values, int32_t n_query,
                                       int64_t q_nnz, int32_t q_features, const int64_t* c_indptr, const int32_t* c_indices,
                                       const float* c_values, int32_t n_corpus, int64_t c_nnz, int32_t c_features, int32_t k,
                                       int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace, int64_t workspace_bytes,
                                       int32_t* idx_out, float* val_out, void* stream) {
  return csr_topk("dae_csr_similarity_topk", q_indptr, q_indices, q_values, n_query, q_nnz, q_features, c_indptr, c_indices, c_values,
                  n_corpus, c_nnz, c_features, k, diag_offset, exclude, splits, workspace, workspace_bytes, idx_out, val_out, false,
                  nullptr, nullptr, 0, nullptr, false, stream);
}

extern "C" int dae_csr_similarity_topk_excl(const int64_t* q_indptr, const int32_t* q_indices, const float* q_values, int32_t n_query,
                                            int64_t q_nnz, int32_t q_features, const int64_t* c_indptr, const int32_t* c_indices,
                                            const float* c_values, int32_t n_corpus, int64_t c_nnz, int32_t c_features, int32_t k,
                                            int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace,
                                            int64_t workspace_bytes, int32_t* idx_out, float* val_out, const int64_t* ex_indptr,
                                            const int32_t* ex_indices, int64_t ex_nnz, void* stream) {
  return csr_topk("dae_csr_similarity_topk_excl", q_indptr, q_indices, q_values, n_query, q_nnz, q_features, c_indptr, c_indices,
                  c_values, n_corpus, c_nnz, c_features, k, diag_offset, exclude, splits, workspace, workspace_bytes, idx_out, val_out,
                  true, ex_indptr, ex_indices, ex_nnz, nullptr, false, stream);
}

extern "C" int dae_csr_similarity_topk_groups(const int64_t* q_indptr, const int32_t* q_indices, const float* q_values, int32_t n_query,
                                              int64_t q_nnz, int32_t q_features, const int64_t* c_indptr, const int32_t* c_indices,
                                              const float* c_values, int32_t n_corpus, int64_t c_nnz, int32_t c_features, int32_t k,
                                              int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace,
                                              int64_t workspace_bytes, int32_t* idx_out, float* val_out, const int64_t* ex_indptr,
                                              const int32_t* ex_indices, int64_t ex_nnz, const int32_t* groups, void* stream) {
  return csr_topk("dae_csr_similarity_topk_groups", q_indptr, q_indices, q_values, n_query, q_nnz, q_features, c_indptr, c_indices,
                  c_values, n_corpus, c_nnz, c_features, k, diag_offset, exclude, splits, workspace, workspace_bytes, idx_out, val_out,
                  true, ex_indptr, ex_indices, ex_nnz, groups, true, stream);
}

extern "C" int dae_csr_similarity_pair_hist_workspace(int32_t n, int64_t nnz, int32_t n_features, int64_t* bytes) {
  DAE_REQUIRE(bytes && n >= 2 && n_features > 0 && nnz >= 0 && nnz < INT32_MAX, "dae_csr_similarity_pair_hist_workspace: bad arguments");
  *bytes = sp_layout(n, n, nnz, n_features, 0, 0).total;
  return DAE_OK;
}

extern "C" int dae_csr_similarity_pair_hist(const int64_t* indptr, const int32_t* indices, const float* values, int32_t n, int64_t nnz,
                                            int32_t n_features, const int32_t* labels, float range, int32_t bins, void* workspace,
                                            int64_t workspace_bytes, uint64_t* hist, double* sums, void* stream) {
  DAE_REQUIRE(indptr && labels && workspace && hist && sums && (nnz == 0 || (indices && values)),
              "dae_csr_similarity_pair_hist: null pointer");
  DAE_REQUIRE(n >= 2 && n_features > 0 && nnz >= 0 && nnz < INT32_MAX,
              "dae_csr_similarity_pair_hist: bad sizes (n = %d >= 2 rows, features > 0 and 0 <= nnz < 2^31 needed)", n);
  DAE_REQUIRE(hist_bins_ok(bins), "dae_csr_similarity_pair_hist: bins = %d is not a power of two in [2^%d, 2^%d]", bins,
              kHistMinLog2Bins, kHistMaxLog2Bins);
  DAE_REQUIRE(hist_range_ok(range), "dae_csr_similarity_pair_hist: range M = %g is not a power of two in [2^-64, 2^64]", (double)range);
  DAE_REQUIRE((uintptr_t)workspace % 16 == 0 && ((uintptr_t)hist | (uintptr_t)sums) % 8 == 0,
              "dae_csr_similarity_pair_hist: workspace must be 16-byte, hist and sums 8-byte aligned");
  const SpLayout L = sp_layout(n, n, nnz, n_features, 0, 0);
  DAE_REQUIRE(workspace_bytes >= L.total,
              "dae_csr_similarity_pair_hist: workspace of %lld bytes, %lld needed (dae_csr_similarity_pair_hist_workspace)",
              (long long)workspace_bytes, (long long)L.total);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  int rc = sp_postings(L, indptr, indices, values, n, n_features, ws, st);
  if (rc) return rc;
  SpParams sp{};
  sp.q_indptr = indptr; sp.q_indices = indices; sp.q_values = values;
  sp.bucket = reinterpret_cast<int32_t*>(ws); sp.post = reinterpret_cast<int2*>(ws + L.off_post);
  sp.n_query = n; sp.n_corpus = n; sp.F = n_features; sp.k = 1; sp.splits = L.splits; sp.ranges = L.ranges; sp.exclude = 0;
  sp.labels = labels; sp.range = range; sp.scale = (float)bins / (2.0f * range); sp.bins = (uint32_t)bins;
  sp.hist = reinterpret_cast<unsigned long long*>(hist); sp.sums = sums;
  if ((rc = sp_launch<kSpHist>(sp, st))) return rc;
  DAE_CHECK_LAUNCH("dae_csr_similarity_pair_hist");
  return DAE_OK;
}

extern "C" int dae_csr_similarity_pairs_workspace(int32_t n_query, int32_t n_corpus, int64_t corpus_nnz, int32_t n_features, int64_t* bytes) {
  DAE_REQUIRE(bytes && n_query > 0 && n_corpus > 0 && n_features > 0 && corpus_nnz >= 0 && corpus_nnz < INT32_MAX,
              "dae_csr_similarity_pairs_workspace: bad arguments");
  *bytes = sp_layout(n_query, n_corpus, corpus_nnz, n_features, 0, 0).total;
  return DAE_OK;
}

extern "C" int dae_csr_similarity_pairs(const int64_t* q_indptr, const int32_t* q_indices, const float* q_values, int32_t n_query,
                                        int64_t q_nnz, int32_t q_features, const int64_t* c_indptr, const int32_t* c_indices,
                                        const float* c_values, int32_t n_corpus, int64_t c_nnz, int32_t c_features, int32_t self,
                                        float threshold, void* workspace, int64_t workspace_bytes, uint64_t* count, int64_t capacity,
                                        int32_t* i_out, int32_t* j_out, float* s_out, void* stream) {
  DAE_REQUIRE(q_indptr && c_indptr && workspace && count && (q_nnz == 0 || (q_indices && q_values)) &&
              (c_nnz == 0 || (c_indices && c_values)), "dae_csr_similarity_pairs: null pointer");
  DAE_REQUIRE(capacity >= 0, "dae_csr_similarity_pairs: capacity = %lld < 0", (long long)capacity);
  DAE_REQUIRE(capacity == 0 || (i_out && j_out && s_out), "dae_csr_similarity_pairs: null output with capacity %lld > 0",
              (long long)capacity);
  DAE_REQUIRE(n_query > 0 && n_corpus > 0 && q_features > 0 && c_features > 0 && q_nnz >= 0 && c_nnz >= 0 && c_nnz < INT32_MAX,
              "dae_csr_similarity_pairs: bad sizes");
  DAE_REQUIRE(q_features == c_features, "dae_csr_similarity_pairs: queries have %d features, the corpus %d", q_features, c_features);
  DAE_REQUIRE(!self || (n_query == n_corpus && q_nnz == c_nnz && q_indptr == c_indptr && q_indices == c_indices && q_values == c_values),
              "dae_csr_similarity_pairs: self mode needs the corpus matrix to be the query matrix");
  DAE_REQUIRE(threshold > 0.0f && pair_threshold_ok(threshold),
              "dae_csr_similarity_pairs: threshold %g must be finite and > 0 (a pair sharing no column scores 0)", (double)threshold);
  DAE_REQUIRE((uintptr_t)workspace % 16 == 0 && (uintptr_t)count % 8 == 0 && ((uintptr_t)i_out | (uintptr_t)j_out | (uintptr_t)s_out) % 4 == 0,
              "dae_csr_similarity_pairs: workspace must be 16-byte, the counter 8-byte and the outputs 4-byte aligned");
  const SpLayout L = sp_layout(n_query, n_corpus, c_nnz, c_features, 0, 0);
  DAE_REQUIRE(workspace_bytes >= L.total, "dae_csr_similarity_pairs: workspace of %lld bytes, %lld needed (dae_csr_similarity_pairs_workspace)",
              (long long)workspace_bytes, (long long)L.total);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  int rc = sp_postings(L, c_indptr, c_indices, c_values, n_corpus, c_features, ws, st);
  if (rc) return rc;
  SpParams sp{};
  sp.q_indptr = q_indptr; sp.q_indices = q_indices; sp.q_values = q_values;
  sp.bucket = reinterpret_cast<int32_t*>(ws); sp.post = reinterpret_cast<int2*>(ws + L.off_post);
  sp.n_query = n_query; sp.n_corpus = n_corpus; sp.F = c_features; sp.k = 1; sp.splits = L.splits; sp.ranges = L.ranges; sp.exclude = 0;
  sp.self = self ? 1 : 0; sp.tau = threshold;
  sp.count = reinterpret_cast<unsigned long long*>(count); sp.capacity = (unsigned long long)capacity;
  sp.pair_i = i_out; sp.pair_j = j_out; sp.pair_s = s_out;
  if ((rc = sp_launch<kSpPairs>(sp, st))) return rc;
  DAE_CHECK_LAUNCH("dae_csr_similarity_pairs");
  return DAE_OK;
}
