// K1 (CSR x dense encode forward) and K5 (encode backward) for sm_90a.
//
// Reference ops replaced: tf.sparse.matmul(x_corr, W) + bh, f(.) - f(bh)  (autoencoder/autoencoder.py:377,389)
// and their autodiff (dense F x H dW from sparse_tensor_dense_matmul's adjoint).
//
// Layout: one CTA (128 threads) per batch row.  The row's (col,val) pairs are staged through shared memory in
// chunks of 128 with masked (zero) entries compacted away, then every thread gathers its 128-bit slice of W[col,:]
// with read-only vector loads, several rows of W in flight per thread.  W (20 MB at F=10k,H=500) is L2 resident,
// so the gather runs at L2 bandwidth; HBM only sees the CSR stream, W once, and the E write.
#include <algorithm>
#include <cstdlib>
#include <cuda_bf16.h>
#include "common.cuh"

namespace dae {

template <int VW> struct Vec;
template <> struct Vec<4> { using T = float4; };
template <> struct Vec<2> { using T = float2; };
template <> struct Vec<1> { using T = float; };

template <int VW>
__device__ __forceinline__ void ldg_vec(const float* p, float (&out)[VW]) {
  if constexpr (VW == 4) { const float4 v = __ldg(reinterpret_cast<const float4*>(p)); out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w; }
  else if constexpr (VW == 2) { const float2 v = __ldg(reinterpret_cast<const float2*>(p)); out[0] = v.x; out[1] = v.y; }
  else { out[0] = __ldg(p); }
}

constexpr int kEncThreads = 128;

// stage up to NT (= CTA size) (col,val) pairs of the row into smem, dropping zeros; returns the number kept.
template <int NT = 128>
__device__ __forceinline__ int stage_row_chunk(const int32_t* __restrict__ indices, const float* __restrict__ values,
                                               int64_t base, int64_t p1, float in_scale, int* s_col, float* s_val,
                                               int* s_wcnt) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int64_t p = base + tid;
  float v = 0.0f;
  int c = 0;
  if (p < p1) { v = __ldg(values + p) * in_scale; c = __ldg(indices + p); }
  const bool keep = (v != 0.0f);
  const unsigned m = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) s_wcnt[w] = __popc(m);
  __syncthreads();
  int off = 0, total = 0;
#pragma unroll
  for (int i = 0; i < NT / 32; ++i) { const int n = s_wcnt[i]; if (i < w) off += n; total += n; }
  if (keep) { const int pos = off + __popc(m & ((1u << lane) - 1u)); s_col[pos] = c; s_val[pos] = v; }
  __syncthreads();
  return total;
}

// One CTA per row, G groups of 128 threads.  A group owns a full copy of the row's H accumulators and takes every G-th staged
// entry, so a row has G x 8 W-row loads in flight: the kernel is bound by the LATENCY of the longest row of the batch (all rows
// are resident at once), not by bandwidth -- real text has rows 10x the mean (UCI: mean 155 words, batch maximum ~1000).
// The group partial sums are combined through shared memory and group 0 applies the epilogue.
template <int ACT, int VW, int NC, int G>
__global__ void __launch_bounds__(kEncThreads * G) encode_fwd_kernel(
    const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const float* __restrict__ values,
    const int32_t* __restrict__ rows, int H, float in_scale, const float* __restrict__ W, const float* __restrict__ bh,
    float* __restrict__ E, int64_t ldE, int32_t* __restrict__ col_count, __nv_bfloat16* __restrict__ e_hi,
    __nv_bfloat16* __restrict__ e_lo, int64_t ld_split) {
  constexpr int NT = kEncThreads * G;
  __shared__ int s_col[NT];
  __shared__ float s_val[NT];
  __shared__ int s_wcnt[NT / 32];
  __shared__ float s_red[(G > 1 ? G - 1 : 1) * kEncThreads * VW];
  const int tid = threadIdx.x;
  const int grp = tid / kEncThreads, gt = tid % kEncThreads;   // group, thread inside the group
  const int r = blockIdx.x;
  const int64_t row = rows ? (int64_t)rows[r] : (int64_t)r;
  const int64_t p0 = indptr[row], p1 = indptr[row + 1];

  float acc[NC][VW];
  int hcol[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    hcol[c] = (gt + c * kEncThreads) * VW;
#pragma unroll
    for (int e = 0; e < VW; ++e) acc[c][e] = 0.0f;
  }

  for (int64_t base = p0; base < p1; base += NT) {
    const int total = stage_row_chunk<NT>(indices, values, base, p1, in_scale, s_col, s_val, s_wcnt);
    if (col_count != nullptr && tid < total) atomicAdd(col_count + s_col[tid], 1);  // per-column entry counts for the backward gather
#pragma unroll 8
    for (int q = grp; q < total; q += G) {
      const float v = s_val[q];
      const float* wrow = W + (int64_t)s_col[q] * H;
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        if (hcol[c] < H) {
          float w[VW];
          ldg_vec<VW>(wrow + hcol[c], w);
#pragma unroll
          for (int e = 0; e < VW; ++e) acc[c][e] = fmaf(v, w[e], acc[c][e]);
        }
      }
    }
    __syncthreads();
  }
  if constexpr (G > 1) {   // fixed summation order (group 0 + 1 + 2 + ...): results do not depend on scheduling
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      if (grp > 0) {
#pragma unroll
        for (int e = 0; e < VW; ++e) s_red[((grp - 1) * kEncThreads + gt) * VW + e] = acc[c][e];
      }
      __syncthreads();
      if (grp == 0) {
#pragma unroll
        for (int g = 1; g < G; ++g) {
#pragma unroll
          for (int e = 0; e < VW; ++e) acc[c][e] += s_red[((g - 1) * kEncThreads + gt) * VW + e];
        }
      }
      __syncthreads();
    }
    if (grp != 0) return;
  }
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    if (hcol[c] < H) {
#pragma unroll
      for (int e = 0; e < VW; ++e) {
        const float b = __ldg(bh + hcol[c] + e);
        const float ev = act_fwd<ACT>(acc[c][e] + b) - act_fwd<ACT>(b);
        E[(int64_t)r * ldE + hcol[c] + e] = ev;
        if (e_hi != nullptr) {  // bf16 hi/lo operand copy for the tensor-core contractions (fuses dae_split_bf16 of E)
          const __nv_bfloat16 h = __float2bfloat16_rn(ev);
          e_hi[(int64_t)r * ld_split + hcol[c] + e] = h;
          e_lo[(int64_t)r * ld_split + hcol[c] + e] = __float2bfloat16_rn(ev - __bfloat162float(h));
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// transform-sized K1: persistent CTAs that keep the HOT rows of W in shared memory.
//
// Word frequencies are Zipfian: a few hundred columns carry about half of all stored entries.  The row-gather kernel above pulls
// every W row (2 kB at H = 500) through L2 -> L1 for every entry -- 20 GB per 100 k articles, 66x the algorithmic bytes, and the
// L2 -> L1 fill path is what it saturates.  Here each CTA (one per SM, 4 row groups of 128 threads) first stages the K most frequent
// rows of W into its shared memory with 1-D bulk-TMA copies (cp.async.bulk, one contiguous W row per copy, completion on an
// mbarrier) and then serves entries of those columns from shared memory; only the cold tail still gathers from L2.
// hot_slot[col] = slot of the column in the staged set, or -1.
// ---------------------------------------------------------------------------------------------------------------------

__device__ __forceinline__ uint32_t enc_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <int ACT, int NC, int kHotGroups>
__global__ void __launch_bounds__(kEncThreads * kHotGroups) encode_fwd_hot_kernel(
    const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const float* __restrict__ values, int n_rows, int H,
    float in_scale, const float* __restrict__ W, const float* __restrict__ bh, float* __restrict__ E, int64_t ldE,
    const int32_t* __restrict__ hot_cols, const int32_t* __restrict__ hot_slot, int K) {
  extern __shared__ __align__(16) uint8_t enc_smem[];
  float* s_w = reinterpret_cast<float*>(enc_smem);                       // [K][H] staged rows of W
  __shared__ int s_col[kHotGroups][kEncThreads];
  __shared__ int s_slot[kHotGroups][kEncThreads];
  __shared__ float s_val[kHotGroups][kEncThreads];
  __shared__ __align__(8) uint64_t s_bar;
  const int tid = threadIdx.x, grp = tid / kEncThreads, gt = tid % kEncThreads;
  const uint32_t bar = enc_smem_u32(&s_bar);
  const uint32_t row_bytes = (uint32_t)H * 4u;
  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(row_bytes * (uint32_t)K) : "memory");
  __syncthreads();
  for (int k = tid; k < K; k += blockDim.x) {   // one bulk copy per hot row: 2 kB contiguous in W, contiguous in shared memory
    const float* src = W + (int64_t)hot_cols[k] * H;
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(enc_smem_u32(s_w + (int64_t)k * H)),
                 "l"(src), "r"(row_bytes), "r"(bar)
                 : "memory");
  }
  {  // everybody waits for the staged rows (phase 0 of the barrier)
    uint32_t ok = 0;
    while (!ok) {
      asm volatile(
          "{\n"
          ".reg .pred p;\n"
          "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n"
          "selp.u32 %0, 1, 0, p;\n"
          "}\n"
          : "=r"(ok)
          : "r"(bar)
          : "memory");
    }
  }
  int hcol[NC];
  float fb[NC][4];
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    hcol[c] = (gt + c * kEncThreads) * 4;
#pragma unroll
    for (int e = 0; e < 4; ++e) fb[c][e] = (hcol[c] < H) ? __ldg(bh + hcol[c] + e) : 0.0f;
  }
  for (int r = blockIdx.x * kHotGroups + grp; r < n_rows; r += gridDim.x * kHotGroups) {
    const int64_t p0 = indptr[r], p1 = indptr[r + 1];
    float acc[NC][4];
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[c][e] = 0.0f;
    for (int64_t base = p0; base < p1; base += kEncThreads) {
      const int64_t p = base + gt;
      int col = 0, slot = -1;
      float v = 0.0f;
      if (p < p1) { col = __ldg(indices + p); v = __ldg(values + p) * in_scale; slot = __ldg(hot_slot + col); }
      s_col[grp][gt] = col; s_slot[grp][gt] = slot; s_val[grp][gt] = v;
      asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "n"(kEncThreads) : "memory");   // the group's 128 threads
      const int cnt = (int)((p1 - base < (int64_t)kEncThreads) ? (p1 - base) : (int64_t)kEncThreads);
#pragma unroll 8
      for (int q = 0; q < cnt; ++q) {
        const float vq = s_val[grp][q];
        const int sq = s_slot[grp][q];                 // uniform over the group: no divergence
        // ONE generic-address load serves both cases (shared-memory window or global): no branch in the loop body, so the
        // unrolled iterations keep 8 independent loads in flight per thread exactly like the row kernel
        const float* src = (sq >= 0) ? (s_w + (int64_t)sq * H) : (W + (int64_t)s_col[grp][q] * H);
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          if (hcol[c] < H) {
            const float4 w = *reinterpret_cast<const float4*>(src + hcol[c]);
            acc[c][0] = fmaf(vq, w.x, acc[c][0]); acc[c][1] = fmaf(vq, w.y, acc[c][1]);
            acc[c][2] = fmaf(vq, w.z, acc[c][2]); acc[c][3] = fmaf(vq, w.w, acc[c][3]);
          }
        }
      }
      asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "n"(kEncThreads) : "memory");
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      if (hcol[c] < H) {
        float4 o;
        o.x = act_fwd<ACT>(acc[c][0] + fb[c][0]) - act_fwd<ACT>(fb[c][0]);
        o.y = act_fwd<ACT>(acc[c][1] + fb[c][1]) - act_fwd<ACT>(fb[c][1]);
        o.z = act_fwd<ACT>(acc[c][2] + fb[c][2]) - act_fwd<ACT>(fb[c][2]);
        o.w = act_fwd<ACT>(acc[c][3] + fb[c][3]) - act_fwd<ACT>(fb[c][3]);
        *reinterpret_cast<float4*>(E + (int64_t)r * ldE + hcol[c]) = o;
      }
    }
  }
}

// backward: dA = dE * f'(A) (A recovered from E + f(bh)), dbh += dA - f'(bh) dE, dW[col,:] += val * dA
template <int ACT, int VW, int NC>
__global__ void __launch_bounds__(kEncThreads) encode_bwd_kernel(
    const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const float* __restrict__ values,
    const int32_t* __restrict__ rows, int H, float in_scale, const float* __restrict__ E, const float* __restrict__ bh,
    float* __restrict__ dE, const float* __restrict__ dE_add, int64_t ldE, float* __restrict__ dW, float* __restrict__ dbh) {
  __shared__ int s_col[kEncThreads];
  __shared__ float s_val[kEncThreads];
  __shared__ int s_wcnt[kEncThreads / 32];
  const int tid = threadIdx.x;
  const int r = blockIdx.x;
  const int64_t row = rows ? (int64_t)rows[r] : (int64_t)r;
  const int64_t p0 = indptr[row], p1 = indptr[row + 1];

  float dA[NC][VW];
  int hcol[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    hcol[c] = (tid + c * kEncThreads) * VW;
#pragma unroll
    for (int e = 0; e < VW; ++e) {
      dA[c][e] = 0.0f;
      const int h = hcol[c] + e;
      if (hcol[c] < H) {
        const float b = __ldg(bh + h);
        const float fb = act_fwd<ACT>(b);
        const float fa = E[(int64_t)r * ldE + h] + fb;
        const float de = dE[(int64_t)r * ldE + h] + (dE_add ? dE_add[(int64_t)r * ldE + h] : 0.0f);
        const float da = de * act_grad_from_y<ACT>(fa);
        dA[c][e] = da;
        dE[(int64_t)r * ldE + h] = da;
        atomicAdd(dbh + h, da - act_grad_from_y<ACT>(fb) * de);
      }
    }
  }
  for (int64_t base = p0; base < p1; base += kEncThreads) {
    const int total = stage_row_chunk(indices, values, base, p1, in_scale, s_col, s_val, s_wcnt);
    for (int q = 0; q < total; ++q) {
      const float v = s_val[q];
      float* wrow = dW + (int64_t)s_col[q] * H;
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        if (hcol[c] < H) {
          if constexpr (VW == 4) {
            atomicAdd(reinterpret_cast<float4*>(wrow + hcol[c]),
                      make_float4(v * dA[c][0], v * dA[c][1], v * dA[c][2], v * dA[c][3]));
          } else if constexpr (VW == 2) {
            atomicAdd(reinterpret_cast<float2*>(wrow + hcol[c]), make_float2(v * dA[c][0], v * dA[c][1]));
          } else {
            atomicAdd(wrow + hcol[c], v * dA[c][0]);
          }
        }
      }
    }
    __syncthreads();
  }
}

// ---- backward without fp32 atomics on dW: the batch's stored entries are bucketed by column (counts come from the forward
// kernel), then every touched row of dW is produced by ONE CTA that gathers v * dA[r,:] over the column's entries.
__global__ void __launch_bounds__(1024) col_scan_kernel(const int32_t* __restrict__ col_count, int F, int32_t* __restrict__ col_start,
                                                       int32_t* __restrict__ col_cursor) {
  // exclusive scan of the per-column counts: chunks of 8192 staged in shared memory (coalesced in / out), 8 consecutive
  // elements per thread, warp-shuffle scan of the thread sums, running carry between chunks
  constexpr int kPer = 8, kChunkElems = 1024 * kPer;
  __shared__ int s[kChunkElems];
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < F; base += kChunkElems) {
    const int n = min(kChunkElems, F - base);
    for (int i = tid; i < kChunkElems; i += 1024) s[i] = (i < n) ? col_count[base + i] : 0;
    __syncthreads();
    int v[kPer], sum = 0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) { v[j] = s[tid * kPer + j]; sum += v[j]; }
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      int w = s_warp[lane], wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += t; }
      s_warp[lane] = wi - w;  // exclusive prefix of the warp totals
    }
    __syncthreads();
    int run = s_carry + s_warp[wid] + incl - sum;
#pragma unroll
    for (int j = 0; j < kPer; ++j) { s[tid * kPer + j] = run; run += v[j]; }
    __syncthreads();
    for (int i = tid; i < n; i += 1024) { const int x = s[i]; col_start[base + i] = x; col_cursor[base + i] = x; }
    __syncthreads();
    if (tid == 1023) s_carry = run;
    __syncthreads();
  }
  if (tid == 0) col_start[F] = s_carry;
}

// per batch row: dA = dE * f'(A), dbh, and the row's kept entries appended to their column buckets.  One WARP per row, kRowsPerCta rows
// per CTA: the rows' dbh contributions are summed through shared memory and leave as one atomic per hidden unit per CTA (the H
// addresses of dbh are otherwise hit by every row of the batch), while the rows still progress in parallel.
constexpr int kRowsPerCta = 4;

// DET (the deterministic mode): the CTA's dbh sum goes to its own row dbh[blockIdx.x * H + h] of a partial buffer instead of an atomic,
// and the entries are bucketed by det_place_kernel instead.
template <int ACT, bool DET = false>
__global__ void __launch_bounds__(32 * kRowsPerCta) encode_bwd_rows_kernel(
    const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const float* __restrict__ values,
    const int32_t* __restrict__ rows, int n_rows, int H, float in_scale, const float* __restrict__ E, const float* __restrict__ bh,
    float* __restrict__ dE, const float* __restrict__ dE_add, int64_t ldE, float* __restrict__ dbh, int32_t* __restrict__ col_cursor, int32_t* __restrict__ ent_col,
    int32_t* __restrict__ ent_row, float* __restrict__ ent_val) {
  extern __shared__ float s_part[];   // [kRowsPerCta][H]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r = blockIdx.x * kRowsPerCta + warp;
  float* part = s_part + (int64_t)warp * H;
  if (r < n_rows) {
    for (int h = lane; h < H; h += 32) {
      const float fb = act_fwd<ACT>(__ldg(bh + h));
      const float fa = E[(int64_t)r * ldE + h] + fb;
      const float de = dE[(int64_t)r * ldE + h] + (dE_add ? dE_add[(int64_t)r * ldE + h] : 0.0f);
      const float da = de * act_grad_from_y<ACT>(fa);
      dE[(int64_t)r * ldE + h] = da;
      part[h] = da - act_grad_from_y<ACT>(fb) * de;
    }
  } else {
    for (int h = lane; h < H; h += 32) part[h] = 0.0f;
  }
  __syncthreads();
  for (int h = tid; h < H; h += 32 * kRowsPerCta) {
    float t = 0.0f;
#pragma unroll
    for (int w = 0; w < kRowsPerCta; ++w) t += s_part[(int64_t)w * H + h];
    if constexpr (DET) dbh[(int64_t)blockIdx.x * H + h] = t;
    else atomicAdd(dbh + h, t);
  }
  if constexpr (DET) return;
  if (r < n_rows) {
    const int64_t row = rows ? (int64_t)rows[r] : (int64_t)r;
    const int64_t p0 = indptr[row], p1 = indptr[row + 1];
    for (int64_t p = p0 + lane; p < p1; p += 32) {
      const float v = __ldg(values + p) * in_scale;
      if (v != 0.0f) {
        const int col = __ldg(indices + p);
        const int slot = atomicAdd(col_cursor + col, 1);
        ent_col[slot] = col;
        ent_row[slot] = r;
        ent_val[slot] = v;
      }
    }
  }
}

// Entries are bucketed by column (ent_* sorted by column).  Work is split by ENTRIES, not by columns (word frequencies are
// Zipfian: a few columns hold hundreds of entries): each CTA takes chunks of kChunk consecutive entries, accumulates
// v * dA[r,:] in registers while the column stays the same and flushes one vector red.global.add per (chunk, column) run --
// about (#touched columns + #chunks) vector atomics per step instead of one per entry.
constexpr int kChunk = 32;

template <int VW, int NC>
__global__ void __launch_bounds__(kEncThreads) encode_bwd_gather_kernel(const int32_t* __restrict__ col_start, int F,
                                                                        const int32_t* __restrict__ ent_col,
                                                                        const int32_t* __restrict__ ent_row,
                                                                        const float* __restrict__ ent_val, int H,
                                                                        const float* __restrict__ dA, int64_t ldE,
                                                                        float* __restrict__ dW) {
  __shared__ int s_c[kChunk];
  __shared__ int s_r[kChunk];
  __shared__ float s_v[kChunk];
  const int tid = threadIdx.x;
  const int total = col_start[F];
  int hcol[NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) hcol[c] = (tid + c * kEncThreads) * VW;

  for (int base = blockIdx.x * kChunk; base < total; base += gridDim.x * kChunk) {
    const int n = min(kChunk, total - base);
    __syncthreads();
    if (tid < n) { s_c[tid] = ent_col[base + tid]; s_r[tid] = ent_row[base + tid]; s_v[tid] = ent_val[base + tid]; }
    __syncthreads();
    float acc[NC][VW];
#pragma unroll
    for (int c = 0; c < NC; ++c)
#pragma unroll
      for (int k = 0; k < VW; ++k) acc[c][k] = 0.0f;
    int cur = s_c[0];
    for (int q0 = 0; q0 < n; q0 += 8) {
      float a[8][NC][VW];
#pragma unroll
      for (int u = 0; u < 8; ++u) {   // eight rows of dA in flight per thread
        const int q = min(q0 + u, n - 1);
        const float* arow = dA + (int64_t)s_r[q] * ldE;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          if (hcol[c] < H) ldg_vec<VW>(arow + hcol[c], a[u][c]);
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int q = q0 + u;
        if (q < n) {
          const int col = s_c[q];
          if (col != cur) {           // column run ended: flush (uniform branch, every thread sees the same column list)
            float* wrow = dW + (int64_t)cur * H;
#pragma unroll
            for (int c = 0; c < NC; ++c) {
              if (hcol[c] < H) {
                if constexpr (VW == 4) atomicAdd(reinterpret_cast<float4*>(wrow + hcol[c]), make_float4(acc[c][0], acc[c][1], acc[c][2], acc[c][3]));
                else if constexpr (VW == 2) atomicAdd(reinterpret_cast<float2*>(wrow + hcol[c]), make_float2(acc[c][0], acc[c][1]));
                else atomicAdd(wrow + hcol[c], acc[c][0]);
              }
#pragma unroll
              for (int k = 0; k < VW; ++k) acc[c][k] = 0.0f;
            }
            cur = col;
          }
          const float v = s_v[q];
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            if (hcol[c] < H) {
#pragma unroll
              for (int k = 0; k < VW; ++k) acc[c][k] = fmaf(v, a[u][c][k], acc[c][k]);
            }
          }
        }
      }
    }
    float* wrow = dW + (int64_t)cur * H;
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      if (hcol[c] < H) {
        if constexpr (VW == 4) atomicAdd(reinterpret_cast<float4*>(wrow + hcol[c]), make_float4(acc[c][0], acc[c][1], acc[c][2], acc[c][3]));
        else if constexpr (VW == 2) atomicAdd(reinterpret_cast<float2*>(wrow + hcol[c]), make_float2(acc[c][0], acc[c][1]));
        else atomicAdd(wrow + hcol[c], acc[c][0]);
      }
    }
  }
}

// ---- deterministic encode backward (DESIGN 4.7) -------------------------------------------------------------------------------------
// Stable bucketing: the batch rows are cut into T tiles of RT consecutive rows.  (1) every tile counts its entries per column
// (integer atomics: exact); (2) one thread per column turns its T counts into the tile's first slot in the column's bucket
// (col_start[c] + the counts of the earlier tiles); (3) one warp per tile walks its rows IN ORDER and hands each entry the next slot of
// its column.  A canonical CSR row holds a column at most once, so the lanes of one row never share a column.  Each bucket then lists
// its entries in batch-row order, whatever the timing.
constexpr int kDbhGroup = 32;

struct DetLayout {
  int T, RT, CH;          // row tiles, rows per tile, entries per gather chunk
  int64_t n_chunks, n_cta, n_groups;   // dbh: n_cta row sums of 4-row CTAs, added in groups of kDbhGroup, then the groups
  int64_t off_start, off_cursor, off_col, off_row, off_val, off_tile, off_dbh, off_colsum, off_parts, off_dbh2, bytes;
};

static DetLayout det_layout(int n_rows, int F, int H, int64_t cap) {
  DetLayout L{};
  const int64_t max_tiles = std::max<int64_t>(1, ((int64_t)1 << 24) / F);      // the tile table stays under 64 MB
  L.T = (int)std::min<int64_t>((n_rows + 7) / 8, max_tiles);
  if (L.T < 1) L.T = 1;
  L.RT = (n_rows + L.T - 1) / L.T;
  if (L.RT < 1) L.RT = 1;
  L.T = (n_rows + L.RT - 1) / L.RT;
  if (L.T < 1) L.T = 1;
  L.CH = 64;                                                                   // the chunk partials stay under 256 MB
  while (((cap + L.CH - 1) / L.CH) * 2 * (int64_t)H * 4 > ((int64_t)256 << 20)) L.CH *= 2;
  L.n_chunks = std::max<int64_t>(1, (cap + L.CH - 1) / L.CH);
  L.n_cta = (n_rows + kRowsPerCta - 1) / kRowsPerCta;
  L.n_groups = (L.n_cta + kDbhGroup - 1) / kDbhGroup;
  auto al = [](int64_t b) { return (b + 255) / 256 * 256; };
  int64_t o = 0;
  L.off_start = o; o += al(4 * ((int64_t)F + 1));
  L.off_cursor = o; o += al(4 * (int64_t)F);
  L.off_col = o; o += al(4 * cap);
  L.off_row = o; o += al(4 * cap);
  L.off_val = o; o += al(4 * cap);
  L.off_tile = o; o += al(4 * (int64_t)L.T * F);
  L.off_dbh = o; o += al(4 * std::max<int64_t>(1, L.n_cta) * H);
  L.off_colsum = o; o += al(4 * (int64_t)F * H);
  L.off_parts = o; o += al(4 * L.n_chunks * 2 * H);
  L.off_dbh2 = o; o += al(4 * std::max<int64_t>(1, L.n_groups) * H);
  L.bytes = o;
  return L;
}

// first level of the fixed-order dbh sum: out[g][h] = parts[32 g][h] + parts[32 g + 1][h] + ... (in order); dae_reduce_parts then adds
// the groups in order.  Two levels keep the serial chain short at large batches (100 000 rows: 782 + 32 adds instead of 25 000).
__global__ void det_group_sum_kernel(const float* __restrict__ parts, int n_parts, int H, float* __restrict__ out) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x, g = blockIdx.y;
  if (h >= H) return;
  const int p0 = g * kDbhGroup, p1 = min(n_parts, p0 + kDbhGroup);
  float s = parts[(int64_t)p0 * H + h];
  for (int p = p0 + 1; p < p1; ++p) s = __fadd_rn(s, parts[(int64_t)p * H + h]);
  out[(int64_t)g * H + h] = s;
}

__global__ void det_tile_count_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                      const float* __restrict__ values, const int32_t* __restrict__ rows, int n_rows, int F, int RT,
                                      float in_scale, int32_t* __restrict__ tile_cnt) {
  const int r = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  const int64_t row = rows ? (int64_t)rows[r] : (int64_t)r;
  int32_t* cnt = tile_cnt + (int64_t)(r / RT) * F;
  for (int64_t p = indptr[row] + lane; p < indptr[row + 1]; p += 32)
    if (__ldg(values + p) * in_scale != 0.0f) atomicAdd(cnt + __ldg(indices + p), 1);
}

__global__ void det_tile_scan_kernel(int32_t* __restrict__ tile, int T, int F, const int32_t* __restrict__ col_start) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= F) return;
  int run = col_start[c];
  for (int t = 0; t < T; ++t) { const int x = tile[(int64_t)t * F + c]; tile[(int64_t)t * F + c] = run; run += x; }
}

__global__ void det_place_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices, const float* __restrict__ values,
                                 const int32_t* __restrict__ rows, int n_rows, int F, int RT, int T, float in_scale,
                                 int32_t* __restrict__ tile, int32_t* __restrict__ ent_col, int32_t* __restrict__ ent_row,
                                 float* __restrict__ ent_val) {
  const int t = (int)((blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (t >= T) return;
  int32_t* cur = tile + (int64_t)t * F;
  const int r1 = min(n_rows, (t + 1) * RT);
  for (int r = t * RT; r < r1; ++r) {
    const int64_t row = rows ? (int64_t)rows[r] : (int64_t)r;
    for (int64_t p = indptr[row] + lane; p < indptr[row + 1]; p += 32) {
      const float v = __ldg(values + p) * in_scale;
      if (v != 0.0f) {
        const int col = __ldg(indices + p);
        const int slot = cur[col];
        cur[col] = slot + 1;
        ent_col[slot] = col; ent_row[slot] = r; ent_val[slot] = v;
      }
    }
    __syncwarp();   // the next row's lanes read the cursors this row advanced
  }
}

// Sparse dW in fixed order: chunks of CH consecutive bucketed entries (fixed positions).  Inside a chunk a run of one column is summed
// in entry (= batch-row) order with separately rounded multiplies and adds.  A run that is its column's whole bucket is stored to
// colsum[col]; a run cut by a chunk boundary is the chunk's first run (slot 0) or its last (slot 1) and goes to parts[chunk][slot].
// Every thread walks the same entry list for its own VW columns of H, so any H works and no thread waits for another.
template <int VW>
__global__ void __launch_bounds__(kEncThreads) encode_bwd_gather_det_kernel(const int32_t* __restrict__ col_start, int F,
                                                                            const int32_t* __restrict__ ent_col,
                                                                            const int32_t* __restrict__ ent_row,
                                                                            const float* __restrict__ ent_val, int H,
                                                                            const float* __restrict__ dA, int64_t ldE, int CH,
                                                                            float* __restrict__ colsum, float* __restrict__ parts) {
  const int total = col_start[F];
  for (int64_t chunk = blockIdx.x; chunk * CH < total; chunk += gridDim.x) {
    const int base = (int)(chunk * CH), end = min(base + CH, total);
    for (int h0 = threadIdx.x * VW; h0 < H; h0 += kEncThreads * VW) {
      float acc[VW];
#pragma unroll
      for (int k = 0; k < VW; ++k) acc[k] = 0.0f;
      int cur = __ldg(ent_col + base), a = base;
      auto flush = [&](int b) {
        const bool whole = (a == __ldg(col_start + cur)) && (b == __ldg(col_start + cur + 1));
        float* dst = whole ? colsum + (int64_t)cur * H : parts + (chunk * 2 + (a == base ? 0 : 1)) * H;
#pragma unroll
        for (int k = 0; k < VW; ++k) dst[h0 + k] = acc[k];
      };
      for (int q0 = base; q0 < end; q0 += 8) {
        float x[8][VW];
        float v[8];
        int cc[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {   // eight rows of dA in flight per thread
          const int q = min(q0 + u, end - 1);
          v[u] = __ldg(ent_val + q);
          cc[u] = __ldg(ent_col + q);
          ldg_vec<VW>(dA + (int64_t)__ldg(ent_row + q) * ldE + h0, x[u]);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          if (q0 + u < end) {
            if (cc[u] != cur) {
              flush(q0 + u);
#pragma unroll
              for (int k = 0; k < VW; ++k) acc[k] = 0.0f;
              cur = cc[u];
              a = q0 + u;
            }
#pragma unroll
            for (int k = 0; k < VW; ++k) acc[k] = __fadd_rn(acc[k], __fmul_rn(v[u], x[u][k]));
          }
        }
      }
      flush(end);
    }
  }
}

// After the dense dW is in place: dW[c, :] += the column's sparse sum -- colsum[c], or its chunk partials added in chunk order.
__global__ void encode_sparse_dw_add_kernel(const int32_t* __restrict__ col_start, int F, int H, int CH, const float* __restrict__ colsum,
                                            const float* __restrict__ parts, float* __restrict__ dW) {
  for (int c = blockIdx.x; c < F; c += gridDim.x) {
    const int s = col_start[c], e = col_start[c + 1];
    if (s == e) continue;
    const int k0 = s / CH, k1 = (e - 1) / CH;
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
      float v;
      if (k0 == k1) {
        v = colsum[(int64_t)c * H + h];
      } else {
        v = parts[((int64_t)k0 * 2 + (s == k0 * CH ? 0 : 1)) * H + h];
        for (int k = k0 + 1; k <= k1; ++k) v = __fadd_rn(v, parts[(int64_t)k * 2 * H + h]);
      }
      dW[(int64_t)c * H + h] = __fadd_rn(dW[(int64_t)c * H + h], v);
    }
  }
}

template <int ACT, int VW>
static int launch_fwd_nc(int nc, int groups, dim3 grid, cudaStream_t st, const int64_t* indptr, const int32_t* indices, const float* values,
                         const int32_t* rows, int H, float in_scale, const float* W, const float* bh, float* E, int64_t ldE,
                         int32_t* col_count, void* e_hi, void* e_lo, int64_t ld_split) {
#define DAE_FWD(NC, G) encode_fwd_kernel<ACT, VW, NC, G><<<grid, kEncThreads * G, 0, st>>>(indptr, indices, values, rows, H, in_scale, W, bh, E, ldE, \
    col_count, (__nv_bfloat16*)e_hi, (__nv_bfloat16*)e_lo, ld_split)
  if (groups == 4) {
    switch (nc) {
      case 1: DAE_FWD(1, 4); break;
      case 2: DAE_FWD(2, 4); break;
      case 4: DAE_FWD(4, 4); break;
      default: DAE_FWD(8, 4); break;
    }
  } else {
    switch (nc) {
      case 1: DAE_FWD(1, 1); break;
      case 2: DAE_FWD(2, 1); break;
      case 4: DAE_FWD(4, 1); break;
      default: DAE_FWD(8, 1); break;
    }
  }
#undef DAE_FWD
  return 0;
}

template <int ACT, int VW>
static int launch_bwd_nc(int nc, dim3 grid, cudaStream_t st, const int64_t* indptr, const int32_t* indices, const float* values,
                         const int32_t* rows, int H, float in_scale, const float* E, const float* bh, float* dE, const float* dE_add,
                         int64_t ldE, float* dW, float* dbh) {
  switch (nc) {
    case 1: encode_bwd_kernel<ACT, VW, 1><<<grid, kEncThreads, 0, st>>>(indptr, indices, values, rows, H, in_scale, E, bh, dE, dE_add, ldE, dW, dbh); break;
    case 2: encode_bwd_kernel<ACT, VW, 2><<<grid, kEncThreads, 0, st>>>(indptr, indices, values, rows, H, in_scale, E, bh, dE, dE_add, ldE, dW, dbh); break;
    case 4: encode_bwd_kernel<ACT, VW, 4><<<grid, kEncThreads, 0, st>>>(indptr, indices, values, rows, H, in_scale, E, bh, dE, dE_add, ldE, dW, dbh); break;
    default: encode_bwd_kernel<ACT, VW, 8><<<grid, kEncThreads, 0, st>>>(indptr, indices, values, rows, H, in_scale, E, bh, dE, dE_add, ldE, dW, dbh); break;
  }
  return 0;
}

static inline int pick_vw(int H, int64_t ld, const void* p) {
  if (H % 4 == 0 && ld % 4 == 0 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) return 4;
  if (H % 2 == 0 && ld % 2 == 0 && (reinterpret_cast<uintptr_t>(p) & 7) == 0) return 2;
  return 1;
}
static inline int pick_nc(int H, int vw) {
  const int need = (H + vw * kEncThreads - 1) / (vw * kEncThreads);
  if (need <= 1) return 1;
  if (need <= 2) return 2;
  if (need <= 4) return 4;
  if (need <= 8) return 8;
  return -1;
}

}  // namespace dae

namespace dae {

// dae_encode_csr_fwd and dae_encode_csr_fwd_groups: `groups` thread groups of 128 per row (1 or 4); messages under `name`.
static int encode_fwd(const char* name, const int64_t* indptr, const int32_t* indices, const float* values, const int32_t* rows,
                      int32_t n_rows, int32_t F, int32_t H, float in_scale, const float* W, const float* bh, int32_t enc_act, float* E,
                      int64_t ldE, int32_t* col_count, void* e_hi, void* e_lo, int64_t ld_split, int groups, void* stream) {
  DAE_REQUIRE(indptr && indices && values && W && bh && E, "%s: null pointer", name);
  DAE_REQUIRE(n_rows >= 0 && F > 0 && H > 0 && ldE >= H, "%s: bad shape n_rows=%d F=%d H=%d ldE=%lld", name, n_rows, F, H, (long long)ldE);
  DAE_REQUIRE(!e_hi || (e_lo && ld_split >= H), "%s: bad split outputs", name);
  if (n_rows == 0) return DAE_OK;
  const int vw = pick_vw(H, H, W);
  const int nc = pick_nc(H, vw);
  if (nc < 0) { set_error("%s: H=%d too large for vector width %d", name, H, vw); return DAE_ERR_UNSUPPORTED; }
  cudaStream_t st = (cudaStream_t)stream;
  if (col_count) DAE_CUDA(cudaMemsetAsync(col_count, 0, sizeof(int32_t) * F, st));
  dim3 grid(n_rows);
  DAE_DISPATCH_ACT(enc_act, ACT, {
    if (vw == 4) launch_fwd_nc<ACT, 4>(nc, groups, grid, st, indptr, indices, values, rows, H, in_scale, W, bh, E, ldE, col_count, e_hi, e_lo, ld_split);
    else if (vw == 2) launch_fwd_nc<ACT, 2>(nc, groups, grid, st, indptr, indices, values, rows, H, in_scale, W, bh, E, ldE, col_count, e_hi, e_lo, ld_split);
    else launch_fwd_nc<ACT, 1>(nc, groups, grid, st, indptr, indices, values, rows, H, in_scale, W, bh, E, ldE, col_count, e_hi, e_lo, ld_split);
  });
  DAE_CHECK_LAUNCH(name);
  return DAE_OK;
}

}  // namespace dae

extern "C" int dae_encode_csr_fwd(const int64_t* indptr, const int32_t* indices, const float* values, const int32_t* rows,
                                  int32_t n_rows, int32_t F, int32_t H, float in_scale, const float* W, const float* bh,
                                  int32_t enc_act, float* E, int64_t ldE, int32_t* col_count, void* e_hi, void* e_lo,
                                  int64_t ld_split, void* stream) {
  using namespace dae;
  // Few rows (a training batch): every row is resident at once and the launch lasts as long as its longest row -> split rows over
  // 4 thread groups.  Many rows (transform): throughput-bound, one group per row keeps more rows in flight.
  const int groups = (n_rows <= sm_count() * 32) ? 4 : 1;
  return encode_fwd("dae_encode_csr_fwd", indptr, indices, values, rows, n_rows, F, H, in_scale, W, bh, enc_act, E, ldE, col_count, e_hi,
                    e_lo, ld_split, groups, stream);
}

// The same with the group count given (1 or 4) instead of chosen from n_rows: a row's output bits depend on the group count only,
// so a caller that pins it gets the same row whether it encodes the row alone, in a subset or in the whole set (DESIGN 4.19).
extern "C" int dae_encode_csr_fwd_groups(const int64_t* indptr, const int32_t* indices, const float* values, const int32_t* rows,
                                         int32_t n_rows, int32_t F, int32_t H, float in_scale, const float* W, const float* bh,
                                         int32_t enc_act, float* E, int64_t ldE, int32_t* col_count, void* e_hi, void* e_lo,
                                         int64_t ld_split, int32_t groups, void* stream) {
  using namespace dae;
  DAE_REQUIRE(groups == 1 || groups == 4, "dae_encode_csr_fwd_groups: groups = %d, 1 or 4", groups);
  return encode_fwd("dae_encode_csr_fwd_groups", indptr, indices, values, rows, n_rows, F, H, in_scale, W, bh, enc_act, E, ldE, col_count,
                    e_hi, e_lo, ld_split, groups, stream);
}

extern "C" int dae_encode_csr_bwd(const int64_t* indptr, const int32_t* indices, const float* values, const int32_t* rows,
                                  int32_t n_rows, int32_t F, int32_t H, float in_scale, const float* E, const float* bh,
                                  int32_t enc_act, float* dE, const float* dE_add, int64_t ldE, float* dW, float* dbh, int32_t dbh_zeroed,
                                  void* stream) {
  using namespace dae;
  DAE_REQUIRE(indptr && indices && values && E && bh && dE && dW && dbh, "dae_encode_csr_bwd: null pointer");
  DAE_REQUIRE(n_rows >= 0 && F > 0 && H > 0 && ldE >= H, "dae_encode_csr_bwd: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  if (!dbh_zeroed) DAE_CUDA(cudaMemsetAsync(dbh, 0, sizeof(float) * H, st));
  if (n_rows == 0) return DAE_OK;
  const int vw = pick_vw(H, H, dW);
  const int nc = pick_nc(H, vw);
  if (nc < 0) { set_error("dae_encode_csr_bwd: H=%d too large", H); return DAE_ERR_UNSUPPORTED; }
  dim3 grid(n_rows);
  DAE_DISPATCH_ACT(enc_act, ACT, {
    if (vw == 4) launch_bwd_nc<ACT, 4>(nc, grid, st, indptr, indices, values, rows, H, in_scale, E, bh, dE, dE_add, ldE, dW, dbh);
    else if (vw == 2) launch_bwd_nc<ACT, 2>(nc, grid, st, indptr, indices, values, rows, H, in_scale, E, bh, dE, dE_add, ldE, dW, dbh);
    else launch_bwd_nc<ACT, 1>(nc, grid, st, indptr, indices, values, rows, H, in_scale, E, bh, dE, dE_add, ldE, dW, dbh);
  });
  DAE_CHECK_LAUNCH("dae_encode_csr_bwd");
  return DAE_OK;
}

extern "C" int dae_encode_csr_bwd_gather(const int64_t* indptr, const int32_t* indices, const float* values, const int32_t* rows,
                                         int32_t n_rows, int32_t F, int32_t H, float in_scale, const float* E, const float* bh,
                                         int32_t enc_act, float* dE, const float* dE_add, int64_t ldE, float* dW, float* dbh,
                                         int32_t dbh_zeroed, const int32_t* col_count, int32_t* col_start, int32_t* col_cursor,
                                         int32_t* ent_col, int32_t* ent_row, float* ent_val, void* stream) {
  using namespace dae;
  DAE_REQUIRE(indptr && indices && values && E && bh && dE && dW && dbh && col_start && col_cursor && ent_col && ent_row && ent_val,
              "dae_encode_csr_bwd_gather: null pointer");
  DAE_REQUIRE(n_rows >= 0 && F > 0 && H > 0 && ldE >= H, "dae_encode_csr_bwd_gather: bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  if (!dbh_zeroed) DAE_CUDA(cudaMemsetAsync(dbh, 0, sizeof(float) * H, st));
  if (n_rows == 0) return DAE_OK;
  int vw = pick_vw(H, ldE, dE);
  if (pick_vw(H, H, dW) < vw) vw = pick_vw(H, H, dW);
  const int nc = pick_nc(H, vw);
  if (nc < 0 || nc > 2) { set_error("dae_encode_csr_bwd_gather: H=%d not supported (use dae_encode_csr_bwd)", H); return DAE_ERR_UNSUPPORTED; }
  if (col_count) col_scan_kernel<<<1, 1024, 0, st>>>(col_count, F, col_start, col_cursor);  // NULL: dae_col_scan already ran
  DAE_DISPATCH_ACT(enc_act, ACT, {
    encode_bwd_rows_kernel<ACT><<<(n_rows + kRowsPerCta - 1) / kRowsPerCta, 32 * kRowsPerCta, sizeof(float) * kRowsPerCta * H, st>>>(indptr, indices, values, rows, n_rows, H, in_scale, E, bh, dE, dE_add, ldE, dbh, col_cursor,
                                                               ent_col, ent_row, ent_val);
  });
#define DAE_GATHER(VW, NC) encode_bwd_gather_kernel<VW, NC><<<sm_count() * 16, kEncThreads, 0, st>>>(col_start, F, ent_col, ent_row, ent_val, H, dE, ldE, dW)
#define DAE_GATHER_NC(VW) \
  do { if (nc == 1) DAE_GATHER(VW, 1); else DAE_GATHER(VW, 2); } while (0)
  if (vw == 4) DAE_GATHER_NC(4); else if (vw == 2) DAE_GATHER_NC(2); else DAE_GATHER_NC(1);
#undef DAE_GATHER_NC
#undef DAE_GATHER
  DAE_CHECK_LAUNCH("dae_encode_csr_bwd_gather");
  return DAE_OK;
}

extern "C" int dae_col_scan(const int32_t* col_count, int32_t F, int32_t* col_start, int32_t* col_cursor, void* stream) {
  using namespace dae;
  DAE_REQUIRE(col_count && col_start && col_cursor && F > 0, "dae_col_scan: bad arguments");
  col_scan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(col_count, F, col_start, col_cursor);
  DAE_CHECK_LAUNCH("dae_col_scan");
  return DAE_OK;
}

extern "C" int dae_encode_csr_fwd_hot(const int64_t* indptr, const int32_t* indices, const float* values, int32_t n_rows, int32_t F,
                                      int32_t H, float in_scale, const float* W, const float* bh, int32_t enc_act, float* E, int64_t ldE,
                                      const int32_t* hot_cols, const int32_t* hot_slot, int32_t K, int32_t groups, void* stream) {
  using namespace dae;
  DAE_REQUIRE(indptr && indices && values && W && bh && E && hot_cols && hot_slot, "dae_encode_csr_fwd_hot: null pointer");
  DAE_REQUIRE(n_rows >= 0 && F > 0 && H > 0 && ldE >= H && K >= 1, "dae_encode_csr_fwd_hot: bad shape");
  DAE_REQUIRE(H % 4 == 0 && ldE % 4 == 0 && ((uintptr_t)W & 15) == 0 && ((uintptr_t)E & 15) == 0 && H <= 8 * kEncThreads,
              "dae_encode_csr_fwd_hot: needs H %% 4 == 0, H <= 1024 and 16-byte aligned W / E (use dae_encode_csr_fwd otherwise)");
  const size_t smem = (size_t)K * H * 4;
  DAE_REQUIRE(smem <= 200 * 1024, "dae_encode_csr_fwd_hot: K * H * 4 = %zu bytes of staged rows exceed 200 KB", smem);
  if (n_rows == 0) return DAE_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int sms = sm_count();
  const int nc = (H + 4 * kEncThreads - 1) / (4 * kEncThreads);
  const int G = (groups >= 8) ? 8 : 4;
  // CTAs per SM follow from the staged set: one for K * H * 4 > 100 KB, two up to 100 KB, three up to 64 KB ...
  int per_sm = (int)((220 * 1024) / (smem + 8 * 1024));
  if (per_sm < 1) per_sm = 1;
  if (per_sm * G * kEncThreads > 2048) per_sm = 2048 / (G * kEncThreads);
  const int want = (n_rows + G - 1) / G;
  const int grid = want < sms * per_sm ? want : sms * per_sm;
#define DAE_HOT(ACT, NC, GG)                                                                                                       \
  do {                                                                                                                            \
    auto kern = encode_fwd_hot_kernel<ACT, NC, GG>;                                                                               \
    DAE_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));                                \
    kern<<<grid, kEncThreads * GG, smem, st>>>(indptr, indices, values, n_rows, H, in_scale, W, bh, E, ldE, hot_cols, hot_slot, K); \
  } while (0)
  DAE_DISPATCH_ACT(enc_act, ACT, {
    if (G == 8) { if (nc <= 1) DAE_HOT(ACT, 1, 8); else DAE_HOT(ACT, 2, 8); }
    else { if (nc <= 1) DAE_HOT(ACT, 1, 4); else DAE_HOT(ACT, 2, 4); }
  });
#undef DAE_HOT
  DAE_CHECK_LAUNCH("dae_encode_csr_fwd_hot");
  return DAE_OK;
}

extern "C" int dae_encode_csr_bwd_det_workspace(int32_t n_rows, int32_t F, int32_t H, int64_t cap_nnz, int64_t* bytes) {
  using namespace dae;
  DAE_REQUIRE(bytes && n_rows >= 1 && F > 0 && H > 0 && cap_nnz >= 0, "dae_encode_csr_bwd_det_workspace: bad arguments");
  *bytes = det_layout(n_rows, F, H, cap_nnz).bytes;
  return DAE_OK;
}

extern "C" int dae_encode_csr_bwd_det(const int64_t* indptr, const int32_t* indices, const float* values, const int32_t* rows,
                                      int32_t n_rows, int32_t F, int32_t H, float in_scale, const float* E, const float* bh,
                                      int32_t enc_act, float* dE, const float* dE_add, int64_t ldE, float* dbh, const int32_t* col_count,
                                      int64_t cap_nnz, void* workspace, int64_t workspace_bytes, void* stream) {
  using namespace dae;
  DAE_REQUIRE(indptr && indices && values && E && bh && dE && dbh && col_count && workspace, "dae_encode_csr_bwd_det: null pointer");
  DAE_REQUIRE(n_rows >= 1 && F > 0 && H > 0 && ldE >= H && cap_nnz >= 0, "dae_encode_csr_bwd_det: bad shape");
  const DetLayout L = det_layout(n_rows, F, H, cap_nnz);
  DAE_REQUIRE(workspace_bytes >= L.bytes, "dae_encode_csr_bwd_det: workspace of %lld bytes, need %lld", (long long)workspace_bytes,
              (long long)L.bytes);
  const size_t smem = sizeof(float) * kRowsPerCta * H;
  DAE_REQUIRE(smem <= 200 * 1024, "dae_encode_csr_bwd_det: H=%d too large", H);
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = (uint8_t*)workspace;
  int32_t* col_start = (int32_t*)(w + L.off_start);
  int32_t* tile = (int32_t*)(w + L.off_tile);
  int32_t* ent_col = (int32_t*)(w + L.off_col);
  int32_t* ent_row = (int32_t*)(w + L.off_row);
  float* ent_val = (float*)(w + L.off_val);
  float* dbh_part = (float*)(w + L.off_dbh);
  col_scan_kernel<<<1, 1024, 0, st>>>(col_count, F, col_start, (int32_t*)(w + L.off_cursor));
  DAE_CUDA(cudaMemsetAsync(tile, 0, sizeof(int32_t) * (size_t)L.T * F, st));
  det_tile_count_kernel<<<(n_rows + 7) / 8, 256, 0, st>>>(indptr, indices, values, rows, n_rows, F, L.RT, in_scale, tile);
  det_tile_scan_kernel<<<(F + 255) / 256, 256, 0, st>>>(tile, L.T, F, col_start);
  det_place_kernel<<<(L.T + 3) / 4, 128, 0, st>>>(indptr, indices, values, rows, n_rows, F, L.RT, L.T, in_scale, tile, ent_col, ent_row, ent_val);
  DAE_DISPATCH_ACT(enc_act, ACT, {
    auto kern = encode_bwd_rows_kernel<ACT, true>;
    if (smem > 48 * 1024) DAE_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)L.n_cta, 32 * kRowsPerCta, smem, st>>>(indptr, indices, values, rows, n_rows, H, in_scale, E, bh, dE, dE_add, ldE,
                                                            dbh_part, nullptr, nullptr, nullptr, nullptr);
  });
  float* dbh_group = (float*)(w + L.off_dbh2);   // dbh = the CTAs' sums in groups of kDbhGroup, then the groups, each level in order
  det_group_sum_kernel<<<dim3((H + 127) / 128, (unsigned)L.n_groups), 128, 0, st>>>(dbh_part, (int)L.n_cta, H, dbh_group);
  int rc = dae_reduce_parts(dbh_group, (int32_t)L.n_groups, H, dbh, stream);
  if (rc) return rc;
  const int vw = (H % 4 == 0 && ldE % 4 == 0 && ((uintptr_t)dE & 15) == 0) ? 4 : ((H % 2 == 0 && ldE % 2 == 0 && ((uintptr_t)dE & 7) == 0) ? 2 : 1);
  const int64_t want = L.n_chunks;
  const int grid = (int)std::min<int64_t>(want, (int64_t)sm_count() * 16);
  float* colsum = (float*)(w + L.off_colsum);
  float* parts = (float*)(w + L.off_parts);
  if (vw == 4) encode_bwd_gather_det_kernel<4><<<grid, kEncThreads, 0, st>>>(col_start, F, ent_col, ent_row, ent_val, H, dE, ldE, L.CH, colsum, parts);
  else if (vw == 2) encode_bwd_gather_det_kernel<2><<<grid, kEncThreads, 0, st>>>(col_start, F, ent_col, ent_row, ent_val, H, dE, ldE, L.CH, colsum, parts);
  else encode_bwd_gather_det_kernel<1><<<grid, kEncThreads, 0, st>>>(col_start, F, ent_col, ent_row, ent_val, H, dE, ldE, L.CH, colsum, parts);
  DAE_CHECK_LAUNCH("dae_encode_csr_bwd_det");
  return DAE_OK;
}

extern "C" int dae_encode_sparse_dw_add(int32_t n_rows, int32_t F, int32_t H, int64_t cap_nnz, const void* workspace, int64_t workspace_bytes,
                                        float* dW, void* stream) {
  using namespace dae;
  DAE_REQUIRE(workspace && dW && n_rows >= 1 && F > 0 && H > 0 && cap_nnz >= 0, "dae_encode_sparse_dw_add: bad arguments");
  const DetLayout L = det_layout(n_rows, F, H, cap_nnz);
  DAE_REQUIRE(workspace_bytes >= L.bytes, "dae_encode_sparse_dw_add: workspace of %lld bytes, need %lld", (long long)workspace_bytes,
              (long long)L.bytes);
  const uint8_t* w = (const uint8_t*)workspace;
  encode_sparse_dw_add_kernel<<<std::min(F, 65535), 128, 0, (cudaStream_t)stream>>>((const int32_t*)(w + L.off_start), F, H, L.CH,
                                                                                   (const float*)(w + L.off_colsum),
                                                                                   (const float*)(w + L.off_parts), dW);
  DAE_CHECK_LAUNCH("dae_encode_sparse_dw_add");
  return DAE_OK;
}
