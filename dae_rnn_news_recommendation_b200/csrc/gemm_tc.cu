// wgmma / TMA / mbarrier GEMM for the dense contractions of the DAE step, fp32-accurate through a 3-pass bf16 split.
//
// Reference ops replaced: tf.matmul(encode, tf.transpose(W)) (autoencoder/autoencoder.py:411) and its autodiff
// (dW = dZ^T.E, dE = dZ.W), and tf.matmul(encode, tf.transpose(encode)) (autoencoder/triplet_loss_utils.py:93,219).
//
// Numerics: every fp32 operand x is carried as two bf16 arrays, hi = bf16(x) and lo = bf16(x - hi) (|x - hi - lo| <= 2^-17 |x|).
//   D += A_hi.B_hi + A_lo.B_hi + A_hi.B_lo      (three bf16 wgmma per k-step, fp32 accumulation in registers)
// The dropped lo.lo term is <= 2^-18 relative, so the product is fp32-grade (1e-5 rel. worst case vs the 1e-4 budget).
//
// Structure (one CTA per SM, persistent over output tiles):
//   store GEMM (dae_gemm_bf16x3, dae_gemm_sym_bf16x3; 384 threads = three warpgroups):
//   warpgroup 0   : TMA producer -- one lane issues cp.async.bulk.tensor.2d, 128B swizzle, into a STAGES-deep smem ring (hi and lo
//                   tiles); the other warps only take part in the CTA-wide barriers
//   warpgroups 1-2: consumers    -- each owns 64 rows of the 128-row tile: wgmma.mma_async m64 x BLOCK_N x k16 from shared-memory
//                   descriptors, then the store epilogue from a shared-memory staging tile; meanwhile the producer already fills the
//                   ring with the next tile's operands.
//   fused decode (dae_decode_fused_bf16x3; 640 threads = five warpgroups, see decode_fused_kernel): the same producer, two MMA
//                   warpgroups that only run the main loop, and two epilogue warpgroups that run the loss epilogue of tile i from
//                   the staging tile while the MMA warpgroups accumulate tile i + 1.
//   similarity top-k (dae_similarity_topk_bf16x3; see topk_kernel): the fused decode's five warpgroups with a k-best selection
//                   epilogue instead of the loss, so the similarity matrix never leaves the SM.
//   pair histogram (dae_similarity_pair_hist_bf16x3; see pair_hist_kernel): the same five warpgroups over the lower-triangle tiles
//                   of X.X^T, binning related / unrelated pair scores into uint64 histograms for the AUROC.
//   thresholded pairs (dae_similarity_pairs_bf16x3; see pairs_kernel): the same five warpgroups, emitting every pair with a score
//                   at or above a threshold (near-duplicates) into caller-sized arrays through a warp-aggregated 64-bit counter.
// Operands may be K-major (K contiguous) or MN-major (M/N contiguous) -- both straight from row-major arrays (wgmma's transpose
// bits), so no transposed copies of dZ / E / W are ever made.
#include <cuda.h>
#include <cuda_bf16.h>
#include <type_traits>
#include "common.cuh"
#include "pair_hist.cuh"
#include "pairs.cuh"
#include "topk.cuh"

namespace dae {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;    // 64 bf16 = 128 bytes = one swizzle row
constexpr int WGMMA_K = 16;
constexpr int kThreads = 384;
constexpr int kDecodeN = 128;  // column tile of the fused decode kernel (dae_decode_prepare lays tile_ptr out for it)

// ---------------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Spin, then back off with nanosleep; a wait that lasts longer than ~4 s (a lost TMA / arrival: a programming error, not a
// slow peer) traps so the failure surfaces on the host at the next synchronisation instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > 4096u) {
      __nanosleep(64);
      if (spins > (1u << 26)) __trap();
    }
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// ---- CTA pair: a cluster of two CTAs works on two vertically adjacent 128-row tiles with the SAME B tile.  Each CTA loads its own
// A tile and HALF of the B tile, multicast into the shared memory of both CTAs (completing bytes on the mbarrier at the same offset
// in each), so a k-block costs each SM 48 KB of L2 -> SM traffic instead of 64 KB.  A ring stage is refilled only when the
// consumers of BOTH CTAs have released it (the peer's multicast writes into it).
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void tma_load_2d_mc(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
          smem_u32(dst)),
      "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
// arrive on the mbarrier at this offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
  uint32_t raddr;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(smem_u32(bar)), "r"(rank));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(raddr) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {   // acquire at cluster scope (remote arrivals)
  uint32_t spins = 0;
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (ok) return;
    if (++spins > 4096u) { __nanosleep(64); if (spins > (1u << 26)) __trap(); }
  }
}

__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Shared-memory matrix descriptor (sm_90 wgmma), 128-byte swizzle (layout 1) or, for 32-wide K-major k-blocks, 64-byte swizzle (layout 2).
//   K-major : rows of 128 B (64 B), 8-row groups 1024 B (512 B) apart (SBO); LBO unused (1).
//   MN-major: 64-element (128 B) column slabs, 8 k-rows per 1024 B group (SBO), next slab LBO bytes further.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout = 1) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)layout << 62;
  return d;
}

// D (+)= A.B for one warpgroup: m64 x n x k16, bf16 operands from shared memory, fp32 accumulators d[n / 2] in the wgmma fragment
// layout (thread t of the warpgroup: rows 16 (t / 32) + (t % 32) / 4 + {0, 8}, columns 8 j + 2 (t % 4) + {0, 1}).
// TA / TB: the operand is MN-major (transposed).  scale_d = 0 overwrites D.

template <int TA, int TB>
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

template <int TA, int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d), "n"(TA), "n"(TB));
}

// ---------------------------------------------------------------------------------------------------------------------
// kernel parameters
// ---------------------------------------------------------------------------------------------------------------------
struct GemmParams {
  int M, N, K;           // logical sizes (TMA zero-fills out-of-range rows / columns)
  int k_splits;          // > 1: uniform split-K
  int stream_k;          // 1: stream-K -- the CTAs share the (tile, k-block) units evenly, partial tiles are added with atomics
  int atomic;            // accumulate into C with fp32 atomics (split-K / stream-K, or C += ...)
  int a_mn, b_mn;        // operand majorness
  int a_sym_kb;          // > 0: C = (A + A^T).B -- k-blocks [0, a_sym_kb) read the square A K-major, k-blocks [a_sym_kb, 2 a_sym_kb) read it
                         // MN-major (= A^T) through the second pair of tensor maps, and B's k index wraps (both halves multiply B)
  float alpha;
  float* C;              // store GEMM: fp32 output [M x ldc]
  int64_t ldc;
  int n_store;           // columns < n_store are stored
  int special_col;       // store GEMM: this column (the all-ones column of [E | 1]) goes to special_out[m] instead; -1 = none
  float* special_out;
  // fused decode loss (M = batch rows, N = features)
  const int64_t* indptr; const int32_t* indices; const float* values; const int32_t* rows;
  const float* bv; const float* weight; const double* stats;
  __nv_bfloat16* dz_hi; __nv_bfloat16* dz_lo; int64_t ld_dz;
  float* row_loss_part;  // [M] row losses, accumulated with fp32 atomics (zeroed by the launcher)
  const int32_t* tile_ptr; // [M x (2 * n_tiles_n + 1)]: first CSR entry of every half tile, relative to the row start
  // deterministic mode (see DESIGN 4.7)
  float* sk_ws;          // stream-K: a segment that covers part of a tile stores it to slot [cta][first ? 0 : 1] of this
                         // [n_cta][2][BLOCK_M][BLOCK_N] workspace instead of adding it to C; sk_fixup_kernel sums the slots in k order
  int loss_parts;        // fused decode: row_loss_part is [2 * n_tiles_n][M], one store per (half tile, row) instead of an atomic
};

// Work distribution, walked identically by every warpgroup of a CTA.
//   classic : work item w = (tile, k split), items blockIdx.x, blockIdx.x + gridDim.x, ...
//   stream-K: the tiles x k-blocks units are cut into gridDim.x equal contiguous ranges; a CTA's range covers the tail of one
//             tile, whole tiles, and the head of another -- every segment is one accumulator pass + one (atomic) epilogue.
//             Balances shapes whose tile count does not fill the SMs evenly (dW: 316 tiles on an H100 SXM's 132) without shrinking the tiles.
struct Sched {
  int tiles_m, tiles, kb_total, kb_per_split, n_work, stream, w, n_cta;
  long long u, u_end;
  // pair != 0: the two CTAs of a cluster walk the SAME list; an m index then names a pair of 128-row tiles
  __device__ __forceinline__ void init(const GemmParams& p, int block_n, int pair = 0, int block_k = BLOCK_K) {
    const int cta = pair ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
    n_cta = pair ? (int)(gridDim.x >> 1) : (int)gridDim.x;
    tiles_m = (p.M + BLOCK_M - 1) / BLOCK_M;
    if (pair) tiles_m = (tiles_m + 1) / 2;
    tiles = tiles_m * ((p.N + block_n - 1) / block_n);
    kb_total = (p.K + block_k - 1) / block_k;
    stream = p.stream_k;
    kb_per_split = (kb_total + p.k_splits - 1) / p.k_splits;
    n_work = tiles * p.k_splits;
    w = cta;
    const long long U = (long long)tiles * kb_total;
    u = (long long)cta * U / n_cta;
    u_end = (long long)(cta + 1) * U / n_cta;
  }
  __device__ __forceinline__ bool next(int& mb, int& nb, int& kb0, int& kb1) {
    int tile;
    if (stream) {
      if (u >= u_end) return false;
      tile = (int)(u / kb_total);
      kb0 = (int)(u - (long long)tile * kb_total);
      const long long left = u_end - u;
      kb1 = (left < (long long)(kb_total - kb0)) ? kb0 + (int)left : kb_total;
      u += kb1 - kb0;
    } else {
      if (w >= n_work) return false;
      tile = w % tiles;
      kb0 = (w / tiles) * kb_per_split;
      kb1 = min(kb_total, kb0 + kb_per_split);
      w += n_cta;
    }
    mb = tile % tiles_m;
    nb = tile / tiles_m;
    return true;
  }
};

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&v);
}
__device__ __forceinline__ float f_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float f_lg2(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float f_ex2(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
constexpr float kLog2e = 1.4426950408889634f;

// decoder activation on the MUFU pipe (relative error ~1e-6, inside the 1e-4 parity budget)
template <int ACT>
__device__ __forceinline__ float act_fast(float z) {
  if (ACT == DAE_ACT_SIGMOID) return f_rcp(1.0f + f_ex2(-kLog2e * z));
  if (ACT == DAE_ACT_TANH) return 1.0f - 2.0f * f_rcp(1.0f + f_ex2(2.0f * kLog2e * z));
  return z;
}


// r[j] for a runtime j in [0,16) without dynamic register indexing
__device__ __forceinline__ float select16(const uint32_t (&r)[16], int j) {
  uint32_t v = r[0];
#pragma unroll
  for (int k = 1; k < 16; ++k) v = (j == k) ? r[k] : v;
  return __uint_as_float(v);
}

// One 16-column chunk of the fused decode epilogue, evaluated as if every target x were 0 (99 % of a bag-of-words row is):
// z = acc + bv -> D = g(z) -> loss term -> dZ = sc * dloss/dz, packed as bf16 hi / lo pairs.  `lsum`: CE in log2 units, MSE plain.
template <int ACT, int LOSS>
__device__ __forceinline__ void decode_chunk_generic(const uint32_t (&r)[16], const float* __restrict__ bias, float sc, bool edge,
                                                     int n_lim, int nc, uint32_t (&hpk)[8], uint32_t (&lpk)[8], float& lsum) {
#pragma unroll
  for (int j2 = 0; j2 < 8; ++j2) {
    float dzp[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int j = 2 * j2 + e;
      const float z = __uint_as_float(r[j]) + bias[j];
      const float d = act_fast<ACT>(z);
      float dz, lt;
      if (LOSS == DAE_LOSS_CE) {
        const float omd = 1.0f - d;
        const float b = omd + kEps;                 // 1. - decode + 1e-16, left to right (:269)
        lt = -f_lg2(b);
        // dl * g' = d * omd / b; omd / b == 1 exactly in fp32 unless omd == 0 (then the product is 0)
        dz = (ACT == DAE_ACT_SIGMOID) ? ((omd != 0.0f) ? sc * d : 0.0f) : sc * act_grad_from_y<ACT>(d) * f_rcp(b);
      } else {
        lt = d * d;
        dz = 2.0f * sc * d * act_grad_from_y<ACT>(d);
      }
      if (edge) { const bool in = (nc + j < n_lim); lt = in ? lt : 0.0f; dz = in ? dz : 0.0f; }  // uniform branch
      lsum += lt;
      dzp[e] = dz;
    }
    const uint32_t hp = pack_bf16(dzp[0], dzp[1]);
    hpk[j2] = hp;
    lpk[j2] = pack_bf16(dzp[0] - __uint_as_float(hp << 16), dzp[1] - __uint_as_float(hp & 0xffff0000u));
  }
}

// sigmoid + cross-entropy fast path (x = 0): with t = e^z,  1 - D = 1/(1+t),  -log(1 - D) = log(1+t),  dZ = sc * t/(1+t).
// Four columns share ONE reciprocal (Montgomery batch inversion of P = prod(1+t)) and ONE logarithm (log2 P): 1.5 MUFU per
// element instead of 3.  Valid while every z <= 10 (P <= e^10 bounds each factor, all factors being >= 1): there the fp32
// reference's own `1 - decode` rounding (2^-25 / (1 - D) relative) stays far below the parity budget; the caller re-evaluates the
// chunk with decode_chunk_generic when this returns false.
__device__ __forceinline__ bool decode_chunk_sigmoid_ce(const uint32_t (&r)[16], const float* __restrict__ biasc, float sc,
                                                        uint32_t (&hpk)[8], uint32_t (&lpk)[8], float& lsum) {
  bool ok = true;
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    float t[4], a[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      t[j] = f_ex2(fmaf(__uint_as_float(r[4 * g + j]), kLog2e, biasc[4 * g + j]));   // biasc = bv * log2(e)
      a[j] = 1.0f + t[j];
    }
    const float p01 = a[0] * a[1], p23 = a[2] * a[3], P = p01 * p23;
    ok = ok && (P <= 22026.0f);                         // false for NaN / inf as well
    const float Rs = f_rcp(P) * sc;
    lsum += f_lg2(P);
    const float r23 = Rs * p23, r01 = Rs * p01;
    const float dz0 = t[0] * (r23 * a[1]), dz1 = t[1] * (r23 * a[0]), dz2 = t[2] * (r01 * a[3]), dz3 = t[3] * (r01 * a[2]);
    const uint32_t h0 = pack_bf16(dz0, dz1), h1 = pack_bf16(dz2, dz3);
    hpk[2 * g] = h0; hpk[2 * g + 1] = h1;
    lpk[2 * g] = pack_bf16(dz0 - __uint_as_float(h0 << 16), dz1 - __uint_as_float(h0 & 0xffff0000u));
    lpk[2 * g + 1] = pack_bf16(dz2 - __uint_as_float(h1 << 16), dz3 - __uint_as_float(h1 & 0xffff0000u));
  }
  return ok;
}

// One k-block (BK / 16 k16 steps) of a warpgroup's 64 x BLOCK_N tile: lo.hi, hi.lo, hi.hi per step, small terms first.
// K-major: 128-byte swizzle at BK = 64, 64-byte swizzle at BK = 32 (rows of BK bf16, 8-row groups SBO apart).
// MN-major: 128-byte swizzle at either BK, 64-element column slabs of BK k-rows (LBO = slab stride 64 BK 2 bytes).
template <int BLOCK_N, int TA, int TB, int BK = BLOCK_K>
__device__ __forceinline__ void mma_kblock(float (&acc)[BLOCK_N / 2], uint32_t sa_hi, uint32_t sa_lo, uint32_t sb_hi, uint32_t sb_lo,
                                           bool first) {
  static_assert(BK == 64 || BK == 32, "k-blocks are 32 or 64 wide");
  constexpr uint32_t kmaj_layout = BK == 64 ? 1u : 2u, kmaj_sbo = BK == 64 ? 1024u : 512u, mn_lbo = 64u * BK * 2u;
  constexpr uint32_t a_layout = TA ? 1u : kmaj_layout, b_layout = TB ? 1u : kmaj_layout;
  constexpr uint32_t a_sbo = TA ? 1024u : kmaj_sbo, b_sbo = TB ? 1024u : kmaj_sbo;
  constexpr uint32_t a_lbo = TA ? mn_lbo : 16u, b_lbo = TB ? mn_lbo : 16u;
  constexpr uint32_t a_step = TA ? 2048u : 32u, b_step = TB ? 2048u : 32u;  // bytes per WGMMA_K
#pragma unroll
  for (int k = 0; k < BK / WGMMA_K; ++k) {
    const uint64_t da_hi = make_desc(sa_hi + k * a_step, a_lbo, a_sbo, a_layout), da_lo = make_desc(sa_lo + k * a_step, a_lbo, a_sbo, a_layout);
    const uint64_t db_hi = make_desc(sb_hi + k * b_step, b_lbo, b_sbo, b_layout), db_lo = make_desc(sb_lo + k * b_step, b_lbo, b_sbo, b_layout);
    const uint32_t sc = (first && k == 0) ? 0u : 1u;
    if constexpr (BLOCK_N == 128) {
      wgmma_n128<TA, TB>(acc, da_lo, db_hi, sc);
      wgmma_n128<TA, TB>(acc, da_hi, db_lo, 1u);
      wgmma_n128<TA, TB>(acc, da_hi, db_hi, 1u);
    } else {
      wgmma_n64<TA, TB>(acc, da_lo, db_hi, sc);
      wgmma_n64<TA, TB>(acc, da_hi, db_lo, 1u);
      wgmma_n64<TA, TB>(acc, da_hi, db_hi, 1u);
    }
  }
}

// 16 consecutive staged accumulator values of one row
__device__ __forceinline__ void stage_ld16(const float* src, uint32_t (&r)[16]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 v = reinterpret_cast<const float4*>(src)[q];
    r[4 * q] = __float_as_uint(v.x); r[4 * q + 1] = __float_as_uint(v.y); r[4 * q + 2] = __float_as_uint(v.z); r[4 * q + 3] = __float_as_uint(v.w);
  }
}

// ---- the two halves of the main loop, shared by the store GEMM and the fused decode

// TMA producer (one lane): fills the STAGES-deep ring with the A and B k-blocks (hi and lo) of every work item of `sched`, in order.
// PAIR = 1: two-CTA cluster sharing the B tile through TMA multicast (see the PTX wrappers above).
// SchedT: Sched, or any walker with the same next(mb, nb, kb0, kb1) (TopkSched).
template <int BLOCK_N, int STAGES, int PAIR, int BK = BLOCK_K, class SchedT>
__device__ __forceinline__ void tma_produce(const GemmParams& p, SchedT& sched, uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                            uint32_t crank, const CUtensorMap* tm_a_hi, const CUtensorMap* tm_a_lo,
                                            const CUtensorMap* tm_b_hi, const CUtensorMap* tm_b_lo, const CUtensorMap* tm_at_hi,
                                            const CUtensorMap* tm_at_lo) {
  constexpr int A_TILE = BLOCK_M * BK * 2;        // bytes of one bf16 A tile (16 KB at BK = 64)
  constexpr int B_TILE = BLOCK_N * BK * 2;
  constexpr int STAGE_BYTES = 2 * A_TILE + 2 * B_TILE;
  int stage = 0; uint32_t phase = 0;
  int mb, nb, kb0, kb1;
  while (sched.next(mb, nb, kb0, kb1)) {
    for (int kb = kb0; kb < kb1; ++kb) {
      if (PAIR) mbar_wait_cluster(&empty_bar[stage], phase ^ 1); else mbar_wait(&empty_bar[stage], phase ^ 1);
      uint8_t* sa_hi = smem + stage * STAGE_BYTES;
      uint8_t* sa_lo = sa_hi + A_TILE;
      uint8_t* sb_hi = sa_lo + A_TILE;
      uint8_t* sb_lo = sb_hi + B_TILE;
      const int mt = PAIR ? mb * 2 + (int)crank : mb;            // this CTA's 128-row m tile
      mbar_expect_tx(&full_bar[stage], STAGE_BYTES);             // PAIR: half of the B bytes come from the peer's multicast
      if (p.a_sym_kb > 0 && kb >= p.a_sym_kb) {      // second half of (A + A^T).B: the same square array read M-contiguous
#pragma unroll
        for (int j = 0; j < BLOCK_M / 64; ++j) {
          tma_load_2d(tm_at_hi, &full_bar[stage], sa_hi + j * (64 * BK * 2), mt * BLOCK_M + j * 64, (kb - p.a_sym_kb) * BK);
          tma_load_2d(tm_at_lo, &full_bar[stage], sa_lo + j * (64 * BK * 2), mt * BLOCK_M + j * 64, (kb - p.a_sym_kb) * BK);
        }
      } else if (!p.a_mn) {
        tma_load_2d(tm_a_hi, &full_bar[stage], sa_hi, kb * BK, mt * BLOCK_M);
        tma_load_2d(tm_a_lo, &full_bar[stage], sa_lo, kb * BK, mt * BLOCK_M);
      } else {
#pragma unroll
        for (int j = 0; j < BLOCK_M / 64; ++j) {
          tma_load_2d(tm_a_hi, &full_bar[stage], sa_hi + j * (64 * BK * 2), mt * BLOCK_M + j * 64, kb * BK);
          tma_load_2d(tm_a_lo, &full_bar[stage], sa_lo + j * (64 * BK * 2), mt * BLOCK_M + j * 64, kb * BK);
        }
      }
      const int kbb = (p.a_sym_kb > 0 && kb >= p.a_sym_kb) ? kb - p.a_sym_kb : kb;   // B's k block
      if (PAIR) {   // this CTA's 64-row half of the B tile, into both CTAs (K-major: rows 64 crank..; MN-major: slab crank)
        const int off = (int)crank * 8192, n_half = nb * BLOCK_N + (int)crank * 64;
        if (!p.b_mn) {
          tma_load_2d_mc(tm_b_hi, &full_bar[stage], sb_hi + off, kbb * BK, n_half, 0x3);
          tma_load_2d_mc(tm_b_lo, &full_bar[stage], sb_lo + off, kbb * BK, n_half, 0x3);
        } else {
          tma_load_2d_mc(tm_b_hi, &full_bar[stage], sb_hi + off, n_half, kbb * BK, 0x3);
          tma_load_2d_mc(tm_b_lo, &full_bar[stage], sb_lo + off, n_half, kbb * BK, 0x3);
        }
      } else if (!p.b_mn) {
        tma_load_2d(tm_b_hi, &full_bar[stage], sb_hi, kbb * BK, nb * BLOCK_N);
        tma_load_2d(tm_b_lo, &full_bar[stage], sb_lo, kbb * BK, nb * BLOCK_N);
      } else {
#pragma unroll
        for (int j = 0; j < BLOCK_N / 64; ++j) {
          tma_load_2d(tm_b_hi, &full_bar[stage], sb_hi + j * (64 * BK * 2), nb * BLOCK_N + j * 64, kbb * BK);
          tma_load_2d(tm_b_lo, &full_bar[stage], sb_lo + j * (64 * BK * 2), nb * BLOCK_N + j * 64, kbb * BK);
        }
      }
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
  }
}

// The k-blocks [kb0, kb1) of one work item for MMA warpgroup wg (rows [64 wg, 64 wg + 64) of the tile): wgmma into acc, each ring stage
// released to the producer (of both CTAs of a pair) once its wgmma have retired.  stage / phase carry the ring position across work items.
// MAJ: bit 0 = A MN-major, bit 1 = B MN-major, bit 2 = (A + A^T).B (A K-major for k-blocks < a_sym_kb, MN-major after).  A
// compile-time constant, because a runtime choice between wgmma variants inside the k loop makes ptxas serialise the wgmma.
template <int BLOCK_N, int STAGES, int PAIR, int MAJ, int BK = BLOCK_K>
__device__ __forceinline__ void mma_work_item(float (&acc)[BLOCK_N / 2], const GemmParams& p, uint8_t* smem, uint64_t* full_bar,
                                              uint64_t* empty_bar, int wg, int lane, uint32_t crank, int& stage, uint32_t& phase,
                                              int kb0, int kb1) {
  constexpr int A_TILE = BLOCK_M * BK * 2;
  constexpr int B_TILE = BLOCK_N * BK * 2;
  constexpr int STAGE_BYTES = 2 * A_TILE + 2 * B_TILE;
  auto release = [&](int s) {   // this warp is done reading ring stage s (its wgmma have retired)
    __syncwarp();
    if (lane == 0) { mbar_arrive(&empty_bar[s]); if (PAIR) mbar_arrive_cluster(&empty_bar[s], crank ^ 1u); }
  };
  int prev = -1;
  auto run_k = [&](auto ta, auto tb, int kb_begin, int kb_end) {   // k-blocks [kb_begin, kb_end) with fixed majorness
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa_hi = smem_u32(smem + stage * STAGE_BYTES) + wg * (64 * BK * 2);   // K-major: 64 rows x 2 BK B; MN-major: slab wg
      const uint32_t sa_lo = sa_hi + A_TILE;
      const uint32_t sb_hi = smem_u32(smem + stage * STAGE_BYTES) + 2 * A_TILE, sb_lo = sb_hi + B_TILE;
      wgmma_fence();
      mma_kblock<BLOCK_N, decltype(ta)::value, decltype(tb)::value, BK>(acc, sa_hi, sa_lo, sb_hi, sb_lo, kb == kb0);
      wgmma_commit();
      wgmma_wait<1>();                     // the previous k-block's wgmma have retired: its stage can be refilled
      if (prev >= 0) release(prev);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
  };
  using K0 = std::integral_constant<int, 0>;
  using K1 = std::integral_constant<int, 1>;
  if constexpr ((MAJ & 4) != 0) {
    run_k(K0{}, K1{}, kb0, min(kb1, p.a_sym_kb));
    run_k(K1{}, K1{}, max(kb0, p.a_sym_kb), kb1);
  } else {
    run_k(std::integral_constant<int, MAJ & 1>{}, std::integral_constant<int, (MAJ >> 1) & 1>{}, kb0, kb1);
  }
  wgmma_wait<0>();
  if (prev >= 0) release(prev);
}

// ---------------------------------------------------------------------------------------------------------------------
// store GEMM: C (+)= alpha A.B, 384 threads = producer + two consumer warpgroups that run the main loop and then the store epilogue
// ---------------------------------------------------------------------------------------------------------------------
template <int BLOCK_N, int STAGES, int PAIR, int MAJ, int BK = BLOCK_K>
__global__ void __launch_bounds__(kThreads, 1) gemm_bf16x3_kernel(const __grid_constant__ CUtensorMap tm_a_hi,
                                                                   const __grid_constant__ CUtensorMap tm_a_lo,
                                                                   const __grid_constant__ CUtensorMap tm_b_hi,
                                                                   const __grid_constant__ CUtensorMap tm_b_lo,
                                                                   const __grid_constant__ CUtensorMap tm_at_hi,   // A^T views (a_sym_kb > 0)
                                                                   const __grid_constant__ CUtensorMap tm_at_lo,
                                                                   const GemmParams p) {
  static_assert(!PAIR || BLOCK_N == 128, "CTA pairs split the B tile into two 64-row halves");
  constexpr int STAGE_BYTES = 2 * BLOCK_M * BK * 2 + 2 * BLOCK_N * BK * 2;
  constexpr int SROW = BLOCK_N + 4;               // staging row stride (floats): conflict-free 16-byte row reads
  constexpr int kParts = 2;                       // column parts per tile (one per epilogue warp of a 32-row quarter)
  constexpr int HALF_N = BLOCK_N / kParts;        // columns handled by one epilogue warp
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* stg = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);   // [BLOCK_M][SROW] accumulator staging
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  Sched sched;
  sched.init(p, BLOCK_N, PAIR, BK);
  const uint32_t crank = PAIR ? cluster_ctarank() : 0u;

  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tm_a_hi); prefetch_tmap(&tm_a_lo); prefetch_tmap(&tm_b_hi); prefetch_tmap(&tm_b_lo);
    if (p.a_sym_kb > 0) { prefetch_tmap(&tm_at_hi); prefetch_tmap(&tm_at_lo); }
  }
  if (warp == 1 && lane == 0) {
    // empty: one arrival per consumer warp (of both CTAs of a pair)
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], PAIR ? 16 : 8); }
    fence_barrier_init();
  }
  if (PAIR) cluster_sync_all(); else __syncthreads();   // the peer's barriers must be initialised before anything signals them

  if (warp == 0) {
    if (lane == 0)
      tma_produce<BLOCK_N, STAGES, PAIR, BK>(p, sched, smem, full_bar, empty_bar, crank, &tm_a_hi, &tm_a_lo, &tm_b_hi, &tm_b_lo, &tm_at_hi,
                                         &tm_at_lo);
  } else if (warp >= 4) {
    // ===================== consumers: wgmma main loop, then the store epilogue =====================
    const int wg = (warp >> 2) - 1;          // consumer warpgroup: rows [64 wg, 64 wg + 64) of the tile
    const int wi = warp & 3;                 // warp within the warpgroup
    const int quarter = wg * 2 + (wi & 1);   // 32-row quarter of the tile this warp's epilogue handles
    const int half = wi >> 1;                // which column part of the tile
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.0f;
    int stage = 0; uint32_t phase = 0;
    int mb, nb, kb0, kb1;
    int seg = 0;                             // segments of this CTA so far (deterministic stream-K: slot of a partial tile)
    while (sched.next(mb, nb, kb0, kb1)) {
      if (PAIR) mb = mb * 2 + (int)crank;     // this CTA's 128-row m tile of the pair
      mma_work_item<BLOCK_N, STAGES, PAIR, MAJ, BK>(acc, p, smem, full_bar, empty_bar, wg, lane, crank, stage, phase, kb0, kb1);
      float* ws_tile = nullptr;              // partial tile of the deterministic mode: goes to the CTA's workspace slot
      if (p.sk_ws != nullptr && !(kb0 == 0 && kb1 == sched.kb_total))
        ws_tile = p.sk_ws + ((int64_t)blockIdx.x * 2 + (seg == 0 ? 0 : 1)) * (BLOCK_M * BLOCK_N);
      ++seg;

      // accumulators -> staging rows (the previous tile's epilogue of this warpgroup must be done with them)
      named_bar_sync(1 + wg, 128);
      {
        const int r0 = wg * 64 + wi * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < BLOCK_N / 8; ++j) {
          *reinterpret_cast<float2*>(&stg[r0 * SROW + 8 * j + c0]) = make_float2(acc[4 * j], acc[4 * j + 1]);
          *reinterpret_cast<float2*>(&stg[(r0 + 8) * SROW + 8 * j + c0]) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
      }
      named_bar_sync(1 + wg, 128);
      const int n0 = nb * BLOCK_N + half * HALF_N;
      const float* tr = stg + (quarter * 32) * SROW + half * HALF_N;   // the warp's 32 rows
      const int m_base = mb * BLOCK_M + quarter * 32;
      const bool vec_ok = ((p.ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0);
#pragma unroll 1
      for (int c = 0; c < HALF_N / 16; ++c) {
        const int nc = n0 + c * 16;   // first column of this 16-wide chunk
        if (ws_tile != nullptr) {     // deterministic stream-K: the whole 32 x 16 block, scaled, into the slot (rows of 64 B)
          const int rsub = lane >> 4, csub = lane & 15;
          float* dst = ws_tile + (int64_t)(quarter * 32) * BLOCK_N + half * HALF_N + c * 16 + csub;
#pragma unroll 4
          for (int i = 0; i < 16; ++i) {
            const int rr = 2 * i + rsub;
            dst[(int64_t)rr * BLOCK_N] = p.alpha * tr[rr * SROW + c * 16 + csub];
          }
          continue;
        }
        const bool interior = vec_ok && (m_base + 32 <= p.M) && (nc + 16 <= p.n_store) && (p.special_col < nc || p.special_col >= nc + 16);
        if (interior) {               // fast path: 8 rows x 64 B per store instruction, 128-bit accesses
          const int rsub = lane >> 2, c4 = (lane & 3) * 4;
          float* dst = p.C + (int64_t)(m_base + rsub) * p.ldc + nc + c4;
          const int64_t step = 8 * p.ldc;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            float4 v = *reinterpret_cast<const float4*>(&tr[(rsub + 8 * i) * SROW + c * 16 + c4]);
            v.x *= p.alpha; v.y *= p.alpha; v.z *= p.alpha; v.w *= p.alpha;
            if (p.atomic) atomicAdd(reinterpret_cast<float4*>(dst), v); else *reinterpret_cast<float4*>(dst) = v;
            dst += step;
          }
        } else {                      // edge tiles / the [dW | dbv] column / unaligned C
          const int rsub = lane >> 4, csub = lane & 15;
          const int n = nc + csub;
          for (int i = 0; i < 16; ++i) {
            const int rr = 2 * i + rsub;
            const int mm = m_base + rr;
            const float v = p.alpha * tr[rr * SROW + c * 16 + csub];
            if (mm < p.M) {
              if (n == p.special_col) {
                if (p.atomic) atomicAdd(p.special_out + mm, v); else p.special_out[mm] = v;
              } else if (n < p.n_store) {
                float* dst = p.C + (int64_t)mm * p.ldc + n;
                if (p.atomic) atomicAdd(dst, v); else *dst = v;
              }
            }
          }
        }
      }
    }
  }

  if (PAIR) cluster_sync_all();   // nobody leaves while the peer may still multicast into this CTA or arrive on its barriers
}

// ---------------------------------------------------------------------------------------------------------------------
// fused decode: D = g(E.W^T + bv), row loss, dZ (bf16 hi / lo), 640 threads = five warpgroups with one role each
//   warpgroup 0   : TMA producer (one lane), as in the store GEMM
//   warpgroups 1-2: MMA   -- rows [64 h, 64 h + 64) of the tile (h = warpgroup - 1): the wgmma main loop only; the finished accumulators
//                   go to their half of the staging tile, and the warpgroup starts on the next tile at once
//   warpgroups 3-4: epilogue -- the loss epilogue of staging half h = warpgroup - 3, one batch row per thread
// Each staging half is handed over through an mbarrier pair: staged[h] (4 arrivals: the MMA warps of half h have written it) and
// drained[h] (4 arrivals: the epilogue warps of half h have read it), with the same phase discipline as the operand ring.  So the
// epilogue of tile i runs while the tensor cores accumulate tile i + 1, and a tile costs max(MMA, epilogue) instead of their sum.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kDecodeThreads = 640;
// Operand ring of 32-wide k-blocks (64B swizzle, 32 KB per stage) x 4 stages: the same 128 KB as 2 stages of 64, but three stages
// (96 KB) in flight behind the one being multiplied instead of one (64 KB).  With K = H = 500 the main loop waits on L2 -> shared
// memory latency, not on the tensor cores, so the extra bytes in flight shorten it (H100 SXM, C2: 95 -> 76 us per launch).
constexpr int kDecodeBK = 32;
constexpr int kDecodeStages = 4;
// setmaxnreg budgets (the launch gives every thread 65536 / 640 -> 96 registers; the sum may not exceed 640 x 96): the producer
// needs next to nothing, the MMA warps keep 64 accumulators + descriptors, the epilogue warps take the rest
constexpr int kRegsProducer = 32, kRegsMma = 104, kRegsEpilogue = 120;
static_assert(128 * kRegsProducer + 256 * kRegsMma + 256 * kRegsEpilogue <= kDecodeThreads * 96, "register budget");

template <int R> __device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

template <int ACT, int LOSS>
__global__ void __launch_bounds__(kDecodeThreads, 1) decode_fused_kernel(const __grid_constant__ CUtensorMap tm_a_hi,
                                                                         const __grid_constant__ CUtensorMap tm_a_lo,
                                                                         const __grid_constant__ CUtensorMap tm_b_hi,
                                                                         const __grid_constant__ CUtensorMap tm_b_lo,
                                                                         const GemmParams p) {
  constexpr int BLOCK_N = kDecodeN, STAGES = kDecodeStages, BK = kDecodeBK;
  constexpr int STAGE_BYTES = 2 * BLOCK_M * BK * 2 + 2 * BLOCK_N * BK * 2;
  constexpr int SROW = BLOCK_N + 4;               // staging row stride (floats): conflict-free 16-byte row reads
  constexpr int kParts = 2;                       // column parts per tile (one per epilogue warp of a 32-row quarter)
  constexpr int HALF_N = BLOCK_N / kParts;        // columns handled by one epilogue warp
  constexpr bool kFast = (ACT == DAE_ACT_SIGMOID) && (LOSS == DAE_LOSS_CE);
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* stg = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);   // [BLOCK_M][SROW] accumulator staging
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES], staged_bar[2], drained_bar[2];
  __shared__ float s_bias[2][BLOCK_N];            // per epilogue warpgroup
  __shared__ float s_biasc[kFast ? 2 : 1][kFast ? BLOCK_N : 1];   // bv * log2(e) for the sigmoid/CE fast path
  __shared__ __align__(16) uint8_t s_stage[8][2][32][48];  // per epilogue warp: bf16 hi / lo dZ blocks [32 rows x 16 cols], rows padded to 48 B

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int role = warp >> 2;                     // warpgroup: 0 producer, 1-2 MMA, 3-4 epilogue
  Sched sched;                                    // initialised by each role after its register budget is set

  if (warp == 0 && lane == 0) { prefetch_tmap(&tm_a_hi); prefetch_tmap(&tm_a_lo); prefetch_tmap(&tm_b_hi); prefetch_tmap(&tm_b_lo); }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }   // empty: one arrival per MMA warp
    for (int h = 0; h < 2; ++h) { mbar_init(&staged_bar[h], 4); mbar_init(&drained_bar[h], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (role == 0) {
    // ===================== TMA producer =====================
    regs_dec<kRegsProducer>();
    sched.init(p, BLOCK_N, 0, BK);
    if (warp == 0 && lane == 0)
      tma_produce<BLOCK_N, STAGES, 0, BK>(p, sched, smem, full_bar, empty_bar, 0u, &tm_a_hi, &tm_a_lo, &tm_b_hi, &tm_b_lo, &tm_a_hi, &tm_a_lo);
  } else if (role <= 2) {
    // ===================== MMA: wgmma main loop -> staging half =====================
    regs_inc<kRegsMma>();
    sched.init(p, BLOCK_N, 0, BK);
    const int h = role - 1;
    const int wi = warp & 3;
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.0f;
    int stage = 0; uint32_t phase = 0, tphase = 0;
    int mb, nb, kb0, kb1;
    while (sched.next(mb, nb, kb0, kb1)) {
      mma_work_item<BLOCK_N, STAGES, 0, 0, BK>(acc, p, smem, full_bar, empty_bar, h, lane, 0u, stage, phase, kb0, kb1);
      mbar_wait(&drained_bar[h], tphase ^ 1);   // the epilogue is done with the previous tile's rows
      const int r0 = h * 64 + wi * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        *reinterpret_cast<float2*>(&stg[r0 * SROW + 8 * j + c0]) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(&stg[(r0 + 8) * SROW + 8 * j + c0]) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&staged_bar[h]);
      tphase ^= 1;
    }
  } else {
    // ===================== epilogue: D = g(Z + bv); row loss; dZ -> bf16 hi/lo (autoencoder.py:411, triplet_loss_utils.py:269-275)
    regs_inc<kRegsEpilogue>();
    sched.init(p, BLOCK_N, 0, BK);
    const int h = role - 3;                  // staging half: rows [64 h, 64 h + 64)
    const int ew = warp - 12;                // epilogue warp 0..7 (its dZ transpose buffer)
    const int wi = warp & 3;
    const int quarter = h * 2 + (wi & 1);    // 32-row quarter of the tile this warp handles
    const int half = wi >> 1;                // which column part of the tile
    const int row_in_tile = quarter * 32 + lane;
    const int tid = threadIdx.x - 128 * role;
    const int tiles_n = (p.N + BLOCK_N - 1) / BLOCK_N;
    uint8_t* stg_hi = reinterpret_cast<uint8_t*>(&s_stage[ew][0][0][0]);
    uint8_t* stg_lo = reinterpret_cast<uint8_t*>(&s_stage[ew][1][0][0]);
    const int rsub = lane >> 1, csub = lane & 1;          // write-out mapping: 16 rows x 2 x 16 B per instruction
    uint32_t tphase = 0;
    int mb, nb, kb0, kb1;
    while (sched.next(mb, nb, kb0, kb1)) {
      const float* srow = stg + row_in_tile * SROW + half * HALF_N;   // this thread's row, this warp's column part
      const int m = mb * BLOCK_M + row_in_tile;
      const int n0 = nb * BLOCK_N + half * HALF_N;
      // 99 % of a bag-of-words target row is zero, so each 16-column chunk is first evaluated branch-free as if x == 0,
      // stored, and then the row's few stored entries inside the chunk are re-evaluated exactly and patched in place.  The clean
      // CSR row is walked with a cursor (columns are sorted) that keeps the next THREE entries (c0,v0),(c1,v1),(c2,v2) in
      // registers.  The cursor, the row scale and the bias slice depend only on the tile's coordinates, so they are loaded
      // while the MMA warps are still accumulating this tile.
      int64_t pc = 0, pe = 0;
      int c0 = 0x7fffffff, c1 = 0x7fffffff, c2 = 0x7fffffff;
      float v0 = 0.0f, v1 = 0.0f, v2 = 0.0f;
      float sc = 0.0f;
      if (m < p.M) {
        const int64_t row = p.rows ? (int64_t)p.rows[m] : (int64_t)m;
        const int64_t rbeg = p.indptr[row];
        const int32_t* tp = p.tile_ptr + (int64_t)m * (kParts * tiles_n + 1) + nb * kParts + half;
        pc = rbeg + tp[0]; pe = rbeg + tp[1];     // entries of this row that fall into this half tile
        if (pc < pe) { c0 = p.indices[pc]; v0 = p.values[pc]; }
        if (pc + 1 < pe) { c1 = p.indices[pc + 1]; v1 = p.values[pc + 1]; }
        if (pc + 2 < pe) { c2 = p.indices[pc + 2]; v2 = p.values[pc + 2]; }
        sc = (p.weight ? p.weight[m] : 1.0f) / ((float)p.stats[DAE_STAT_SUM_W] + kEps);
      }
      named_bar_sync(1 + h, 128);   // every warp of this warpgroup is done with the previous tile's bias slice
      {  // this tile's visible-bias slice (BLOCK_N = 128 = one column per thread)
        const float b = (nb * BLOCK_N + tid < p.N) ? p.bv[nb * BLOCK_N + tid] : 0.0f;
        s_bias[h][tid] = b;
        if (kFast) s_biasc[h][tid] = b * kLog2e;
      }
      mbar_wait(&staged_bar[h], tphase);
      named_bar_sync(1 + h, 128);
      const float inv_sc = (sc != 0.0f) ? 1.0f / sc : 0.0f;
      const bool edge = (n0 + HALF_N > p.N);   // only the last column tile has out-of-range columns
      float lsum = 0.0f;   // CE: accumulated in log2 units, scaled by ln2 at the end
      // dZ leaves through a per-warp shared-memory transpose: each thread (= batch row) drops the bf16 hi and lo parts of its
      // 16 values into its two staging rows (patching the row's stored entries there), then the warp writes both 32 x 16
      // blocks with full 32-byte sectors (16 rows per store instruction).
      const int m_base = mb * BLOCK_M + quarter * 32;
      const int n_lim = edge ? p.N : 0x7fffffff;
#pragma unroll 1
      for (int c = 0; c < HALF_N / 16; ++c) {
        uint32_t r[16];
        stage_ld16(srow + c * 16, r);
        const int nc = n0 + c * 16;
        if (m < p.M) {
          const float* bias = &s_bias[h][half * HALF_N + c * 16];
          uint32_t hpk[8], lpk[8];
          bool fast_ok = false;   // this chunk went through the sigmoid/CE fast path: staged dZ = sc * D exactly
          if (kFast && !edge) {
            const float l0 = lsum;
            fast_ok = decode_chunk_sigmoid_ce(r, &s_biasc[h][half * HALF_N + c * 16], sc, hpk, lpk, lsum);
            if (!fast_ok) { lsum = l0; decode_chunk_generic<ACT, LOSS>(r, bias, sc, edge, n_lim, nc, hpk, lpk, lsum); }
          } else {
            decode_chunk_generic<ACT, LOSS>(r, bias, sc, edge, n_lim, nc, hpk, lpk, lsum);
          }
          uint4* sh = reinterpret_cast<uint4*>(stg_hi + lane * 48);
          uint4* sl = reinterpret_cast<uint4*>(stg_lo + lane * 48);
          sh[0] = make_uint4(hpk[0], hpk[1], hpk[2], hpk[3]); sh[1] = make_uint4(hpk[4], hpk[5], hpk[6], hpk[7]);
          sl[0] = make_uint4(lpk[0], lpk[1], lpk[2], lpk[3]); sl[1] = make_uint4(lpk[4], lpk[5], lpk[6], lpk[7]);
          // exact re-evaluation of the stored entries of this row inside the group (densified target, :264)
          while (c0 < nc + 16) {
            const float x = v0;
            const int j = c0 - nc;
            __nv_bfloat16* ph = reinterpret_cast<__nv_bfloat16*>(stg_hi + lane * 48) + j;
            __nv_bfloat16* pl = reinterpret_cast<__nv_bfloat16*>(stg_lo + lane * 48) + j;
            float d;
            if (kFast && fast_ok && sc != 0.0f) d = (__bfloat162float(*ph) + __bfloat162float(*pl)) * inv_sc;   // D back from the staged sc * D
            else d = act_fast<ACT>(select16(r, j) + bias[j]);
            const float gp = act_grad_from_y<ACT>(d);
            float dz;
            if (LOSS == DAE_LOSS_CE) {
              const float a = d + kEps, b = (1.0f - d) + kEps;
              const float la = f_lg2(a), lb = f_lg2(b);
              lsum += lb - (x * la + (1.0f - x) * lb);      // replace the x == 0 term by the exact one
              dz = sc * gp * ((1.0f - x) * f_rcp(b) - x * f_rcp(a));
            } else {
              const float e2 = x - d;
              lsum += e2 * e2 - d * d;
              dz = -2.0f * sc * e2 * gp;
            }
            const __nv_bfloat16 hb = __float2bfloat16_rn(dz);
            *ph = hb;
            *pl = __float2bfloat16_rn(dz - __bfloat162float(hb));
            ++pc;
            c0 = c1; v0 = v1; c1 = c2; v1 = v2;
            c2 = 0x7fffffff;
            if (pc + 2 < pe) { c2 = p.indices[pc + 2]; v2 = p.values[pc + 2]; }
          }
        }
        __syncwarp();
        if (nc < p.ld_dz) {  // ld_dz is a multiple of 32 (launcher), so whole 16-column groups are in range
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int rr = rsub + 16 * i;
            if (m_base + rr < p.M) {
              const int64_t off = (int64_t)(m_base + rr) * p.ld_dz + nc + csub * 8;
              *reinterpret_cast<uint4*>(p.dz_hi + off) = *reinterpret_cast<const uint4*>(stg_hi + rr * 48 + csub * 16);
              *reinterpret_cast<uint4*>(p.dz_lo + off) = *reinterpret_cast<const uint4*>(stg_lo + rr * 48 + csub * 16);
            }
          }
        }
        __syncwarp();
      }
      if (lane == 0) mbar_arrive(&drained_bar[h]);   // this warp's staging rows may be overwritten (the loop ends in __syncwarp)
      tphase ^= 1;
      if (m < p.M) {   // 2 * tiles_n partials per row
        const float l = (LOSS == DAE_LOSS_CE) ? lsum * 0.6931471805599453f : lsum;
        if (p.loss_parts) p.row_loss_part[(int64_t)(nb * kParts + half) * p.M + m] = l;
        else atomicAdd(p.row_loss_part + m, l);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// fused similarity + k-best selection (dae_similarity_topk_bf16x3): for every query row i the k largest S[i, j] = Q_i . C_j and their
// corpus indices, without writing S.  The five warpgroups, register split and staged / drained hand-off of the fused decode; the
// schedule, the epilogue and the shape of the operand ring differ.
//   work item: (128-row block of Q, contiguous range of column tiles) -- split s of `splits`.  A CTA sweeps its range left to right
//              and its epilogue threads keep their running lists over the whole sweep.
//   epilogue : thread = (row, 64-column half of every tile), as in the decode.  A list of KMAX (score, index) pairs sorted by
//              (score desc, index asc) lives in registers, every index into it unrolled.  Four staged values cost one compare
//              against the current k-th score; only a value that beats it is inserted.  Columns arrive in increasing order and an
//              equal score never displaces an entry, so among equal scores the lower index stays first.  At the end of the item
//              the first k entries go to the workspace (2 * splits lists per row) and topk_merge_kernel merges them.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kTopkMaxK = 32;
constexpr int kTopkMaxSplits = 32;   // 2 * splits lists per row: at most two per lane of the merging warp
constexpr int kTopkMinTiles = 4;     // automatic splits sweep at least this many column tiles (amortises the list flush)
// Operand ring: 2 stages of 64-wide k-blocks (128B swizzle, 64 KB each), as the store GEMM, not the decode's 4 x 32.  Measured on an
// H100 SXM (700 W) at Nq = Nc = 100 000, H = 500, k = 10: 81 ms per call with 2 x 64, 92 ms with 3 x 32, 113 ms with 4 x 32.
constexpr int kTopkBK = 64;
constexpr int kTopkStages = 2;

struct TopkParams {
  GemmParams g;                      // M = queries, N = corpus rows, K = dim
  int k, splits;
  int exclude;                       // != 0: column i + diag_offset is not a candidate of row i
  int64_t diag_offset;
  float* ws_val; int32_t* ws_idx;    // [M x 2 splits x k] partial lists
  // topk_kernel<KMAX, true>: per-row exclusion lists (CSR structure, rows sorted, no duplicates, indices in [0, N)).  Last, so the
  // fields above keep their parameter offsets in the plain instantiations.
  const int64_t* ex_indptr; const int32_t* ex_indices;
  // topk_kernel<KMAX, true, true>: groups[c] >= 0 is corpus row c's group label; only one row per group enters a list
  const int32_t* groups;
};

// (row block, column-tile range) work items, items blockIdx.x, blockIdx.x + gridDim.x, ...; next() returns one column tile at a time,
// with `first` / `last` marking the ends of an item.  Every range is non-empty (the launcher keeps splits <= column tiles).
struct TopkSched {
  int tiles_n, splits, kb_total, n_work, n_cta, w;
  int mb, split, t, t_end;
  bool first, last;
  __device__ __forceinline__ void init(const TopkParams& tp, int block_n, int block_k) {
    const int tiles_m = (tp.g.M + BLOCK_M - 1) / BLOCK_M;
    tiles_n = (tp.g.N + block_n - 1) / block_n;
    splits = tp.splits;
    kb_total = (tp.g.K + block_k - 1) / block_k;
    n_work = tiles_m * splits;
    n_cta = (int)gridDim.x;
    w = (int)blockIdx.x - n_cta;
    mb = split = t = t_end = 0;
    first = last = false;
  }
  __device__ __forceinline__ bool next(int& mb_, int& nb, int& kb0, int& kb1) {
    first = false;
    if (t >= t_end) {
      w += n_cta;
      if (w >= n_work) return false;
      mb = w / splits;
      split = w - mb * splits;
      t = split * tiles_n / splits;                 // 32-bit: splits <= 32 and tiles_n < 2^24
      t_end = (split + 1) * tiles_n / splits;
      first = true;
    }
    mb_ = mb; nb = t; kb0 = 0; kb1 = kb_total;
    last = (++t == t_end);
    return true;
  }
};

// offer (v, col) to a sorted list whose k-th score is thr: inserted if it beats thr and is a candidate
template <int KMAX>
__device__ __forceinline__ void topk_offer(float (&sv)[KMAX], int (&si)[KMAX], float& thr, int k, float v, int col, int n_lim,
                                           int excl) {
  if (!(v > thr) || col >= n_lim || col == excl) return;
#pragma unroll
  for (int j = KMAX - 1; j >= 0; --j) {   // downwards: sv[j - 1] still holds its old value when entry j is rewritten
    const bool up = (j > 0) && (v > sv[j > 0 ? j - 1 : 0]);
    const bool here = v > sv[j];
    si[j] = up ? si[j > 0 ? j - 1 : 0] : (here ? col : si[j]);
    sv[j] = up ? sv[j > 0 ? j - 1 : 0] : (here ? v : sv[j]);
  }
  // thr = sv[k - 1].  The select is PTX so that the compiler cannot fold the unrolled chain back into a dynamic index, which
  // would move sv to local memory.
  float t = sv[0];
#pragma unroll
  for (int j = 1; j < KMAX; ++j)
    asm("{\n.reg .pred q;\nsetp.eq.s32 q, %1, %2;\nselp.f32 %0, %3, %0, q;\n}\n" : "+f"(t) : "r"(j), "r"(k - 1), "f"(sv[j]));
  thr = t;
}

// GROUPS: offer (v, col) of group g to a list whose first k entries hold distinct groups, each its best so far.  If entry gp < k
// holds g, v replaces it only if it beats it, moving up over the entries in between (entries after gp stay); otherwise (v, col)
// goes through the ordinary insert.  Slots k..KMAX-1 hold shifted-out entries and never block a group: a group whose best left the
// first k can only come back above thr, and then that value is its best so far.  The entries' groups live in registers (sg, REG)
// or are reloaded from `groups` on this rare path (!REG: KMAX = 32, whose 64-register list leaves no room for 32 more).
template <int KMAX, bool REG>
__device__ __forceinline__ void topk_offer_group(float (&sv)[KMAX], int (&si)[KMAX], int (&sg)[REG ? KMAX : 1], float& thr, int k,
                                                 float v, int col, int g, int n_lim, int excl, const int32_t* __restrict__ groups) {
  if (!(v > thr) || col >= n_lim || col == excl) return;
  int gp = KMAX - 1;                      // the last entry that may move
  bool drop = false;
#pragma unroll
  for (int j = 0; j < KMAX; ++j) {
    if (j < k) {
      const int gj = REG ? sg[REG ? j : 0] : (si[j] >= 0 ? __ldg(groups + si[j]) : -1);
      if (gj == g) { gp = j; drop = !(v > sv[j]); }
    }
  }
  if (drop) return;
#pragma unroll
  for (int j = KMAX - 1; j >= 0; --j) {   // topk_offer's update, on entries 0..gp only
    const bool up = (j > 0) && j <= gp && (v > sv[j > 0 ? j - 1 : 0]);
    const bool here = j <= gp && v > sv[j];
    si[j] = up ? si[j > 0 ? j - 1 : 0] : (here ? col : si[j]);
    if constexpr (REG) sg[REG ? j : 0] = up ? sg[REG && j > 0 ? j - 1 : 0] : (here ? g : sg[REG ? j : 0]);
    sv[j] = up ? sv[j > 0 ? j - 1 : 0] : (here ? v : sv[j]);
  }
  float t = sv[0];
#pragma unroll
  for (int j = 1; j < KMAX; ++j)
    asm("{\n.reg .pred q;\nsetp.eq.s32 q, %1, %2;\nselp.f32 %0, %3, %0, q;\n}\n" : "+f"(t) : "r"(j), "r"(k - 1), "f"(sv[j]));
  thr = t;
}

// EXCL: the columns in row m's exclusion list are never candidates.  Before scanning a tile, the epilogue thread writes -inf over
// the listed columns of its own (row, 64-column half) staging run -- its alone until it arrives on `drained` -- and -inf never beats
// thr.  A cursor into the sorted list, placed by binary search at the item's first column, only moves forward during the item; the
// next listed column waits in a register, so a tile without a listed column costs one compare.
// GROUPS (with EXCL; ex_indptr may be null: no lists): the list holds the k best group representatives of the columns seen
// (topk_offer_group), the groups of its entries in registers.  Each epilogue warp copies the labels of its 64 columns of the tile
// to shared memory, as pair_hist_kernel does; they are read only on the rare path behind the unchanged `max > thr` filter.
template <int KMAX, bool EXCL = false, bool GROUPS = false>
__global__ void __launch_bounds__(kDecodeThreads, 1) topk_kernel(const __grid_constant__ CUtensorMap tm_a_hi,
                                                                 const __grid_constant__ CUtensorMap tm_a_lo,
                                                                 const __grid_constant__ CUtensorMap tm_b_hi,
                                                                 const __grid_constant__ CUtensorMap tm_b_lo,
                                                                 const TopkParams tp) {
  constexpr int BLOCK_N = kDecodeN, STAGES = kTopkStages, BK = kTopkBK;
  constexpr int STAGE_BYTES = 2 * BLOCK_M * BK * 2 + 2 * BLOCK_N * BK * 2;
  constexpr int SROW = BLOCK_N + 4;               // staging row stride (floats): conflict-free 16-byte row reads
  constexpr int HALF_N = BLOCK_N / 2;             // columns handled by one epilogue thread per tile
  const GemmParams& p = tp.g;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* stg = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);   // [BLOCK_M][SROW] accumulator staging
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES], staged_bar[2], drained_bar[2];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int role = warp >> 2;                     // warpgroup: 0 producer, 1-2 MMA, 3-4 epilogue
  TopkSched sched;

  if (warp == 0 && lane == 0) { prefetch_tmap(&tm_a_hi); prefetch_tmap(&tm_a_lo); prefetch_tmap(&tm_b_hi); prefetch_tmap(&tm_b_lo); }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    for (int h = 0; h < 2; ++h) { mbar_init(&staged_bar[h], 4); mbar_init(&drained_bar[h], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (role == 0) {
    // ===================== TMA producer =====================
    regs_dec<kRegsProducer>();
    sched.init(tp, BLOCK_N, BK);
    if (warp == 0 && lane == 0)
      tma_produce<BLOCK_N, STAGES, 0, BK>(p, sched, smem, full_bar, empty_bar, 0u, &tm_a_hi, &tm_a_lo, &tm_b_hi, &tm_b_lo, &tm_a_hi, &tm_a_lo);
  } else if (role <= 2) {
    // ===================== MMA: wgmma main loop -> staging half =====================
    regs_inc<kRegsMma>();
    sched.init(tp, BLOCK_N, BK);
    const int h = role - 1;
    const int wi = warp & 3;
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.0f;
    int stage = 0; uint32_t phase = 0, tphase = 0;
    int mb, nb, kb0, kb1;
    while (sched.next(mb, nb, kb0, kb1)) {
      mma_work_item<BLOCK_N, STAGES, 0, 0, BK>(acc, p, smem, full_bar, empty_bar, h, lane, 0u, stage, phase, kb0, kb1);
      mbar_wait(&drained_bar[h], tphase ^ 1);   // the epilogue is done with the previous tile's rows
      const int r0 = h * 64 + wi * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        *reinterpret_cast<float2*>(&stg[r0 * SROW + 8 * j + c0]) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(&stg[(r0 + 8) * SROW + 8 * j + c0]) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&staged_bar[h]);
      tphase ^= 1;
    }
  } else {
    // ===================== epilogue: running k-best list of one (row, column half) =====================
    regs_inc<kRegsEpilogue>();
    sched.init(tp, BLOCK_N, BK);
    const int h = role - 3;                  // staging half: rows [64 h, 64 h + 64)
    const int wi = warp & 3;
    const int quarter = h * 2 + (wi & 1);    // 32-row quarter of the tile this warp handles
    const int half = wi >> 1;                // which column half of the tile
    const int row_in_tile = quarter * 32 + lane;
    const int k = tp.k;
    const float* srow = stg + row_in_tile * SROW + half * HALF_N;
    float sv[KMAX];
    int si[KMAX];
    constexpr bool REG_GROUPS = GROUPS && KMAX <= 16;
    [[maybe_unused]] int sg[REG_GROUPS ? KMAX : 1];                   // GROUPS, KMAX = 16: the group of each entry
    [[maybe_unused]] __shared__ __align__(16) int32_t s_grp[8][HALF_N];   // GROUPS: per epilogue warp, its 64 columns' labels
    [[maybe_unused]] const int ew = warp - 12;                        // epilogue warp 0..7
    float thr = neg_inf();
    int m = 0, excl = -1;
    [[maybe_unused]] int64_t ex_cur = 0, ex_end = 0;   // EXCL: cursor into row m's list and its end
    [[maybe_unused]] int ex_next = INT_MAX;            // EXCL: the list entry at the cursor (INT_MAX past the end)
    uint32_t tphase = 0;
    int mb, nb, kb0, kb1;
    while (sched.next(mb, nb, kb0, kb1)) {
      if (sched.first) {
#pragma unroll
        for (int j = 0; j < KMAX; ++j) { sv[j] = neg_inf(); si[j] = -1; }
        if constexpr (REG_GROUPS) {
#pragma unroll
          for (int j = 0; j < KMAX; ++j) sg[j] = -1;
        }
        thr = neg_inf();
        m = mb * BLOCK_M + row_in_tile;
        const int64_t e = (int64_t)m + tp.diag_offset;
        excl = (tp.exclude && e >= 0 && e < p.N) ? (int)e : -1;
        if constexpr (EXCL) {
          ex_next = INT_MAX;
          if (m < p.M && (!GROUPS || tp.ex_indptr)) {
            const int c_first = nb * BLOCK_N + half * HALF_N;   // the first column this thread sees in the item
            int64_t lo = tp.ex_indptr[m], hi = tp.ex_indptr[m + 1];
            ex_end = hi;
            while (lo < hi) {
              const int64_t mid = lo + ((hi - lo) >> 1);
              if (tp.ex_indices[mid] < c_first) lo = mid + 1; else hi = mid;
            }
            ex_cur = lo;
            if (ex_cur < ex_end) ex_next = tp.ex_indices[ex_cur];
          }
        }
      }
      const int n0 = nb * BLOCK_N + half * HALF_N;
      if constexpr (GROUPS) {   // the previous tile's reads ended at the __syncwarp before `drained`
        const int j0 = n0 + lane, j1 = n0 + 32 + lane;
        s_grp[ew][lane] = j0 < p.N ? tp.groups[j0] : -1;
        s_grp[ew][lane + 32] = j1 < p.N ? tp.groups[j1] : -1;
        __syncwarp();
      }
      mbar_wait(&staged_bar[h], tphase);
      if (m < p.M) {
        if constexpr (EXCL) {
          float* wrow = stg + row_in_tile * SROW + half * HALF_N;
          while (ex_next < n0 + HALF_N) {   // listed columns of the other half (ex_next < n0) are skipped
            if (ex_next >= n0) wrow[ex_next - n0] = neg_inf();
            ex_next = (++ex_cur < ex_end) ? tp.ex_indices[ex_cur] : INT_MAX;
          }
        }
#pragma unroll 1
        for (int c = 0; c < HALF_N; c += 4) {
          const float4 v = *reinterpret_cast<const float4*>(srow + c);
          if (fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)) > thr) {   // rare once the list has filled
            if constexpr (GROUPS) {
              const int4 g = *reinterpret_cast<const int4*>(&s_grp[ew][c]);
              topk_offer_group<KMAX, REG_GROUPS>(sv, si, sg, thr, k, v.x, n0 + c, g.x, p.N, excl, tp.groups);
              topk_offer_group<KMAX, REG_GROUPS>(sv, si, sg, thr, k, v.y, n0 + c + 1, g.y, p.N, excl, tp.groups);
              topk_offer_group<KMAX, REG_GROUPS>(sv, si, sg, thr, k, v.z, n0 + c + 2, g.z, p.N, excl, tp.groups);
              topk_offer_group<KMAX, REG_GROUPS>(sv, si, sg, thr, k, v.w, n0 + c + 3, g.w, p.N, excl, tp.groups);
            } else {
              topk_offer<KMAX>(sv, si, thr, k, v.x, n0 + c, p.N, excl);
              topk_offer<KMAX>(sv, si, thr, k, v.y, n0 + c + 1, p.N, excl);
              topk_offer<KMAX>(sv, si, thr, k, v.z, n0 + c + 2, p.N, excl);
              topk_offer<KMAX>(sv, si, thr, k, v.w, n0 + c + 3, p.N, excl);
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&drained_bar[h]);   // this warp's staging rows may be overwritten
      tphase ^= 1;
      if (sched.last && m < p.M) {
        const int64_t base = ((int64_t)m * (2 * sched.splits) + 2 * sched.split + half) * k;
#pragma unroll
        for (int j = 0; j < KMAX; ++j)
          if (j < k) { tp.ws_val[base + j] = sv[j]; tp.ws_idx[base + j] = si[j]; }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// related / unrelated pair histogram (dae_similarity_pair_hist_bf16x3): for every pair i > j of rows of X with labels >= 0 the
// bf16x3 score S[i, j] = X_i . X_j is binned into hist[related ? 0 : 1][bin], without writing S.  topk_kernel's five warpgroups,
// operand ring and staged / drained hand-off; a different schedule and epilogue.
//   work item: one 128 x 128 tile with nb <= mb (the lower triangle and the diagonal: half of the tiles of S), dealt round-robin.
//   epilogue : thread = (row, 64-column half), as in top-k.  Each warp copies the labels of its 64 columns to shared memory, then
//              walks its row's columns in order, skips j >= i and label -1, and adds runs of equal (group, bin) to hist with one
//              red.global.add.u64 each.  The fp64 score sums of the two groups stay in registers and are flushed once per tile.
// ---------------------------------------------------------------------------------------------------------------------
struct PairHistParams {
  GemmParams g;                      // M = N = rows of X, K = dim
  const int32_t* labels;             // [N], -1 = no label
  float range, scale;                // M of the grid and bins / (2M)
  uint32_t bins;
  unsigned long long* hist;          // [2 x bins]
  double* sums;                      // [2]
};

// tiles t = mb (mb + 1) / 2 + nb, nb <= mb, items blockIdx.x, blockIdx.x + gridDim.x, ...
struct PairHistSched {
  long long t, n_tiles;
  int n_cta, kb_total;
  __device__ __forceinline__ void init(const PairHistParams& hp, int block_k) {
    const long long tm = (hp.g.M + BLOCK_M - 1) / BLOCK_M;
    n_tiles = tm * (tm + 1) / 2;
    kb_total = (hp.g.K + block_k - 1) / block_k;
    n_cta = (int)gridDim.x;
    t = blockIdx.x;
  }
  __device__ __forceinline__ bool next(int& mb, int& nb, int& kb0, int& kb1) {
    if (t >= n_tiles) return false;
    long long r = (long long)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
    while (r * (r + 1) / 2 > t) --r;
    while ((r + 1) * (r + 2) / 2 <= t) ++r;
    mb = (int)r;
    nb = (int)(t - r * (r + 1) / 2);
    kb0 = 0; kb1 = kb_total;
    t += n_cta;
    return true;
  }
};

__global__ void __launch_bounds__(kDecodeThreads, 1) pair_hist_kernel(const __grid_constant__ CUtensorMap tm_a_hi,
                                                                      const __grid_constant__ CUtensorMap tm_a_lo,
                                                                      const __grid_constant__ CUtensorMap tm_b_hi,
                                                                      const __grid_constant__ CUtensorMap tm_b_lo,
                                                                      const PairHistParams hp) {
  constexpr int BLOCK_N = kDecodeN, STAGES = kTopkStages, BK = kTopkBK;
  constexpr int STAGE_BYTES = 2 * BLOCK_M * BK * 2 + 2 * BLOCK_N * BK * 2;
  constexpr int SROW = BLOCK_N + 4;
  constexpr int HALF_N = BLOCK_N / 2;
  const GemmParams& p = hp.g;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* stg = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);   // [BLOCK_M][SROW] accumulator staging
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES], staged_bar[2], drained_bar[2];
  __shared__ __align__(16) int32_t s_lab[8][HALF_N];   // per epilogue warp: the labels of its 64 columns of the current tile

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int role = warp >> 2;                     // warpgroup: 0 producer, 1-2 MMA, 3-4 epilogue
  PairHistSched sched;

  if (warp == 0 && lane == 0) { prefetch_tmap(&tm_a_hi); prefetch_tmap(&tm_a_lo); prefetch_tmap(&tm_b_hi); prefetch_tmap(&tm_b_lo); }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    for (int h = 0; h < 2; ++h) { mbar_init(&staged_bar[h], 4); mbar_init(&drained_bar[h], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (role == 0) {
    // ===================== TMA producer =====================
    regs_dec<kRegsProducer>();
    sched.init(hp, BK);
    if (warp == 0 && lane == 0)
      tma_produce<BLOCK_N, STAGES, 0, BK>(p, sched, smem, full_bar, empty_bar, 0u, &tm_a_hi, &tm_a_lo, &tm_b_hi, &tm_b_lo, &tm_a_hi, &tm_a_lo);
  } else if (role <= 2) {
    // ===================== MMA: wgmma main loop -> staging half =====================
    regs_inc<kRegsMma>();
    sched.init(hp, BK);
    const int h = role - 1;
    const int wi = warp & 3;
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.0f;
    int stage = 0; uint32_t phase = 0, tphase = 0;
    int mb, nb, kb0, kb1;
    while (sched.next(mb, nb, kb0, kb1)) {
      mma_work_item<BLOCK_N, STAGES, 0, 0, BK>(acc, p, smem, full_bar, empty_bar, h, lane, 0u, stage, phase, kb0, kb1);
      mbar_wait(&drained_bar[h], tphase ^ 1);   // the epilogue is done with the previous tile's rows
      const int r0 = h * 64 + wi * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        *reinterpret_cast<float2*>(&stg[r0 * SROW + 8 * j + c0]) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(&stg[(r0 + 8) * SROW + 8 * j + c0]) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&staged_bar[h]);
      tphase ^= 1;
    }
  } else {
    // ===================== epilogue: bin the lower-triangle pairs of one (row, column half) =====================
    regs_inc<kRegsEpilogue>();
    sched.init(hp, BK);
    const int h = role - 3;                  // staging half: rows [64 h, 64 h + 64)
    const int ew = warp - 12;                // epilogue warp 0..7 (its label buffer)
    const int wi = warp & 3;
    const int quarter = h * 2 + (wi & 1);    // 32-row quarter of the tile this warp handles
    const int half = wi >> 1;                // which column half of the tile
    const int row_in_tile = quarter * 32 + lane;
    const float* srow = stg + row_in_tile * SROW + half * HALF_N;
    const float range = hp.range, scale = hp.scale;
    const uint32_t bins = hp.bins;
    uint32_t tphase = 0;
    int mb, nb, kb0, kb1;
    while (sched.next(mb, nb, kb0, kb1)) {
      const int i = mb * BLOCK_M + row_in_tile;
      const int n0 = nb * BLOCK_N + half * HALF_N;
      {
        const int j0 = n0 + lane, j1 = n0 + 32 + lane;
        s_lab[ew][lane] = j0 < p.N ? hp.labels[j0] : -1;
        s_lab[ew][lane + 32] = j1 < p.N ? hp.labels[j1] : -1;
      }
      const int li = i < p.N ? hp.labels[i] : -1;
      const int c_end = li < 0 ? 0 : min(HALF_N, i - n0);   // columns j < i only (j < i < N)
      __syncwarp();
      double sum_rel = 0.0, sum_unrel = 0.0;
      uint32_t run_key = 0, run_n = 0;
      auto offer = [&](float s, int lj, bool in) {
        if (!in || lj < 0) return;
        const bool rel = (lj == li);
        const uint32_t key = (rel ? 0u : bins) + pair_bin(s, range, scale, bins);
        if (rel) sum_rel += (double)s; else sum_unrel += (double)s;
        if (key != run_key && run_n) { red_add_u64(hp.hist + run_key, run_n); run_n = 0; }
        run_key = key;
        ++run_n;
      };
      mbar_wait(&staged_bar[h], tphase);
#pragma unroll 1
      for (int c = 0; c < c_end; c += 4) {   // 16-byte row reads: conflict-free with the SROW padding
        const float4 v = *reinterpret_cast<const float4*>(srow + c);
        const int4 l = *reinterpret_cast<const int4*>(&s_lab[ew][c]);
        offer(v.x, l.x, true);
        offer(v.y, l.y, c + 1 < c_end);
        offer(v.z, l.z, c + 2 < c_end);
        offer(v.w, l.w, c + 3 < c_end);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&drained_bar[h]);   // this warp's staging rows (and its label buffer) may be overwritten
      tphase ^= 1;
      if (run_n) red_add_u64(hp.hist + run_key, run_n);
      sum_rel = warp_sum(sum_rel);
      sum_unrel = warp_sum(sum_unrel);
      if (lane == 0) {
        if (sum_rel != 0.0) atomicAdd(hp.sums, sum_rel);
        if (sum_unrel != 0.0) atomicAdd(hp.sums + 1, sum_unrel);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// thresholded pairs (dae_similarity_pairs_bf16x3): every (i, j) with S[i, j] = Q_i . C_j >= tau as an (i, j, s) triple, without
// writing S.  topk_kernel's five warpgroups, operand ring, tile shape and k16 order, so every score has the bits
// dae_similarity_topk_bf16x3 computes for the same (i, j); a different schedule and epilogue.
//   work item: one 128 x 128 tile, dealt round-robin: self mode (Q is C) the tiles with nb <= mb, as pair_hist_kernel; corpus mode
//              all of them.
//   epilogue : thread = (row, 64-column half), as in top-k.  Pass 1 counts the row's qualifying columns (j < i in self mode, j < N
//              in corpus mode): per float4 one max and compare against tau, the common case.  A warp with any hit reserves its
//              slots with one atomicAdd on the 64-bit counter (pair_slots) and pass 2 writes the triples to the slots below capacity.
// ---------------------------------------------------------------------------------------------------------------------
struct PairsParams {
  GemmParams g;                      // M = queries, N = corpus rows, K = dim
  int self;                          // != 0: Q is C; tiles nb <= mb, columns j < i
  float tau;
  unsigned long long* count;         // caller-zeroed, accumulated: the number of qualifying pairs
  unsigned long long capacity;       // slots of i_out / j_out / s_out
  int32_t* i_out; int32_t* j_out; float* s_out;
  // pairs_kernel<true> (long top-k lists, corpus-mode tiles): row i's threshold row_tau[i] (at least -FLT_MAX, so -inf and NaN
  // never qualify), column i + diag_offset left out when `exclude`, per-row exclusion lists (may be null) and per-row counts
  // row_count[i] (caller-zeroed, accumulated).  Last, so the fields above keep their parameter offsets in pairs_kernel<false>.
  const float* row_tau;
  int64_t diag_offset;
  int exclude;
  const int64_t* ex_indptr; const int32_t* ex_indices;
  unsigned int* row_count;
};

// self: tiles t = mb (mb + 1) / 2 + nb, nb <= mb (PairHistSched's order); corpus: t = mb * tiles_n + nb.  Items blockIdx.x,
// blockIdx.x + gridDim.x, ...
struct PairsSched {
  long long t, n_tiles;
  int tiles_n, self, n_cta, kb_total;
  __device__ __forceinline__ void init(const PairsParams& pp, int block_n, int block_k) {
    const long long tm = (pp.g.M + BLOCK_M - 1) / BLOCK_M;
    tiles_n = (pp.g.N + block_n - 1) / block_n;
    self = pp.self;
    n_tiles = self ? tm * (tm + 1) / 2 : tm * tiles_n;
    kb_total = (pp.g.K + block_k - 1) / block_k;
    n_cta = (int)gridDim.x;
    t = blockIdx.x;
  }
  __device__ __forceinline__ bool next(int& mb, int& nb, int& kb0, int& kb1) {
    if (t >= n_tiles) return false;
    if (self) {
      long long r = (long long)((sqrt(8.0 * (double)t + 1.0) - 1.0) * 0.5);
      while (r * (r + 1) / 2 > t) --r;
      while ((r + 1) * (r + 2) / 2 <= t) ++r;
      mb = (int)r;
      nb = (int)(t - r * (r + 1) / 2);
    } else {
      mb = (int)(t / tiles_n);
      nb = (int)(t - (long long)mb * tiles_n);
    }
    kb0 = 0; kb1 = kb_total;
    t += n_cta;
    return true;
  }
};

// ROWS: the collect stage of the long top-k lists -- a threshold per row; the self match and the listed columns are written as -inf
// over the thread's own staging run before the scan (topk_kernel<KMAX, true>'s trick, with a binary search per tile since the
// tiles of one row are not swept in one item), and -inf is below every threshold.
template <bool ROWS = false>
__global__ void __launch_bounds__(kDecodeThreads, 1) pairs_kernel(const __grid_constant__ CUtensorMap tm_a_hi,
                                                                  const __grid_constant__ CUtensorMap tm_a_lo,
                                                                  const __grid_constant__ CUtensorMap tm_b_hi,
                                                                  const __grid_constant__ CUtensorMap tm_b_lo,
                                                                  const PairsParams pp) {
  constexpr int BLOCK_N = kDecodeN, STAGES = kTopkStages, BK = kTopkBK;
  constexpr int STAGE_BYTES = 2 * BLOCK_M * BK * 2 + 2 * BLOCK_N * BK * 2;
  constexpr int SROW = BLOCK_N + 4;
  constexpr int HALF_N = BLOCK_N / 2;
  const GemmParams& p = pp.g;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* stg = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);   // [BLOCK_M][SROW] accumulator staging
  __shared__ __align__(8) uint64_t full_bar[STAGES], empty_bar[STAGES], staged_bar[2], drained_bar[2];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int role = warp >> 2;                     // warpgroup: 0 producer, 1-2 MMA, 3-4 epilogue
  PairsSched sched;

  if (warp == 0 && lane == 0) { prefetch_tmap(&tm_a_hi); prefetch_tmap(&tm_a_lo); prefetch_tmap(&tm_b_hi); prefetch_tmap(&tm_b_lo); }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    for (int h = 0; h < 2; ++h) { mbar_init(&staged_bar[h], 4); mbar_init(&drained_bar[h], 4); }
    fence_barrier_init();
  }
  __syncthreads();

  if (role == 0) {
    // ===================== TMA producer =====================
    regs_dec<kRegsProducer>();
    sched.init(pp, BLOCK_N, BK);
    if (warp == 0 && lane == 0)
      tma_produce<BLOCK_N, STAGES, 0, BK>(p, sched, smem, full_bar, empty_bar, 0u, &tm_a_hi, &tm_a_lo, &tm_b_hi, &tm_b_lo, &tm_a_hi, &tm_a_lo);
  } else if (role <= 2) {
    // ===================== MMA: wgmma main loop -> staging half =====================
    regs_inc<kRegsMma>();
    sched.init(pp, BLOCK_N, BK);
    const int h = role - 1;
    const int wi = warp & 3;
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.0f;
    int stage = 0; uint32_t phase = 0, tphase = 0;
    int mb, nb, kb0, kb1;
    while (sched.next(mb, nb, kb0, kb1)) {
      mma_work_item<BLOCK_N, STAGES, 0, 0, BK>(acc, p, smem, full_bar, empty_bar, h, lane, 0u, stage, phase, kb0, kb1);
      mbar_wait(&drained_bar[h], tphase ^ 1);   // the epilogue is done with the previous tile's rows
      const int r0 = h * 64 + wi * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        *reinterpret_cast<float2*>(&stg[r0 * SROW + 8 * j + c0]) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(&stg[(r0 + 8) * SROW + 8 * j + c0]) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&staged_bar[h]);
      tphase ^= 1;
    }
  } else {
    // ===================== epilogue: emit the qualifying pairs of one (row, column half) =====================
    regs_inc<kRegsEpilogue>();
    sched.init(pp, BLOCK_N, BK);
    const int h = role - 3;                  // staging half: rows [64 h, 64 h + 64)
    const int wi = warp & 3;
    const int quarter = h * 2 + (wi & 1);    // 32-row quarter of the tile this warp handles
    const int half = wi >> 1;                // which column half of the tile
    const int row_in_tile = quarter * 32 + lane;
    const float* srow = stg + row_in_tile * SROW + half * HALF_N;
    const float tau = pp.tau;
    uint32_t tphase = 0;
    int mb, nb, kb0, kb1;
    while (sched.next(mb, nb, kb0, kb1)) {
      const int i = mb * BLOCK_M + row_in_tile;
      const int n0 = nb * BLOCK_N + half * HALF_N;
      const int lim = pp.self ? i : p.N;                          // columns j < lim (self: i < M = N)
      const int c_end = i < p.M ? max(0, min(HALF_N, lim - n0)) : 0;
      mbar_wait(&staged_bar[h], tphase);
      [[maybe_unused]] float tau_i = tau;
      if constexpr (ROWS) {
        if (i < p.M) {
          tau_i = fmaxf(pp.row_tau[i], -FLT_MAX);
          float* wrow = stg + row_in_tile * SROW + half * HALF_N;
          const int64_t e = (int64_t)i + pp.diag_offset;
          if (pp.exclude && e >= n0 && e < n0 + HALF_N) wrow[e - n0] = neg_inf();
          if (pp.ex_indptr) {
            int64_t lo = pp.ex_indptr[i], hi = pp.ex_indptr[i + 1];
            while (lo < hi) {
              const int64_t mid = lo + ((hi - lo) >> 1);
              if (pp.ex_indices[mid] < n0) lo = mid + 1; else hi = mid;
            }
            for (; lo < pp.ex_indptr[i + 1] && pp.ex_indices[lo] < n0 + HALF_N; ++lo) wrow[pp.ex_indices[lo] - n0] = neg_inf();
          }
        }
      }
      const float thr = ROWS ? tau_i : tau;
      int hits = 0;
#pragma unroll 1
      for (int c = 0; c < c_end; c += 4) {   // NaN never qualifies: fmaxf drops it and every compare with it is false
        const float4 v = *reinterpret_cast<const float4*>(srow + c);
        if (fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)) >= thr)   // rare at a near-duplicate threshold
          hits += (v.x >= thr) + (c + 1 < c_end && v.y >= thr) + (c + 2 < c_end && v.z >= thr) + (c + 3 < c_end && v.w >= thr);
      }
      if constexpr (ROWS) {
        if (hits) atomicAdd(pp.row_count + i, (unsigned int)hits);
      }
      if (__any_sync(0xffffffffu, hits != 0)) {
        unsigned long long slot = pair_slots(pp.count, hits);
        if (hits) {
#pragma unroll 1
          for (int c = 0; c < c_end; ++c) {
            const float s = srow[c];
            if (s >= thr) pair_put(slot++, pp.capacity, i, n0 + c, s, pp.i_out, pp.j_out, pp.s_out);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&drained_bar[h]);   // this warp's staging rows may be overwritten
      tphase ^= 1;
    }
  }
}

// tile_ptr[m][t] = number of stored entries of batch row m with column < t * half_n (t = 0 .. n_half_tiles): where each
// half tile of the fused decode epilogue starts in the (sorted) clean CSR row.  One thread per (row, t).
__global__ void decode_tile_ptr_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                       const int32_t* __restrict__ rows, int M, int n_half_tiles, int half_n,
                                       int32_t* __restrict__ tile_ptr) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > n_half_tiles) return;
  for (int m = blockIdx.y; m < M; m += gridDim.y) {   // grid.y <= 65 535: batches above that loop over their rows
    const int64_t row = rows ? (int64_t)rows[m] : (int64_t)m;
    const int64_t b = indptr[row], e = indptr[row + 1];
    const int target = t * half_n;
    int64_t lo = b, hi = e;
    while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (indices[mid] < target) lo = mid + 1; else hi = mid; }
    tile_ptr[(int64_t)m * (n_half_tiles + 1) + t] = (int32_t)(lo - b);
  }
}

// fp32 -> (bf16 hi, bf16 lo) split, row by row, zero padding up to ld_dst columns; optional 1.0 in column `ones_col`.
__global__ void split_bf16_kernel(const float* __restrict__ src, int rows, int cols, int64_t ld_src, __nv_bfloat16* __restrict__ hi,
                                  __nv_bfloat16* __restrict__ lo, int64_t ld_dst, int ones_col, float scale) {
  const int64_t total = (int64_t)rows * ld_dst;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / ld_dst;
    const int c = (int)(i - r * ld_dst);
    float v = (c < cols) ? src[r * ld_src + c] * scale : 0.0f;
    if (c == ones_col) v = 1.0f;
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    hi[i] = h;
    lo[i] = __float2bfloat16_rn(v - __bfloat162float(h));
  }
}

// GG = alpha * (G + G^T) split to bf16 hi/lo (B x ld), for dE_tri = GG . E
__global__ void sym_split_kernel(const float* __restrict__ G, int B, int64_t ldg, float alpha, __nv_bfloat16* __restrict__ hi,
                                 __nv_bfloat16* __restrict__ lo, int64_t ld) {
  __shared__ float t[32][33];
  const int bx = blockIdx.x * 32, by = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int r = bx + j, c = by + tx;            // read G^T tile: G[bx + j][by + tx]
    t[j][tx] = (r < B && c < B) ? G[(int64_t)r * ldg + c] : 0.0f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int r = by + j, c = bx + tx;            // output element (r, c) = G[r][c] + G[c][r]
    if (r < B && c < ld) {
      float v = 0.0f;
      if (c < B) v = alpha * (G[(int64_t)r * ldg + c] + t[tx][j]);
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      hi[(int64_t)r * ld + c] = h;
      lo[(int64_t)r * ld + c] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// host side: tensor maps + launch
// ---------------------------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(sym);
  }
  return fn;
}

// 2-D bf16 tensor [outer x inner] (inner contiguous), row stride ld elements; box = {box_inner, box_outer}: 64 inner elements with the
// 128B swizzle, 32 with the 64B swizzle.
static int make_map(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, uint64_t ld, uint32_t box_outer,
                    uint32_t box_inner = 64) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point not found"); return DAE_ERR_CUDA; }
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, box_inner == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d): inner=%llu outer=%llu ld=%llu", (int)r,
                                     (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)ld); return DAE_ERR_CUDA; }
  return DAE_OK;
}

struct Operand { const void* hi; const void* lo; int64_t ld; int mn_major; };

// cudaFuncSetAttribute is per device: remember which devices have been configured for this instantiation
template <typename Kern>
static int ensure_smem_attr(Kern kern, int smem, bool (&done)[64]) {
  int dev = 0;
  DAE_CUDA(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64 || !done[dev]) {
    DAE_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    if (dev >= 0 && dev < 64) done[dev] = true;
  }
  return DAE_OK;
}


static int g_pair_mode = -1;   // -1 (default) and 0: never; 1: whenever the shape allows (dae_gemm_config)
static int g_lean = 0;         // 1: 128 x 64 tiles with 2-stage rings for dae_gemm_bf16x3 (~130 KB of shared memory instead of ~195 KB)

template <int BLOCK_N, int STAGES, int PAIR, int MAJ, int BK = BLOCK_K>
static int launch_gemm_maj(const Operand& A, const Operand& B, GemmParams p, cudaStream_t st, int* grid_out = nullptr) {
  CUtensorMap ta_hi, ta_lo, tb_hi, tb_lo;
  int rc;
  constexpr int B_ROWS = PAIR ? BLOCK_N / 2 : BLOCK_N;   // n rows of the B tile one CTA loads
  // K-major: tensor [rows=MN x cols=K], box {BK k, tile rows};  MN-major: tensor [rows=K x cols=MN], box {64 mn, BK k}
  if (!A.mn_major) {
    const uint64_t a_cols = p.a_sym_kb > 0 ? (uint64_t)p.M : (uint64_t)p.K;   // (A + A^T).B: A is M x M, K = 2 x (padded M)
    if ((rc = make_map(&ta_hi, A.hi, a_cols, p.M, A.ld, BLOCK_M, BK))) return rc;
    if ((rc = make_map(&ta_lo, A.lo, a_cols, p.M, A.ld, BLOCK_M, BK))) return rc;
  } else {
    if ((rc = make_map(&ta_hi, A.hi, p.M, p.K, A.ld, BK))) return rc;
    if ((rc = make_map(&ta_lo, A.lo, p.M, p.K, A.ld, BK))) return rc;
  }
  if (!B.mn_major) {
    if ((rc = make_map(&tb_hi, B.hi, p.K, p.N, B.ld, B_ROWS, BK))) return rc;
    if ((rc = make_map(&tb_lo, B.lo, p.K, p.N, B.ld, B_ROWS, BK))) return rc;
  } else {
    const uint64_t b_rows = p.a_sym_kb > 0 ? (uint64_t)p.M : (uint64_t)p.K;
    if ((rc = make_map(&tb_hi, B.hi, p.N, b_rows, B.ld, BK))) return rc;
    if ((rc = make_map(&tb_lo, B.lo, p.N, b_rows, B.ld, BK))) return rc;
  }
  p.a_mn = A.mn_major; p.b_mn = B.mn_major;
  CUtensorMap tat_hi = ta_hi, tat_lo = ta_lo;
  if (p.a_sym_kb > 0) {   // A is a square [M x M] array read K-major above; these are its M-contiguous (transposed) views
    if (PAIR || A.mn_major) { set_error("dae_gemm_sym_bf16x3: unsupported configuration"); return DAE_ERR_UNSUPPORTED; }
    if ((rc = make_map(&tat_hi, A.hi, p.M, p.M, A.ld, 64))) return rc;
    if ((rc = make_map(&tat_lo, A.lo, p.M, p.M, A.ld, 64))) return rc;
  }
  // operand ring + accumulator staging tile + alignment slack
  constexpr int smem = STAGES * (2 * BLOCK_M * BK * 2 + 2 * BLOCK_N * BK * 2) + BLOCK_M * (BLOCK_N + 4) * 4 + 1024;
  int tiles_m = (p.M + BLOCK_M - 1) / BLOCK_M;
  if (PAIR) tiles_m = (tiles_m + 1) / 2;
  const int tiles_n = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int kblocks = (p.K + BK - 1) / BK;
  auto kern = gemm_bf16x3_kernel<BLOCK_N, STAGES, PAIR, MAJ, BK>;
  static bool attr_done[64] = {false};
  if ((rc = ensure_smem_attr(kern, smem, attr_done))) return rc;
  const int slots = PAIR ? sm_count() / 2 : sm_count();   // CTAs, or CTA pairs, resident at once
  int n;
  if (p.stream_k) {   // segments of at least 6 k-blocks of 64 (12 of 32): a shorter main loop does not amortise its (atomic) epilogue
    const long long units = (long long)tiles_m * tiles_n * kblocks;
    long long g = units / (6 * BLOCK_K / BK);
    if (g < 1) g = 1;
    n = (int)(g < slots ? g : slots);
  } else {
    const int items = tiles_m * tiles_n * p.k_splits;
    n = items < slots ? items : slots;
  }
  if (grid_out) *grid_out = n;
  if (!PAIR) {
    kern<<<n, kThreads, smem, st>>>(ta_hi, ta_lo, tb_hi, tb_lo, tat_hi, tat_lo, p);
  } else {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(2 * n); cfg.blockDim = dim3(kThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    DAE_CUDA(cudaLaunchKernelEx(&cfg, kern, ta_hi, ta_lo, tb_hi, tb_lo, tat_hi, tat_lo, p));
  }
  return DAE_OK;
}

// the plain GEMMs take any majorness; (A + A^T).B goes through launch_gemm_maj directly
template <int BLOCK_N, int STAGES, int PAIR, int BK = BLOCK_K>
static int launch_gemm(const Operand& A, const Operand& B, GemmParams p, cudaStream_t st, int* grid_out = nullptr) {
  if (!A.mn_major && !B.mn_major) return launch_gemm_maj<BLOCK_N, STAGES, PAIR, 0, BK>(A, B, p, st, grid_out);
  if (A.mn_major && !B.mn_major) return launch_gemm_maj<BLOCK_N, STAGES, PAIR, 1, BK>(A, B, p, st, grid_out);
  if (!A.mn_major) return launch_gemm_maj<BLOCK_N, STAGES, PAIR, 2, BK>(A, B, p, st, grid_out);
  return launch_gemm_maj<BLOCK_N, STAGES, PAIR, 3, BK>(A, B, p, st, grid_out);
}

// Deterministic stream-K, after the GEMM: kFixupSlices CTAs per output tile, each over a slice of its rows.  A tile that one CTA
// covered was stored by that CTA; a tile cut between CTAs c0 < c1 < ... is the sum of their workspace slots in that (= k) order,
// stored (or added, C += ...) once.  The CTA
// ranges are recomputed exactly as Sched::init cuts them (u_c = c U / n_cta); CTA c's segment in the tile is its first one (slot 0)
// iff its range starts inside the tile.
constexpr int kMaxFixupCtas = 1024;   // CTAs of one stream-K launch (at most one per SM) the fixup can list for a tile
constexpr int kFixupSlices = 16;      // CTAs per tile: the slot reads of a split tile spread over the SMs (latency, not bandwidth)

template <int BLOCK_N>
__global__ void __launch_bounds__(256) sk_fixup_kernel(const GemmParams p, int tiles_m, int tiles, int kb_total, int n_cta) {
  __shared__ int s_slot[kMaxFixupCtas];   // workspace slots of the CTAs that cover this tile, in k order
  __shared__ int s_n;
  const int t = blockIdx.x;
  if (threadIdx.x == 0) {   // the CTA ranges are found once per tile, not per element (64-bit divisions)
    const long long U = (long long)tiles * kb_total, T0 = (long long)t * kb_total, T1 = T0 + kb_total;
    auto u_of = [&](int c) { return (long long)c * U / n_cta; };
    int c0 = (int)(T0 * n_cta / U);
    while (c0 + 1 < n_cta && u_of(c0 + 1) <= T0) ++c0;
    while (c0 > 0 && u_of(c0) > T0) --c0;
    int n = 0;
    if (u_of(c0 + 1) < T1) {   // otherwise one CTA covered the whole tile and stored it
      for (int c = c0; c < n_cta && u_of(c) < T1; ++c) {
        if (u_of(c + 1) == u_of(c)) continue;   // an empty range has no segment
        s_slot[n++] = 2 * c + (u_of(c) >= T0 ? 0 : 1);
      }
    }
    s_n = n;
  }
  __syncthreads();
  const int n = s_n;
  if (n == 0) return;
  const int mb = t % tiles_m, nb = t / tiles_m;
  constexpr int kPer = BLOCK_M * BLOCK_N / kFixupSlices;   // blockIdx.y: one slice of 128 / kFixupSlices rows of the tile
  for (int e = blockIdx.y * kPer + threadIdx.x; e < (blockIdx.y + 1) * kPer; e += blockDim.x) {
    const int m = mb * BLOCK_M + e / BLOCK_N, col = nb * BLOCK_N + e % BLOCK_N;
    if (m >= p.M || (col != p.special_col && col >= p.n_store)) continue;
    float s = p.sk_ws[(int64_t)s_slot[0] * (BLOCK_M * BLOCK_N) + e];
    for (int i = 1; i < n; ++i) s = s + p.sk_ws[(int64_t)s_slot[i] * (BLOCK_M * BLOCK_N) + e];
    float* dst = (col == p.special_col) ? p.special_out + m : p.C + (int64_t)m * p.ldc + col;
    *dst = p.atomic ? *dst + s : s;   // (atomic = accumulate here: this is the only writer of the element)
  }
}

static int64_t sk_workspace_bytes() { return (int64_t)2 * sm_count() * BLOCK_M * 128 * (int64_t)sizeof(float); }

// the fused decode, top-k, pair-histogram and pairs kernels: A [M x K] and B [N x K] (M, N and K from g), both K-major, in 128-row
// and kDecodeN-row boxes; one persistent CTA per SM over the kernel's work items.  Templated on the kernel itself, not its type, so
// that every kernel has its own attr_done (topk_kernel<16, false> and <32, false> share a type).
template <auto Kern, int BK, int STAGES, class Params>
static int launch_persistent(const Operand& A, const Operand& B, const GemmParams& g, const Params& kp, long long items,
                             cudaStream_t st) {
  CUtensorMap ta_hi, ta_lo, tb_hi, tb_lo;
  int rc;
  if ((rc = make_map(&ta_hi, A.hi, g.K, g.M, A.ld, BLOCK_M, BK))) return rc;
  if ((rc = make_map(&ta_lo, A.lo, g.K, g.M, A.ld, BLOCK_M, BK))) return rc;
  if ((rc = make_map(&tb_hi, B.hi, g.K, g.N, B.ld, kDecodeN, BK))) return rc;
  if ((rc = make_map(&tb_lo, B.lo, g.K, g.N, B.ld, kDecodeN, BK))) return rc;
  // operand ring + accumulator staging tile + alignment slack (the decode's dZ transpose blocks are static)
  constexpr int smem = STAGES * (2 * BLOCK_M * BK * 2 + 2 * kDecodeN * BK * 2) + BLOCK_M * (kDecodeN + 4) * 4 + 1024;
  static bool attr_done[64] = {false};
  if ((rc = ensure_smem_attr(Kern, smem, attr_done))) return rc;
  const int n = items < sm_count() ? (int)items : sm_count();
  Kern<<<n, kDecodeThreads, smem, st>>>(ta_hi, ta_lo, tb_hi, tb_lo, kp);
  return DAE_OK;
}

// the fused decode: E [M x K] and W [N x K]; work items: the 128 x kDecodeN output tiles
template <int LOSS>
static int launch_decode(int dec_act, const Operand& A, const Operand& B, const GemmParams& p, cudaStream_t st) {
  const long long tiles = (long long)((p.M + BLOCK_M - 1) / BLOCK_M) * ((p.N + kDecodeN - 1) / kDecodeN);
  if (dec_act == DAE_ACT_SIGMOID)
    return launch_persistent<decode_fused_kernel<DAE_ACT_SIGMOID, LOSS>, kDecodeBK, kDecodeStages>(A, B, p, p, tiles, st);
  if (dec_act == DAE_ACT_TANH)
    return launch_persistent<decode_fused_kernel<DAE_ACT_TANH, LOSS>, kDecodeBK, kDecodeStages>(A, B, p, p, tiles, st);
  return launch_persistent<decode_fused_kernel<DAE_ACT_NONE, LOSS>, kDecodeBK, kDecodeStages>(A, B, p, p, tiles, st);
}

// fused similarity + k-best: Q [M x K] and C [N x K]; work items: (row block, split); the kernel keeps lists of 16 or 32 >= tp.k
template <bool EXCL, bool GROUPS>
static int launch_topk(const Operand& A, const Operand& B, const TopkParams& tp, cudaStream_t st) {
  const long long items = (long long)((tp.g.M + BLOCK_M - 1) / BLOCK_M) * tp.splits;
  if (tp.k <= 16) return launch_persistent<topk_kernel<16, EXCL, GROUPS>, kTopkBK, kTopkStages>(A, B, tp.g, tp, items, st);
  return launch_persistent<topk_kernel<32, EXCL, GROUPS>, kTopkBK, kTopkStages>(A, B, tp.g, tp, items, st);
}

// thresholded pairs: Q [M x K] and C [N x K]; work items: the tiles (self: the lower triangle)
template <bool ROWS>
static int launch_pairs(const Operand& A, const Operand& B, const PairsParams& pp, cudaStream_t st) {
  const long long tm = (pp.g.M + BLOCK_M - 1) / BLOCK_M, tn = (pp.g.N + kDecodeN - 1) / kDecodeN;
  return launch_persistent<pairs_kernel<ROWS>, kTopkBK, kTopkStages>(A, B, pp.g, pp, pp.self ? tm * (tm + 1) / 2 : tm * tn, st);
}

// column splits of dae_similarity_topk_bf16x3: `requested` (> 0), or the fewest that give every SM a work item while each split
// still sweeps kTopkMinTiles column tiles; always within [1, min(column tiles, kTopkMaxSplits)]
static int topk_splits(int n_query, int n_corpus, int requested) {
  const int tiles_m = (n_query + BLOCK_M - 1) / BLOCK_M, tiles_n = (n_corpus + kDecodeN - 1) / kDecodeN;
  int s = requested;
  if (s <= 0) {
    s = (sm_count() + tiles_m - 1) / tiles_m;
    const int by_len = tiles_n / kTopkMinTiles;
    if (s > by_len) s = by_len;
  }
  if (s > tiles_n) s = tiles_n;
  if (s > kTopkMaxSplits) s = kTopkMaxSplits;
  return s < 1 ? 1 : s;
}

static int64_t topk_workspace_bytes(int n_query, int k, int splits) {
  return (int64_t)n_query * 2 * splits * k * (int64_t)(sizeof(float) + sizeof(int32_t));
}

// CTA pairs cut the L2 -> SM traffic of the B operand by a quarter, but the multicast ties the two CTAs' pipelines together: measured
// on an H100 SXM (700 W) at C2, a training step takes 0.384 ms without pairs and 0.476 ms with them, so they run only when forced
static bool use_pair() { return g_pair_mode == 1 && !g_lean; }

}  // namespace dae

using namespace dae;

extern "C" int dae_split_bf16(const float* src, int32_t rows, int32_t cols, int64_t ld_src, void* hi, void* lo, int64_t ld_dst,
                              int32_t ones_col, float scale, void* stream) {
  DAE_REQUIRE(src && hi && lo && rows > 0 && cols > 0 && ld_src >= cols && ld_dst >= cols, "dae_split_bf16: bad arguments");
  const int64_t total = (int64_t)rows * ld_dst;
  const int cap = sm_count() * 16;
  const int blocks = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
  split_bf16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(src, rows, cols, ld_src, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, ld_dst,
                                                              ones_col, scale);
  DAE_CHECK_LAUNCH("dae_split_bf16");
  return DAE_OK;
}

extern "C" int dae_sym_split_bf16(const float* G, int32_t B, int64_t ldg, float alpha, void* hi, void* lo, int64_t ld, void* stream) {
  DAE_REQUIRE(G && hi && lo && B > 0 && ldg >= B && ld >= B, "dae_sym_split_bf16: bad arguments");
  dim3 grid((unsigned)((ld + 31) / 32), (B + 31) / 32), block(32, 8);
  sym_split_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(G, B, ldg, alpha, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, ld);
  DAE_CHECK_LAUNCH("dae_sym_split_bf16");
  return DAE_OK;
}

// test hook: pair_mode 1 = CTA pairs (two-CTA clusters sharing the B tile) for dae_gemm_bf16x3 wherever the shape allows, otherwise
// never; lean = 1: 128 x 64 tiles with 2-stage rings for dae_gemm_bf16x3.  The fused decode has one configuration.
extern "C" int dae_gemm_config(int32_t pair_mode, int32_t lean) {
  dae::g_pair_mode = pair_mode < 0 ? -1 : (pair_mode ? 1 : 0);
  dae::g_lean = lean ? 1 : 0;
  return DAE_OK;
}

// dae_gemm_bf16x3 and, with det, dae_gemm_bf16x3_det: the same schedules and main loops without the CTA-pair and lean engines;
// partial stream-K tiles go through the workspace and sk_fixup_kernel instead of atomic adds into a zeroed C
static int gemm_bf16x3(const char* fn, bool det, int32_t M, int32_t N, int32_t K, float alpha, const void* a_hi, const void* a_lo,
                       int64_t lda, int32_t a_mn_major, const void* b_hi, const void* b_lo, int64_t ldb, int32_t b_mn_major, float* C,
                       int64_t ldc, int32_t n_store, int32_t special_col, float* special_out, int32_t k_splits, int32_t accumulate,
                       void* workspace, int64_t workspace_bytes, void* stream) {
  DAE_REQUIRE(a_hi && a_lo && b_hi && b_lo && C && M > 0 && N > 0 && K > 0, "%s: bad arguments", fn);
  DAE_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "%s: operand leading dimensions must be multiples of 8 (TMA 16-byte strides)", fn);
  DAE_REQUIRE(((uintptr_t)a_hi | (uintptr_t)a_lo | (uintptr_t)b_hi | (uintptr_t)b_lo) % 16 == 0, "%s: operands must be 16-byte aligned",
              fn);
  DAE_REQUIRE(!det || k_splits == 1 || k_splits == -1, "%s: k_splits must be 1 or -1 (stream-K), got %d", fn, k_splits);
  cudaStream_t st = (cudaStream_t)stream;
  if (n_store <= 0 || n_store > N) n_store = N;
  DAE_REQUIRE(ldc >= n_store, "%s: ldc %lld below n_store %d", fn, (long long)ldc, n_store);
  DAE_REQUIRE(!special_out || (special_col >= n_store && special_col < N), "%s: special_col %d outside [n_store, N) = [%d, %d)", fn,
              special_col, n_store, N);
  DAE_REQUIRE(!det || (workspace && workspace_bytes >= sk_workspace_bytes()), "%s: workspace of %lld bytes, need %lld", fn,
              (long long)workspace_bytes, (long long)sk_workspace_bytes());
  const int kblocks = (K + BLOCK_K - 1) / BLOCK_K;
  const int tm = (M + 127) / 128, tn128 = (N + 127) / 128, tn64 = (N + 63) / 64;
  const int sms = sm_count();
  int stream_k = 0;
  if (k_splits < 0) {   // auto: stream-K unless the 128 x 128 tiling already fills the SMs in whole waves
    const int t = tm * tn128;
    stream_k = (t % sms == 0) ? 0 : 1;
    k_splits = 1;
  }
  if (k_splits < 1) k_splits = 1;
  if (k_splits > kblocks) k_splits = kblocks;
  {  // no empty splits
    const int per = (kblocks + k_splits - 1) / k_splits;
    k_splits = (kblocks + per - 1) / per;
  }
  const bool partial = (k_splits > 1) || stream_k;
  if (!det && partial && !accumulate) {
    DAE_CUDA(cudaMemset2DAsync(C, ldc * sizeof(float), 0, (size_t)n_store * sizeof(float), M, st));
    if (special_col >= 0 && special_out) DAE_CUDA(cudaMemsetAsync(special_out, 0, sizeof(float) * M, st));
  }
  GemmParams p{};
  p.M = M; p.N = N; p.K = K; p.k_splits = k_splits; p.stream_k = stream_k; p.alpha = alpha;
  p.atomic = ((partial && !det) || accumulate) ? 1 : 0;   // det: every element has one writer, the GEMM or the fixup
  p.C = C; p.ldc = ldc; p.n_store = n_store;
  p.special_col = (special_out ? special_col : -1); p.special_out = special_out;
  Operand A{a_hi, a_lo, lda, a_mn_major}, B{b_hi, b_lo, ldb, b_mn_major};
  // 128 x 128 tiles move fewer operand bytes per output, 128 x 64 tiles quantise better onto the SMs: pick the variant with the
  // smaller (waves x relative tile cost).  Stream-K balances by construction, so it always takes the 128 x 128 tiles, with a ring of
  // 4 stages of 32-wide k-blocks: the same 128 KB as 2 x 64, but three stages (96 KB) in flight behind the one being multiplied
  // instead of one (64 KB), which the L2 -> shared-memory latency of dE / dW needs (see DESIGN 4.1).  The lean and pair test
  // configurations keep the 2 x 64 rings.
  int rc, n = 0;
  const int tiles128 = tm * tn128 * k_splits, tiles64 = tm * tn64 * k_splits;
  const float cost128 = 2.0f * (float)((tiles128 + sms - 1) / sms), cost64 = 1.1f * (float)((tiles64 + sms - 1) / sms);
  if (det && stream_k) p.sk_ws = (float*)workspace;
  if (!det && g_lean) rc = launch_gemm<64, 2, 0>(A, B, p, st);
  else if (!det && use_pair()) rc = launch_gemm<128, 2, 1>(A, B, p, st);
  else if (stream_k) rc = launch_gemm<128, 4, 0, 32>(A, B, p, st, &n);
  else if (cost64 < cost128) rc = launch_gemm<64, 3, 0>(A, B, p, st);
  else rc = launch_gemm<128, 2, 0>(A, B, p, st);
  if (rc) return rc;
  if (det && stream_k) {
    DAE_REQUIRE(n <= kMaxFixupCtas, "%s: %d stream-K CTAs exceed the fixup's %d", fn, n, kMaxFixupCtas);
    sk_fixup_kernel<128><<<dim3(tm * tn128, kFixupSlices), 256, 0, st>>>(p, tm, tm * tn128, (K + 31) / 32, n);
  }
  DAE_CHECK_LAUNCH(fn);
  return DAE_OK;
}

extern "C" int dae_gemm_bf16x3(int32_t M, int32_t N, int32_t K, float alpha, const void* a_hi, const void* a_lo, int64_t lda,
                               int32_t a_mn_major, const void* b_hi, const void* b_lo, int64_t ldb, int32_t b_mn_major, float* C,
                               int64_t ldc, int32_t n_store, int32_t special_col, float* special_out, int32_t k_splits,
                               int32_t accumulate, void* stream) {
  return gemm_bf16x3("dae_gemm_bf16x3", false, M, N, K, alpha, a_hi, a_lo, lda, a_mn_major, b_hi, b_lo, ldb, b_mn_major, C, ldc, n_store,
                     special_col, special_out, k_splits, accumulate, nullptr, 0, stream);
}

extern "C" int dae_gemm_bf16x3_det(int32_t M, int32_t N, int32_t K, float alpha, const void* a_hi, const void* a_lo, int64_t lda,
                                   int32_t a_mn_major, const void* b_hi, const void* b_lo, int64_t ldb, int32_t b_mn_major, float* C,
                                   int64_t ldc, int32_t n_store, int32_t special_col, float* special_out, int32_t k_splits,
                                   int32_t accumulate, void* workspace, int64_t workspace_bytes, void* stream) {
  return gemm_bf16x3("dae_gemm_bf16x3_det", true, M, N, K, alpha, a_hi, a_lo, lda, a_mn_major, b_hi, b_lo, ldb, b_mn_major, C, ldc,
                     n_store, special_col, special_out, k_splits, accumulate, workspace, workspace_bytes, stream);
}

// C[m, n] (+)= alpha * sum_k (G[m, k] + G[k, m]) * B[k, n] for a square G [M x M] (bf16 hi / lo, row-major, ld = ldg) and B stored
// [M x ldb] row-major (n contiguous).  ONE launch: the k loop runs over G's columns and then over G's rows (the same array through
// an M-contiguous tensor map), so G + G^T is never formed.  dE2 = alpha (G + G^T) E of the batch_all / batch_hard backward.
// det (dae_gemm_sym_bf16x3_det): partial stream-K tiles go through the workspace and sk_fixup_kernel instead of atomics.
static int gemm_sym_bf16x3(const char* fn, bool det, int32_t M, int32_t N, float alpha, const void* g_hi, const void* g_lo, int64_t ldg,
                           const void* b_hi, const void* b_lo, int64_t ldb, float* C, int64_t ldc, int32_t accumulate, void* workspace,
                           int64_t workspace_bytes, void* stream) {
  DAE_REQUIRE(g_hi && g_lo && b_hi && b_lo && C && M > 0 && N > 0, "%s: bad arguments", fn);
  DAE_REQUIRE(ldg % 8 == 0 && ldb % 8 == 0 && ldg >= M && ldb >= N, "%s: leading dimensions must be multiples of 8 and cover the matrices",
              fn);
  DAE_REQUIRE(((uintptr_t)g_hi | (uintptr_t)g_lo | (uintptr_t)b_hi | (uintptr_t)b_lo) % 16 == 0, "%s: operands must be 16-byte aligned",
              fn);
  DAE_REQUIRE(!det || (workspace && workspace_bytes >= sk_workspace_bytes()), "%s: workspace of %lld bytes, need %lld", fn,
              (long long)workspace_bytes, (long long)sk_workspace_bytes());
  cudaStream_t st = (cudaStream_t)stream;
  GemmParams p{};
  const int kb_half = (M + BLOCK_K - 1) / BLOCK_K;
  // stream-K: 28 tiles of 128 x 128 at B = 800 would leave 104 SMs idle for a 26-k-block main loop; ~6 k-blocks per CTA instead
  p.M = M; p.N = N; p.K = 2 * kb_half * BLOCK_K; p.k_splits = 1; p.stream_k = 1; p.atomic = (!det || accumulate) ? 1 : 0; p.alpha = alpha;
  p.C = C; p.ldc = ldc; p.n_store = N; p.special_col = -1; p.special_out = nullptr; p.a_sym_kb = kb_half;
  if (det) p.sk_ws = (float*)workspace;
  else if (!accumulate) DAE_CUDA(cudaMemset2DAsync(C, ldc * sizeof(float), 0, (size_t)N * sizeof(float), M, st));
  Operand A{g_hi, g_lo, ldg, 0}, B{b_hi, b_lo, ldb, 1};
  int n = 0;
  int rc = launch_gemm_maj<128, 2, 0, 6>(A, B, p, st, &n);
  if (rc) return rc;
  if (det) {
    DAE_REQUIRE(n <= kMaxFixupCtas, "%s: %d stream-K CTAs exceed the fixup's %d", fn, n, kMaxFixupCtas);
    const int tm = (M + 127) / 128, tn = (N + 127) / 128;
    sk_fixup_kernel<128><<<dim3(tm * tn, kFixupSlices), 256, 0, st>>>(p, tm, tm * tn, 2 * kb_half, n);
  }
  DAE_CHECK_LAUNCH(fn);
  return DAE_OK;
}

extern "C" int dae_gemm_sym_bf16x3(int32_t M, int32_t N, float alpha, const void* g_hi, const void* g_lo, int64_t ldg, const void* b_hi,
                                   const void* b_lo, int64_t ldb, float* C, int64_t ldc, int32_t accumulate, void* stream) {
  return gemm_sym_bf16x3("dae_gemm_sym_bf16x3", false, M, N, alpha, g_hi, g_lo, ldg, b_hi, b_lo, ldb, C, ldc, accumulate, nullptr, 0,
                         stream);
}

extern "C" int dae_gemm_sym_bf16x3_det(int32_t M, int32_t N, float alpha, const void* g_hi, const void* g_lo, int64_t ldg, const void* b_hi,
                                       const void* b_lo, int64_t ldb, float* C, int64_t ldc, int32_t accumulate, void* workspace,
                                       int64_t workspace_bytes, void* stream) {
  return gemm_sym_bf16x3("dae_gemm_sym_bf16x3_det", true, M, N, alpha, g_hi, g_lo, ldg, b_hi, b_lo, ldb, C, ldc, accumulate, workspace,
                         workspace_bytes, stream);
}

extern "C" int dae_gemm_det_workspace(int64_t* bytes) {
  DAE_REQUIRE(bytes, "dae_gemm_det_workspace: null pointer");
  *bytes = sk_workspace_bytes();
  return DAE_OK;
}

extern "C" int dae_decode_prepare(int32_t Brows, int32_t F, const int64_t* indptr, const int32_t* indices, const int32_t* rows,
                                  float* row_loss_part, int32_t* tile_ptr, void* stream) {
  DAE_REQUIRE(Brows > 0 && F > 0 && indptr && indices && row_loss_part && tile_ptr, "dae_decode_prepare: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  DAE_CUDA(cudaMemsetAsync(row_loss_part, 0, sizeof(float) * Brows, st));
  const int n_half = 2 * ((F + kDecodeN - 1) / kDecodeN);            // two column parts per tile of the fused decode kernel
  dim3 grid((n_half + 1 + 127) / 128, Brows < 65535 ? Brows : 65535);
  decode_tile_ptr_kernel<<<grid, 128, 0, st>>>(indptr, indices, rows, Brows, n_half, kDecodeN / 2, tile_ptr);
  DAE_CHECK_LAUNCH("dae_decode_prepare");
  return DAE_OK;
}

// dae_decode_fused_bf16x3 and, with det, dae_decode_fused_bf16x3_det: row_loss_part is then [dae_decode_loss_parts][Brows], one store
// per (half tile, row) instead of an atomic add per row
static int decode_fused(const char* fn, bool det, int32_t Brows, int32_t F, int32_t K, const void* e_hi, const void* e_lo, int64_t lde,
                        const void* w_hi, const void* w_lo, int64_t ldw, const int64_t* indptr, const int32_t* indices,
                        const float* values, const int32_t* rows, const float* bv, int32_t dec_act, int32_t loss_func,
                        const float* weight, const double* stats, void* dz_hi, void* dz_lo, int64_t ld_dz, float* row_loss_part,
                        int32_t* tile_ptr, int32_t prepared, void* stream) {
  DAE_REQUIRE(e_hi && e_lo && w_hi && w_lo && indptr && indices && values && bv && stats && dz_hi && dz_lo && row_loss_part && tile_ptr,
              "%s: null pointer", fn);
  DAE_REQUIRE(loss_func == DAE_LOSS_CE || loss_func == DAE_LOSS_MSE, "%s: cosine loss uses the unfused path", fn);
  DAE_REQUIRE(lde % 8 == 0 && ldw % 8 == 0 && ld_dz % 32 == 0 && ld_dz >= F, "%s: bad leading dimensions", fn);
  cudaStream_t st = (cudaStream_t)stream;
  GemmParams p{};
  p.M = Brows; p.N = F; p.K = K; p.k_splits = 1; p.alpha = 1.0f; p.special_col = -1;
  p.indptr = indptr; p.indices = indices; p.values = values; p.rows = rows; p.bv = bv; p.weight = weight; p.stats = stats;
  p.dz_hi = (__nv_bfloat16*)dz_hi; p.dz_lo = (__nv_bfloat16*)dz_lo; p.ld_dz = ld_dz; p.row_loss_part = row_loss_part;
  p.tile_ptr = tile_ptr; p.loss_parts = det ? 1 : 0;
  // dae_decode_prepare not issued by the caller (e.g. on a parallel graph branch): do it in line.  (det: its zeroing of the first
  // Brows floats is harmless, every part is stored)
  if (!prepared) {
    int rc0 = dae_decode_prepare(Brows, F, indptr, indices, rows, row_loss_part, tile_ptr, stream);
    if (rc0) return rc0;
  }
  Operand A{e_hi, e_lo, lde, 0}, B{w_hi, w_lo, ldw, 0};
  int rc = (loss_func == DAE_LOSS_CE) ? launch_decode<DAE_LOSS_CE>(dec_act, A, B, p, st)
                                      : launch_decode<DAE_LOSS_MSE>(dec_act, A, B, p, st);
  if (rc) return rc;
  DAE_CHECK_LAUNCH(fn);
  return DAE_OK;
}

extern "C" int dae_decode_fused_bf16x3(int32_t Brows, int32_t F, int32_t K, const void* e_hi, const void* e_lo, int64_t lde,
                                       const void* w_hi, const void* w_lo, int64_t ldw, const int64_t* indptr, const int32_t* indices,
                                       const float* values, const int32_t* rows, const float* bv, int32_t dec_act, int32_t loss_func,
                                       const float* weight, const double* stats, void* dz_hi, void* dz_lo, int64_t ld_dz,
                                       float* row_loss_part, int32_t* tile_ptr, int32_t prepared, void* stream) {
  return decode_fused("dae_decode_fused_bf16x3", false, Brows, F, K, e_hi, e_lo, lde, w_hi, w_lo, ldw, indptr, indices, values, rows, bv,
                      dec_act, loss_func, weight, stats, dz_hi, dz_lo, ld_dz, row_loss_part, tile_ptr, prepared, stream);
}

extern "C" int dae_decode_fused_bf16x3_det(int32_t Brows, int32_t F, int32_t K, const void* e_hi, const void* e_lo, int64_t lde,
                                           const void* w_hi, const void* w_lo, int64_t ldw, const int64_t* indptr, const int32_t* indices,
                                           const float* values, const int32_t* rows, const float* bv, int32_t dec_act, int32_t loss_func,
                                           const float* weight, const double* stats, void* dz_hi, void* dz_lo, int64_t ld_dz,
                                           float* row_loss_parts, int32_t* tile_ptr, int32_t prepared, void* stream) {
  return decode_fused("dae_decode_fused_bf16x3_det", true, Brows, F, K, e_hi, e_lo, lde, w_hi, w_lo, ldw, indptr, indices, values, rows,
                      bv, dec_act, loss_func, weight, stats, dz_hi, dz_lo, ld_dz, row_loss_parts, tile_ptr, prepared, stream);
}

extern "C" int dae_decode_loss_parts(int32_t F, int32_t* n_parts) {
  DAE_REQUIRE(F > 0 && n_parts, "dae_decode_loss_parts: bad arguments");
  *n_parts = 2 * ((F + kDecodeN - 1) / kDecodeN);
  return DAE_OK;
}

extern "C" int dae_similarity_topk_workspace(int32_t n_query, int32_t n_corpus, int32_t k, int32_t splits, int64_t* bytes) {
  DAE_REQUIRE(bytes && n_query > 0 && n_corpus > 0, "dae_similarity_topk_workspace: bad arguments");
  DAE_REQUIRE(k >= 1 && k <= kTopkMaxK, "dae_similarity_topk_workspace: k = %d is outside the supported range 1 <= k <= %d", k, kTopkMaxK);
  *bytes = topk_workspace_bytes(n_query, k, topk_splits(n_query, n_corpus, splits));
  return DAE_OK;
}

// the leading-dimension and alignment checks of the similarity exports over Q [n_query x dim] and C [n_corpus x dim] (bf16 hi / lo,
// K-major, read by TMA); a16 / a8 / a4: the export's other pointers that must be 16- / 8- / 4-byte aligned, or-ed together
static int check_operands(const char* fn, int32_t dim, const void* q_hi, const void* q_lo, int64_t ldq, const void* c_hi, const void* c_lo,
                          int64_t ldc, uintptr_t a16, uintptr_t a8, uintptr_t a4, const char* alignment) {
  DAE_REQUIRE(ldq >= dim && ldc >= dim && ldq % 8 == 0 && ldc % 8 == 0,
              "%s: leading dimensions must cover dim and be multiples of 8 (TMA 16-byte strides)", fn);
  DAE_REQUIRE(((uintptr_t)q_hi | (uintptr_t)q_lo | (uintptr_t)c_hi | (uintptr_t)c_lo | a16) % 16 == 0 && a8 % 8 == 0 && a4 % 4 == 0,
              "%s: %s", fn, alignment);
  return DAE_OK;
}

// the partial lists of k in `workspace`: 2 s per query row
static TopkParams topk_params(int32_t n_query, int32_t n_corpus, int32_t dim, int k, int s, int64_t diag_offset, int32_t exclude,
                              void* workspace) {
  TopkParams tp{};
  tp.g.M = n_query; tp.g.N = n_corpus; tp.g.K = dim; tp.g.k_splits = 1; tp.g.alpha = 1.0f; tp.g.special_col = -1;
  tp.k = k; tp.splits = s; tp.exclude = exclude ? 1 : 0; tp.diag_offset = diag_offset;
  tp.ws_val = reinterpret_cast<float*>(workspace);
  tp.ws_idx = reinterpret_cast<int32_t*>(reinterpret_cast<float*>(workspace) + (int64_t)n_query * 2 * s * k);
  return tp;
}

// dae_similarity_topk_bf16x3 (excl false), dae_similarity_topk_excl_bf16x3 (excl true, the lists ex_indptr / ex_indices) and
// dae_similarity_topk_groups_bf16x3 (excl true, groups non-null; ex_indptr may be null when ex_nnz = 0: no lists)
static int dense_topk(const char* fn, int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo, int64_t ldq,
                      const void* c_hi, const void* c_lo, int64_t ldc, int32_t k, int64_t diag_offset, int32_t exclude, int32_t splits,
                      void* workspace, int64_t workspace_bytes, int32_t* idx_out, float* val_out, bool excl, const int64_t* ex_indptr,
                      const int32_t* ex_indices, int64_t ex_nnz, const int32_t* groups, bool grouped, void* stream) {
  DAE_REQUIRE(q_hi && q_lo && c_hi && c_lo && workspace && idx_out && val_out &&
              (!excl || (grouped ? (groups && (ex_nnz == 0 || (ex_indptr && ex_indices))) : (ex_indptr && (ex_nnz == 0 || ex_indices)))),
              "%s: null pointer", fn);
  DAE_REQUIRE(n_query > 0 && n_corpus > 0 && dim > 0 && (!excl || ex_nnz >= 0), "%s: bad sizes", fn);
  DAE_REQUIRE(k >= 1 && k <= kTopkMaxK, "%s: k = %d is outside the supported range 1 <= k <= %d", fn, k, kTopkMaxK);
  int rc = check_operands(fn, dim, q_hi, q_lo, ldq, c_hi, c_lo, ldc, (uintptr_t)workspace, (uintptr_t)ex_indptr,
                          (uintptr_t)ex_indices | (uintptr_t)groups,
                          !excl     ? "operands and workspace must be 16-byte aligned"
                          : grouped ? "operands and workspace must be 16-byte, ex_indptr 8-byte, ex_indices and groups 4-byte aligned"
                                    : "operands and workspace must be 16-byte, ex_indptr 8-byte, ex_indices 4-byte aligned");
  if (rc) return rc;
  const int s = topk_splits(n_query, n_corpus, splits);
  const int64_t need = topk_workspace_bytes(n_query, k, s);
  DAE_REQUIRE(workspace_bytes >= need, "%s: workspace of %lld bytes, %lld needed (dae_similarity_topk_workspace)", fn,
              (long long)workspace_bytes, (long long)need);
  cudaStream_t st = (cudaStream_t)stream;
  TopkParams tp = topk_params(n_query, n_corpus, dim, k, s, diag_offset, exclude, workspace);
  tp.ex_indptr = ex_indptr; tp.ex_indices = ex_indices; tp.groups = groups;
  Operand A{q_hi, q_lo, ldq, 0}, B{c_hi, c_lo, ldc, 0};
  rc = !excl ? launch_topk<false, false>(A, B, tp, st) : !grouped ? launch_topk<true, false>(A, B, tp, st)
                                                         : launch_topk<true, true>(A, B, tp, st);
  if (rc) return rc;
  DAE_CHECK_LAUNCH(fn);
  if (grouped)
    topk_merge_groups_kernel<<<(n_query + 7) / 8, 256, 0, st>>>(tp.ws_val, tp.ws_idx, groups, n_query, 2 * s, k, idx_out, val_out);
  else
    topk_merge_kernel<<<(n_query + 7) / 8, 256, 0, st>>>(tp.ws_val, tp.ws_idx, n_query, 2 * s, k, idx_out, val_out);
  const cudaError_t e = cudaGetLastError();   // DAE_CHECK_LAUNCH with the name "<fn> (merge)"
  if (e != cudaSuccess) {
    set_error("%s (merge): %s", fn, cudaGetErrorString(e));
    return DAE_ERR_CUDA;
  }
  return DAE_OK;
}

extern "C" int dae_similarity_topk_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo, int64_t ldq,
                                          const void* c_hi, const void* c_lo, int64_t ldc, int32_t k, int64_t diag_offset, int32_t exclude,
                                          int32_t splits, void* workspace, int64_t workspace_bytes, int32_t* idx_out, float* val_out,
                                          void* stream) {
  return dense_topk("dae_similarity_topk_bf16x3", n_query, n_corpus, dim, q_hi, q_lo, ldq, c_hi, c_lo, ldc, k, diag_offset, exclude,
                    splits, workspace, workspace_bytes, idx_out, val_out, false, nullptr, nullptr, 0, nullptr, false, stream);
}

extern "C" int dae_similarity_topk_excl_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo,
                                               int64_t ldq, const void* c_hi, const void* c_lo, int64_t ldc, int32_t k,
                                               int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace,
                                               int64_t workspace_bytes, int32_t* idx_out, float* val_out, const int64_t* ex_indptr,
                                               const int32_t* ex_indices, int64_t ex_nnz, void* stream) {
  return dense_topk("dae_similarity_topk_excl_bf16x3", n_query, n_corpus, dim, q_hi, q_lo, ldq, c_hi, c_lo, ldc, k, diag_offset, exclude,
                    splits, workspace, workspace_bytes, idx_out, val_out, true, ex_indptr, ex_indices, ex_nnz, nullptr, false, stream);
}

extern "C" int dae_similarity_topk_groups_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo,
                                                 int64_t ldq, const void* c_hi, const void* c_lo, int64_t ldc, int32_t k,
                                                 int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace,
                                                 int64_t workspace_bytes, int32_t* idx_out, float* val_out, const int64_t* ex_indptr,
                                                 const int32_t* ex_indices, int64_t ex_nnz, const int32_t* groups, void* stream) {
  return dense_topk("dae_similarity_topk_groups_bf16x3", n_query, n_corpus, dim, q_hi, q_lo, ldq, c_hi, c_lo, ldc, k, diag_offset,
                    exclude, splits, workspace, workspace_bytes, idx_out, val_out, true, ex_indptr, ex_indices, ex_nnz, groups, true,
                    stream);
}

extern "C" int dae_similarity_pair_hist_bf16x3(int32_t n, int32_t dim, const void* x_hi, const void* x_lo, int64_t ldx,
                                               const int32_t* labels, float range, int32_t bins, uint64_t* hist, double* sums,
                                               void* stream) {
  DAE_REQUIRE(x_hi && x_lo && labels && hist && sums, "dae_similarity_pair_hist_bf16x3: null pointer");
  DAE_REQUIRE(n >= 2 && dim > 0, "dae_similarity_pair_hist_bf16x3: bad sizes (n = %d >= 2 rows and dim = %d > 0 needed)", n, dim);
  DAE_REQUIRE(hist_bins_ok(bins), "dae_similarity_pair_hist_bf16x3: bins = %d is not a power of two in [2^%d, 2^%d]", bins,
              kHistMinLog2Bins, kHistMaxLog2Bins);
  DAE_REQUIRE(hist_range_ok(range), "dae_similarity_pair_hist_bf16x3: range M = %g is not a power of two in [2^-64, 2^64]", (double)range);
  DAE_REQUIRE(ldx >= dim && ldx % 8 == 0,
              "dae_similarity_pair_hist_bf16x3: the leading dimension must cover dim and be a multiple of 8 (TMA 16-byte strides)");
  DAE_REQUIRE(((uintptr_t)x_hi | (uintptr_t)x_lo) % 16 == 0 && ((uintptr_t)hist | (uintptr_t)sums) % 8 == 0 && (uintptr_t)labels % 4 == 0,
              "dae_similarity_pair_hist_bf16x3: operands must be 16-byte, hist and sums 8-byte, labels 4-byte aligned");
  PairHistParams hp{};
  hp.g.M = n; hp.g.N = n; hp.g.K = dim; hp.g.k_splits = 1; hp.g.alpha = 1.0f; hp.g.special_col = -1;
  hp.labels = labels; hp.range = range; hp.scale = (float)bins / (2.0f * range); hp.bins = (uint32_t)bins;
  hp.hist = reinterpret_cast<unsigned long long*>(hist); hp.sums = sums;
  Operand X{x_hi, x_lo, ldx, 0};
  const long long tm = (n + BLOCK_M - 1) / BLOCK_M;   // work items: the lower-triangle tiles
  int rc = launch_persistent<pair_hist_kernel, kTopkBK, kTopkStages>(X, X, hp.g, hp, tm * (tm + 1) / 2, (cudaStream_t)stream);
  if (rc) return rc;
  DAE_CHECK_LAUNCH("dae_similarity_pair_hist_bf16x3");
  return DAE_OK;
}

// the PairsParams common to dae_similarity_pairs_bf16x3 and the collect stage of long top-k lists
static PairsParams pairs_params(int32_t n_query, int32_t n_corpus, int32_t dim, uint64_t* count, int64_t capacity, int32_t* i_out,
                                int32_t* j_out, float* s_out) {
  PairsParams pp{};
  pp.g.M = n_query; pp.g.N = n_corpus; pp.g.K = dim; pp.g.k_splits = 1; pp.g.alpha = 1.0f; pp.g.special_col = -1;
  pp.count = reinterpret_cast<unsigned long long*>(count); pp.capacity = (unsigned long long)capacity;
  pp.i_out = i_out; pp.j_out = j_out; pp.s_out = s_out;
  return pp;
}

extern "C" int dae_similarity_pairs_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo, int64_t ldq,
                                           const void* c_hi, const void* c_lo, int64_t ldc, int32_t self, float threshold, uint64_t* count,
                                           int64_t capacity, int32_t* i_out, int32_t* j_out, float* s_out, void* stream) {
  DAE_REQUIRE(q_hi && q_lo && c_hi && c_lo && count, "dae_similarity_pairs_bf16x3: null pointer");
  DAE_REQUIRE(capacity >= 0, "dae_similarity_pairs_bf16x3: capacity = %lld < 0", (long long)capacity);
  DAE_REQUIRE(capacity == 0 || (i_out && j_out && s_out), "dae_similarity_pairs_bf16x3: null output with capacity %lld > 0",
              (long long)capacity);
  DAE_REQUIRE(n_query > 0 && n_corpus > 0 && dim > 0, "dae_similarity_pairs_bf16x3: bad sizes");
  DAE_REQUIRE(!self || (n_query == n_corpus && q_hi == c_hi && q_lo == c_lo && ldq == ldc),
              "dae_similarity_pairs_bf16x3: self mode needs the corpus operands to be the query operands");
  DAE_REQUIRE(pair_threshold_ok(threshold), "dae_similarity_pairs_bf16x3: threshold %g is not finite", (double)threshold);
  int rc = check_operands("dae_similarity_pairs_bf16x3", dim, q_hi, q_lo, ldq, c_hi, c_lo, ldc, 0, (uintptr_t)count,
                          (uintptr_t)i_out | (uintptr_t)j_out | (uintptr_t)s_out,
                          "operands must be 16-byte, the counter 8-byte and the outputs 4-byte aligned");
  if (rc) return rc;
  PairsParams pp = pairs_params(n_query, n_corpus, dim, count, capacity, i_out, j_out, s_out);
  pp.self = self ? 1 : 0; pp.tau = threshold;
  Operand A{q_hi, q_lo, ldq, 0}, B{c_hi, c_lo, ldc, 0};
  rc = launch_pairs<false>(A, B, pp, (cudaStream_t)stream);
  if (rc) return rc;
  DAE_CHECK_LAUNCH("dae_similarity_pairs_bf16x3");
  return DAE_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// long top-k lists (k up to kTopkLongMaxK, DESIGN 4.14): bound, collect, select.  The bound runs topk_kernel<32> with enough splits
// that the 2 * splits partial lists of 32 hold at least 2k entries; their k-th best is a lower bound tau_i on the row's k-th score.
// The collect stage (pairs_kernel<true>) lists every candidate with s >= tau_i, so every answer; dae_pairs_sort makes each row's
// candidates contiguous in increasing column order, and the select stage ranks them.  All scores come from the same tiles and
// k16 order as topk_kernel's, so they are its bits.
// ---------------------------------------------------------------------------------------------------------------------
static int topk_bound_splits(int n_query, int n_corpus, int k, int requested) {
  const int s = topk_splits(n_query, n_corpus, requested);
  const int need = (k + 31) / 32;
  return topk_splits(n_query, n_corpus, s > need ? s : need);
}

// rank chunk L of topk_bound_kernel / topk_select_kernel: a power of two >= k, and a multiple of the block size
static int rank_chunk(int k) {
  int L = kRankThreads;
  while (L < k) L <<= 1;
  return L;
}

extern "C" int dae_similarity_topk_bound_workspace(int32_t n_query, int32_t n_corpus, int32_t k, int32_t splits, int64_t* bytes) {
  DAE_REQUIRE(bytes && n_query > 0 && n_corpus > 0, "dae_similarity_topk_bound_workspace: bad arguments");
  DAE_REQUIRE(k >= 1 && k <= kTopkLongMaxK, "dae_similarity_topk_bound_workspace: k = %d is outside the supported range 1 <= k <= %d", k,
              kTopkLongMaxK);
  *bytes = topk_workspace_bytes(n_query, kTopkMaxK, topk_bound_splits(n_query, n_corpus, k, splits));
  return DAE_OK;
}

extern "C" int dae_similarity_topk_bound_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo,
                                                int64_t ldq, const void* c_hi, const void* c_lo, int64_t ldc, int32_t k,
                                                int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace,
                                                int64_t workspace_bytes, const int64_t* ex_indptr, const int32_t* ex_indices,
                                                int64_t ex_nnz, const int32_t* groups, float* tau, void* stream) {
  DAE_REQUIRE(q_hi && q_lo && c_hi && c_lo && workspace && tau && (ex_nnz == 0 || (ex_indptr && ex_indices)),
              "dae_similarity_topk_bound_bf16x3: null pointer");
  DAE_REQUIRE(n_query > 0 && n_corpus > 0 && dim > 0 && ex_nnz >= 0, "dae_similarity_topk_bound_bf16x3: bad sizes");
  DAE_REQUIRE(k >= 1 && k <= kTopkLongMaxK, "dae_similarity_topk_bound_bf16x3: k = %d is outside the supported range 1 <= k <= %d", k,
              kTopkLongMaxK);
  int rc = check_operands("dae_similarity_topk_bound_bf16x3", dim, q_hi, q_lo, ldq, c_hi, c_lo, ldc, (uintptr_t)workspace,
                          (uintptr_t)ex_indptr, (uintptr_t)ex_indices | (uintptr_t)groups | (uintptr_t)tau,
                          "operands and workspace must be 16-byte, ex_indptr 8-byte, ex_indices, groups and tau 4-byte aligned");
  if (rc) return rc;
  const int s = topk_bound_splits(n_query, n_corpus, k, splits);
  const int64_t need = topk_workspace_bytes(n_query, kTopkMaxK, s);
  DAE_REQUIRE(workspace_bytes >= need,
              "dae_similarity_topk_bound_bf16x3: workspace of %lld bytes, %lld needed (dae_similarity_topk_bound_workspace)",
              (long long)workspace_bytes, (long long)need);
  cudaStream_t st = (cudaStream_t)stream;
  TopkParams tp = topk_params(n_query, n_corpus, dim, kTopkMaxK, s, diag_offset, exclude, workspace);
  tp.ex_indptr = ex_nnz ? ex_indptr : nullptr; tp.ex_indices = ex_indices; tp.groups = groups;
  Operand A{q_hi, q_lo, ldq, 0}, B{c_hi, c_lo, ldc, 0};
  rc = groups ? launch_topk<true, true>(A, B, tp, st)
              : (tp.ex_indptr ? launch_topk<true, false>(A, B, tp, st) : launch_topk<false, false>(A, B, tp, st));
  if (rc) return rc;
  DAE_CHECK_LAUNCH("dae_similarity_topk_bound_bf16x3");
  const int L = rank_chunk(k);
  if (groups)
    topk_bound_kernel<true><<<n_query, kRankThreads, 4 * L * 8, st>>>(tp.ws_val, tp.ws_idx, 2 * s, kTopkMaxK, k, L, groups, tau);
  else
    topk_bound_kernel<false><<<n_query, kRankThreads, 2 * L * 8, st>>>(tp.ws_val, tp.ws_idx, 2 * s, kTopkMaxK, k, L, nullptr, tau);
  DAE_CHECK_LAUNCH("dae_similarity_topk_bound_bf16x3 (bound)");
  return DAE_OK;
}

extern "C" int dae_similarity_topk_collect_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo,
                                                  int64_t ldq, const void* c_hi, const void* c_lo, int64_t ldc, int64_t diag_offset,
                                                  int32_t exclude, const float* tau, const int64_t* ex_indptr, const int32_t* ex_indices,
                                                  int64_t ex_nnz, uint64_t* count, uint32_t* row_count, int64_t capacity, int32_t* i_out,
                                                  int32_t* j_out, float* s_out, void* stream) {
  DAE_REQUIRE(q_hi && q_lo && c_hi && c_lo && tau && count && row_count && (ex_nnz == 0 || (ex_indptr && ex_indices)),
              "dae_similarity_topk_collect_bf16x3: null pointer");
  DAE_REQUIRE(capacity >= 0, "dae_similarity_topk_collect_bf16x3: capacity = %lld < 0", (long long)capacity);
  DAE_REQUIRE(capacity == 0 || (i_out && j_out && s_out), "dae_similarity_topk_collect_bf16x3: null output with capacity %lld > 0",
              (long long)capacity);
  DAE_REQUIRE(n_query > 0 && n_corpus > 0 && dim > 0 && ex_nnz >= 0, "dae_similarity_topk_collect_bf16x3: bad sizes");
  int rc = check_operands("dae_similarity_topk_collect_bf16x3", dim, q_hi, q_lo, ldq, c_hi, c_lo, ldc, 0,
                          (uintptr_t)count | (uintptr_t)ex_indptr,
                          (uintptr_t)tau | (uintptr_t)row_count | (uintptr_t)ex_indices | (uintptr_t)i_out | (uintptr_t)j_out |
                              (uintptr_t)s_out,
                          "operands must be 16-byte, the counter and ex_indptr 8-byte, the other arrays 4-byte aligned");
  if (rc) return rc;
  PairsParams pp = pairs_params(n_query, n_corpus, dim, count, capacity, i_out, j_out, s_out);
  pp.row_tau = tau; pp.diag_offset = diag_offset; pp.exclude = exclude ? 1 : 0;
  pp.ex_indptr = ex_nnz ? ex_indptr : nullptr; pp.ex_indices = ex_indices; pp.row_count = row_count;
  Operand A{q_hi, q_lo, ldq, 0}, B{c_hi, c_lo, ldc, 0};
  rc = launch_pairs<true>(A, B, pp, (cudaStream_t)stream);
  if (rc) return rc;
  DAE_CHECK_LAUNCH("dae_similarity_topk_collect_bf16x3");
  return DAE_OK;
}

extern "C" int dae_similarity_topk_select(int32_t n_query, int64_t n_pairs, const int32_t* i_sorted, const int32_t* j_sorted,
                                          const float* s_sorted, int32_t k, const int32_t* groups, int32_t* idx_out, float* val_out,
                                          void* stream) {
  DAE_REQUIRE(idx_out && val_out && (n_pairs == 0 || (i_sorted && j_sorted && s_sorted)), "dae_similarity_topk_select: null pointer");
  DAE_REQUIRE(n_query > 0 && n_pairs >= 0 && n_pairs <= INT32_MAX, "dae_similarity_topk_select: bad sizes");
  DAE_REQUIRE(k >= 1 && k <= kTopkLongMaxK, "dae_similarity_topk_select: k = %d is outside the supported range 1 <= k <= %d", k,
              kTopkLongMaxK);
  DAE_REQUIRE(((uintptr_t)i_sorted | (uintptr_t)j_sorted | (uintptr_t)s_sorted | (uintptr_t)groups | (uintptr_t)idx_out |
               (uintptr_t)val_out) % 4 == 0,
              "dae_similarity_topk_select: arrays must be 4-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int L = rank_chunk(k);
  if (groups)
    topk_select_kernel<true><<<n_query, kRankThreads, 4 * L * 8, st>>>(i_sorted, j_sorted, s_sorted, n_pairs, k, L, groups, idx_out,
                                                                        val_out);
  else
    topk_select_kernel<false><<<n_query, kRankThreads, 2 * L * 8, st>>>(i_sorted, j_sorted, s_sorted, n_pairs, k, L, nullptr, idx_out,
                                                                         val_out);
  DAE_CHECK_LAUNCH("dae_similarity_topk_select");
  return DAE_OK;
}
