// K4: online triplet mining on the Gram matrix S = E.E^T -- loss, statistics and G = dL_tri/dS, fused, with no
// B^3 storage.
//
// Reference ops replaced: the B x B x B broadcast / mask / softplus / reduce chain of batch_all_triplet_loss
// (autoencoder/triplet_loss_utils.py:96-131) and the row reductions of batch_hard_triplet_loss (:219-259), plus
// their autodiff; and the row-wise explicit-triplet loss (autoencoder/autoencoder_triplet.py:308-311).
//
// batch_all: rows are label sorted (dae_batch_prepare), so for anchor i the positives are the contiguous segment
// [lo,hi) \ {i} and the negatives the rest.  One CTA per anchor sweeps the n_pos x n_neg rectangle in registers:
//   softplus(S_ik - S_ij) = log(1 + u_j v_k),  u_j = exp(m - S_ij), v_k = exp(S_ik - m)   (one FFMA + 2 MUFU per triplet)
// The sweep is bound by the MUFU pipe (lg2 + rcp per triplet), not by HBM or tensor throughput.
#include <cuda_bf16.h>
#include "common.cuh"

namespace dae {

constexpr int kTY = 8, kTX = 32, kTJ = 4, kTK = 4;
constexpr int kJTile = kTY * kTJ;   // 32 positives per j-tile
constexpr int kKTile = kTX * kTK;   // 128 negatives per k-tile
constexpr int kTripThreads = kTY * kTX;

__device__ __forceinline__ float fast_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float fast_lg2(float x) { float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float fast_ex2(float x) { float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

// ---- fp32 register pairs: the tier-0 tile packs its 4 x 4 triplets as 2 row pairs x 4 columns and runs every multiply / add on
// pairs.  sm_90 has no packed fp32x2 instructions, so each pair operation is two round-to-nearest scalar ops (no contraction into
// FMAs the formulation does not have).
typedef float2 f2;
__device__ __forceinline__ f2 pk(float lo, float hi) { return make_float2(lo, hi); }
__device__ __forceinline__ void upk(f2 v, float& lo, float& hi) { lo = v.x; hi = v.y; }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

// TIER 0 on row pairs: U = (u_a, u_a'), V[b] = (v_b, v_b).  Same arithmetic as triplet_tile<0> below (e = u v, t = 1 + e, one
// log2 and one reciprocal per four t's of a ROW), lane-wise.  rs += row sums of sigma (pair), cs[b] += column sums (pair: the two
// rows still separate), lg += sum of log2(1 + e).
__device__ __forceinline__ void triplet_pair_tile(f2 U, const f2 (&V)[kTK], f2& rs, f2 (&cs)[kTK], float& lg) {
  const f2 one = pk(1.0f, 1.0f);
  f2 e[kTK], t[kTK];
#pragma unroll
  for (int b = 0; b < kTK; ++b) { e[b] = mul2(U, V[b]); t[b] = fma2(U, V[b], one); }
  const f2 p01 = mul2(t[0], t[1]), p23 = mul2(t[2], t[3]), P = mul2(p01, p23);
  float Px, Py;
  upk(P, Px, Py);
  lg += fast_lg2(Px) + fast_lg2(Py);
  const f2 r = pk(fast_rcp(Px), fast_rcp(Py));
  const f2 r01 = mul2(r, p23), r23 = mul2(r, p01);
  const f2 s0 = mul2(e[0], mul2(r01, t[1])), s1 = mul2(e[1], mul2(r01, t[0]));
  const f2 s2 = mul2(e[2], mul2(r23, t[3])), s3 = mul2(e[3], mul2(r23, t[2]));
  rs = add2(rs, add2(add2(s0, s1), add2(s2, s3)));
  cs[0] = add2(cs[0], s0); cs[1] = add2(cs[1], s1); cs[2] = add2(cs[2], s2); cs[3] = add2(cs[3], s3);
}

// One 4 x 4 register tile of triplets: sg[a][b] = sigmoid(x_ab) = e/(1+e) with e = exp(x_ab) = u_a v_b (computed as e * 1/(1+e),
// which keeps full relative accuracy when sigmoid is tiny), lg += sum of log2(1 + e).
//   TIER 0 (row range < 10): t = 1 + e <= 2.2e4, so products of four t's stay finite: ONE lg2 and ONE rcp per four
//                            triplets (log of the product; Montgomery batch inversion) -> 0.5 MUFU per triplet.  x >= -10 here,
//                            so e >= 4.5e-5 and fp32's t = 1 + e keeps the term.
//   TIER 1 (row range < 80): one lg2 + one rcp per triplet on the factorised exponentials.
//   TIER 2                 : direct, overflow-safe evaluation (3 MUFU per triplet).
// In tiers 1 and 2, log2(1 + e) for e < 2^-12 is the series (e - e^2 / 2) / ln 2, within e^2 / 3 <= 2^-25 of the term: fp32's
// 1 + e is 1 for e < 2^-24 (x < -16.6), so lg2(t) would drop a well-separated triplet's loss term, and lg2.approx's 2^-22 absolute
// error is already 2^-10.5 of log2(1 + e) at e = 2^-12.  Only the loss changes: sigma = e * rcp(t) keeps full relative accuracy.
constexpr float kSeriesMax = 0x1p-12f;
__device__ __forceinline__ float ln_1p_small(float e) { return fmaf(-0.5f * e, e, e); }   // e - e^2 / 2

template <int TIER>
__device__ __forceinline__ void triplet_tile(const float (&s_j)[kTJ], const float (&u_j)[kTJ], const float (&s_k)[kTK],
                                             const float (&v_k)[kTK], float (&sg)[kTJ][kTK], float& lg) {
#pragma unroll
  for (int a = 0; a < kTJ; ++a) {
    if (TIER == 0) {
      const float e0 = u_j[a] * v_k[0], e1 = u_j[a] * v_k[1], e2 = u_j[a] * v_k[2], e3 = u_j[a] * v_k[3];
      const float t0 = e0 + 1.0f, t1 = e1 + 1.0f, t2 = e2 + 1.0f, t3 = e3 + 1.0f;
      const float p01 = t0 * t1, p23 = t2 * t3, P = p01 * p23;
      lg += fast_lg2(P);
      const float r = fast_rcp(P);
      const float r01 = r * p23, r23 = r * p01;
      sg[a][0] = e0 * (r01 * t1); sg[a][1] = e1 * (r01 * t0); sg[a][2] = e2 * (r23 * t3); sg[a][3] = e3 * (r23 * t2);
    } else if (TIER == 1) {
#pragma unroll
      for (int b = 0; b < kTK; ++b) {
        const float e = u_j[a] * v_k[b];
        const float t = e + 1.0f;
        if (e < kSeriesMax) lg = fmaf(ln_1p_small(e), kLog2e, lg); else lg += fast_lg2(t);
        sg[a][b] = e * fast_rcp(t);
      }
    } else if (TIER == 3) {   // pos_triplets_only (triplet_loss_utils.py:118-120): softplus and COUNTS over positive triplets only
#pragma unroll
      for (int b = 0; b < kTK; ++b) {
        const bool pos = (s_j[a] < 1.0e38f) && (s_k[b] > s_j[a]);   // s_j is the positive test's threshold (pos_threshold)
        const float x = s_k[b] - s_j[a];
        const float em = fast_ex2(-fabsf(x) * kLog2e);
        lg += pos ? (fmaxf(x, 0.0f) * kLog2e + fast_lg2(1.0f + em)) : 0.0f;
        sg[a][b] = pos ? 1.0f : 0.0f;
      }
    } else {
#pragma unroll
      for (int b = 0; b < kTK; ++b) {
        const bool valid = (s_j[a] < 1.0e38f) && (s_k[b] > -1.0e38f);
        const float x = s_k[b] - s_j[a];
        const float em = fast_ex2(-fabsf(x) * kLog2e);
        const float t = 1.0f + em;
        const float r = fast_rcp(t);
        const float l1p = (em < kSeriesMax) ? ln_1p_small(em) * kLog2e : fast_lg2(t);
        lg += valid ? (fmaxf(x, 0.0f) * kLog2e + l1p) : 0.0f;
        sg[a][b] = valid ? (x >= 0.0f ? r : em * r) : 0.0f;
      }
    }
  }
}

// The reference counts a triplet as positive when fp32(S_ik - S_ij) > 1e-16f (triplet_loss_utils.py:114).  fp32(b - a) is monotone
// in b, so that test is S_ik > t(S_ij) with t(a) = the largest fp32 b for which fp32(b - a) <= 1e-16f: one compare per triplet.
// t(a) = a whenever |a| >= 2^-29 (one ulp of a exceeds 1e-16f).  Below, a bisection on the ordered-integer encoding of fp32 finds it
// (stepping ulp by ulp would take ~2^23 steps near a = -1e-16); the staging loops run it once per positive, not per triplet.
__device__ __forceinline__ int f32_ordered(float f) { const int b = __float_as_int(f); return b < 0 ? -(b & 0x7fffffff) : b; }
__device__ __forceinline__ float f32_from_ordered(int o) { return __int_as_float(o < 0 ? ((-o) | (int)0x80000000) : o); }
__device__ __noinline__ float pos_threshold_small(float a) {
  int lo = f32_ordered(a), hi = f32_ordered(__fadd_rn(a, 1e-15f));   // fp32(a - a) = 0 passes, fp32(hi - a) ~ 1e-15 fails
  while (hi - lo > 1) {
    const int mid = lo + ((hi - lo) >> 1);
    if (__fsub_rn(f32_from_ordered(mid), a) <= 1e-16f) lo = mid; else hi = mid;
  }
  return f32_from_ordered(lo);
}
__device__ __forceinline__ float pos_threshold(float a) { return fabsf(a) >= 0x1p-29f ? a : pos_threshold_small(a); }

// smem layout (floats): sj[Pj] uj[Pj] gj[Pj] | sk[Pk] vk[Pk] | gk[kTY][Pk]      Pj, Pk = padded counts
// sj holds pos_threshold(S_ij), so that the reference's positive test is one compare per triplet.
template <int TIER>
__device__ __forceinline__ void triplet_sweep(const float* sj, const float* uj, float* gj, const float* sk, const float* vk, float* gk,
                                              int Pj, int Pk, int Pk_max, int tx, int ty, float& lacc, int& npos) {
  for (int jt = 0; jt < Pj; jt += kJTile) {
    float s_j[kTJ], u_j[kTJ], rs[kTJ];
#pragma unroll
    for (int a = 0; a < kTJ; ++a) { s_j[a] = sj[jt + ty * kTJ + a]; u_j[a] = uj[jt + ty * kTJ + a]; rs[a] = 0.0f; }
    if (TIER == 0) {   // packed fp32x2 path
      const f2 U01 = pk(u_j[0], u_j[1]), U23 = pk(u_j[2], u_j[3]);
      f2 rs01 = pk(0.0f, 0.0f), rs23 = pk(0.0f, 0.0f);
      for (int kt = 0; kt < Pk; kt += kKTile) {
        const int q0 = kt + tx * kTK;
        const float4 s4 = *reinterpret_cast<const float4*>(sk + q0);
        const float4 v4 = *reinterpret_cast<const float4*>(vk + q0);
        const float s_k[kTK] = {s4.x, s4.y, s4.z, s4.w};
        const f2 V[kTK] = {pk(v4.x, v4.x), pk(v4.y, v4.y), pk(v4.z, v4.z), pk(v4.w, v4.w)};
        f2 cs[kTK] = {pk(0.0f, 0.0f), pk(0.0f, 0.0f), pk(0.0f, 0.0f), pk(0.0f, 0.0f)};
        triplet_pair_tile(U01, V, rs01, cs, lacc);
        triplet_pair_tile(U23, V, rs23, cs, lacc);
#pragma unroll
        for (int a = 0; a < kTJ; ++a) {
#pragma unroll
          for (int b = 0; b < kTK; ++b)   // fp32(S_ik - S_ij) > 1e-16 (triplet_loss_utils.py:114): one compare + one predicated add
            asm("{ .reg .pred p; setp.gt.f32 p, %1, %2; @p add.s32 %0, %0, 1; }" : "+r"(npos) : "f"(s_k[b]), "f"(s_j[a]));
        }
        float4* g = reinterpret_cast<float4*>(gk + ty * Pk_max + q0);
        float4 o = *g;
        float lo, hi;
        upk(cs[0], lo, hi); o.x += lo + hi;
        upk(cs[1], lo, hi); o.y += lo + hi;
        upk(cs[2], lo, hi); o.z += lo + hi;
        upk(cs[3], lo, hi); o.w += lo + hi;
        *g = o;
      }
      upk(rs01, rs[0], rs[1]);
      upk(rs23, rs[2], rs[3]);
    } else
    for (int kt = 0; kt < Pk; kt += kKTile) {
      const int q0 = kt + tx * kTK;
      const float4 s4 = *reinterpret_cast<const float4*>(sk + q0);
      const float4 v4 = *reinterpret_cast<const float4*>(vk + q0);
      const float s_k[kTK] = {s4.x, s4.y, s4.z, s4.w};
      const float v_k[kTK] = {v4.x, v4.y, v4.z, v4.w};
      float sg[kTJ][kTK];
      triplet_tile<TIER>(s_j, u_j, s_k, v_k, sg, lacc);
      float cs[kTK] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
      for (int a = 0; a < kTJ; ++a) {
#pragma unroll
        for (int b = 0; b < kTK; ++b) {
          // fp32(S_ik - S_ij) > 1e-16 (triplet_loss_utils.py:114): one compare + one predicated add
          asm("{ .reg .pred p; setp.gt.f32 p, %1, %2; @p add.s32 %0, %0, 1; }" : "+r"(npos) : "f"(s_k[b]), "f"(s_j[a]));
          rs[a] += sg[a][b];
          cs[b] += sg[a][b];
        }
      }
      float4* g = reinterpret_cast<float4*>(gk + ty * Pk_max + q0);
      float4 o = *g;
      o.x += cs[0]; o.y += cs[1]; o.z += cs[2]; o.w += cs[3];
      *g = o;
    }
#pragma unroll
    for (int a = 0; a < kTJ; ++a) {
      const float t = warp_sum(rs[a]);
      if (tx == 0) gj[jt + ty * kTJ + a] = t;
    }
  }
}

__global__ void __launch_bounds__(kTripThreads) triplet_batch_all_kernel(const float* __restrict__ S, int64_t lds, int B,
                                                                         const int32_t* __restrict__ seg_lo,
                                                                         const int32_t* __restrict__ seg_hi, float* __restrict__ G,
                                                                         int64_t ldg, double* __restrict__ stats, int Pj_max, int Pk_max,
                                                                         int pos_only, __nv_bfloat16* __restrict__ g_hi,
                                                                         __nv_bfloat16* __restrict__ g_lo, int64_t ld_split,
                                                                         double* __restrict__ loss_slots) {
  extern __shared__ __align__(16) float smem[];
  __shared__ float red_f[32];
  __shared__ double red_d[32];
  const int i = blockIdx.x;
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  const int lo = seg_lo[i], hi = seg_hi[i];
  const int nj = hi - lo;       // segment length (includes the anchor itself, neutralised with u = 0)
  const int nk = B - nj;        // negatives
  const float* srow = S + (int64_t)i * lds;
  float* grow = G + (int64_t)i * ldg;

  if (nj <= 1 || nk == 0) {  // no valid triplet with this anchor
    if (loss_slots && tid == 0) loss_slots[i] = 0.0;   // (deterministic mode: its slot adds 0, as the atomic path does)
    for (int c = tid; c < B; c += kTripThreads) {
      grow[c] = 0.0f;
      if (g_hi) { g_hi[(int64_t)i * ld_split + c] = __float2bfloat16_rn(0.0f); g_lo[(int64_t)i * ld_split + c] = __float2bfloat16_rn(0.0f); }
    }
    return;
  }
  // the row's value range picks the evaluation tier
  float mx = -3.0e38f, mn = 3.0e38f;
  for (int c = tid; c < B; c += kTripThreads) { const float s = srow[c]; mx = fmaxf(mx, s); mn = fminf(mn, s); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); }
  if (tx == 0) { red_f[ty] = mx; red_f[8 + ty] = mn; }
  __syncthreads();
  mx = red_f[0]; mn = red_f[8];
#pragma unroll
  for (int w = 1; w < kTY; ++w) { mx = fmaxf(mx, red_f[w]); mn = fminf(mn, red_f[8 + w]); }
  const float range = mx - mn;
  const int tier = pos_only ? 3 : ((range < 10.0f) ? 0 : ((range < 80.0f) ? 1 : 2));
  const float mid = 0.5f * (mx + mn);

  const int Pj = (nj + kJTile - 1) / kJTile * kJTile;
  const int Pk = (nk + kKTile - 1) / kKTile * kKTile;
  float* sj = smem;
  float* uj = sj + Pj_max;
  float* gj = uj + Pj_max;
  float* sk = gj + Pj_max;
  float* vk = sk + Pk_max;
  float* gk = vk + Pk_max;  // [kTY][Pk_max]

  for (int p = tid; p < Pj; p += kTripThreads) {
    const int c = lo + p;
    const bool ok = (p < nj) && (c != i);
    const float s = ok ? srow[c] : 3.0e38f;               // +huge: never "positive", contributes 0
    sj[p] = ok ? pos_threshold(s) : s;   // fp32(S_ik - S_ij) > 1e-16 becomes one compare per triplet
    uj[p] = ok ? fast_ex2((mid - s) * kLog2e) : 0.0f;
    gj[p] = 0.0f;
  }
  for (int q = tid; q < Pk; q += kTripThreads) {
    const int c = (q < lo) ? q : q + nj;
    const bool ok = q < nk;
    const float s = ok ? srow[c] : -3.0e38f;
    sk[q] = s;
    vk[q] = ok ? fast_ex2((s - mid) * kLog2e) : 0.0f;
  }
  for (int e = tid; e < kTY * Pk; e += kTripThreads) gk[(e / Pk) * Pk_max + (e % Pk)] = 0.0f;
  __syncthreads();

  float lacc = 0.0f;   // sum of log2(1 + e^x)
  int npos = 0;
  if (tier == 0) triplet_sweep<0>(sj, uj, gj, sk, vk, gk, Pj, Pk, Pk_max, tx, ty, lacc, npos);
  else if (tier == 1) triplet_sweep<1>(sj, uj, gj, sk, vk, gk, Pj, Pk, Pk_max, tx, ty, lacc, npos);
  else if (tier == 2) triplet_sweep<2>(sj, uj, gj, sk, vk, gk, Pj, Pk, Pk_max, tx, ty, lacc, npos);
  else triplet_sweep<3>(sj, uj, gj, sk, vk, gk, Pj, Pk, Pk_max, tx, ty, lacc, npos);
  __syncthreads();
  const float inv = pos_only ? 1.0f : (float)(1.0 / (stats[DAE_STAT_N_VALID] + 1e-16));  // pos_only: G holds raw counts
  for (int c = tid; c < B; c += kTripThreads) {
    float g;
    if (c >= lo && c < hi) {
      g = -gj[c - lo] * inv;      // -sum_k sigma(S_ik - S_ij); the anchor's own slot has u = 0 -> 0
    } else {
      const int q = (c < lo) ? c : c - nj;
      float t = 0.0f;
#pragma unroll
      for (int w = 0; w < kTY; ++w) t += gk[w * Pk_max + q];
      g = t * inv;                // +sum_j sigma(S_ik - S_ij)
    }
    grow[c] = g;
    if (g_hi) {   // the bf16 hi / lo operand copy the (G + G^T).E GEMM reads (no separate split pass)
      const __nv_bfloat16 h = __float2bfloat16_rn(g);
      g_hi[(int64_t)i * ld_split + c] = h;
      g_lo[(int64_t)i * ld_split + c] = __float2bfloat16_rn(g - __bfloat162float(h));
    }
  }
  const double lsum = block_sum((double)lacc * (double)kLn2, red_d);
  const double psum = block_sum((double)npos, red_d);
  if (tid == 0) {   // loss_slots (deterministic mode): the anchor's loss goes to its own slot, summed in anchor order later
    if (loss_slots) loss_slots[blockIdx.x] = lsum; else atomicAdd(stats + DAE_STAT_TRIPLET_SUM, lsum);
    atomicAdd(stats + DAE_STAT_NUM, psum);   // an integer count: exact in any order
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// batch_all above 4096 rows: the same per-anchor sweep with shared memory that does not grow with B.  The anchor's negatives stream
// through chunks of kChunkK (s, v and the per-warp column-sum slabs), its positives through chunks of kChunkJ (s, u, row sums).  For
// each negative chunk every positive chunk is swept; the chunk's column sums are then complete and leave as their G entries.  The
// positives' row sums carry across negative chunks in the CTA's own row of G (one thread per entry, chunks in order: deterministic).
// The chunk sizes are multiples of the register tiles, so the column sums are accumulated in the same order as in
// triplet_batch_all_kernel (bit-identical negative entries of G); row sums and the loss differ by fp32 rounding of the chunk partials.
// The per-thread log accumulator is flushed into fp64 after every (positive, negative) chunk pair.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kChunkJ = 512;    // positives per chunk (16 j-tiles)
constexpr int kChunkK = 1024;   // negatives per chunk (8 k-tiles)
static_assert(kChunkJ % kJTile == 0 && kChunkK % kKTile == 0, "chunks must hold whole register tiles");

// Anchor i = row0 + blockIdx.x lives in row blockIdx.x of S / G / g_hi / g_lo (row0 = 0: the whole B x B matrices; row0 > 0: an
// anchor-row block of them, see dae_triplet_batch_all_rows); segments are indexed by the anchor.
__global__ void __launch_bounds__(kTripThreads) triplet_batch_all_tiled_kernel(const float* __restrict__ S, int64_t lds, int row0, int B,
                                                                               const int32_t* __restrict__ seg_lo,
                                                                               const int32_t* __restrict__ seg_hi, float* G, int64_t ldg,
                                                                               double* __restrict__ stats, int pos_only,
                                                                               __nv_bfloat16* __restrict__ g_hi,
                                                                               __nv_bfloat16* __restrict__ g_lo, int64_t ld_split,
                                                                               double* __restrict__ loss_slots) {
  __shared__ __align__(16) float sj[kChunkJ];
  __shared__ __align__(16) float uj[kChunkJ];
  __shared__ __align__(16) float gj[kChunkJ];
  __shared__ __align__(16) float sk[kChunkK];
  __shared__ __align__(16) float vk[kChunkK];
  __shared__ __align__(16) float gk[kTY * kChunkK];
  __shared__ float red_f[32];
  __shared__ double red_d[32];
  const int r = blockIdx.x, i = row0 + r;
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  const int lo = seg_lo[i], hi = seg_hi[i];
  const int nj = hi - lo;
  const int nk = B - nj;
  const float* srow = S + (int64_t)r * lds;
  float* grow = G + (int64_t)r * ldg;

  if (nj <= 1 || nk == 0) {
    if (loss_slots && tid == 0) loss_slots[i] = 0.0;   // (deterministic mode: its slot adds 0, as the atomic path does)
    for (int c = tid; c < B; c += kTripThreads) {
      grow[c] = 0.0f;
      if (g_hi) { g_hi[(int64_t)r * ld_split + c] = __float2bfloat16_rn(0.0f); g_lo[(int64_t)r * ld_split + c] = __float2bfloat16_rn(0.0f); }
    }
    return;
  }
  // the tier is chosen from the whole row's range
  float mx = -3.0e38f, mn = 3.0e38f;
  for (int c = tid; c < B; c += kTripThreads) { const float s = srow[c]; mx = fmaxf(mx, s); mn = fminf(mn, s); }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); }
  if (tx == 0) { red_f[ty] = mx; red_f[8 + ty] = mn; }
  __syncthreads();
  mx = red_f[0]; mn = red_f[8];
#pragma unroll
  for (int w = 1; w < kTY; ++w) { mx = fmaxf(mx, red_f[w]); mn = fminf(mn, red_f[8 + w]); }
  const float range = mx - mn;
  const int tier = pos_only ? 3 : ((range < 10.0f) ? 0 : ((range < 80.0f) ? 1 : 2));
  const float mid = 0.5f * (mx + mn);
  const float inv = pos_only ? 1.0f : (float)(1.0 / (stats[DAE_STAT_N_VALID] + 1e-16));

  double lsum = 0.0;   // sum of log2(1 + e^x), fp64 across chunks
  int npos = 0;
  for (int k0 = 0; k0 < nk; k0 += kChunkK) {
    const int ck = min(kChunkK, nk - k0);
    const int Pk = (ck + kKTile - 1) / kKTile * kKTile;
    __syncthreads();   // the previous chunk's readers of sk / vk / gk are done
    for (int q = tid; q < Pk; q += kTripThreads) {
      const int qq = k0 + q;
      const int c = (qq < lo) ? qq : qq + nj;
      const bool ok = q < ck;
      const float s = ok ? srow[c] : -3.0e38f;
      sk[q] = s;
      vk[q] = ok ? fast_ex2((s - mid) * kLog2e) : 0.0f;
    }
    for (int e = tid; e < kTY * Pk; e += kTripThreads) gk[(e / Pk) * kChunkK + (e % Pk)] = 0.0f;
    for (int j0 = 0; j0 < nj; j0 += kChunkJ) {
      const int cj = min(kChunkJ, nj - j0);
      const int Pj = (cj + kJTile - 1) / kJTile * kJTile;
      __syncthreads();   // sj / uj / gj of the previous positive chunk are consumed
      for (int p = tid; p < Pj; p += kTripThreads) {
        const int c = lo + j0 + p;
        const bool ok = (p < cj) && (c != i);
        const float s = ok ? srow[c] : 3.0e38f;
        sj[p] = ok ? pos_threshold(s) : s;
        uj[p] = ok ? fast_ex2((mid - s) * kLog2e) : 0.0f;
        gj[p] = 0.0f;
      }
      __syncthreads();
      float lacc = 0.0f;
      if (tier == 0) triplet_sweep<0>(sj, uj, gj, sk, vk, gk, Pj, Pk, kChunkK, tx, ty, lacc, npos);
      else if (tier == 1) triplet_sweep<1>(sj, uj, gj, sk, vk, gk, Pj, Pk, kChunkK, tx, ty, lacc, npos);
      else if (tier == 2) triplet_sweep<2>(sj, uj, gj, sk, vk, gk, Pj, Pk, kChunkK, tx, ty, lacc, npos);
      else triplet_sweep<3>(sj, uj, gj, sk, vk, gk, Pj, Pk, kChunkK, tx, ty, lacc, npos);
      lsum += (double)lacc;
      __syncthreads();
      // raw row sums of this chunk pair, carried in G; entry lo + j0 + p is always owned by thread p % kTripThreads
      for (int p = tid; p < cj; p += kTripThreads) {
        float* g = grow + lo + j0 + p;
        *g = (k0 == 0 ? 0.0f : *g) + gj[p];
      }
    }
    __syncthreads();   // the column-sum slabs of this negative chunk are complete
    for (int q = tid; q < ck; q += kTripThreads) {
      const int qq = k0 + q;
      const int c = (qq < lo) ? qq : qq + nj;
      float t = 0.0f;
#pragma unroll
      for (int w = 0; w < kTY; ++w) t += gk[w * kChunkK + q];
      const float g = t * inv;    // +sum_j sigma(S_ik - S_ij)
      grow[c] = g;
      if (g_hi) {
        const __nv_bfloat16 h = __float2bfloat16_rn(g);
        g_hi[(int64_t)r * ld_split + c] = h;
        g_lo[(int64_t)r * ld_split + c] = __float2bfloat16_rn(g - __bfloat162float(h));
      }
    }
  }
  for (int p = tid; p < nj; p += kTripThreads) {   // same owner thread as the carries above
    const int c = lo + p;
    const float g = -grow[c] * inv;    // -sum_k sigma(S_ik - S_ij); the anchor's own slot has u = 0 -> 0
    grow[c] = g;
    if (g_hi) {
      const __nv_bfloat16 h = __float2bfloat16_rn(g);
      g_hi[(int64_t)r * ld_split + c] = h;
      g_lo[(int64_t)r * ld_split + c] = __float2bfloat16_rn(g - __bfloat162float(h));
    }
  }
  const double ls = block_sum(lsum * (double)kLn2, red_d);
  const double ps = block_sum((double)npos, red_d);
  if (tid == 0) {   // loss_slots (deterministic mode): the anchor's loss goes to its own slot, summed in anchor order later
    if (loss_slots) loss_slots[row0 + (int64_t)blockIdx.x] = ls; else atomicAdd(stats + DAE_STAT_TRIPLET_SUM, ls);
    atomicAdd(stats + DAE_STAT_NUM, ps);     // an integer count: exact in any order
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// batch_hard: one CTA per anchor row.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kHardThreads = 256;

__device__ __forceinline__ float block_max(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) r = fmaxf(r, red[w]);
  __syncthreads();
  return r;
}

// Anchor a = row0 + blockIdx.x lives in row blockIdx.x of S / G (row0 = 0: the whole matrices; see dae_triplet_batch_hard_rows).
__global__ void __launch_bounds__(kHardThreads) triplet_batch_hard_kernel(const float* __restrict__ S, int64_t lds, int row0, int B,
                                                                          const float* __restrict__ labels, float* __restrict__ G,
                                                                          int64_t ldg, float* __restrict__ weight,
                                                                          double* __restrict__ stats, double* __restrict__ loss_slots) {
  __shared__ float red[32];
  __shared__ float redi[32];
  const int a = row0 + (int)blockIdx.x, tid = threadIdx.x;
  const float* srow = S + (int64_t)blockIdx.x * lds;
  float* grow = G + (int64_t)blockIdx.x * ldg;
  const float la = labels[a];
  // m = row max (triplet_loss_utils.py:227); hn = max(an * S) (:240-243)
  float m = -3.0e38f, hn = -3.0e38f;
  for (int c = tid; c < B; c += kHardThreads) {
    const float s = srow[c];
    m = fmaxf(m, s);
    const float an = (labels[c] != la) ? 1.0f : 0.0f;
    hn = fmaxf(hn, an * s);
  }
  m = block_max(m, red);
  hn = block_max(hn, red);
  // hp = min(S + m * (1 - ap)) (:228-231)
  float hpn = -3.0e38f;  // max of the negated values
  for (int c = tid; c < B; c += kHardThreads) {
    const float ap = (c != a && labels[c] == la) ? 1.0f : 0.0f;
    hpn = fmaxf(hpn, -(srow[c] + m * (1.0f - ap)));
  }
  const float hp = -block_max(hpn, red);
  const float td = fmaxf(hn - hp, 0.0f);   // :247
  const bool active = td > 0.0f;           // :249
  // tie counts for the reduce_min / reduce_max gradients (TF splits the gradient equally among ties)
  float tp = 0.0f, tn = 0.0f, tm = 0.0f, tp_masked = 0.0f;
  for (int c = tid; c < B; c += kHardThreads) {
    const float s = srow[c];
    const float ap = (c != a && labels[c] == la) ? 1.0f : 0.0f;
    const float an = (labels[c] != la) ? 1.0f : 0.0f;
    if (s + m * (1.0f - ap) == hp) { tp += 1.0f; if (ap == 0.0f) tp_masked += 1.0f; }
    if (an * s == hn) tn += 1.0f;
    if (s == m) tm += 1.0f;
  }
  tp = block_sum(tp, red);
  tn = block_sum(tn, redi);
  tm = block_sum(tm, red);
  tp_masked = block_sum(tp_masked, redi);
  // dL/dtd_a (unnormalised by 1/(sum c + eps): applied by triplet_hard_scale_kernel)
  const float q = active ? 1.0f / (1.0f + expf(-td)) : 0.0f;
  const float dm = -q * tp_masked / tp;  // gradient reaching the row max through masked argmin entries
  for (int c = tid; c < B; c += kHardThreads) {
    const float s = srow[c];
    const float ap = (c != a && labels[c] == la) ? 1.0f : 0.0f;
    const float an = (labels[c] != la) ? 1.0f : 0.0f;
    float g = 0.0f;
    if (active) {
      if (s + m * (1.0f - ap) == hp) g -= q / tp;
      if (an * s == hn) g += an * q / tn;
      if (s == m) g += dm / tm;
      // data weight (:251-253): equality is tested on the raw dot products over the whole row
      float w = 0.0f;
      if (s == hp) w += 1.0f;
      if (s == hn) w += 1.0f;
      if (c == a) w += 1.0f;
      if (w != 0.0f) atomicAdd(weight + c, w);
    }
    grow[c] = g;
  }
  if (tid == 0 && loss_slots) loss_slots[a] = active ? (double)(fmaxf(td, 0.0f) + log1pf(expf(-td))) : 0.0;
  if (tid == 0 && active) {
    if (!loss_slots) atomicAdd(stats + DAE_STAT_TRIPLET_SUM, (double)(fmaxf(td, 0.0f) + log1pf(expf(-td))));  // softplus(td), td > 0
    atomicAdd(stats + DAE_STAT_N_ACTIVE, 1.0);
  }
}

// after all rows: sum_w, and G *= 1/(sum c + eps)
__global__ void triplet_hard_scale_kernel(float* __restrict__ G, int64_t ldg, int B, const float* __restrict__ weight,
                                          double* __restrict__ stats) {
  const float inv = (float)(1.0 / (stats[DAE_STAT_N_ACTIVE] + 1e-16));
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = blockIdx.y;
  if (c < B) G[(int64_t)r * ldg + c] *= inv;
  if (r == 0 && blockIdx.x == 0) {
    __shared__ double red[32];
    double s = 0.0;
    for (int i = threadIdx.x; i < B; i += blockDim.x) s += (double)weight[i];
    s = block_sum(s, red);
    if (threadIdx.x == 0) stats[DAE_STAT_SUM_W] = s;
  }
}

// block-mined batch_hard, after the last anchor block: sum_w (block 0, the summation order of triplet_hard_scale_kernel) and
// dE2 *= 1/(sum c + eps) -- the blocks' dE2 GEMMs ran on the unscaled G.
__global__ void triplet_hard_finish_kernel(const float* __restrict__ weight, int B, double* __restrict__ stats, float* __restrict__ dE2,
                                           int H, int64_t ld) {
  if (blockIdx.x == 0) {
    __shared__ double red[32];
    double s = 0.0;
    for (int i = threadIdx.x; i < B; i += blockDim.x) s += (double)weight[i];
    s = block_sum(s, red);
    if (threadIdx.x == 0) stats[DAE_STAT_SUM_W] = s;
  }
  if (!dE2) return;
  const float inv = (float)(1.0 / (stats[DAE_STAT_N_ACTIVE] + 1e-16));
  const int64_t total = (int64_t)B * H;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / H;
    dE2[r * ld + (e - r * H)] *= inv;
  }
}

// explicit triplets: one warp per row
__global__ void triplet_explicit_kernel(const float* __restrict__ E, const float* __restrict__ Ep, const float* __restrict__ En,
                                        int B, int H, int64_t ld, float alpha, float* __restrict__ dE, float* __restrict__ dEp,
                                        float* __restrict__ dEn, double* __restrict__ stats, double* __restrict__ loss_slots) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= B) return;
  const float* e = E + (int64_t)r * ld;
  const float* ep = Ep + (int64_t)r * ld;
  const float* en = En + (int64_t)r * ld;
  float dp = 0.0f;
  for (int h = lane; h < H; h += 32) dp += e[h] * ep[h] - e[h] * en[h];  // autoencoder_triplet.py:308-311
  dp = warp_sum(dp);
  const float x = -dp;                       // loss = softplus(x) = -log_sigmoid(dp)
  const float sp = fmaxf(x, 0.0f) + log1pf(expf(-fabsf(x)));
  const float sg = 1.0f / (1.0f + expf(-x)); // d softplus / dx
  const float c = alpha * sg / (float)B;     // d(alpha * mean)/dx
  for (int h = lane; h < H; h += 32) {
    const float ev = e[h];
    dE[(int64_t)r * ld + h] += c * (en[h] - ep[h]);   // accumulated on top of the reconstruction gradient
    dEp[(int64_t)r * ld + h] += -c * ev;
    dEn[(int64_t)r * ld + h] += c * ev;
  }
  if (lane == 0) { if (loss_slots) loss_slots[r] = (double)sp; else atomicAdd(stats + DAE_STAT_TRIPLET_SUM, (double)sp); }
  if (r == 0 && lane == 0) stats[DAE_STAT_N_ACTIVE] = (double)B;
}

constexpr int kSmemSweepMaxB = 4096;   // triplet_batch_all_kernel serves B up to here, triplet_batch_all_tiled_kernel above
static int g_force_tiled = 0;           // test hook (dae_triplet_config): the tiled sweep at every B

}  // namespace dae

extern "C" int dae_triplet_config(int32_t force_tiled) {
  dae::g_force_tiled = force_tiled ? 1 : 0;
  return DAE_OK;
}

static int dae_triplet_batch_all_impl(const float* S, int64_t lds, int32_t B, const int32_t* seg_lo, const int32_t* seg_hi, float* G,
                                     int64_t ldg, double* stats, int32_t pos_only, void* g_hi, void* g_lo, int64_t ld_split, void* stream, double* loss_slots) {
  using namespace dae;
  DAE_REQUIRE(S && seg_lo && seg_hi && G && stats && B >= 1 && lds >= B && ldg >= B, "dae_triplet_batch_all: bad arguments");
  DAE_REQUIRE(B <= DAE_MAX_TRIPLET_BATCH, "dae_triplet_batch_all: B <= %d rows, the cap of the B x B mining buffers (got %d)",
              DAE_MAX_TRIPLET_BATCH, B);
  DAE_REQUIRE(!g_hi || (g_lo && ld_split >= B), "dae_triplet_batch_all: bad split outputs");
  cudaStream_t st = (cudaStream_t)stream;
  if (B > kSmemSweepMaxB || g_force_tiled) {
    triplet_batch_all_tiled_kernel<<<B, kTripThreads, 0, st>>>(S, lds, 0, B, seg_lo, seg_hi, G, ldg, stats, pos_only, (__nv_bfloat16*)g_hi,
                                                               (__nv_bfloat16*)g_lo, ld_split, loss_slots);
    DAE_CHECK_LAUNCH("dae_triplet_batch_all(tiled)");
    return DAE_OK;
  }
  const int Pj = (B + kJTile - 1) / kJTile * kJTile;
  const int Pk = (B + kKTile - 1) / kKTile * kKTile;
  const size_t smem = sizeof(float) * ((size_t)3 * Pj + (size_t)2 * Pk + (size_t)kTY * Pk);
  DAE_REQUIRE(smem + 1024 <= 227 * 1024, "dae_triplet_batch_all: B=%d needs %zu B of shared memory", B, smem);
  {   // opt in to > 48 KB of dynamic shared memory: a per-DEVICE function attribute, remembered per device (grown monotonically)
    static size_t attr_smem[64] = {0};
    int dev = 0;
    DAE_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || smem > attr_smem[dev]) {
      DAE_CUDA(cudaFuncSetAttribute(triplet_batch_all_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      if (dev >= 0 && dev < 64) attr_smem[dev] = smem;
    }
  }
  triplet_batch_all_kernel<<<B, kTripThreads, smem, st>>>(S, lds, B, seg_lo, seg_hi, G, ldg, stats, Pj, Pk, pos_only, (__nv_bfloat16*)g_hi,
                                                          (__nv_bfloat16*)g_lo, ld_split, loss_slots);
  DAE_CHECK_LAUNCH("dae_triplet_batch_all");
  return DAE_OK;
}

static int dae_triplet_batch_hard_impl(const float* S, int64_t lds, int32_t B, const float* labels, float* G, int64_t ldg,
                                      float* weight, double* stats, void* stream, double* loss_slots) {
  using namespace dae;
  DAE_REQUIRE(S && labels && G && weight && stats && B >= 1 && lds >= B && ldg >= B, "dae_triplet_batch_hard: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  DAE_CUDA(cudaMemsetAsync(weight, 0, sizeof(float) * B, st));
  triplet_batch_hard_kernel<<<B, kHardThreads, 0, st>>>(S, lds, 0, B, labels, G, ldg, weight, stats, loss_slots);
  dim3 grid((B + 255) / 256, B);
  triplet_hard_scale_kernel<<<grid, 256, 0, st>>>(G, ldg, B, weight, stats);
  DAE_CHECK_LAUNCH("dae_triplet_batch_hard");
  return DAE_OK;
}

static int dae_triplet_batch_all_rows_impl(const float* S_blk, int64_t lds, int32_t row0, int32_t n_rows, int32_t B, const int32_t* seg_lo,
                                          const int32_t* seg_hi, float* G_blk, int64_t ldg, double* stats, int32_t pos_only, void* g_hi,
                                          void* g_lo, int64_t ld_split, void* stream, double* loss_slots) {
  using namespace dae;
  DAE_REQUIRE(S_blk && seg_lo && seg_hi && G_blk && stats && B >= 1 && lds >= B && ldg >= B,
              "dae_triplet_batch_all_rows: bad arguments");
  DAE_REQUIRE(B <= DAE_MAX_BLOCKED_BATCH, "dae_triplet_batch_all_rows: B <= %d rows (got %d)", DAE_MAX_BLOCKED_BATCH, B);
  DAE_REQUIRE(row0 >= 0 && n_rows >= 1 && (int64_t)row0 + n_rows <= B,
              "dae_triplet_batch_all_rows: anchor rows [%d, %lld) outside the batch of %d", row0, (long long)row0 + n_rows, B);
  DAE_REQUIRE(!g_hi || (g_lo && ld_split >= B), "dae_triplet_batch_all_rows: bad split outputs");
  triplet_batch_all_tiled_kernel<<<n_rows, kTripThreads, 0, (cudaStream_t)stream>>>(S_blk, lds, row0, B, seg_lo, seg_hi, G_blk, ldg, stats,
                                                                                    pos_only, (__nv_bfloat16*)g_hi, (__nv_bfloat16*)g_lo,
                                                                                    ld_split, loss_slots);
  DAE_CHECK_LAUNCH("dae_triplet_batch_all_rows");
  return DAE_OK;
}

static int dae_triplet_batch_hard_rows_impl(const float* S_blk, int64_t lds, int32_t row0, int32_t n_rows, int32_t B, const float* labels,
                                           float* G_blk, int64_t ldg, float* weight, double* stats, void* stream, double* loss_slots) {
  using namespace dae;
  DAE_REQUIRE(S_blk && labels && G_blk && weight && stats && B >= 1 && lds >= B && ldg >= B, "dae_triplet_batch_hard_rows: bad arguments");
  DAE_REQUIRE(B <= DAE_MAX_BLOCKED_BATCH, "dae_triplet_batch_hard_rows: B <= %d rows (got %d)", DAE_MAX_BLOCKED_BATCH, B);
  DAE_REQUIRE(row0 >= 0 && n_rows >= 1 && (int64_t)row0 + n_rows <= B,
              "dae_triplet_batch_hard_rows: anchor rows [%d, %lld) outside the batch of %d", row0, (long long)row0 + n_rows, B);
  triplet_batch_hard_kernel<<<n_rows, kHardThreads, 0, (cudaStream_t)stream>>>(S_blk, lds, row0, B, labels, G_blk, ldg, weight, stats, loss_slots);
  DAE_CHECK_LAUNCH("dae_triplet_batch_hard_rows");
  return DAE_OK;
}

extern "C" int dae_triplet_batch_hard_finish(const float* weight, int32_t B, double* stats, float* dE2, int32_t H, int64_t ld, void* stream) {
  using namespace dae;
  DAE_REQUIRE(weight && stats && B >= 1 && B <= DAE_MAX_BLOCKED_BATCH, "dae_triplet_batch_hard_finish: bad arguments");
  DAE_REQUIRE(!dE2 || (H >= 1 && ld >= H), "dae_triplet_batch_hard_finish: bad dE2 shape");
  int blocks = 1;
  if (dE2) {
    const int64_t want = ((int64_t)B * H + 255) / 256;
    blocks = (int)(want < 4096 ? want : 4096);
  }
  triplet_hard_finish_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(weight, B, stats, dE2, H, ld);
  DAE_CHECK_LAUNCH("dae_triplet_batch_hard_finish");
  return DAE_OK;
}

static int dae_triplet_explicit_impl(const float* E, const float* Ep, const float* En, int32_t B, int32_t H, int64_t ld, float alpha,
                                    float* dE, float* dEp, float* dEn, double* stats, void* stream, double* loss_slots) {
  using namespace dae;
  DAE_REQUIRE(E && Ep && En && dE && dEp && dEn && stats && B >= 1 && H >= 1 && ld >= H, "dae_triplet_explicit: bad arguments");
  triplet_explicit_kernel<<<(B + 7) / 8, 256, 0, (cudaStream_t)stream>>>(E, Ep, En, B, H, ld, alpha, dE, dEp, dEn, stats, loss_slots);
  DAE_CHECK_LAUNCH("dae_triplet_explicit");
  return DAE_OK;
}

extern "C" int dae_triplet_batch_all(const float* S, int64_t lds, int32_t B, const int32_t* seg_lo, const int32_t* seg_hi, float* G,
                                     int64_t ldg, double* stats, int32_t pos_only, void* g_hi, void* g_lo, int64_t ld_split, void* stream) {
  return dae_triplet_batch_all_impl(S, lds, B, seg_lo, seg_hi, G, ldg, stats, pos_only, g_hi, g_lo, ld_split, stream, nullptr);
}
extern "C" int dae_triplet_batch_all_det(const float* S, int64_t lds, int32_t B, const int32_t* seg_lo, const int32_t* seg_hi, float* G,
                                     int64_t ldg, double* stats, int32_t pos_only, void* g_hi, void* g_lo, int64_t ld_split, double* loss_slots, void* stream) {
  DAE_REQUIRE(loss_slots, "dae_triplet_batch_all_det: null loss_slots");
  return dae_triplet_batch_all_impl(S, lds, B, seg_lo, seg_hi, G, ldg, stats, pos_only, g_hi, g_lo, ld_split, stream, loss_slots);
}

extern "C" int dae_triplet_batch_hard(const float* S, int64_t lds, int32_t B, const float* labels, float* G, int64_t ldg,
                                      float* weight, double* stats, void* stream) {
  return dae_triplet_batch_hard_impl(S, lds, B, labels, G, ldg, weight, stats, stream, nullptr);
}
extern "C" int dae_triplet_batch_hard_det(const float* S, int64_t lds, int32_t B, const float* labels, float* G, int64_t ldg,
                                      float* weight, double* stats, double* loss_slots, void* stream) {
  DAE_REQUIRE(loss_slots, "dae_triplet_batch_hard_det: null loss_slots");
  return dae_triplet_batch_hard_impl(S, lds, B, labels, G, ldg, weight, stats, stream, loss_slots);
}

extern "C" int dae_triplet_batch_all_rows(const float* S_blk, int64_t lds, int32_t row0, int32_t n_rows, int32_t B, const int32_t* seg_lo,
                                          const int32_t* seg_hi, float* G_blk, int64_t ldg, double* stats, int32_t pos_only, void* g_hi,
                                          void* g_lo, int64_t ld_split, void* stream) {
  return dae_triplet_batch_all_rows_impl(S_blk, lds, row0, n_rows, B, seg_lo, seg_hi, G_blk, ldg, stats, pos_only, g_hi, g_lo, ld_split, stream, nullptr);
}
extern "C" int dae_triplet_batch_all_rows_det(const float* S_blk, int64_t lds, int32_t row0, int32_t n_rows, int32_t B, const int32_t* seg_lo,
                                          const int32_t* seg_hi, float* G_blk, int64_t ldg, double* stats, int32_t pos_only, void* g_hi,
                                          void* g_lo, int64_t ld_split, double* loss_slots, void* stream) {
  DAE_REQUIRE(loss_slots, "dae_triplet_batch_all_rows_det: null loss_slots");
  return dae_triplet_batch_all_rows_impl(S_blk, lds, row0, n_rows, B, seg_lo, seg_hi, G_blk, ldg, stats, pos_only, g_hi, g_lo, ld_split, stream, loss_slots);
}

extern "C" int dae_triplet_batch_hard_rows(const float* S_blk, int64_t lds, int32_t row0, int32_t n_rows, int32_t B, const float* labels,
                                           float* G_blk, int64_t ldg, float* weight, double* stats, void* stream) {
  return dae_triplet_batch_hard_rows_impl(S_blk, lds, row0, n_rows, B, labels, G_blk, ldg, weight, stats, stream, nullptr);
}
extern "C" int dae_triplet_batch_hard_rows_det(const float* S_blk, int64_t lds, int32_t row0, int32_t n_rows, int32_t B, const float* labels,
                                           float* G_blk, int64_t ldg, float* weight, double* stats, double* loss_slots, void* stream) {
  DAE_REQUIRE(loss_slots, "dae_triplet_batch_hard_rows_det: null loss_slots");
  return dae_triplet_batch_hard_rows_impl(S_blk, lds, row0, n_rows, B, labels, G_blk, ldg, weight, stats, stream, loss_slots);
}

extern "C" int dae_triplet_explicit(const float* E, const float* Ep, const float* En, int32_t B, int32_t H, int64_t ld, float alpha,
                                    float* dE, float* dEp, float* dEn, double* stats, void* stream) {
  return dae_triplet_explicit_impl(E, Ep, En, B, H, ld, alpha, dE, dEp, dEn, stats, stream, nullptr);
}
extern "C" int dae_triplet_explicit_det(const float* E, const float* Ep, const float* En, int32_t B, int32_t H, int64_t ld, float alpha,
                                    float* dE, float* dEp, float* dEn, double* stats, double* loss_slots, void* stream) {
  DAE_REQUIRE(loss_slots, "dae_triplet_explicit_det: null loss_slots");
  return dae_triplet_explicit_impl(E, Ep, En, B, H, ld, alpha, dE, dEp, dEn, stats, stream, loss_slots);
}

namespace dae {
// deterministic mode: stats[TRIPLET_SUM] += the per-anchor (per-row) losses in a fixed order -- each thread its strided slots in index
// order, then block_sum's fixed tree
__global__ void __launch_bounds__(1024) triplet_loss_sum_kernel(const double* __restrict__ slots, int n, double* __restrict__ stats) {
  __shared__ double red[32];
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += slots[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) stats[DAE_STAT_TRIPLET_SUM] += s;
}
}  // namespace dae

extern "C" int dae_triplet_loss_sum(const double* loss_slots, int32_t n, double* stats, void* stream) {
  using namespace dae;
  DAE_REQUIRE(loss_slots && stats && n >= 1, "dae_triplet_loss_sum: bad arguments");
  triplet_loss_sum_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(loss_slots, n, stats);
  DAE_CHECK_LAUNCH("dae_triplet_loss_sum");
  return DAE_OK;
}
