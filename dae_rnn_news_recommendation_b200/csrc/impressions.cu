// Impression logs (DESIGN 4.13, 4.16): the pairwise and the sampled-softmax impression losses of the user encoders and the
// per-impression ranking metrics.
//
// An impression is a list of shown articles items[indptr[i] .. indptr[i + 1]) with a click flag per article.  Both kernels give
// one warp to one row of work and score the candidates with warp dot products (lane j takes the columns j, j + 32, ...), so a
// candidate list of any length is walked in chunks of kImpChunk scores held in shared memory per warp.
#include "common.cuh"
#include "impression_rank.cuh"

namespace dae {

constexpr int kImpWarps = 4;

// sigma(x) with the approximate divide (2 ulp, no slow-path subroutine: the pair loop keeps its state in registers)
__device__ __forceinline__ float imp_sigmoid(float x) { return __fdividef(1.0f, 1.0f + expf(-x)); }

// 1 / x for an integer-valued x in [1, 2^62]: the fp32 approximation refined by two Newton steps to fp64 accuracy, inline
__device__ __forceinline__ double imp_recip(double x) {
  double r = (double)__fdividef(1.0f, (float)x);
  r = r * (2.0 - x * r);
  return r * (2.0 - x * r);
}

__device__ __forceinline__ float warp_dot(const float* __restrict__ a, const float* __restrict__ b, int H, int lane) {
  float s = 0.0f;
#pragma unroll 1   // unrolled, the loss kernel's nested loops spill to local memory
  for (int j = lane; j < H; j += 32) s = fmaf(a[j], b[j], s);
  return warp_sum(s);
}

// Scores h . e(items[k]) of candidates [k0, k0 + n) into s[0, n) and their click flags into f[0, n) (shared, one warp).
__device__ __forceinline__ void score_chunk(const float* __restrict__ h, const float* __restrict__ emb, int64_t ld_emb, int H,
                                            const int32_t* __restrict__ items, const uint8_t* __restrict__ clicked, int64_t k0, int n,
                                            float* s, uint8_t* f, int lane) {
  for (int t = 0; t < n; ++t) {
    const float v = warp_dot(h, emb + (int64_t)items[k0 + t] * ld_emb, H, lane);
    if (lane == 0) s[t] = v;
  }
  for (int t = lane; t < n; t += 32) f[t] = clicked[k0 + t] != 0;
  __syncwarp();
}

// One warp per packed position p: dh_p = sum over the impressions q in [pos_indptr[p], pos_indptr[p + 1]) (in that order) of
// scale / (|C_q| |N_q|) sum_j w_j e_j with w_n = sum_c s(s_n - s_c), w_c = -sum_n s(s_n - s_c); *loss_sum += the impressions'
// 1 / (|C| |N|) sum_{c, n} softplus(s_n - s_c).  Impressions without a click or without a non-click add nothing; a position
// without impressions gets dh_p = 0.  The warp owns row p of dh: no atomics, the result does not depend on the schedule.
// Candidates are taken kImpChunk at a time (chunk A, whose weights are summed in shared memory) against every chunk B of the
// same impression, whose scores are recomputed when the impression has more than one chunk.
// DEMB (dae_impression_rank_loss_grad, DESIGN 4.19): each candidate's coefficient g also adds g h_p into demb[items[j]] by fp32
// atomics; the DEMB = false instance is dae_impression_rank_loss's kernel, its code unchanged by the flag.
// DET (the *_det exports, DESIGN 4.21): position p's loss (the warp sum of its lanes' terms) is stored to loss_slots[p] instead of
// added, and with DEMB candidate k of the packed items gets the triple (items[k], p, g) at index k (slot -1 in an impression without
// a click or without a non-click) for dae_ordered_rows.  dh's arithmetic is the same in every instance.
// The DET instances hold the loss-slot and triple pointers too: 8 CTAs per SM give them 64 registers and no spill (0: no minimum,
// the default instances' bounds).
template <bool DEMB, bool DET = false>
__global__ void __launch_bounds__(kImpWarps * 32, DET ? 8 : 0) impression_rank_loss_kernel(
    const float* __restrict__ h, int64_t ld_h, const float* __restrict__ emb, int64_t ld_emb, int H, const int64_t* __restrict__ pos_indptr,
    int64_t n_pos, const int64_t* __restrict__ imp_indptr, const int32_t* __restrict__ items, const uint8_t* __restrict__ clicked,
    float scale, float* __restrict__ dh, int64_t ld_dh, double* __restrict__ loss_sum, float* __restrict__ demb, int64_t ld_demb,
    double* __restrict__ loss_slots, int32_t* __restrict__ t_slot, int32_t* __restrict__ t_row, float* __restrict__ t_coef) {
  __shared__ float s_a[kImpWarps][kImpChunk], s_b[kImpWarps][kImpChunk], s_w[kImpWarps][kImpChunk];
  __shared__ uint8_t f_a[kImpWarps][kImpChunk], f_b[kImpWarps][kImpChunk];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double acc = 0.0;
  for (int64_t p = (int64_t)blockIdx.x * kImpWarps + w; p < n_pos; p += (int64_t)gridDim.x * kImpWarps) {
    float* d = dh + p * ld_dh;
    for (int j = lane; j < H; j += 32) d[j] = 0.0f;
    const float* hp = h + p * ld_h;
    for (int64_t q = pos_indptr[p]; q < pos_indptr[p + 1]; ++q) {
      const int64_t b0 = imp_indptr[q], m = imp_indptr[q + 1] - b0;
      const int nc = count_clicked(clicked + b0, m, lane);
      const int64_t nn = m - nc;
      if (nc == 0 || nn == 0) {
        if constexpr (DEMB && DET) {
          for (int64_t k = lane; k < m; k += 32) t_slot[b0 + k] = -1;
        }
        continue;
      }
      const double inv = imp_recip((double)nc * (double)nn);
      const float coef = (float)((double)scale * inv);
      double l_imp = 0.0;
      for (int64_t a0 = 0; a0 < m; a0 += kImpChunk) {
        const int na = (int)min((int64_t)kImpChunk, m - a0);
        score_chunk(hp, emb, ld_emb, H, items + b0, clicked + b0, a0, na, s_a[w], f_a[w], lane);
        for (int t = lane; t < na; t += 32) s_w[w][t] = 0.0f;
        for (int64_t c0 = 0; c0 < m; c0 += kImpChunk) {
          const int nb = (int)min((int64_t)kImpChunk, m - c0);
          const float* sb = s_a[w];
          const uint8_t* fb = f_a[w];
          if (c0 != a0) {
            score_chunk(hp, emb, ld_emb, H, items + b0, clicked + b0, c0, nb, s_b[w], f_b[w], lane);
            sb = s_b[w];
            fb = f_b[w];
          }
          for (int t = lane; t < na; t += 32) {
            const float sj = s_a[w][t];
            const uint8_t cj = f_a[w][t];
            float wj = s_w[w][t], lj = 0.0f;
            for (int k = 0; k < nb; ++k) {
              if (fb[k] == cj) continue;
              if (cj) {   // j clicked, k not: x = s_k - s_j
                const float x = sb[k] - sj;
                wj -= imp_sigmoid(x);
                lj += fmaxf(x, 0.0f) + log1pf(expf(-fabsf(x)));
              } else {    // j not clicked, k clicked: x = s_j - s_k
                wj += imp_sigmoid(sj - sb[k]);
              }
            }
            s_w[w][t] = wj;
            l_imp += (double)lj;
          }
          __syncwarp();
        }
        for (int t = 0; t < na; ++t) {
          const float g = coef * s_w[w][t];
          const float* e = emb + (int64_t)items[b0 + a0 + t] * ld_emb;
#pragma unroll 1
          for (int j = lane; j < H; j += 32) d[j] = fmaf(g, e[j], d[j]);
          if constexpr (DEMB && DET) {
            if (lane == 0) {
              const int64_t k = b0 + a0 + t;
              t_slot[k] = items[k]; t_row[k] = (int32_t)p; t_coef[k] = g;
            }
          } else if constexpr (DEMB) {
            float* de = demb + (int64_t)items[b0 + a0 + t] * ld_demb;
#pragma unroll 1
            for (int j = lane; j < H; j += 32) atomicAdd(de + j, g * hp[j]);
          }
        }
        __syncwarp();
      }
      acc += l_imp * inv;
    }
    if constexpr (DET) {
      const double l = warp_sum(acc);
      if (lane == 0) loss_slots[p] = l;
      acc = 0.0;
    }
  }
  if constexpr (DET) return;
  acc = warp_sum(acc);
  if (lane == 0 && acc != 0.0) atomicAdd(loss_sum, acc);
}

// One warp per impression i: scores[k] = q_i . e(items[k]) (cosine: divided by |q_i| |e|, 0 when either is zero) for every k in
// [indptr[i], indptr[i + 1]), then metrics[i] = (AUC, MRR, nDCG@5, nDCG@10) from those fp32 scores (impression_rank_metrics).
__global__ void __launch_bounds__(kImpWarps * 32) impression_metrics_kernel(
    const float* __restrict__ qv, int64_t ld_q, const float* __restrict__ emb, int64_t ld_emb, int H, int cosine,
    const int64_t* __restrict__ indptr, const int32_t* __restrict__ items, const uint8_t* __restrict__ clicked, int64_t n_imp,
    float* scores, double* __restrict__ metrics) {
  __shared__ float s_s[kImpWarps][kImpChunk];
  __shared__ uint8_t s_f[kImpWarps][kImpChunk];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int64_t i = (int64_t)blockIdx.x * kImpWarps + w; i < n_imp; i += (int64_t)gridDim.x * kImpWarps) {
    const int64_t b0 = indptr[i], m = indptr[i + 1] - b0;
    const float* q = qv + i * ld_q;
    float qn = 0.0f;
    if (cosine) qn = sqrtf(warp_dot(q, q, H, lane));
    for (int64_t k = 0; k < m; ++k) {
      const float* e = emb + (int64_t)items[b0 + k] * ld_emb;
      float dot = 0.0f, ee = 0.0f;
      for (int j = lane; j < H; j += 32) {
        const float x = e[j];
        dot = fmaf(q[j], x, dot);
        ee = fmaf(x, x, ee);
      }
      dot = warp_sum(dot);
      float s = dot;
      if (cosine) {
        ee = warp_sum(ee);
        s = (qn > 0.0f && ee > 0.0f) ? dot / (qn * sqrtf(ee)) : 0.0f;
      }
      if (lane == 0) scores[b0 + k] = s;
    }
    __syncwarp();   // the scores written by lane 0 are read by every lane below
    impression_rank_metrics(scores, clicked, b0, m, s_s[w], s_f[w], metrics + i * 4, lane);
  }
}

constexpr int kImpMaxNegatives = 32;   // K <= 32: one draw per lane

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Draw d of click r (its ordinal among the impression's clicks) of global impression id: word d & 3 of Philox4x32-10 with key
// (seed lo, seed hi) and counter (id, r, epoch lo, d >> 2).  It depends on nothing else: not on the batch, the position or the grid.
__device__ __forceinline__ uint32_t softmax_draw(uint64_t seed, uint64_t epoch, uint32_t id, uint32_t r, int d) {
  uint32_t c[4] = {id, r, (uint32_t)epoch, (uint32_t)(d >> 2)};
  uint32_t k[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
#pragma unroll
  for (int i = 0; i < 10; ++i) philox_round(c, k);
  const uint32_t lo = (d & 1) ? c[1] : c[0], hi = (d & 1) ? c[3] : c[2];
  return (d & 2) ? hi : lo;
}

// One warp per packed position p, its impressions q in [pos_indptr[p], pos_indptr[p + 1]) in that order.  For each click c of a
// usable impression (|C|, |N| >= 1), with r its ordinal in C: S_c = N if K = 0 or K >= |N|, else K distinct non-clicks by
// Floyd's algorithm (d = 0 .. K - 1: j = |N| - K + d, t = floor(u_d (j + 1) / 2^32), take j if t is taken, else t; ordinals into N
// in item order).  *loss_sum += l_c = log(e^{s_c} + sum_{S_c} e^{s_n}) - s_c (max subtracted; fp64 atomics, one per warp) and
// dh_p += scale sum_c sum_{j in {c} + S_c} (p_cj - [j = c]) e_j.  The weights are summed per candidate first (ws: two 4-byte words
// per shown article, word 0 the weight, word 1 the non-click list), then each candidate's row is read once, in item order; rows
// of zero weight are skipped.  With S_c = N the impression is scored once: every click shares T = sum_N e^{s_n - M_N}, so the
// work is O(m H + |C|).  Otherwise only the click and its K draws are scored, one draw per lane; Floyd's membership test is a
// warp vote.  The warp owns row p of dh: no atomics on dh, the result does not depend on the schedule.  Launch bounds of 8 CTAs
// per SM let ptxas use 64 registers; at its default of 48 it spilled the draw loop's state to the stack.
// DEMB (dae_impression_softmax_loss_grad, DESIGN 4.19): each candidate's weight g also adds g h_p into demb[it[k]] by fp32 atomics;
// the DEMB = false instance is dae_impression_softmax_loss's kernel, its code unchanged by the flag.
// DET (the *_det exports, DESIGN 4.21): position p's loss is stored to loss_slots[p], and with DEMB shown article k gets the triple
// (it[k], p, g) at its index in the packed items, g being its weight summed over the impression's clicks in click order (slot -1
// where g = 0 or in an impression without a click or without a non-click).  dh's arithmetic is the same in every instance.
template <bool DEMB, bool DET = false>
__global__ void __launch_bounds__(kImpWarps * 32, 8) impression_softmax_loss_kernel(
    const float* __restrict__ h, int64_t ld_h, const float* __restrict__ emb, int64_t ld_emb, int H, const int64_t* __restrict__ pos_indptr,
    int64_t n_pos, const int64_t* __restrict__ imp_indptr, const int32_t* __restrict__ items, const uint8_t* __restrict__ clicked,
    const int64_t* __restrict__ imp_ids, int K, uint64_t seed, uint64_t epoch, float scale, float* __restrict__ dh, int64_t ld_dh,
    double* __restrict__ loss_sum, float* ws, float* __restrict__ demb, int64_t ld_demb, double* __restrict__ loss_slots,
    int32_t* __restrict__ t_slot, int32_t* __restrict__ t_row, float* __restrict__ t_coef) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const float neg_inf = __int_as_float(0xff800000);
  double acc = 0.0;
  for (int64_t p = (int64_t)blockIdx.x * kImpWarps + w; p < n_pos; p += (int64_t)gridDim.x * kImpWarps) {
    float* d = dh + p * ld_dh;
    for (int j = lane; j < H; j += 32) d[j] = 0.0f;
    const float* hp = h + p * ld_h;
    for (int64_t q = pos_indptr[p]; q < pos_indptr[p + 1]; ++q) {
      const int64_t b0 = imp_indptr[q];
      const int m = (int)(imp_indptr[q + 1] - b0);   // < 2^31: an impression's articles are distinct int32 rows
      const int32_t* it = items + b0;
      const uint8_t* cl = clicked + b0;
      const int nc = count_clicked(cl, m, lane), nn = m - nc;
      if (nc == 0 || nn == 0) {
        if constexpr (DEMB && DET) {
          for (int k = lane; k < m; k += 32) t_slot[b0 + k] = -1;
        }
        continue;
      }
      float* wq = ws + 2 * b0;                           // wq[2 k]: candidate k's weight
      int32_t* nq = reinterpret_cast<int32_t*>(ws) + 2 * b0 + 1;   // nq[2 o]: the position of the o-th non-click
      if (K == 0 || K >= nn) {
        for (int k = 0; k < m; ++k) {
          const float v = warp_dot(hp, emb + (int64_t)it[k] * ld_emb, H, lane);
          if (lane == 0) wq[2 * k] = v;
        }
        __syncwarp();
        float mx = neg_inf;
        for (int k = lane; k < m; k += 32)
          if (!cl[k]) mx = fmaxf(mx, wq[2 * k]);
        const float mn = warp_max(mx);
        float t = 0.0f;
        for (int k = lane; k < m; k += 32)
          if (!cl[k]) t += expf(wq[2 * k] - mn);
        const float tn = warp_sum(t);
        float r = 0.0f;
        for (int k = lane; k < m; k += 32) {
          if (!cl[k]) continue;
          const float sc = wq[2 * k], mc = fmaxf(sc, mn), xc = sc - mc, ec = expf(xc), en = expf(mn - mc);
          const float z = fmaf(en, tn, ec), rz = __fdividef(1.0f, z);
          acc += (double)(logf(z) - xc);
          r = fmaf(en, rz, r);
          wq[2 * k] = fmaf(ec, rz, -1.0f);
        }
        const float rn = warp_sum(r);
        for (int k = lane; k < m; k += 32)
          if (!cl[k]) wq[2 * k] = expf(wq[2 * k] - mn) * rn;
      } else {
        int base = 0;
        for (int k0 = 0; k0 < m; k0 += 32) {
          const int k = k0 + lane;
          const bool nonc = k < m && !cl[k];
          const unsigned b = __ballot_sync(0xffffffffu, nonc);
          if (nonc) nq[2 * (base + __popc(b & ((1u << lane) - 1u)))] = k;
          if (k < m) wq[2 * k] = 0.0f;
          base += __popc(b);
        }
        __syncwarp();
        const uint32_t id = (uint32_t)imp_ids[q];
        uint32_t r = 0;
        for (int k0 = 0; k0 < m; k0 += 32) {
          for (unsigned bits = __ballot_sync(0xffffffffu, k0 + lane < m && cl[k0 + lane]); bits; bits &= bits - 1u, ++r) {
            const int c = k0 + __ffs(bits) - 1;
            const uint32_t u = lane < K ? softmax_draw(seed, epoch, id, r, lane) : 0u;
            int sel = -1;
            for (int dd = 0; dd < K; ++dd) {
              const int j = nn - K + dd;
              const int t = (int)(((uint64_t)__shfl_sync(0xffffffffu, u, dd) * (uint64_t)(j + 1)) >> 32);
              const bool taken = __any_sync(0xffffffffu, lane < dd && sel == t);
              if (lane == dd) sel = taken ? j : t;
            }
            const int pos = lane < K ? nq[2 * sel] : 0;
            float s = 0.0f;
            for (int dd = 0; dd < K; ++dd) {
              const float v = warp_dot(hp, emb + (int64_t)it[__shfl_sync(0xffffffffu, pos, dd)] * ld_emb, H, lane);
              if (lane == dd) s = v;
            }
            const float sc = warp_dot(hp, emb + (int64_t)it[c] * ld_emb, H, lane);
            const float mc = fmaxf(sc, warp_max(lane < K ? s : neg_inf)), xc = sc - mc, ec = expf(xc);
            const float e = lane < K ? expf(s - mc) : 0.0f;
            const float z = warp_sum(e) + ec, rz = __fdividef(1.0f, z);
            if (lane < K) wq[2 * pos] += e * rz;
            if (lane == 0) {
              wq[2 * c] = fmaf(ec, rz, -1.0f);
              acc += (double)(logf(z) - xc);
            }
            __syncwarp();
          }
        }
      }
      __syncwarp();
      for (int k = 0; k < m; ++k) {
        const float g = scale * wq[2 * k];
        if constexpr (DEMB && DET) {
          if (lane == 0) { t_slot[b0 + k] = g == 0.0f ? -1 : it[k]; t_row[b0 + k] = (int32_t)p; t_coef[b0 + k] = g; }
        }
        if (g == 0.0f) continue;
        const float* e = emb + (int64_t)it[k] * ld_emb;
#pragma unroll 1
        for (int j = lane; j < H; j += 32) d[j] = fmaf(g, e[j], d[j]);
        if constexpr (DEMB && !DET) {
          float* de = demb + (int64_t)it[k] * ld_demb;
#pragma unroll 1
          for (int j = lane; j < H; j += 32) atomicAdd(de + j, g * hp[j]);
        }
      }
      __syncwarp();   // the next impression of this warp may write ws entries that lanes read above
    }
    if constexpr (DET) {
      const double l = warp_sum(acc);
      if (lane == 0) loss_slots[p] = l;
      acc = 0.0;
    }
  }
  if constexpr (DET) return;
  acc = warp_sum(acc);
  if (lane == 0 && acc != 0.0) atomicAdd(loss_sum, acc);
}

static int imp_grid(int64_t rows) {
  const int64_t b = (rows + kImpWarps - 1) / kImpWarps, cap = (int64_t)sm_count() * 16;
  return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

}  // namespace dae

using namespace dae;

extern "C" int dae_impression_rank_loss(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int64_t* pos_indptr,
                                        int64_t n_pos, const int64_t* imp_indptr, const int32_t* items, const uint8_t* clicked, float scale,
                                        float* dh, int64_t ld_dh, double* loss_sum, void* stream) {
  DAE_REQUIRE(h && emb && pos_indptr && imp_indptr && items && clicked && dh && loss_sum && H > 0 && n_pos > 0 && ld_h >= H &&
              ld_emb >= H && ld_dh >= H, "dae_impression_rank_loss: bad arguments");
  impression_rank_loss_kernel<false><<<imp_grid(n_pos), kImpWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos_indptr, n_pos, imp_indptr, items, clicked, scale, dh, ld_dh, loss_sum, nullptr, 0, nullptr, nullptr, nullptr,
      nullptr);
  DAE_CHECK_LAUNCH("dae_impression_rank_loss");
  return DAE_OK;
}

extern "C" int dae_impression_rank_loss_grad(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H,
                                             const int64_t* pos_indptr, int64_t n_pos, const int64_t* imp_indptr, const int32_t* items,
                                             const uint8_t* clicked, float scale, float* dh, int64_t ld_dh, double* loss_sum, float* demb,
                                             int64_t ld_demb, void* stream) {
  DAE_REQUIRE(h && emb && pos_indptr && imp_indptr && items && clicked && dh && loss_sum && demb && H > 0 && n_pos > 0 && ld_h >= H &&
              ld_emb >= H && ld_dh >= H && ld_demb >= H, "dae_impression_rank_loss_grad: bad arguments");
  impression_rank_loss_kernel<true><<<imp_grid(n_pos), kImpWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos_indptr, n_pos, imp_indptr, items, clicked, scale, dh, ld_dh, loss_sum, demb, ld_demb, nullptr, nullptr, nullptr,
      nullptr);
  DAE_CHECK_LAUNCH("dae_impression_rank_loss_grad");
  return DAE_OK;
}

extern "C" int dae_impression_softmax_loss(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H,
                                           const int64_t* pos_indptr, int64_t n_pos, const int64_t* imp_indptr, const int32_t* items,
                                           const uint8_t* clicked, const int64_t* imp_ids, int32_t K, uint64_t seed, uint64_t epoch,
                                           float scale, float* dh, int64_t ld_dh, double* loss_sum, void* workspace, void* stream) {
  DAE_REQUIRE(h && emb && pos_indptr && imp_indptr && items && clicked && imp_ids && dh && loss_sum && workspace && H > 0 && n_pos > 0 &&
              ld_h >= H && ld_emb >= H && ld_dh >= H && K >= 0 && K <= kImpMaxNegatives, "dae_impression_softmax_loss: bad arguments");
  impression_softmax_loss_kernel<false><<<imp_grid(n_pos), kImpWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos_indptr, n_pos, imp_indptr, items, clicked, imp_ids, K, seed, epoch, scale, dh, ld_dh, loss_sum,
      (float*)workspace, nullptr, 0, nullptr, nullptr, nullptr, nullptr);
  DAE_CHECK_LAUNCH("dae_impression_softmax_loss");
  return DAE_OK;
}

extern "C" int dae_impression_softmax_loss_grad(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H,
                                                const int64_t* pos_indptr, int64_t n_pos, const int64_t* imp_indptr, const int32_t* items,
                                                const uint8_t* clicked, const int64_t* imp_ids, int32_t K, uint64_t seed, uint64_t epoch,
                                                float scale, float* dh, int64_t ld_dh, double* loss_sum, void* workspace, float* demb,
                                                int64_t ld_demb, void* stream) {
  DAE_REQUIRE(h && emb && pos_indptr && imp_indptr && items && clicked && imp_ids && dh && loss_sum && workspace && demb && H > 0 &&
              n_pos > 0 && ld_h >= H && ld_emb >= H && ld_dh >= H && ld_demb >= H && K >= 0 && K <= kImpMaxNegatives,
              "dae_impression_softmax_loss_grad: bad arguments");
  impression_softmax_loss_kernel<true><<<imp_grid(n_pos), kImpWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos_indptr, n_pos, imp_indptr, items, clicked, imp_ids, K, seed, epoch, scale, dh, ld_dh, loss_sum,
      (float*)workspace, demb, ld_demb, nullptr, nullptr, nullptr, nullptr);
  DAE_CHECK_LAUNCH("dae_impression_softmax_loss_grad");
  return DAE_OK;
}

extern "C" int dae_impression_metrics(const float* q, int64_t ld_q, const float* emb, int64_t ld_emb, int32_t H, int32_t cosine,
                                      const int64_t* indptr, const int32_t* items, const uint8_t* clicked, int64_t n_imp, float* scores,
                                      double* metrics, void* stream) {
  DAE_REQUIRE(q && emb && indptr && items && clicked && scores && metrics && H > 0 && n_imp > 0 && ld_q >= H && ld_emb >= H &&
              (cosine == 0 || cosine == 1), "dae_impression_metrics: bad arguments");
  impression_metrics_kernel<<<imp_grid(n_imp), kImpWarps * 32, 0, (cudaStream_t)stream>>>(
      q, ld_q, emb, ld_emb, H, cosine, indptr, items, clicked, n_imp, scores, metrics);
  DAE_CHECK_LAUNCH("dae_impression_metrics");
  return DAE_OK;
}

// ---- deterministic mode (DESIGN 4.21) ------------------------------------------------------------------------------------------
static bool imp_det_aligned(const double* loss_slots, const int32_t* t_slot, const int32_t* t_row, const float* t_coef) {
  return ((uintptr_t)loss_slots & 7) == 0 && (((uintptr_t)t_slot | (uintptr_t)t_row | (uintptr_t)t_coef) & 3) == 0;
}

extern "C" int dae_impression_rank_loss_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H,
                                            const int64_t* pos_indptr, int64_t n_pos, const int64_t* imp_indptr, const int32_t* items,
                                            const uint8_t* clicked, float scale, float* dh, int64_t ld_dh, double* loss_slots,
                                            void* stream) {
  DAE_REQUIRE(h && emb && pos_indptr && imp_indptr && items && clicked && dh && loss_slots && H > 0 && n_pos > 0 && ld_h >= H &&
              ld_emb >= H && ld_dh >= H, "dae_impression_rank_loss_det: bad arguments");
  DAE_REQUIRE(imp_det_aligned(loss_slots, nullptr, nullptr, nullptr), "dae_impression_rank_loss_det: loss_slots must be 8-byte aligned");
  impression_rank_loss_kernel<false, true><<<imp_grid(n_pos), kImpWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos_indptr, n_pos, imp_indptr, items, clicked, scale, dh, ld_dh, nullptr, nullptr, 0, loss_slots,
      nullptr, nullptr, nullptr);
  DAE_CHECK_LAUNCH("dae_impression_rank_loss_det");
  return DAE_OK;
}

extern "C" int dae_impression_rank_loss_grad_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H,
                                                 const int64_t* pos_indptr, int64_t n_pos, const int64_t* imp_indptr,
                                                 const int32_t* items, const uint8_t* clicked, float scale, float* dh, int64_t ld_dh,
                                                 double* loss_slots, int32_t* t_slot, int32_t* t_row, float* t_coef, void* stream) {
  DAE_REQUIRE(h && emb && pos_indptr && imp_indptr && items && clicked && dh && loss_slots && t_slot && t_row && t_coef && H > 0 &&
              n_pos > 0 && n_pos < (1LL << 31) && ld_h >= H && ld_emb >= H && ld_dh >= H,
              "dae_impression_rank_loss_grad_det: bad arguments");
  DAE_REQUIRE(imp_det_aligned(loss_slots, t_slot, t_row, t_coef), "dae_impression_rank_loss_grad_det: misaligned loss_slots or triples");
  impression_rank_loss_kernel<true, true><<<imp_grid(n_pos), kImpWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos_indptr, n_pos, imp_indptr, items, clicked, scale, dh, ld_dh, nullptr, nullptr, 0, loss_slots,
      t_slot, t_row, t_coef);
  DAE_CHECK_LAUNCH("dae_impression_rank_loss_grad_det");
  return DAE_OK;
}

extern "C" int dae_impression_softmax_loss_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H,
                                               const int64_t* pos_indptr, int64_t n_pos, const int64_t* imp_indptr, const int32_t* items,
                                               const uint8_t* clicked, const int64_t* imp_ids, int32_t K, uint64_t seed, uint64_t epoch,
                                               float scale, float* dh, int64_t ld_dh, double* loss_slots, void* workspace,
                                               void* stream) {
  DAE_REQUIRE(h && emb && pos_indptr && imp_indptr && items && clicked && imp_ids && dh && loss_slots && workspace && H > 0 &&
              n_pos > 0 && ld_h >= H && ld_emb >= H && ld_dh >= H && K >= 0 && K <= kImpMaxNegatives,
              "dae_impression_softmax_loss_det: bad arguments");
  DAE_REQUIRE(imp_det_aligned(loss_slots, nullptr, nullptr, nullptr) && ((uintptr_t)workspace & 3) == 0,
              "dae_impression_softmax_loss_det: misaligned loss_slots or workspace");
  impression_softmax_loss_kernel<false, true><<<imp_grid(n_pos), kImpWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos_indptr, n_pos, imp_indptr, items, clicked, imp_ids, K, seed, epoch, scale, dh, ld_dh, nullptr,
      (float*)workspace, nullptr, 0, loss_slots, nullptr, nullptr, nullptr);
  DAE_CHECK_LAUNCH("dae_impression_softmax_loss_det");
  return DAE_OK;
}

extern "C" int dae_impression_softmax_loss_grad_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H,
                                                    const int64_t* pos_indptr, int64_t n_pos, const int64_t* imp_indptr,
                                                    const int32_t* items, const uint8_t* clicked, const int64_t* imp_ids, int32_t K,
                                                    uint64_t seed, uint64_t epoch, float scale, float* dh, int64_t ld_dh,
                                                    double* loss_slots, void* workspace, int32_t* t_slot, int32_t* t_row,
                                                    float* t_coef, void* stream) {
  DAE_REQUIRE(h && emb && pos_indptr && imp_indptr && items && clicked && imp_ids && dh && loss_slots && workspace && t_slot && t_row &&
              t_coef && H > 0 && n_pos > 0 && n_pos < (1LL << 31) && ld_h >= H && ld_emb >= H && ld_dh >= H && K >= 0 &&
              K <= kImpMaxNegatives, "dae_impression_softmax_loss_grad_det: bad arguments");
  DAE_REQUIRE(imp_det_aligned(loss_slots, t_slot, t_row, t_coef) && ((uintptr_t)workspace & 3) == 0,
              "dae_impression_softmax_loss_grad_det: misaligned loss_slots, workspace or triples");
  impression_softmax_loss_kernel<true, true><<<imp_grid(n_pos), kImpWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos_indptr, n_pos, imp_indptr, items, clicked, imp_ids, K, seed, epoch, scale, dh, ld_dh, nullptr,
      (float*)workspace, nullptr, 0, loss_slots, t_slot, t_row, t_coef);
  DAE_CHECK_LAUNCH("dae_impression_softmax_loss_grad_det");
  return DAE_OK;
}
