// GRU user encoder (DESIGN 4.10): the elementwise kernels around the bf16x3 GEMMs of a GRU over packed reading sequences.
//
// A batch of users is ordered by length, descending (the PackedSequence layout): at step t the users still reading are the prefix
// [0, n_t) and their positions are the rows off_t .. off_t + n_t - 1 of every packed [positions x ...] buffer.  The GEMMs
// (dae_gemm_bf16x3) produce the projections XP = [X | 1].[W_ih | b_ih]^T and HP_t = [h_{t-1} | 1].[W_hh | b_hh]^T; the cell kernels
// apply the gates (torch.nn.GRU convention, gate order r, z, n) and emit the next GEMM operands as bf16 hi / lo pairs directly.
#include <cuda_bf16.h>
#include "common.cuh"

namespace dae {

__device__ __forceinline__ void split_store(float v, __nv_bfloat16* hi, __nv_bfloat16* lo, int64_t o) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[o] = h;
  lo[o] = __float2bfloat16_rn(v - __bfloat162float(h));
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// hi / lo [n_rows x ld_dst] <- src rows rows[r] (columns [0, cols)), column ones_col = 1, every other column 0
__global__ void __launch_bounds__(256) gather_split_kernel(const float* __restrict__ src, int64_t ld_src, const int32_t* __restrict__ rows,
                                                           int n_rows, int cols, __nv_bfloat16* __restrict__ hi,
                                                           __nv_bfloat16* __restrict__ lo, int64_t ld_dst, int ones_col) {
  const int64_t total = (int64_t)n_rows * ld_dst, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += stride) {
    const int64_t r = q / ld_dst, c = q - r * ld_dst;
    const float v = c < cols ? src[(int64_t)rows[r] * ld_src + c] : (c == ones_col ? 1.0f : 0.0f);
    split_store(v, hi, lo, q);
  }
}

// One step forward for rows [0, n): r = s(xr + hr), z = s(xz + hz), n = tanh(xn + r hn), h = (1 - z) n + z h_prev.
// h_prev == nullptr: h_prev = 0.  h_out may be h_prev (each element is read, then written, by the same thread).
// Rows i < n_split also go to the bf16 hi / lo operand of the next step's recurrent GEMM; gates (optional) <- [r | z | n | hn].
__global__ void __launch_bounds__(256) gru_cell_fwd_kernel(int n, int H, const float* __restrict__ xp, int64_t ld_xp,
                                                           const float* __restrict__ hp, int64_t ld_hp, const float* h_prev,
                                                           int64_t ld_hprev, float* h_out, int64_t ld_h, int n_split,
                                                           __nv_bfloat16* __restrict__ h_hi, __nv_bfloat16* __restrict__ h_lo,
                                                           int64_t ld_split, float* __restrict__ gates, int64_t ld_gates) {
  const int64_t total = (int64_t)n * H, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += stride) {
    const int i = (int)(q / H), j = (int)(q - (int64_t)i * H);
    const float* x = xp + (int64_t)i * ld_xp;
    const float* g = hp + (int64_t)i * ld_hp;
    const float hprev = h_prev ? h_prev[(int64_t)i * ld_hprev + j] : 0.0f;
    const float r = sigmoidf_(x[j] + g[j]);
    const float z = sigmoidf_(x[H + j] + g[H + j]);
    const float hn = g[2 * H + j];
    const float nn = tanhf(x[2 * H + j] + r * hn);
    const float h = (1.0f - z) * nn + z * hprev;
    h_out[(int64_t)i * ld_h + j] = h;
    if (h_hi && i < n_split) split_store(h, h_hi, h_lo, (int64_t)i * ld_split + j);
    if (gates) {
      float* s = gates + (int64_t)i * ld_gates;
      s[j] = r; s[H + j] = z; s[2 * H + j] = nn; s[3 * H + j] = hn;
    }
  }
}

// One step backward for rows [0, n): dh = carry + dh_in.  dXP = [dr^, dz^, dn^] and dHP = [dr^, dz^, r dn^] (bf16 hi / lo rows of the
// packed operands), carry <- dh z (the recurrent GEMM then adds dHP . W_hh onto it).
__global__ void __launch_bounds__(256) gru_cell_bwd_kernel(int n, int H, const float* __restrict__ dh_in, int64_t ld_dh_in,
                                                           float* __restrict__ carry, int64_t ld_carry, const float* __restrict__ gates,
                                                           int64_t ld_gates, const float* __restrict__ h_prev, int64_t ld_hprev,
                                                           __nv_bfloat16* __restrict__ dxp_hi, __nv_bfloat16* __restrict__ dxp_lo,
                                                           __nv_bfloat16* __restrict__ dhp_hi, __nv_bfloat16* __restrict__ dhp_lo,
                                                           int64_t ld_g) {
  const int64_t total = (int64_t)n * H, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += stride) {
    const int i = (int)(q / H), j = (int)(q - (int64_t)i * H);
    float* c = carry + (int64_t)i * ld_carry + j;
    const float dh = *c + (dh_in ? dh_in[(int64_t)i * ld_dh_in + j] : 0.0f);
    const float* s = gates + (int64_t)i * ld_gates;
    const float r = s[j], z = s[H + j], nn = s[2 * H + j], hn = s[3 * H + j];
    const float hprev = h_prev ? h_prev[(int64_t)i * ld_hprev + j] : 0.0f;
    const float dn = dh * (1.0f - z) * (1.0f - nn * nn);
    const float dz = dh * (hprev - nn) * z * (1.0f - z);
    const float dr = dn * hn * r * (1.0f - r);
    const int64_t o = (int64_t)i * ld_g;
    split_store(dr, dxp_hi, dxp_lo, o + j);
    split_store(dz, dxp_hi, dxp_lo, o + H + j);
    split_store(dn, dxp_hi, dxp_lo, o + 2 * H + j);
    split_store(dr, dhp_hi, dhp_lo, o + j);
    split_store(dz, dhp_hi, dhp_lo, o + H + j);
    split_store(r * dn, dhp_hi, dhp_lo, o + 2 * H + j);
    *c = dh * z;
  }
}

// neg[p] = (pos[p] + 1 + floor(u (N - 1))) mod N with u = c / 2^32, c the first word of Philox4x32-10 keyed by seed at counter
// (p, batch, epoch): uniform over the N - 1 other articles, never pos[p].  pos[p] < 0 (no next read): neg[p] = -1.
__global__ void __launch_bounds__(256) seq_negatives_kernel(const int32_t* __restrict__ pos, int64_t n_pos, int32_t n_items,
                                                            uint64_t seed, uint64_t epoch, uint64_t batch, int32_t* __restrict__ neg) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n_pos; p += stride) {
    const int32_t a = pos[p];
    if (a < 0) { neg[p] = -1; continue; }
    uint32_t c[4] = {(uint32_t)p, (uint32_t)batch, (uint32_t)epoch, (uint32_t)(epoch >> 32)};
    uint32_t k[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
#pragma unroll
    for (int r = 0; r < 10; ++r) philox_round(c, k);
    const uint32_t off = (uint32_t)(((uint64_t)c[0] * (uint64_t)(n_items - 1)) >> 32);
    neg[p] = (int32_t)(((int64_t)a + 1 + off) % n_items);
  }
}

// One warp per position p: s+ = h_p . e(pos), s- = h_p . e(neg), loss softplus(s- - s+) (summed into *loss_sum in fp64),
// dh_p = scale sigma(s- - s+) (e(neg) - e(pos)).  Positions without a next read (pos < 0) get dh_p = 0.
// DEMB (dae_seq_rank_loss_grad, DESIGN 4.19): also demb[neg] += g h_p and demb[pos] -= g h_p with g = scale sigma(s- - s+), by fp32
// atomics; the DEMB = false instance is dae_seq_rank_loss's kernel, its code unchanged by the flag.
// DET (the *_det exports, DESIGN 4.21): the loss term of position p is stored to loss_slots[p] (0 without a next read) instead of
// added, and with DEMB the article gradient is emitted as triples (t_slot, t_row, t_coef) at 2p = (neg, p, +g) and
// 2p + 1 = (pos, p, -g) (slot -1 without a next read) for dae_ordered_rows; dh's arithmetic is the same in every instance.
constexpr int kLossWarps = 8;
template <bool DEMB, bool DET = false>
__global__ void __launch_bounds__(kLossWarps * 32) seq_rank_loss_kernel(const float* __restrict__ h, int64_t ld_h,
                                                                        const float* __restrict__ emb, int64_t ld_emb, int H,
                                                                        const int32_t* __restrict__ pos, const int32_t* __restrict__ neg,
                                                                        int64_t n_pos, float scale, float* __restrict__ dh,
                                                                        int64_t ld_dh, double* __restrict__ loss_sum,
                                                                        float* __restrict__ demb, int64_t ld_demb,
                                                                        double* __restrict__ loss_slots, int32_t* __restrict__ t_slot,
                                                                        int32_t* __restrict__ t_row, float* __restrict__ t_coef) {
  __shared__ double s_loss[kLossWarps];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double acc = 0.0;
  for (int64_t p = (int64_t)blockIdx.x * kLossWarps + w; p < n_pos; p += (int64_t)gridDim.x * kLossWarps) {
    const int32_t a = pos[p];
    float* d = dh + p * ld_dh;
    if (a < 0) {
      for (int j = lane; j < H; j += 32) d[j] = 0.0f;
      if constexpr (DET) {
        if (lane == 0) {
          loss_slots[p] = 0.0;
          if constexpr (DEMB) { t_slot[2 * p] = -1; t_slot[2 * p + 1] = -1; }
        }
      }
      continue;
    }
    const float* hp = h + p * ld_h;
    const float* ep = emb + (int64_t)a * ld_emb;
    const float* en = emb + (int64_t)neg[p] * ld_emb;
    float sp = 0.0f, sn = 0.0f;
    for (int j = lane; j < H; j += 32) { const float x = hp[j]; sp = fmaf(x, ep[j], sp); sn = fmaf(x, en[j], sn); }
    sp = warp_sum(sp);
    sn = warp_sum(sn);
    const float x = sn - sp;
    const float g = scale * sigmoidf_(x);
    for (int j = lane; j < H; j += 32) d[j] = g * (en[j] - ep[j]);
    if constexpr (DEMB && DET) {
      if (lane == 0) {
        t_slot[2 * p] = neg[p]; t_row[2 * p] = (int32_t)p; t_coef[2 * p] = g;
        t_slot[2 * p + 1] = a; t_row[2 * p + 1] = (int32_t)p; t_coef[2 * p + 1] = -g;
      }
    } else if constexpr (DEMB) {
      float* dp = demb + (int64_t)a * ld_demb;
      float* dn = demb + (int64_t)neg[p] * ld_demb;
      for (int j = lane; j < H; j += 32) {
        const float x = g * hp[j];
        atomicAdd(dn + j, x);
        atomicAdd(dp + j, -x);
      }
    }
    if constexpr (DET) {
      if (lane == 0) loss_slots[p] = (double)(fmaxf(x, 0.0f) + log1pf(expf(-fabsf(x))));
    } else {
      if (lane == 0) acc += (double)(fmaxf(x, 0.0f) + log1pf(expf(-fabsf(x))));
    }
  }
  if constexpr (DET) return;
  if (lane == 0) s_loss[w] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < kLossWarps; ++k) t += s_loss[k];
    if (t != 0.0) atomicAdd(loss_sum, t);
  }
}

// *out += the sum of slots[0, n) in a fixed order: thread t of kSlotSumThreads adds slots t, t + kSlotSumThreads, ... in index
// order from +0, then thread 0 adds the kSlotSumThreads partials in thread order from +0, then adds that total to *out.
constexpr int kSlotSumThreads = 256;
__global__ void __launch_bounds__(kSlotSumThreads) loss_slots_sum_kernel(const double* __restrict__ slots, int64_t n,
                                                                          double* __restrict__ out) {
  __shared__ double part[kSlotSumThreads];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += kSlotSumThreads) s += slots[i];
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int k = 0; k < kSlotSumThreads; ++k) t += part[k];
    *out += t;
  }
}

static int grid_for(int64_t work, int per_block, int cap_per_sm) {
  const int64_t b = (work + per_block - 1) / per_block, cap = (int64_t)sm_count() * cap_per_sm;
  return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

}  // namespace dae

using namespace dae;

extern "C" int dae_gather_split_bf16(const float* src, int64_t ld_src, const int32_t* rows, int32_t n_rows, int32_t cols, void* hi, void* lo,
                                     int64_t ld_dst, int32_t ones_col, void* stream) {
  DAE_REQUIRE(src && rows && hi && lo && n_rows > 0 && cols > 0 && ld_src >= cols && ld_dst >= cols && ones_col < ld_dst,
              "dae_gather_split_bf16: bad arguments");
  gather_split_kernel<<<grid_for((int64_t)n_rows * ld_dst, 256, 16), 256, 0, (cudaStream_t)stream>>>(
      src, ld_src, rows, n_rows, cols, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo, ld_dst, ones_col);
  DAE_CHECK_LAUNCH("dae_gather_split_bf16");
  return DAE_OK;
}

extern "C" int dae_gru_cell_fwd(int32_t n, int32_t H, const float* xp, int64_t ld_xp, const float* hp, int64_t ld_hp, const float* h_prev,
                                int64_t ld_hprev, float* h_out, int64_t ld_h, int32_t n_split, void* h_hi, void* h_lo, int64_t ld_split,
                                float* gates, int64_t ld_gates, void* stream) {
  DAE_REQUIRE(n > 0 && H > 0 && xp && hp && h_out && ld_xp >= 3 * H && ld_hp >= 3 * H && ld_h >= H && (!h_prev || ld_hprev >= H),
              "dae_gru_cell_fwd: bad arguments");
  DAE_REQUIRE(!h_hi || (h_lo && ld_split >= H && n_split >= 0 && n_split <= n), "dae_gru_cell_fwd: bad split arguments");
  DAE_REQUIRE(!gates || ld_gates >= 4 * H, "dae_gru_cell_fwd: ld_gates < 4H");
  gru_cell_fwd_kernel<<<grid_for((int64_t)n * H, 256, 16), 256, 0, (cudaStream_t)stream>>>(
      n, H, xp, ld_xp, hp, ld_hp, h_prev, ld_hprev, h_out, ld_h, n_split, (__nv_bfloat16*)h_hi, (__nv_bfloat16*)h_lo, ld_split, gates,
      ld_gates);
  DAE_CHECK_LAUNCH("dae_gru_cell_fwd");
  return DAE_OK;
}

extern "C" int dae_gru_cell_bwd(int32_t n, int32_t H, const float* dh_in, int64_t ld_dh_in, float* carry, int64_t ld_carry,
                                const float* gates, int64_t ld_gates, const float* h_prev, int64_t ld_hprev, void* dxp_hi, void* dxp_lo,
                                void* dhp_hi, void* dhp_lo, int64_t ld_g, void* stream) {
  DAE_REQUIRE(n > 0 && H > 0 && carry && gates && dxp_hi && dxp_lo && dhp_hi && dhp_lo && ld_carry >= H && ld_gates >= 4 * H &&
              ld_g >= 3 * H && (!dh_in || ld_dh_in >= H) && (!h_prev || ld_hprev >= H), "dae_gru_cell_bwd: bad arguments");
  gru_cell_bwd_kernel<<<grid_for((int64_t)n * H, 256, 16), 256, 0, (cudaStream_t)stream>>>(
      n, H, dh_in, ld_dh_in, carry, ld_carry, gates, ld_gates, h_prev, ld_hprev, (__nv_bfloat16*)dxp_hi, (__nv_bfloat16*)dxp_lo,
      (__nv_bfloat16*)dhp_hi, (__nv_bfloat16*)dhp_lo, ld_g);
  DAE_CHECK_LAUNCH("dae_gru_cell_bwd");
  return DAE_OK;
}

extern "C" int dae_seq_negatives(const int32_t* pos, int64_t n_pos, int32_t n_items, uint64_t seed, uint64_t epoch, uint64_t batch,
                                 int32_t* neg, void* stream) {
  DAE_REQUIRE(pos && neg && n_pos > 0 && n_items >= 2, "dae_seq_negatives: bad arguments (n_pos = %lld, n_items = %d >= 2 needed)",
              (long long)n_pos, n_items);
  seq_negatives_kernel<<<grid_for(n_pos, 256, 16), 256, 0, (cudaStream_t)stream>>>(pos, n_pos, n_items, seed, epoch, batch, neg);
  DAE_CHECK_LAUNCH("dae_seq_negatives");
  return DAE_OK;
}

extern "C" int dae_seq_rank_loss(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int32_t* pos,
                                 const int32_t* neg, int64_t n_pos, float scale, float* dh, int64_t ld_dh, double* loss_sum, void* stream) {
  DAE_REQUIRE(h && emb && pos && neg && dh && loss_sum && H > 0 && n_pos > 0 && ld_h >= H && ld_emb >= H && ld_dh >= H,
              "dae_seq_rank_loss: bad arguments");
  seq_rank_loss_kernel<false><<<grid_for(n_pos, kLossWarps, 16), kLossWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos, neg, n_pos, scale, dh, ld_dh, loss_sum, nullptr, 0, nullptr, nullptr, nullptr, nullptr);
  DAE_CHECK_LAUNCH("dae_seq_rank_loss");
  return DAE_OK;
}

extern "C" int dae_seq_rank_loss_grad(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int32_t* pos,
                                      const int32_t* neg, int64_t n_pos, float scale, float* dh, int64_t ld_dh, double* loss_sum,
                                      float* demb, int64_t ld_demb, void* stream) {
  DAE_REQUIRE(h && emb && pos && neg && dh && loss_sum && demb && H > 0 && n_pos > 0 && ld_h >= H && ld_emb >= H && ld_dh >= H &&
              ld_demb >= H, "dae_seq_rank_loss_grad: bad arguments");
  seq_rank_loss_kernel<true><<<grid_for(n_pos, kLossWarps, 16), kLossWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos, neg, n_pos, scale, dh, ld_dh, loss_sum, demb, ld_demb, nullptr, nullptr, nullptr, nullptr);
  DAE_CHECK_LAUNCH("dae_seq_rank_loss_grad");
  return DAE_OK;
}

extern "C" int dae_seq_rank_loss_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int32_t* pos,
                                     const int32_t* neg, int64_t n_pos, float scale, float* dh, int64_t ld_dh, double* loss_slots,
                                     void* stream) {
  DAE_REQUIRE(h && emb && pos && neg && dh && loss_slots && H > 0 && n_pos > 0 && ld_h >= H && ld_emb >= H && ld_dh >= H,
              "dae_seq_rank_loss_det: bad arguments");
  DAE_REQUIRE(((uintptr_t)loss_slots & 7) == 0, "dae_seq_rank_loss_det: loss_slots must be 8-byte aligned");
  seq_rank_loss_kernel<false, true><<<grid_for(n_pos, kLossWarps, 16), kLossWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos, neg, n_pos, scale, dh, ld_dh, nullptr, nullptr, 0, loss_slots, nullptr, nullptr, nullptr);
  DAE_CHECK_LAUNCH("dae_seq_rank_loss_det");
  return DAE_OK;
}

extern "C" int dae_seq_rank_loss_grad_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int32_t* pos,
                                          const int32_t* neg, int64_t n_pos, float scale, float* dh, int64_t ld_dh, double* loss_slots,
                                          int32_t* t_slot, int32_t* t_row, float* t_coef, void* stream) {
  DAE_REQUIRE(h && emb && pos && neg && dh && loss_slots && t_slot && t_row && t_coef && H > 0 && n_pos > 0 && n_pos < (1LL << 30) &&
              ld_h >= H && ld_emb >= H && ld_dh >= H, "dae_seq_rank_loss_grad_det: bad arguments");
  DAE_REQUIRE(((uintptr_t)loss_slots & 7) == 0 && (((uintptr_t)t_slot | (uintptr_t)t_row | (uintptr_t)t_coef) & 3) == 0,
              "dae_seq_rank_loss_grad_det: misaligned loss_slots or triples");
  seq_rank_loss_kernel<true, true><<<grid_for(n_pos, kLossWarps, 16), kLossWarps * 32, 0, (cudaStream_t)stream>>>(
      h, ld_h, emb, ld_emb, H, pos, neg, n_pos, scale, dh, ld_dh, nullptr, nullptr, 0, loss_slots, t_slot, t_row, t_coef);
  DAE_CHECK_LAUNCH("dae_seq_rank_loss_grad_det");
  return DAE_OK;
}

extern "C" int dae_loss_slots_sum(const double* loss_slots, int64_t n, double* out, void* stream) {
  DAE_REQUIRE(loss_slots && out && n >= 0, "dae_loss_slots_sum: bad arguments");
  DAE_REQUIRE((((uintptr_t)loss_slots | (uintptr_t)out) & 7) == 0, "dae_loss_slots_sum: pointers must be 8-byte aligned");
  loss_slots_sum_kernel<<<1, kSlotSumThreads, 0, (cudaStream_t)stream>>>(loss_slots, n, out);
  DAE_CHECK_LAUNCH("dae_loss_slots_sum");
  return DAE_OK;
}
