// Attention user encoder (DESIGN 4.17): NRMS's user encoder made causal, over packed reading sequences.
//
// The packed layout is the RNNs' (user_gru.cu, DESIGN 4.10): users ordered by length, descending; position off[t] + i is read t of
// batch user i, and user i has lens[i] reads.  The projections run on dae_gemm_bf16x3: QKV = [X | 1].[W_in | b_in]^T,
// M = [O | 1].[W_out | b_out]^T and Z = [M | 1].[W_a | b_a]^T.  The kernels here are the parts between them:
//   attention: O_t = sum_{s <= t} softmax_s(q_t . k_s / sqrt(d)) v_s per (user, head), d = H / heads;
//   pooling:   a_s = q . tanh(Z_s), u_t = sum_{s <= t} softmax_{s <= t}(a)_s M_s.
// Every output element is written by one thread in a fixed order (no atomics), so the results are the same bits on every run.
#include <cuda_bf16.h>
#include <math.h>
#include "common.cuh"

namespace dae {

constexpr int kAttnTile = 32;          // queries of one work item = keys of one shared-memory tile = lanes
constexpr int kAttnWarps = 8;          // each warp owns kAttnTile / kAttnWarps = 4 rows of a tile
constexpr int kAttnRows = kAttnTile / kAttnWarps;
constexpr int kMaxHeadDim = 128;       // 4 columns per lane in registers
constexpr int kHeadCols = kMaxHeadDim / 32;
constexpr int kMaxSeqLen = 1024;       // the pooling kernels keep 4 floats per read of a user in shared memory
constexpr int kPoolThreads = 256;
constexpr int kDqThreads = 1024;

__device__ __forceinline__ void attn_split_store(float v, __nv_bfloat16* hi, __nv_bfloat16* lo, int64_t o) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[o] = h;
  lo[o] = __float2bfloat16_rn(v - __bfloat162float(h));
}

__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Shared-memory row stride of a d-wide tile: odd, so lane r reading row r, column c hits bank (r * ds + c) mod 32, all distinct.
__host__ __device__ __forceinline__ int attn_ds(int d) { return d | 1; }

// rows [0, n) of a tile: dst[r * ds + c] <- src[(off[t0 + r] + i) * ld + col + c]
__device__ __forceinline__ void attn_load_tile(float* dst, int ds, const float* __restrict__ src, int64_t ld, int col,
                                               const int64_t* __restrict__ off, int i, int t0, int n, int d) {
  for (int e = threadIdx.x; e < n * d; e += blockDim.x) {
    const int r = e / d, c = e - r * d;
    dst[r * ds + c] = src[(off[t0 + r] + i) * ld + col + c];
  }
}

__device__ __forceinline__ float attn_dot(const float* a, const float* b, int d) {
  float s = 0.0f;
  for (int c = 0; c < d; ++c) s = fmaf(a[c], b[c], s);
  return s;
}

// Work item w of B x heads x nb: user i, head h, tile b (of queries in the forward and dQ, of keys in dK / dV).
__device__ __forceinline__ void attn_item(int64_t w, int heads, int nb, int& i, int& h, int& b) {
  i = (int)(w / ((int64_t)heads * nb));
  const int r = (int)(w - (int64_t)i * heads * nb);
  h = r / nb;
  b = r - h * nb;
}

// Forward: per (user, head, query tile) the causal softmax(QK^T / sqrt(d)) V with an online softmax over key tiles of 32.
__global__ void __launch_bounds__(kAttnTile * kAttnWarps) seq_attention_fwd_kernel(
    int B, int nb, const int64_t* __restrict__ off, const int32_t* __restrict__ lens, int H, int heads, float scale,
    const float* __restrict__ qkv, int64_t ld_qkv, float* __restrict__ o, int64_t ld_o, __nv_bfloat16* __restrict__ o_hi,
    __nv_bfloat16* __restrict__ o_lo, int64_t ld_split, float* __restrict__ lse, int64_t ld_lse) {
  extern __shared__ float sm[];
  const int d = H / heads, ds = attn_ds(d), lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* Qs = sm;
  float* Ks = Qs + kAttnTile * ds;
  float* Vs = Ks + kAttnTile * ds;
  for (int64_t w = blockIdx.x; w < (int64_t)B * heads * nb; w += gridDim.x) {
    int i, h, qb;
    attn_item(w, heads, nb, i, h, qb);
    const int L = lens[i], q0 = qb * kAttnTile;
    if (q0 >= L) continue;                                     // uniform over the CTA
    const int nq = min(kAttnTile, L - q0);
    __syncthreads();                                           // the previous item's tiles are no longer read
    attn_load_tile(Qs, ds, qkv, ld_qkv, h * d, off, i, q0, nq, d);
    float m[kAttnRows], l[kAttnRows], acc[kAttnRows][kHeadCols];
#pragma unroll
    for (int k = 0; k < kAttnRows; ++k) {
      m[k] = -INFINITY;
      l[k] = 0.0f;
#pragma unroll
      for (int c = 0; c < kHeadCols; ++c) acc[k][c] = 0.0f;
    }
    for (int kt = 0; kt <= qb; ++kt) {
      const int k0 = kt * kAttnTile, nk = min(kAttnTile, L - k0);
      __syncthreads();
      attn_load_tile(Ks, ds, qkv, ld_qkv, H + h * d, off, i, k0, nk, d);
      attn_load_tile(Vs, ds, qkv, ld_qkv, 2 * H + h * d, off, i, k0, nk, d);
      __syncthreads();
#pragma unroll
      for (int k = 0; k < kAttnRows; ++k) {
        const int r = warp + kAttnWarps * k, t = q0 + r;
        if (r >= nq) break;                                    // uniform over the warp
        const int key = k0 + lane;
        const bool on = key <= t;                              // the causal mask: t attends to s <= t
        const float s = on ? attn_dot(Qs + r * ds, Ks + lane * ds, d) * scale : -INFINITY;
        const float m_new = fmaxf(m[k], warp_max_f(s));        // finite: key k0 <= q0 <= t is always on
        const float corr = expf(m[k] - m_new);
        const float p = on ? expf(s - m_new) : 0.0f;
        l[k] = l[k] * corr + warp_sum(p);
#pragma unroll
        for (int c = 0; c < kHeadCols; ++c) acc[k][c] *= corr;
        const int n_on = min(nk, t - k0 + 1);
        for (int u = 0; u < n_on; ++u) {
          const float pu = __shfl_sync(0xffffffffu, p, u);
#pragma unroll
          for (int c = 0; c < kHeadCols; ++c) {
            const int j = lane + 32 * c;
            if (j < d) acc[k][c] = fmaf(pu, Vs[u * ds + j], acc[k][c]);
          }
        }
        m[k] = m_new;
      }
    }
#pragma unroll
    for (int k = 0; k < kAttnRows; ++k) {
      const int r = warp + kAttnWarps * k;
      if (r >= nq) break;
      const int64_t p = off[q0 + r] + i;
      const float inv = 1.0f / l[k];
#pragma unroll
      for (int c = 0; c < kHeadCols; ++c) {
        const int j = lane + 32 * c;
        if (j < d) {
          const float v = acc[k][c] * inv;
          o[p * ld_o + h * d + j] = v;
          attn_split_store(v, o_hi, o_lo, p * ld_split + h * d + j);
        }
      }
      if (lane == 0) lse[p * ld_lse + h] = m[k] + logf(l[k]);
    }
  }
}

// D_r = dO_r . O_r for rows [0, n) of a tile, one warp per row (lane-strided partial sums, then warp_sum): Ds[r].
__device__ __forceinline__ void attn_rowdot(float* Ds, const float* __restrict__ dout, int64_t ld_do, const float* __restrict__ o,
                                            int64_t ld_o, int col, const int64_t* __restrict__ off, int i, int t0, int n, int d) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = warp; r < n; r += kAttnWarps) {
    const int64_t p = off[t0 + r] + i;
    float s = 0.0f;
    for (int j = lane; j < d; j += 32) s = fmaf(dout[p * ld_do + col + j], o[p * ld_o + col + j], s);
    s = warp_sum(s);
    if (lane == 0) Ds[r] = s;
  }
}

// dQ per (user, head, query tile): dS_ts = P_ts (dO_t . v_s - D_t) with P_ts = exp(scale q_t . k_s - LSE_t), dQ_t = scale sum_s dS_ts k_s.
__global__ void __launch_bounds__(kAttnTile * kAttnWarps, 2) seq_attention_dq_kernel(
    int B, int nb, const int64_t* __restrict__ off, const int32_t* __restrict__ lens, int H, int heads, float scale,
    const float* __restrict__ qkv, int64_t ld_qkv, const float* __restrict__ o, int64_t ld_o, const float* __restrict__ lse,
    int64_t ld_lse, const float* __restrict__ dout, int64_t ld_do, __nv_bfloat16* __restrict__ dq_hi,
    __nv_bfloat16* __restrict__ dq_lo, int64_t ld_dqkv) {
  extern __shared__ float sm[];
  const int d = H / heads, ds = attn_ds(d), lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* Qs = sm;
  float* Gs = Qs + kAttnTile * ds;         // dO rows of the queries
  float* Ks = Gs + kAttnTile * ds;
  float* Vs = Ks + kAttnTile * ds;
  float* Ds = Vs + kAttnTile * ds;
  for (int64_t w = blockIdx.x; w < (int64_t)B * heads * nb; w += gridDim.x) {
    int i, h, qb;
    attn_item(w, heads, nb, i, h, qb);
    const int L = lens[i], q0 = qb * kAttnTile;
    if (q0 >= L) continue;
    const int nq = min(kAttnTile, L - q0);
    __syncthreads();
    attn_load_tile(Qs, ds, qkv, ld_qkv, h * d, off, i, q0, nq, d);
    attn_load_tile(Gs, ds, dout, ld_do, h * d, off, i, q0, nq, d);
    attn_rowdot(Ds, dout, ld_do, o, ld_o, h * d, off, i, q0, nq, d);
    float acc[kAttnRows][kHeadCols];
#pragma unroll
    for (int k = 0; k < kAttnRows; ++k)
#pragma unroll
      for (int c = 0; c < kHeadCols; ++c) acc[k][c] = 0.0f;
    for (int kt = 0; kt <= qb; ++kt) {
      const int k0 = kt * kAttnTile, nk = min(kAttnTile, L - k0);
      __syncthreads();
      attn_load_tile(Ks, ds, qkv, ld_qkv, H + h * d, off, i, k0, nk, d);
      attn_load_tile(Vs, ds, qkv, ld_qkv, 2 * H + h * d, off, i, k0, nk, d);
      __syncthreads();
#pragma unroll
      for (int k = 0; k < kAttnRows; ++k) {
        const int r = warp + kAttnWarps * k, t = q0 + r;
        if (r >= nq) break;
        const int key = k0 + lane;
        float ds_ = 0.0f;
        if (key <= t) {
          const float pr = expf(attn_dot(Qs + r * ds, Ks + lane * ds, d) * scale - lse[(off[t] + i) * ld_lse + h]);
          ds_ = pr * (attn_dot(Gs + r * ds, Vs + lane * ds, d) - Ds[r]);
        }
        const int n_on = min(nk, t - k0 + 1);
        for (int u = 0; u < n_on; ++u) {
          const float g = __shfl_sync(0xffffffffu, ds_, u);
#pragma unroll
          for (int c = 0; c < kHeadCols; ++c) {
            const int j = lane + 32 * c;
            if (j < d) acc[k][c] = fmaf(g, Ks[u * ds + j], acc[k][c]);
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kAttnRows; ++k) {
      const int r = warp + kAttnWarps * k;
      if (r >= nq) break;
      const int64_t p = off[q0 + r] + i;
#pragma unroll
      for (int c = 0; c < kHeadCols; ++c) {
        const int j = lane + 32 * c;
        if (j < d) attn_split_store(acc[k][c] * scale, dq_hi, dq_lo, p * ld_dqkv + h * d + j);
      }
    }
  }
}

// dK, dV per (user, head, key tile): dV_s = sum_{t >= s} P_ts dO_t, dK_s = scale sum_{t >= s} dS_ts q_t, over query tiles of 32.
__global__ void __launch_bounds__(kAttnTile * kAttnWarps) seq_attention_dkv_kernel(
    int B, int nb, const int64_t* __restrict__ off, const int32_t* __restrict__ lens, int H, int heads, float scale,
    const float* __restrict__ qkv, int64_t ld_qkv, const float* __restrict__ o, int64_t ld_o, const float* __restrict__ lse,
    int64_t ld_lse, const float* __restrict__ dout, int64_t ld_do, __nv_bfloat16* __restrict__ dq_hi,
    __nv_bfloat16* __restrict__ dq_lo, int64_t ld_dqkv) {
  extern __shared__ float sm[];
  const int d = H / heads, ds = attn_ds(d), lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* Ks = sm;
  float* Vs = Ks + kAttnTile * ds;
  float* Qs = Vs + kAttnTile * ds;
  float* Gs = Qs + kAttnTile * ds;
  float* Ds = Gs + kAttnTile * ds;
  float* Ls = Ds + kAttnTile;
  for (int64_t w = blockIdx.x; w < (int64_t)B * heads * nb; w += gridDim.x) {
    int i, h, kb;
    attn_item(w, heads, nb, i, h, kb);
    const int L = lens[i], k0 = kb * kAttnTile;
    if (k0 >= L) continue;
    const int nk = min(kAttnTile, L - k0);
    __syncthreads();
    attn_load_tile(Ks, ds, qkv, ld_qkv, H + h * d, off, i, k0, nk, d);
    attn_load_tile(Vs, ds, qkv, ld_qkv, 2 * H + h * d, off, i, k0, nk, d);
    float dk[kAttnRows][kHeadCols], dv[kAttnRows][kHeadCols];
#pragma unroll
    for (int k = 0; k < kAttnRows; ++k)
#pragma unroll
      for (int c = 0; c < kHeadCols; ++c) dk[k][c] = dv[k][c] = 0.0f;
    for (int q0 = k0; q0 < L; q0 += kAttnTile) {
      const int nq = min(kAttnTile, L - q0);
      __syncthreads();
      attn_load_tile(Qs, ds, qkv, ld_qkv, h * d, off, i, q0, nq, d);
      attn_load_tile(Gs, ds, dout, ld_do, h * d, off, i, q0, nq, d);
      attn_rowdot(Ds, dout, ld_do, o, ld_o, h * d, off, i, q0, nq, d);
      for (int r = threadIdx.x; r < nq; r += blockDim.x) Ls[r] = lse[(off[q0 + r] + i) * ld_lse + h];
      __syncthreads();
#pragma unroll
      for (int k = 0; k < kAttnRows; ++k) {
        const int r = warp + kAttnWarps * k, s = k0 + r;
        if (r >= nk) break;
        const int t = q0 + lane;
        float pr = 0.0f, ds_ = 0.0f;
        if (lane < nq && t >= s) {
          pr = expf(attn_dot(Qs + lane * ds, Ks + r * ds, d) * scale - Ls[lane]);
          ds_ = pr * (attn_dot(Gs + lane * ds, Vs + r * ds, d) - Ds[lane]);
        }
        for (int u = max(0, s - q0); u < nq; ++u) {
          const float pu = __shfl_sync(0xffffffffu, pr, u), gu = __shfl_sync(0xffffffffu, ds_, u);
#pragma unroll
          for (int c = 0; c < kHeadCols; ++c) {
            const int j = lane + 32 * c;
            if (j < d) {
              dv[k][c] = fmaf(pu, Gs[u * ds + j], dv[k][c]);
              dk[k][c] = fmaf(gu, Qs[u * ds + j], dk[k][c]);
            }
          }
        }
      }
    }
#pragma unroll
    for (int k = 0; k < kAttnRows; ++k) {
      const int r = warp + kAttnWarps * k;
      if (r >= nk) break;
      const int64_t p = off[k0 + r] + i;
#pragma unroll
      for (int c = 0; c < kHeadCols; ++c) {
        const int j = lane + 32 * c;
        if (j < d) {
          attn_split_store(dk[k][c] * scale, dq_hi, dq_lo, p * ld_dqkv + H + h * d + j);
          attn_split_store(dv[k][c], dq_hi, dq_lo, p * ld_dqkv + 2 * H + h * d + j);
        }
      }
    }
  }
}

// Pooling forward, one CTA per user: a_s = q . tanh(Z_s) (warp per read), the prefix log-sum-exp lse_t of a (one thread, in read
// order), then u_t = acc_t / S_t with acc_t = acc_{t-1} e^{mx_{t-1} - mx_t} + e^{a_t - mx_t} M_t (thread per column).
__global__ void __launch_bounds__(kPoolThreads) seq_pool_fwd_kernel(
    int B, const int64_t* __restrict__ off, const int32_t* __restrict__ lens, int H, int A, const float* __restrict__ z, int64_t ld_z,
    const float* __restrict__ q, const float* __restrict__ m, int64_t ld_m, float* __restrict__ u, int64_t ld_u,
    float* __restrict__ score, float* __restrict__ plse) {
  __shared__ float sa[kMaxSeqLen], smx[kMaxSeqLen], ssum[kMaxSeqLen];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int i = blockIdx.x; i < B; i += gridDim.x) {
    const int L = lens[i];
    __syncthreads();
    for (int s = warp; s < L; s += nw) {
      const int64_t p = off[s] + i;
      float a = 0.0f;
      for (int k = lane; k < A; k += 32) a = fmaf(q[k], tanhf(z[p * ld_z + k]), a);
      a = warp_sum(a);
      if (lane == 0) { sa[s] = a; score[p] = a; }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float mx = -INFINITY, S = 0.0f;
      for (int t = 0; t < L; ++t) {
        const float mn = fmaxf(mx, sa[t]);
        S = S * expf(mx - mn) + expf(sa[t] - mn);
        mx = mn;
        smx[t] = mx;
        ssum[t] = S;
        plse[off[t] + i] = mx + logf(S);
      }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < H; j += blockDim.x) {
      float acc = 0.0f, mx = -INFINITY;
      for (int t = 0; t < L; ++t) {
        const int64_t p = off[t] + i;
        acc = fmaf(expf(sa[t] - smx[t]), m[p * ld_m + j], acc * expf(mx - smx[t]));
        mx = smx[t];
        u[p * ld_u + j] = acc / ssum[t];
      }
    }
  }
}

// Pooling backward, one CTA per user, from dU (du) and the forward's u, M, Z, a and lse.  With w_ts = e^{a_s - lse_t} and
// e_s = e^{lse_s - lse_{s+1}}: R_s = dU_s + e_s R_{s+1} = sum_{t >= s} e^{lse_s - lse_t} dU_t, C_s = dU_s . u_s + e_s C_{s+1}, so
// dM_s (value path) = w_ss R_s and da_s = sum_{t >= s} w_ts dU_t . (M_s - u_t) = w_ss (M_s . R_s - C_s).  Then dZ_s = da_s q (1 - tanh^2 Z_s)
// (bf16 hi / lo) and the user's share of dq, sum_s da_s tanh Z_s, in read order into dq_part[i].
__global__ void __launch_bounds__(kPoolThreads) seq_pool_bwd_kernel(
    int B, const int64_t* __restrict__ off, const int32_t* __restrict__ lens, int H, int A, const float* __restrict__ du,
    int64_t ld_du, const float* __restrict__ u, int64_t ld_u, const float* __restrict__ m, int64_t ld_m, const float* __restrict__ z,
    int64_t ld_z, const float* __restrict__ q, const float* __restrict__ score, const float* __restrict__ plse, float* dm,
    int64_t ld_dm, __nv_bfloat16* __restrict__ dz_hi, __nv_bfloat16* __restrict__ dz_lo, int64_t ld_dz,
    float* __restrict__ dq_part) {
  __shared__ float se[kMaxSeqLen], sc[kMaxSeqLen], sw[kMaxSeqLen], sda[kMaxSeqLen];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int i = blockIdx.x; i < B; i += gridDim.x) {
    const int L = lens[i];
    __syncthreads();
    for (int s = warp; s < L; s += nw) {                       // c_s = dU_s . u_s
      const int64_t p = off[s] + i;
      float c = 0.0f;
      for (int j = lane; j < H; j += 32) c = fmaf(du[p * ld_du + j], u[p * ld_u + j], c);
      c = warp_sum(c);
      if (lane == 0) {
        sc[s] = c;
        sw[s] = expf(score[p] - plse[p]);
        se[s] = s + 1 < L ? expf(plse[p] - plse[off[s + 1] + i]) : 0.0f;
      }
    }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int s = L - 2; s >= 0; --s) sc[s] = fmaf(se[s], sc[s + 1], sc[s]);   // C_s
    for (int j = threadIdx.x; j < H; j += blockDim.x) {      // R_s, kept in dm until the next pass scales it
      float R = 0.0f;
      for (int s = L - 1; s >= 0; --s) {
        const int64_t p = off[s] + i;
        R = fmaf(se[s], R, du[p * ld_du + j]);
        dm[p * ld_dm + j] = R;
      }
    }
    __syncthreads();
    for (int s = warp; s < L; s += nw) {                       // da_s, then dM_s = w_ss R_s in place
      const int64_t p = off[s] + i;
      float r[8];
      float dot = 0.0f;
      for (int j0 = 0; j0 < H; j0 += 256) {
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const int j = j0 + lane + 32 * c;
          r[c] = j < H ? dm[p * ld_dm + j] : 0.0f;
          if (j < H) dot = fmaf(m[p * ld_m + j], r[c], dot);
        }
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const int j = j0 + lane + 32 * c;
          if (j < H) dm[p * ld_dm + j] = sw[s] * r[c];
        }
      }
      dot = warp_sum(dot);
      if (lane == 0) sda[s] = sw[s] * (dot - sc[s]);
    }
    __syncthreads();
    for (int k = threadIdx.x; k < A; k += blockDim.x) {
      float acc = 0.0f;
      const float qk = q[k];
      for (int s = 0; s < L; ++s) {
        const int64_t p = off[s] + i;
        const float T = tanhf(z[p * ld_z + k]);
        attn_split_store(sda[s] * qk * (1.0f - T * T), dz_hi, dz_lo, p * ld_dz + k);
        acc = fmaf(sda[s], T, acc);
      }
      dq_part[(int64_t)i * A + k] = acc;
    }
  }
}

// dq[k] = sum_i dq_part[i][k]: lane -> column, warp w sums users w, w + 32, ... in order, then warp 0 adds the 32 partials in order.
__global__ void __launch_bounds__(kDqThreads) seq_pool_dq_kernel(int B, int A, const float* __restrict__ dq_part, float* __restrict__ dq) {
  __shared__ float part[kDqThreads / 32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, k = blockIdx.x * 32 + lane;
  float s = 0.0f;
  if (k < A)
    for (int i = warp; i < B; i += kDqThreads / 32) s += dq_part[(int64_t)i * A + k];
  part[warp][lane] = s;
  __syncthreads();
  if (warp == 0 && k < A) {
    float t = 0.0f;
    for (int w = 0; w < kDqThreads / 32; ++w) t += part[w][lane];
    dq[k] = t;
  }
}

static int attn_grid(int64_t work, int cap_per_sm) {
  const int64_t cap = (int64_t)sm_count() * cap_per_sm;
  return (int)(work < 1 ? 1 : (work < cap ? work : cap));
}

static int attn_set_smem(const void* fn, size_t bytes) {
  return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) == cudaSuccess;
}

}  // namespace dae

using namespace dae;

#define ATTN_SHAPE_CHECK(fn)                                                                                                           \
  DAE_REQUIRE(B > 0 && T > 0 && T <= kMaxSeqLen && off && lens && H > 0 && heads > 0 && H % heads == 0 && H / heads <= kMaxHeadDim, \
              fn ": bad shape (B = %d, T = %d <= %d, H = %d, heads = %d dividing H with H / heads <= %d)", B, T, kMaxSeqLen, H, heads, \
              kMaxHeadDim)

extern "C" int dae_seq_attention_fwd(int32_t B, int32_t T, const int64_t* off, const int32_t* lens, int32_t H, int32_t heads,
                                     const float* qkv, int64_t ld_qkv, float* o, int64_t ld_o, void* o_hi, void* o_lo, int64_t ld_split,
                                     float* lse, int64_t ld_lse, void* stream) {
  ATTN_SHAPE_CHECK("dae_seq_attention_fwd");
  DAE_REQUIRE(qkv && o && o_hi && o_lo && lse && ld_qkv >= 3 * (int64_t)H && ld_o >= H && ld_split >= H && ld_lse >= heads,
              "dae_seq_attention_fwd: bad arguments");
  const int d = H / heads, nb = (T + kAttnTile - 1) / kAttnTile;
  const size_t smem = (size_t)3 * kAttnTile * attn_ds(d) * sizeof(float);
  DAE_REQUIRE(attn_set_smem((const void*)seq_attention_fwd_kernel, smem), "dae_seq_attention_fwd: shared memory attribute");
  seq_attention_fwd_kernel<<<attn_grid((int64_t)B * heads * nb, 8), kAttnTile * kAttnWarps, smem, (cudaStream_t)stream>>>(
      B, nb, off, lens, H, heads, 1.0f / sqrtf((float)d), qkv, ld_qkv, o, ld_o, (__nv_bfloat16*)o_hi, (__nv_bfloat16*)o_lo,
      ld_split, lse, ld_lse);
  DAE_CHECK_LAUNCH("dae_seq_attention_fwd");
  return DAE_OK;
}

extern "C" int dae_seq_attention_bwd(int32_t B, int32_t T, const int64_t* off, const int32_t* lens, int32_t H, int32_t heads,
                                     const float* qkv, int64_t ld_qkv, const float* o, int64_t ld_o, const float* lse, int64_t ld_lse,
                                     const float* dout, int64_t ld_do, void* dqkv_hi, void* dqkv_lo, int64_t ld_dqkv, void* stream) {
  ATTN_SHAPE_CHECK("dae_seq_attention_bwd");
  DAE_REQUIRE(qkv && o && lse && dout && dqkv_hi && dqkv_lo && ld_qkv >= 3 * (int64_t)H && ld_o >= H && ld_lse >= heads &&
              ld_do >= H && ld_dqkv >= 3 * (int64_t)H, "dae_seq_attention_bwd: bad arguments");
  const int d = H / heads, nb = (T + kAttnTile - 1) / kAttnTile, ds = attn_ds(d);
  const float scale = 1.0f / sqrtf((float)d);
  const size_t smem = ((size_t)4 * kAttnTile * ds + 2 * kAttnTile) * sizeof(float);
  DAE_REQUIRE(attn_set_smem((const void*)seq_attention_dq_kernel, smem) && attn_set_smem((const void*)seq_attention_dkv_kernel, smem),
              "dae_seq_attention_bwd: shared memory attribute");
  const int grid = attn_grid((int64_t)B * heads * nb, 8);
  seq_attention_dq_kernel<<<grid, kAttnTile * kAttnWarps, smem, (cudaStream_t)stream>>>(
      B, nb, off, lens, H, heads, scale, qkv, ld_qkv, o, ld_o, lse, ld_lse, dout, ld_do, (__nv_bfloat16*)dqkv_hi,
      (__nv_bfloat16*)dqkv_lo, ld_dqkv);
  DAE_CHECK_LAUNCH("dae_seq_attention_bwd (dQ)");
  seq_attention_dkv_kernel<<<grid, kAttnTile * kAttnWarps, smem, (cudaStream_t)stream>>>(
      B, nb, off, lens, H, heads, scale, qkv, ld_qkv, o, ld_o, lse, ld_lse, dout, ld_do, (__nv_bfloat16*)dqkv_hi,
      (__nv_bfloat16*)dqkv_lo, ld_dqkv);
  DAE_CHECK_LAUNCH("dae_seq_attention_bwd (dK, dV)");
  return DAE_OK;
}

extern "C" int dae_seq_pool_fwd(int32_t B, int32_t T, const int64_t* off, const int32_t* lens, int32_t H, int32_t A, const float* z,
                                int64_t ld_z, const float* q, const float* m, int64_t ld_m, float* u, int64_t ld_u, float* score,
                                float* plse, void* stream) {
  DAE_REQUIRE(B > 0 && T > 0 && T <= kMaxSeqLen && off && lens && H > 0 && A > 0,
              "dae_seq_pool_fwd: bad shape (B = %d, T = %d <= %d, H = %d, A = %d)", B, T, kMaxSeqLen, H, A);
  DAE_REQUIRE(z && q && m && u && score && plse && ld_z >= A && ld_m >= H && ld_u >= H, "dae_seq_pool_fwd: bad arguments");
  seq_pool_fwd_kernel<<<attn_grid(B, 8), kPoolThreads, 0, (cudaStream_t)stream>>>(B, off, lens, H, A, z, ld_z, q, m, ld_m, u, ld_u,
                                                                                   score, plse);
  DAE_CHECK_LAUNCH("dae_seq_pool_fwd");
  return DAE_OK;
}

extern "C" int dae_seq_pool_bwd(int32_t B, int32_t T, const int64_t* off, const int32_t* lens, int32_t H, int32_t A, const float* du,
                                int64_t ld_du, const float* u, int64_t ld_u, const float* m, int64_t ld_m, const float* z, int64_t ld_z,
                                const float* q, const float* score, const float* plse, float* dm, int64_t ld_dm, void* dz_hi, void* dz_lo,
                                int64_t ld_dz, float* dq, void* workspace, void* stream) {
  DAE_REQUIRE(B > 0 && T > 0 && T <= kMaxSeqLen && off && lens && H > 0 && A > 0,
              "dae_seq_pool_bwd: bad shape (B = %d, T = %d <= %d, H = %d, A = %d)", B, T, kMaxSeqLen, H, A);
  DAE_REQUIRE(du && u && m && z && q && score && plse && dm && dz_hi && dz_lo && dq && workspace && ld_du >= H && ld_u >= H &&
              ld_m >= H && ld_z >= A && ld_dm >= H && ld_dz >= A, "dae_seq_pool_bwd: bad arguments");
  float* part = (float*)workspace;
  seq_pool_bwd_kernel<<<attn_grid(B, 8), kPoolThreads, 0, (cudaStream_t)stream>>>(
      B, off, lens, H, A, du, ld_du, u, ld_u, m, ld_m, z, ld_z, q, score, plse, dm, ld_dm, (__nv_bfloat16*)dz_hi, (__nv_bfloat16*)dz_lo,
      ld_dz, part);
  DAE_CHECK_LAUNCH("dae_seq_pool_bwd");
  seq_pool_dq_kernel<<<(A + 31) / 32, kDqThreads, 0, (cudaStream_t)stream>>>(B, A, part, dq);
  DAE_CHECK_LAUNCH("dae_seq_pool_bwd (dq)");
  return DAE_OK;
}
