// LSTM user encoder (DESIGN 4.15): the elementwise cell kernels around the bf16x3 GEMMs of an LSTM over packed reading sequences.
//
// The packed layout, the GEMMs and everything around the cell are the GRU's (user_gru.cu, DESIGN 4.10): at step t the users still
// reading are rows [0, n_t), XP = [X | 1].[W_ih | b_ih]^T and HP_t = [h_{t-1} | 1].[W_hh | b_hh]^T.  The cell follows
// torch.nn.LSTM (gate order i, f, g, o):
//   i = s(xi + hi), f = s(xf + hf), g = tanh(xg + hg), o = s(xo + ho),  c_t = f c_{t-1} + i g,  h_t = o tanh(c_t).
// The pre-activation of every gate is XP + HP, so one gradient row dA = [di | df | dg | do] is both dXP and dHP.
#include <cuda_bf16.h>
#include "common.cuh"

namespace dae {

__device__ __forceinline__ void lstm_split_store(float v, __nv_bfloat16* hi, __nv_bfloat16* lo, int64_t o) {
  const __nv_bfloat16 h = __float2bfloat16_rn(v);
  hi[o] = h;
  lo[o] = __float2bfloat16_rn(v - __bfloat162float(h));
}

__device__ __forceinline__ float lstm_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// One step forward for rows [0, n).  c_prev == nullptr: c_{t-1} = 0.  c_out may be c_prev (each element is read, then written, by the
// same thread).  The cell never reads h_{t-1}: it enters through HP only, so h_out may be the buffer the step's GEMM operand was
// split from.  Rows i < n_split also go to the bf16 hi / lo operand of the next step's recurrent GEMM; gates (optional) <- [i|f|g|o].
__global__ void __launch_bounds__(256) lstm_cell_fwd_kernel(int n, int H, const float* __restrict__ xp, int64_t ld_xp,
                                                            const float* __restrict__ hp, int64_t ld_hp, const float* c_prev,
                                                            int64_t ld_cprev, float* c_out, int64_t ld_c, float* __restrict__ h_out,
                                                            int64_t ld_h, int n_split, __nv_bfloat16* __restrict__ h_hi,
                                                            __nv_bfloat16* __restrict__ h_lo, int64_t ld_split,
                                                            float* __restrict__ gates, int64_t ld_gates) {
  const int64_t total = (int64_t)n * H, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += stride) {
    const int i = (int)(q / H), j = (int)(q - (int64_t)i * H);
    const float* x = xp + (int64_t)i * ld_xp;
    const float* a = hp + (int64_t)i * ld_hp;
    const float cprev = c_prev ? c_prev[(int64_t)i * ld_cprev + j] : 0.0f;
    const float ig = lstm_sigmoid(x[j] + a[j]);
    const float fg = lstm_sigmoid(x[H + j] + a[H + j]);
    const float gg = tanhf(x[2 * H + j] + a[2 * H + j]);
    const float og = lstm_sigmoid(x[3 * H + j] + a[3 * H + j]);
    const float c = fg * cprev + ig * gg;
    const float h = og * tanhf(c);
    c_out[(int64_t)i * ld_c + j] = c;
    h_out[(int64_t)i * ld_h + j] = h;
    if (h_hi && i < n_split) lstm_split_store(h, h_hi, h_lo, (int64_t)i * ld_split + j);
    if (gates) {
      float* s = gates + (int64_t)i * ld_gates;
      s[j] = ig; s[H + j] = fg; s[2 * H + j] = gg; s[3 * H + j] = og;
    }
  }
}

// One step backward for rows [0, n): dh = carry_h + dh_in, dc = carry_c + dh o (1 - tanh^2 c_t).  Writes dA = [di, df, dg, do]
// (pre-activation gradients) once, as bf16 hi / lo rows of the packed operand, and carry_c <- dc f.  carry_h is only read: the
// caller's GEMM then stores dA . W_hh over it (see dae_lstm_cell_bwd).
__global__ void __launch_bounds__(256) lstm_cell_bwd_kernel(int n, int H, const float* __restrict__ dh_in, int64_t ld_dh_in,
                                                            const float* __restrict__ carry_h, int64_t ld_carry_h, float* carry_c,
                                                            int64_t ld_carry_c, const float* __restrict__ gates, int64_t ld_gates,
                                                            const float* __restrict__ c, int64_t ld_c, const float* __restrict__ c_prev,
                                                            int64_t ld_cprev, __nv_bfloat16* __restrict__ da_hi,
                                                            __nv_bfloat16* __restrict__ da_lo, int64_t ld_da) {
  const int64_t total = (int64_t)n * H, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += stride) {
    const int i = (int)(q / H), j = (int)(q - (int64_t)i * H);
    const float dh = carry_h[(int64_t)i * ld_carry_h + j] + (dh_in ? dh_in[(int64_t)i * ld_dh_in + j] : 0.0f);
    const float* s = gates + (int64_t)i * ld_gates;
    const float ig = s[j], fg = s[H + j], gg = s[2 * H + j], og = s[3 * H + j];
    const float tc = tanhf(c[(int64_t)i * ld_c + j]);
    const float cprev = c_prev ? c_prev[(int64_t)i * ld_cprev + j] : 0.0f;
    float* cc = carry_c + (int64_t)i * ld_carry_c + j;
    const float dc = *cc + dh * og * (1.0f - tc * tc);
    const float di = dc * gg * ig * (1.0f - ig);
    const float df = dc * cprev * fg * (1.0f - fg);
    const float dg = dc * ig * (1.0f - gg * gg);
    const float dd = dh * tc * og * (1.0f - og);
    const int64_t o = (int64_t)i * ld_da;
    lstm_split_store(di, da_hi, da_lo, o + j);
    lstm_split_store(df, da_hi, da_lo, o + H + j);
    lstm_split_store(dg, da_hi, da_lo, o + 2 * H + j);
    lstm_split_store(dd, da_hi, da_lo, o + 3 * H + j);
    *cc = dc * fg;
  }
}

static int lstm_grid(int64_t work) {
  const int64_t b = (work + 255) / 256, cap = (int64_t)sm_count() * 16;
  return (int)(b < 1 ? 1 : (b < cap ? b : cap));
}

}  // namespace dae

using namespace dae;

extern "C" int dae_lstm_cell_fwd(int32_t n, int32_t H, const float* xp, int64_t ld_xp, const float* hp, int64_t ld_hp,
                                 const float* c_prev, int64_t ld_cprev, float* c_out, int64_t ld_c, float* h_out, int64_t ld_h,
                                 int32_t n_split, void* h_hi, void* h_lo, int64_t ld_split, float* gates, int64_t ld_gates,
                                 void* stream) {
  DAE_REQUIRE(n > 0 && H > 0 && xp && hp && c_out && h_out && ld_xp >= 4 * (int64_t)H && ld_hp >= 4 * (int64_t)H && ld_c >= H &&
              ld_h >= H && (!c_prev || ld_cprev >= H), "dae_lstm_cell_fwd: bad arguments");
  DAE_REQUIRE(!c_prev || c_prev != c_out || ld_cprev == ld_c, "dae_lstm_cell_fwd: c_out == c_prev needs ld_c == ld_cprev");
  DAE_REQUIRE(!h_hi || (h_lo && ld_split >= H && n_split >= 0 && n_split <= n), "dae_lstm_cell_fwd: bad split arguments");
  DAE_REQUIRE(!gates || ld_gates >= 4 * (int64_t)H, "dae_lstm_cell_fwd: ld_gates < 4H");
  lstm_cell_fwd_kernel<<<lstm_grid((int64_t)n * H), 256, 0, (cudaStream_t)stream>>>(
      n, H, xp, ld_xp, hp, ld_hp, c_prev, ld_cprev, c_out, ld_c, h_out, ld_h, n_split, (__nv_bfloat16*)h_hi, (__nv_bfloat16*)h_lo,
      ld_split, gates, ld_gates);
  DAE_CHECK_LAUNCH("dae_lstm_cell_fwd");
  return DAE_OK;
}

extern "C" int dae_lstm_cell_bwd(int32_t n, int32_t H, const float* dh_in, int64_t ld_dh_in, const float* carry_h, int64_t ld_carry_h,
                                 float* carry_c, int64_t ld_carry_c, const float* gates, int64_t ld_gates, const float* c, int64_t ld_c,
                                 const float* c_prev, int64_t ld_cprev, void* da_hi, void* da_lo, int64_t ld_da, void* stream) {
  DAE_REQUIRE(n > 0 && H > 0 && carry_h && carry_c && gates && c && da_hi && da_lo && ld_carry_h >= H && ld_carry_c >= H &&
              ld_gates >= 4 * (int64_t)H && ld_c >= H && ld_da >= 4 * (int64_t)H && (!dh_in || ld_dh_in >= H) &&
              (!c_prev || ld_cprev >= H), "dae_lstm_cell_bwd: bad arguments");
  lstm_cell_bwd_kernel<<<lstm_grid((int64_t)n * H), 256, 0, (cudaStream_t)stream>>>(
      n, H, dh_in, ld_dh_in, carry_h, ld_carry_h, carry_c, ld_carry_c, gates, ld_gates, c, ld_c, c_prev, ld_cprev,
      (__nv_bfloat16*)da_hi, (__nv_bfloat16*)da_lo, ld_da);
  DAE_CHECK_LAUNCH("dae_lstm_cell_bwd");
  return DAE_OK;
}
