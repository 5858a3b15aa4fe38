// Long-term user vectors (LSTUR-ini, DESIGN 4.18): the row-sparse optimizer step of the user table P [users x ld].
//
// A training batch touches at most batch_users rows of P (the batch's unmasked users), and P with Adam's two slots is
// 3 x users x H fp32: streaming all of it through dae_optimizer_step would move gigabytes per batch to update a few thousand rows.
// Here one warp updates one listed row with the update rules of dae_optimizer_step; rows not listed, and their slots, are not read
// or written (a lazy update: their slots do not decay).  Adam's bias correction uses the row's own step count.
#include "common.cuh"
#include "optimizer_rules.cuh"

namespace dae {

// VEC = 4: float4 accesses (cols and both leading dimensions multiples of 4, 16-byte aligned buffers); VEC = 1 otherwise.
template <int OPT, int VEC>
__global__ void __launch_bounds__(256) rows_optimizer_kernel(float* __restrict__ table, int64_t ld, int cols,
                                                             const int32_t* __restrict__ rows, int n, const float* __restrict__ grad,
                                                             int64_t ld_grad, float* __restrict__ slot1, float* __restrict__ slot2,
                                                             int32_t* __restrict__ counts, float lr, float momentum) {
  const int lane = threadIdx.x & 31, warps = (gridDim.x * blockDim.x) >> 5;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    const int32_t r = rows[i];
    if (r < 0) continue;
    float lr_t = lr;
    if (counts) {   // each lane reads the count before lane 0 writes it back
      const int32_t t = counts[r] + 1;
      if (OPT == DAE_OPT_ADAM) lr_t = (float)((double)lr * sqrt(1.0 - pow(0.999, (double)t)) / (1.0 - pow(0.9, (double)t)));
      __syncwarp();
      if (lane == 0) counts[r] = t;
    }
    const int64_t o = (int64_t)r * ld;
    const float* g_row = grad + (int64_t)i * ld_grad;
    for (int c = lane * VEC; c < cols; c += 32 * VEC) {
      float p[VEC], g[VEC], s1[VEC], s2[VEC];
      if (VEC == 4) {
        const float4 pv = *reinterpret_cast<const float4*>(table + o + c), gv = *reinterpret_cast<const float4*>(g_row + c);
        p[0] = pv.x; p[1] = pv.y; p[2] = pv.z; p[3] = pv.w;
        g[0] = gv.x; g[1] = gv.y; g[2] = gv.z; g[3] = gv.w;
        if (OPT != DAE_OPT_SGD) { const float4 v = *reinterpret_cast<const float4*>(slot1 + o + c); s1[0] = v.x; s1[1] = v.y; s1[2] = v.z; s1[3] = v.w; }
        if (OPT == DAE_OPT_ADAM) { const float4 v = *reinterpret_cast<const float4*>(slot2 + o + c); s2[0] = v.x; s2[1] = v.y; s2[2] = v.z; s2[3] = v.w; }
      } else {
        p[0] = table[o + c]; g[0] = g_row[c];
        if (OPT != DAE_OPT_SGD) s1[0] = slot1[o + c];
        if (OPT == DAE_OPT_ADAM) s2[0] = slot2[o + c];
      }
#pragma unroll
      for (int e = 0; e < VEC; ++e) p[e] = opt_update<OPT>(p[e], g[e], s1[e], s2[e], lr, momentum, lr_t);
      if (VEC == 4) {
        *reinterpret_cast<float4*>(table + o + c) = make_float4(p[0], p[1], p[2], p[3]);
        if (OPT != DAE_OPT_SGD) *reinterpret_cast<float4*>(slot1 + o + c) = make_float4(s1[0], s1[1], s1[2], s1[3]);
        if (OPT == DAE_OPT_ADAM) *reinterpret_cast<float4*>(slot2 + o + c) = make_float4(s2[0], s2[1], s2[2], s2[3]);
      } else {
        table[o + c] = p[0];
        if (OPT != DAE_OPT_SGD) slot1[o + c] = s1[0];
        if (OPT == DAE_OPT_ADAM) slot2[o + c] = s2[0];
      }
    }
  }
}

}  // namespace dae

extern "C" int dae_rows_optimizer_step(float* table, int64_t ld, int32_t cols, const int32_t* rows, int32_t n, const float* grad,
                                       int64_t ld_grad, float* slot1, float* slot2, int32_t* counts, int32_t opt, float lr,
                                       float momentum, void* stream) {
  using namespace dae;
  DAE_REQUIRE(table && rows && grad && n >= 0 && cols > 0 && ld >= cols && ld_grad >= cols, "dae_rows_optimizer_step: bad arguments");
  DAE_REQUIRE(opt >= DAE_OPT_SGD && opt <= DAE_OPT_ADAM, "dae_rows_optimizer_step: unknown optimizer %d", opt);
  DAE_REQUIRE(opt == DAE_OPT_SGD || slot1, "dae_rows_optimizer_step: slot1 required");
  DAE_REQUIRE(opt != DAE_OPT_ADAM || (slot2 && counts), "dae_rows_optimizer_step: slot2 and counts required for adam");
  if (n == 0) return DAE_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const bool vec = cols % 4 == 0 && ld % 4 == 0 && ld_grad % 4 == 0 && (uintptr_t)table % 16 == 0 && (uintptr_t)grad % 16 == 0 &&
                   (!slot1 || (uintptr_t)slot1 % 16 == 0) && (!slot2 || (uintptr_t)slot2 % 16 == 0);
  const int blocks = (int)(((int64_t)n + 7) / 8);   // one warp per listed row
#define DAE_ROWS_LAUNCH(OPT)                                                                                                        \
  do {                                                                                                                            \
    if (vec) rows_optimizer_kernel<OPT, 4><<<blocks, 256, 0, st>>>(table, ld, cols, rows, n, grad, ld_grad, slot1, slot2, counts, lr, momentum); \
    else rows_optimizer_kernel<OPT, 1><<<blocks, 256, 0, st>>>(table, ld, cols, rows, n, grad, ld_grad, slot1, slot2, counts, lr, momentum);      \
  } while (0)
  switch (opt) {
    case DAE_OPT_SGD: DAE_ROWS_LAUNCH(DAE_OPT_SGD); break;
    case DAE_OPT_ADAGRAD: DAE_ROWS_LAUNCH(DAE_OPT_ADAGRAD); break;
    case DAE_OPT_MOMENTUM: DAE_ROWS_LAUNCH(DAE_OPT_MOMENTUM); break;
    default: DAE_ROWS_LAUNCH(DAE_OPT_ADAM); break;
  }
#undef DAE_ROWS_LAUNCH
  DAE_CHECK_LAUNCH("dae_rows_optimizer_step");
  return DAE_OK;
}
