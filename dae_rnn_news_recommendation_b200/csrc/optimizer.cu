// K6: fused optimizer over the flat parameter buffer, and the masking-noise kernel.
//
// Reference ops replaced: tf.train.{GradientDescent,Adagrad,Momentum,Adam}Optimizer.minimize's apply step
// (autoencoder/autoencoder.py:451-472, TF-1.12 update rules) and utils.masking_noise (autoencoder/utils.py:94-115).
#include <cuda_bf16.h>
#include "common.cuh"
#include "optimizer_rules.cuh"

namespace dae {

// VEC = 4: float4 accesses (n, H multiples of 4 and 16-byte aligned buffers); VEC = 1: scalar tail / odd shapes.
template <int OPT, int VEC>
__global__ void __launch_bounds__(256) optimizer_kernel(float* __restrict__ theta, const float* __restrict__ grad,
                                                        float* __restrict__ slot1, float* __restrict__ slot2, int64_t n, float lr,
                                                        float momentum, float gscale, float lr_t, __nv_bfloat16* __restrict__ w_hi,
                                                        __nv_bfloat16* __restrict__ w_lo, int64_t n_w, int H, int64_t ld_split,
                                                        const int64_t* __restrict__ ctl) {
  if (OPT == DAE_OPT_ADAM && ctl) {  // device-resident step counter (CUDA-graph replay): lr_t = lr sqrt(1-b2^t)/(1-b1^t)
    const double t = (double)ctl[2];
    lr_t = (float)((double)lr * sqrt(1.0 - pow(0.999, t)) / (1.0 - pow(0.9, t)));
  }
  const uint32_t nq = (uint32_t)(n / VEC), stride = gridDim.x * blockDim.x;
  const uint32_t hq = (uint32_t)(H / VEC), nwq = (uint32_t)(n_w / VEC);
  for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += stride) {
    float p[VEC], g[VEC], s1[VEC], s2[VEC];
    if (VEC == 4) {
      const float4 pv = reinterpret_cast<const float4*>(theta)[q], gv = reinterpret_cast<const float4*>(grad)[q];
      p[0] = pv.x; p[1] = pv.y; p[2] = pv.z; p[3] = pv.w;
      g[0] = gv.x; g[1] = gv.y; g[2] = gv.z; g[3] = gv.w;
      if (OPT != DAE_OPT_SGD) { const float4 v = reinterpret_cast<const float4*>(slot1)[q]; s1[0] = v.x; s1[1] = v.y; s1[2] = v.z; s1[3] = v.w; }
      if (OPT == DAE_OPT_ADAM) { const float4 v = reinterpret_cast<const float4*>(slot2)[q]; s2[0] = v.x; s2[1] = v.y; s2[2] = v.z; s2[3] = v.w; }
    } else {
      p[0] = theta[q]; g[0] = grad[q];
      if (OPT != DAE_OPT_SGD) s1[0] = slot1[q];
      if (OPT == DAE_OPT_ADAM) s2[0] = slot2[q];
    }
#pragma unroll
    for (int e = 0; e < VEC; ++e) p[e] = opt_update<OPT>(p[e], g[e] * gscale, s1[e], s2[e], lr, momentum, lr_t);
    if (VEC == 4) {
      reinterpret_cast<float4*>(theta)[q] = make_float4(p[0], p[1], p[2], p[3]);
      if (OPT != DAE_OPT_SGD) reinterpret_cast<float4*>(slot1)[q] = make_float4(s1[0], s1[1], s1[2], s1[3]);
      if (OPT == DAE_OPT_ADAM) reinterpret_cast<float4*>(slot2)[q] = make_float4(s2[0], s2[1], s2[2], s2[3]);
    } else {
      theta[q] = p[0];
      if (OPT != DAE_OPT_SGD) slot1[q] = s1[0];
      if (OPT == DAE_OPT_ADAM) slot2[q] = s2[0];
    }
    if (w_hi != nullptr && q < nwq) {  // refresh the bf16 hi/lo operand copy of W consumed by the tensor-core GEMMs
      const uint32_t r = q / hq;
      const int64_t o = (int64_t)r * ld_split + (int64_t)(q - r * hq) * VEC;
      __nv_bfloat16 h[VEC], l[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) { h[e] = __float2bfloat16_rn(p[e]); l[e] = __float2bfloat16_rn(p[e] - __bfloat162float(h[e])); }
      if (VEC == 4) {
        *reinterpret_cast<uint2*>(w_hi + o) = *reinterpret_cast<const uint2*>(h);
        *reinterpret_cast<uint2*>(w_lo + o) = *reinterpret_cast<const uint2*>(l);
      } else {
        w_hi[o] = h[0]; w_lo[o] = l[0];
      }
    }
  }
}

__global__ void __launch_bounds__(256) mask_values_kernel(const float* __restrict__ values, const uint8_t* __restrict__ keep,
                                                          int64_t nnz, float corr_frac, uint64_t seed, uint64_t epoch,
                                                          float* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q * 4 < nnz; q += stride) {
    float u[4];
    if (!keep) {
      uint32_t c[4] = {(uint32_t)q, (uint32_t)(q >> 32), (uint32_t)epoch, (uint32_t)(epoch >> 32)};
      uint32_t k[2] = {(uint32_t)seed, (uint32_t)(seed >> 32)};
#pragma unroll
      for (int r = 0; r < 10; ++r) philox_round(c, k);
#pragma unroll
      for (int e = 0; e < 4; ++e) u[e] = (float)(c[e] >> 8) * (1.0f / 16777216.0f);  // [0,1)
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int64_t p = q * 4 + e;
      if (p < nnz) {
        const bool k1 = keep ? (keep[p] != 0) : (u[e] >= corr_frac);  // np.random.rand(nnz) >= v  (utils.py:111)
        out[p] = k1 ? values[p] : 0.0f;
      }
    }
  }
}

}  // namespace dae

extern "C" int dae_optimizer_step(float* theta, const float* grad, float* slot1, float* slot2, int64_t n, int32_t opt, float lr,
                                  float momentum, float grad_scale, int32_t step, const int64_t* ctl, void* w_hi, void* w_lo,
                                  int32_t F, int32_t H, int64_t ld_split, void* stream) {
  using namespace dae;
  DAE_REQUIRE(theta && grad && n > 0, "dae_optimizer_step: bad arguments");
  DAE_REQUIRE(opt == DAE_OPT_SGD || slot1, "dae_optimizer_step: slot1 required");
  DAE_REQUIRE(opt != DAE_OPT_ADAM || slot2, "dae_optimizer_step: slot2 required for adam");
  DAE_REQUIRE(!w_hi || (w_lo && F > 0 && H > 0 && ld_split >= H && (int64_t)F * H <= n), "dae_optimizer_step: bad split arguments");
  cudaStream_t st = (cudaStream_t)stream;
  __nv_bfloat16* wh = (__nv_bfloat16*)w_hi; __nv_bfloat16* wl = (__nv_bfloat16*)w_lo;
  const int64_t n_w = w_hi ? (int64_t)F * H : 0;
  DAE_REQUIRE(n < ((int64_t)1 << 31), "dae_optimizer_step: n too large");
  const int cap = sm_count() * 8;
  const int blocks = (int)((n / 4 + 255) / 256 < cap ? (n / 4 + 255) / 256 + 1 : cap);
  float lr_t = lr;
  if (opt == DAE_OPT_ADAM) {
    const double t = (double)(step < 1 ? 1 : step);
    lr_t = (float)((double)lr * sqrt(1.0 - pow(0.999, t)) / (1.0 - pow(0.9, t)));
  }
  // float4 path for the bulk when shapes / alignment allow, scalar kernel for whatever remains (n % 4 tail or odd H)
  const bool vec = ((uintptr_t)theta % 16 == 0) && ((uintptr_t)grad % 16 == 0) && (!slot1 || (uintptr_t)slot1 % 16 == 0) &&
                   (!slot2 || (uintptr_t)slot2 % 16 == 0) && (!w_hi || (H % 4 == 0 && ld_split % 4 == 0 && (uintptr_t)w_hi % 8 == 0 && (uintptr_t)w_lo % 8 == 0));
#define DAE_OPT_LAUNCH(OPT)                                                                                                           \
  do {                                                                                                                              \
    if (vec) {                                                                                                                      \
      const int64_t n4 = n / 4 * 4;                                                                                                 \
      if (n4) optimizer_kernel<OPT, 4><<<blocks, 256, 0, st>>>(theta, grad, slot1, slot2, n4, lr, momentum, grad_scale, lr_t, wh, wl, n_w, H, ld_split, ctl); \
      if (n > n4) optimizer_kernel<OPT, 1><<<1, 32, 0, st>>>(theta + n4, grad + n4, slot1 ? slot1 + n4 : nullptr, slot2 ? slot2 + n4 : nullptr, n - n4, lr, momentum, grad_scale, lr_t, nullptr, nullptr, 0, 1, 0, ctl); \
    } else {                                                                                                                        \
      optimizer_kernel<OPT, 1><<<blocks, 256, 0, st>>>(theta, grad, slot1, slot2, n, lr, momentum, grad_scale, lr_t, wh, wl, n_w, H, ld_split, ctl); \
    }                                                                                                                               \
  } while (0)
  switch (opt) {
    case DAE_OPT_SGD: DAE_OPT_LAUNCH(DAE_OPT_SGD); break;
    case DAE_OPT_ADAGRAD: DAE_OPT_LAUNCH(DAE_OPT_ADAGRAD); break;
    case DAE_OPT_MOMENTUM: DAE_OPT_LAUNCH(DAE_OPT_MOMENTUM); break;
    case DAE_OPT_ADAM: DAE_OPT_LAUNCH(DAE_OPT_ADAM); break;
    default: set_error("dae_optimizer_step: unknown optimizer %d", opt); return DAE_ERR_BAD_ARG;
  }
#undef DAE_OPT_LAUNCH
  DAE_CHECK_LAUNCH("dae_optimizer_step");
  return DAE_OK;
}

extern "C" int dae_mask_values(const float* values, const uint8_t* keep, int64_t nnz, float corr_frac, uint64_t seed, uint64_t epoch,
                               float* values_out, void* stream) {
  using namespace dae;
  DAE_REQUIRE(values && values_out && nnz >= 0, "dae_mask_values: bad arguments");
  if (nnz == 0) return DAE_OK;
  const int64_t quads = (nnz + 3) / 4;
  const int cap = sm_count() * 16;
  const int blocks = (int)((quads + 255) / 256 < cap ? (quads + 255) / 256 : cap);
  mask_values_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(values, keep, nnz, corr_frac, seed, epoch, values_out);
  DAE_CHECK_LAUNCH("dae_mask_values");
  return DAE_OK;
}
