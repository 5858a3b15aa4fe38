// Shared helpers for libdae_sm100.so (built for sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include "../../include/dae_sm100.h"

namespace dae {

void set_error(const char* fmt, ...);

#define DAE_REQUIRE(cond, ...)                     \
  do {                                             \
    if (!(cond)) {                                 \
      dae::set_error(__VA_ARGS__);                 \
      return DAE_ERR_BAD_ARG;                      \
    }                                              \
  } while (0)

#define DAE_CHECK_LAUNCH(name)                                              \
  do {                                                                      \
    cudaError_t e__ = cudaGetLastError();                                   \
    if (e__ != cudaSuccess) {                                               \
      dae::set_error("%s: %s", name, cudaGetErrorString(e__));              \
      return DAE_ERR_CUDA;                                                  \
    }                                                                       \
  } while (0)

#define DAE_CUDA(call)                                                      \
  do {                                                                      \
    cudaError_t e__ = (call);                                               \
    if (e__ != cudaSuccess) {                                               \
      dae::set_error("%s: %s", #call, cudaGetErrorString(e__));             \
      return DAE_ERR_CUDA;                                                  \
    }                                                                       \
  } while (0)

constexpr float kEps = 1e-16f;

// SMs of the current device (cached per device): grid sizes and wave heuristics follow the part the code runs on
inline int sm_count() {
  static int n[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
  if (!n[dev]) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = 132;
    n[dev] = v;
  }
  return n[dev];
}

template <int ACT>
__device__ __forceinline__ float act_fwd(float x) {
  if (ACT == DAE_ACT_SIGMOID) return 1.0f / (1.0f + expf(-x));
  if (ACT == DAE_ACT_TANH) return tanhf(x);
  return x;
}
// derivative expressed through the activation value y = f(x)
template <int ACT>
__device__ __forceinline__ float act_grad_from_y(float y) {
  if (ACT == DAE_ACT_SIGMOID) return y * (1.0f - y);
  if (ACT == DAE_ACT_TANH) return 1.0f - y * y;
  return 1.0f;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum, result valid in thread 0 (and broadcast through smem to all). blockDim <= 1024.
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* smem32) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) smem32[wid] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  T r = (threadIdx.x < nw) ? smem32[threadIdx.x] : T(0);
  if (wid == 0) {
    r = warp_sum(r);
    if (lane == 0) smem32[0] = r;
  }
  __syncthreads();
  return smem32[0];
}

// Philox4x32-10 (Salmon et al. 2011)
__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t (&k)[2]) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u;
  const uint32_t hi0 = __umulhi(M0, c[0]), lo0 = M0 * c[0];
  const uint32_t hi1 = __umulhi(M1, c[2]), lo1 = M1 * c[2];
  const uint32_t n0 = hi1 ^ c[1] ^ k[0], n1 = lo1, n2 = hi0 ^ c[3] ^ k[1], n3 = lo0;
  c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
  k[0] += 0x9E3779B9u; k[1] += 0xBB67AE85u;
}

#define DAE_DISPATCH_ACT(act, ACT, ...)                      \
  switch (act) {                                             \
    case DAE_ACT_SIGMOID: { constexpr int ACT = DAE_ACT_SIGMOID; __VA_ARGS__; } break; \
    case DAE_ACT_TANH:    { constexpr int ACT = DAE_ACT_TANH;    __VA_ARGS__; } break; \
    default:              { constexpr int ACT = DAE_ACT_NONE;    __VA_ARGS__; } break; \
  }

}  // namespace dae
