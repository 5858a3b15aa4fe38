// The per-element update rules of dae_optimizer_step (TF-1.12's GradientDescent, Adagrad, Momentum and Adam apply steps), shared
// with the row-sparse update of the user table (user_long_term.cu).
#pragma once
#include "common.cuh"

namespace dae {

template <int OPT>
__device__ __forceinline__ float opt_update(float p, float g, float& s1, float& s2, float lr, float momentum, float lr_t) {
  if (OPT == DAE_OPT_SGD) {
    p -= lr * g;
  } else if (OPT == DAE_OPT_ADAGRAD) {   // accum += g^2 ; var -= lr * g * rsqrt(accum)   (initial accum 0.1, no epsilon)
    s1 += g * g;
    p -= lr * g / sqrtf(s1);
  } else if (OPT == DAE_OPT_MOMENTUM) {  // accum = mu * accum + g ; var -= lr * accum
    s1 = momentum * s1 + g;
    p -= lr * s1;
  } else {                               // Adam: m, v; var -= lr_t * m / (sqrt(v) + 1e-8)
    s1 = 0.9f * s1 + (1.0f - 0.9f) * g;
    s2 = 0.999f * s2 + (1.0f - 0.999f) * g * g;
    p -= lr_t * s1 / (sqrtf(s2) + 1e-8f);
  }
  return p;
}

}  // namespace dae
