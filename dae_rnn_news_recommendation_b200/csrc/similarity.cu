// "Next" row of the scope table (SURVEY 8f rank 1): pairwise cosine similarity of the embeddings + nearest-article lookup,
// the immediate consumer of transform()'s output.
//
// Reference ops replaced: sklearn.metrics.pairwise.cosine_similarity / linear_kernel as wrapped by helpers.pairwise_similarity
// (helpers.py:11-50) and the np.nanargmax nearest-article lookup (main_autoencoder.py:352-353).
//   sim = normalize(E) . normalize(E)^T   -> the wgmma bf16x3 GEMM (gemm_tc.cu) on row-normalised operands
// This file holds the two small kernels around it: row normalisation fused with the bf16 hi/lo split, and a row arg-max
// that skips the diagonal (so the N x N matrix never has to leave the GPU for the lookup).
#include <cuda_bf16.h>
#include "common.cuh"

namespace dae {

// one warp per row: out_hi/lo[r, :] = split( x[r, :] * s ), s = 1/sqrt(sum x^2) (norm_kind 2), 1/||x||_1 (1), 1/max|x| (3), 1 (0);
// a row whose fp32 norm is 0 is left untouched (s = 1), as sklearn.preprocessing.normalize does -- including a row whose squared
// norm underflows fp32.  A row whose squared norm overflows fp32 (max |x| above ~1.8e19) gets s = 0 and comes out as zeros.
// Columns [cols, ld_dst) of hi / lo are written 0.
__global__ void __launch_bounds__(256) rownorm_split_kernel(const float* __restrict__ X, int rows, int cols, int64_t ld, int norm_kind,
                                                            __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, int64_t ld_dst,
                                                            float* __restrict__ x_out, int64_t ld_out) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  const float* x = X + (int64_t)r * ld;
  float acc = 0.0f;
  for (int c = lane; c < cols; c += 32) {
    const float v = x[c];
    acc = (norm_kind == 2) ? acc + v * v : (norm_kind == 1 ? acc + fabsf(v) : (norm_kind == 3 ? fmaxf(acc, fabsf(v)) : 0.0f));
  }
  if (norm_kind == 3) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc = fmaxf(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  } else {
    acc = warp_sum(acc);
  }
  float s = 1.0f;
  if (norm_kind == 2) s = (acc > 0.0f) ? 1.0f / sqrtf(acc) : 1.0f;   // sklearn.preprocessing.normalize leaves all-zero rows untouched
  else if (norm_kind != 0) s = (acc > 0.0f) ? 1.0f / acc : 1.0f;
  for (int c = lane; c < ld_dst; c += 32) {
    const float v = (c < cols) ? x[c] * s : 0.0f;
    if (hi) {
      const __nv_bfloat16 h = __float2bfloat16_rn(v);
      hi[(int64_t)r * ld_dst + c] = h;
      lo[(int64_t)r * ld_dst + c] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
    if (x_out && c < cols) x_out[(int64_t)r * ld_out + c] = v;
  }
}

// one warp per row: arg-max / max of S[r, :] over the non-NaN entries, skipping column (r + diag_offset): the diagonal is never a
// candidate, so a row whose other scores are all negative returns the best of them (the reference's nanargmax over the
// zero-diagonal matrix would return the row itself with score 0 there).  The first maximum wins (np.argmax); -inf entries are
// candidates.  A row without any candidate (cols = 1 with the diagonal, or all NaN) gets index -1 and value -inf, the top-k
// kernels' padding.  Optionally zeroes the diagonal entry in place.
__global__ void __launch_bounds__(256) row_argmax_kernel(float* __restrict__ S, int rows, int cols, int64_t ld, int64_t diag_offset,
                                                         int zero_diag, int32_t* __restrict__ idx_out, float* __restrict__ val_out) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= rows) return;
  float* s = S + (int64_t)r * ld;
  const int64_t dcol = (int64_t)r + diag_offset;
  float best = -INFINITY;
  int bi = -1;
  for (int c = lane; c < cols; c += 32) {
    if (c == dcol) { if (zero_diag) s[c] = 0.0f; continue; }
    const float v = s[c];
    if (v == v && (bi < 0 || v > best)) { best = v; bi = c; }   // NaN never; the first candidate always, then only a larger one
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oi >= 0 && (bi < 0 || ob > best || (ob == best && oi < bi))) { best = ob; bi = oi; }   // first maximum wins (np.argmax)
  }
  if (lane == 0) {
    if (idx_out) idx_out[r] = bi;
    if (val_out) val_out[r] = best;
  }
}

}  // namespace dae

extern "C" int dae_rownorm_split_bf16(const float* X, int32_t rows, int32_t cols, int64_t ld, int32_t norm_kind, void* hi, void* lo,
                                      int64_t ld_dst, float* x_out, int64_t ld_out, void* stream) {
  using namespace dae;
  DAE_REQUIRE(X && rows > 0 && cols > 0 && ld >= cols && norm_kind >= 0 && norm_kind <= 3, "dae_rownorm_split_bf16: bad arguments");
  DAE_REQUIRE((hi && lo && ld_dst >= cols) || (!hi && !lo), "dae_rownorm_split_bf16: bad split outputs");
  DAE_REQUIRE(hi || x_out, "dae_rownorm_split_bf16: no output requested");
  if (!hi) ld_dst = cols;
  rownorm_split_kernel<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>(X, rows, cols, ld, norm_kind, (__nv_bfloat16*)hi, (__nv_bfloat16*)lo,
                                                                        ld_dst, x_out, ld_out);
  DAE_CHECK_LAUNCH("dae_rownorm_split_bf16");
  return DAE_OK;
}

extern "C" int dae_row_argmax(float* S, int32_t rows, int32_t cols, int64_t ld, int64_t diag_offset, int32_t zero_diag, int32_t* idx_out,
                              float* val_out, void* stream) {
  using namespace dae;
  DAE_REQUIRE(S && rows > 0 && cols > 0 && ld >= cols, "dae_row_argmax: bad arguments");
  row_argmax_kernel<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>(S, rows, cols, ld, diag_offset, zero_diag, idx_out, val_out);
  DAE_CHECK_LAUNCH("dae_row_argmax");
  return DAE_OK;
}
