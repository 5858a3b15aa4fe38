// Canonical (i, j) order of the thresholded pairs (dae_pairs_sort): the output of dae_similarity_pairs_bf16x3 /
// dae_csr_similarity_pairs comes in slot-reservation order.  The unique keys i * n_corpus + j are radix-sorted with the scores as the
// payload, on cub's double-buffer sort, whose scratch is independent of n.  So the sort holds 24 B per pair (two key buffers, two
// score buffers) and no permutation: the key buffer the sort leaves free receives the decoded i and j.
#include <cub/device/device_radix_sort.cuh>
#include "common.cuh"

namespace dae {
namespace {

// keys[t] -> out_i[t] = keys[t] / n_corpus, out_j[t] = keys[t] % n_corpus (int32 halves of the free key buffer)
__global__ void pairs_decode_kernel(const unsigned long long* __restrict__ keys, int64_t n, int32_t n_corpus, int32_t* __restrict__ out_i,
                                    int32_t* __restrict__ out_j) {
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[t];
    const unsigned long long q = k / (unsigned long long)n_corpus;
    out_i[t] = (int32_t)q;
    out_j[t] = (int32_t)(k - q * (unsigned long long)n_corpus);
  }
}

}  // namespace
}  // namespace dae

using namespace dae;

extern "C" int dae_pairs_sort_workspace(int64_t n, int32_t key_bits, int64_t* bytes) {
  DAE_REQUIRE(bytes && n >= 0 && n <= INT32_MAX && key_bits >= 1 && key_bits <= 64, "dae_pairs_sort_workspace: bad arguments");
  cub::DoubleBuffer<unsigned long long> k(nullptr, nullptr);
  cub::DoubleBuffer<float> v(nullptr, nullptr);
  size_t tb = 0;
  DAE_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, k, v, (int)n, 0, key_bits));
  *bytes = (int64_t)tb;
  return DAE_OK;
}

extern "C" int dae_pairs_sort(int64_t n, int32_t n_corpus, int32_t key_bits, uint64_t* keys, uint64_t* keys_alt, float* s, float* s_alt,
                              void* workspace, int64_t workspace_bytes, int32_t* which, void* stream) {
  DAE_REQUIRE(keys && keys_alt && s && s_alt && workspace && which, "dae_pairs_sort: null pointer");
  DAE_REQUIRE(n >= 0 && n <= INT32_MAX && n_corpus > 0 && key_bits >= 1 && key_bits <= 64, "dae_pairs_sort: bad sizes");
  DAE_REQUIRE(keys != keys_alt && s != s_alt, "dae_pairs_sort: the alternate buffers must be distinct");
  DAE_REQUIRE(((uintptr_t)keys | (uintptr_t)keys_alt) % 8 == 0 && ((uintptr_t)s | (uintptr_t)s_alt) % 4 == 0,
              "dae_pairs_sort: keys must be 8-byte and scores 4-byte aligned");
  cub::DoubleBuffer<unsigned long long> k(reinterpret_cast<unsigned long long*>(keys), reinterpret_cast<unsigned long long*>(keys_alt));
  cub::DoubleBuffer<float> v(s, s_alt);
  size_t tb = 0;
  DAE_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tb, k, v, (int)n, 0, key_bits));
  DAE_REQUIRE(workspace_bytes >= (int64_t)tb, "dae_pairs_sort: workspace of %lld bytes, %lld needed (dae_pairs_sort_workspace)",
              (long long)workspace_bytes, (long long)tb);
  cudaStream_t st = (cudaStream_t)stream;
  if (n > 0) DAE_CUDA(cub::DeviceRadixSort::SortPairs(workspace, tb, k, v, (int)n, 0, key_bits, st));
  *which = k.selector;   // 0: sorted data in keys / s, 1: in keys_alt / s_alt
  unsigned long long* out = k.Alternate();
  int32_t* out_i = reinterpret_cast<int32_t*>(out);
  const int blocks = (int)((n + 255) / 256 < sm_count() * 8 ? (n + 255) / 256 : sm_count() * 8);
  if (n > 0) pairs_decode_kernel<<<blocks, 256, 0, st>>>(k.Current(), n, n_corpus, out_i, out_i + n);
  DAE_CHECK_LAUNCH("dae_pairs_sort");
  return DAE_OK;
}
