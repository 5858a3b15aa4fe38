// Error plumbing + batch preparation kernel of libdae_sm100.so.
#include <cstdarg>
#include "common.cuh"

namespace dae {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace dae

extern "C" int dae_version(void) { return 100; }

extern "C" int dae_last_error(char* buf, size_t len) {
  if (!buf || len == 0) return 0;
  strncpy(buf, dae::g_err, len - 1);
  buf[len - 1] = 0;
  return (int)strlen(buf);
}

namespace dae {

// Label classes are those of the reference's tf.equal: -0.0 and +0.0 are one class, and a NaN label equals nothing, itself included,
// so every NaN row is a class of one.  The sorts compare one total-order key per label: the float's bits mapped to an unsigned
// integer that orders like the value, -0.0 folded into +0.0 and every NaN mapped to the largest key, after +inf.  Ties (one class,
// or the NaN rows) are broken by row id, so the order is ascending (label, row id) with the NaN rows last in row-id order.
constexpr uint32_t kNanKey = 0xffffffffu;
__device__ __forceinline__ uint32_t label_key(float x) {
  if (x != x) return kNanKey;
  const uint32_t u = __float_as_uint(x) == 0x80000000u ? 0u : __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ bool pair_greater(uint32_t ka, int va, uint32_t kb, int vb) { return (ka > kb) || (ka == kb && va > vb); }

// class segment of sorted position i: [first index with key k, one past the last) by binary searches in keys[0, B); a NaN row is
// the class [i, i + 1)
__device__ __forceinline__ void class_segment(const uint32_t* keys, int B, int i, int32_t* lo, int32_t* hi) {
  const uint32_t k = keys[i];
  if (k == kNanKey) { lo[i] = i; hi[i] = i + 1; return; }
  int a = 0, b = i;               // lower bound in [0, i]
  while (a < b) { const int m = (a + b) >> 1; if (keys[m] < k) a = m + 1; else b = m; }
  lo[i] = a;
  a = i + 1; b = B;               // upper bound in (i, B]
  while (a < b) { const int m = (a + b) >> 1; if (keys[m] <= k) a = m + 1; else b = m; }
  hi[i] = a;
}

// One CTA. Orders the batch rows by label (bitonic sort in smem), derives class segments and the
// closed-form batch_all data weights:
//   w_i = 2(n-1)(B-n) + sum_{c != c_i} n_c(n_c-1),   N_valid = sum_c n_c(n_c-1)(B-n_c)
// which equal the three axis reductions of the B^3 mask in triplet_loss_utils.py:129 / :111.
constexpr int kMaxB = 4096;

__global__ void __launch_bounds__(1024) batch_prepare_kernel(
    const int32_t* __restrict__ perm, int64_t offset, const int64_t* __restrict__ ctl, int B, const float* __restrict__ labels_all,
    int strategy, int32_t* __restrict__ rows_out, float* __restrict__ labels_out, int32_t* seg_lo,
    int32_t* seg_hi, float* __restrict__ weight_out, double* __restrict__ stats, int64_t n_perm) {
  if (ctl) offset += ctl[0];  // device-resident batch cursor (CUDA-graph replay)
  if (n_perm > 0 && offset + B > n_perm) return;  // staging the batch AFTER the epoch's last one: nothing to prepare
  __shared__ uint32_t keys[kMaxB];
  __shared__ int vals[kMaxB];
  __shared__ double red[32];
  int32_t* lo = seg_lo;
  int32_t* hi = seg_hi;
  const bool labelled = strategy != DAE_TRIPLET_NONE && labels_all;
  const int tid = threadIdx.x, nt = blockDim.x;
  int P = 1;
  while (P < B) P <<= 1;
  for (int i = tid; i < P; i += nt) {
    if (i < B) {
      const int r = perm ? perm[offset + i] : (int)(offset + i);
      vals[i] = r;
      keys[i] = labelled ? label_key(labels_all[r]) : label_key(0.0f);
    } else {
      vals[i] = 0x7fffffff;
      keys[i] = kNanKey;  // (largest key, largest row id): the padding sorts last
    }
  }
  __syncthreads();
  if (strategy != DAE_TRIPLET_NONE && P <= 1024) {
    // bitonic sort with one element per thread held in registers: partner exchange by warp shuffle for strides < 32
    // (40 of the 55 stages at P = 1024), through shared memory otherwise.  Both partners evaluate the one predicate
    // pair_greater(lower, upper), so every compare-exchange swaps the pair or keeps it: the network permutes its inputs.
    uint32_t key = keys[tid < P ? tid : 0];
    int val = vals[tid < P ? tid : 0];
    for (int k = 2; k <= P; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        uint32_t okey; int oval;
        if (j < 32) {
          okey = __shfl_xor_sync(0xffffffffu, key, j);
          oval = __shfl_xor_sync(0xffffffffu, val, j);
        } else {
          __syncthreads();
          if (tid < P) { keys[tid] = key; vals[tid] = val; }
          __syncthreads();
          okey = keys[(tid ^ j) & (P - 1)];
          oval = vals[(tid ^ j) & (P - 1)];
        }
        const bool up = ((tid & k) == 0), is_lower = ((tid & j) == 0);
        const bool gt = is_lower ? pair_greater(key, val, okey, oval) : pair_greater(okey, oval, key, val);
        if (gt == up) { key = okey; val = oval; }
      }
    }
    __syncthreads();
    if (tid < P) { keys[tid] = key; vals[tid] = val; }
    __syncthreads();
  } else if (strategy != DAE_TRIPLET_NONE) {
    for (int k = 2; k <= P; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = tid; i < P; i += nt) {
          const int ixj = i ^ j;
          if (ixj > i) {
            const uint32_t ka = keys[i], kb = keys[ixj];
            const int va = vals[i], vb = vals[ixj];
            const bool up = ((i & k) == 0);
            if (pair_greater(ka, va, kb, vb) == up) {
              keys[i] = kb; keys[ixj] = ka;
              vals[i] = vb; vals[ixj] = va;
            }
          }
        }
        __syncthreads();
      }
    }
  }
  for (int i = tid; i < B; i += nt) class_segment(keys, B, i, lo, hi);
  __syncthreads();
  double t_part = 0.0, nv_part = 0.0;
  for (int i = tid; i < B; i += nt) {
    const double n = (double)(hi[i] - lo[i]);
    t_part += n - 1.0;
    nv_part += (n - 1.0) * ((double)B - n);
  }
  const double T = block_sum(t_part, red);
  const double NV = block_sum(nv_part, red);
  for (int i = tid; i < B; i += nt) {
    const double n = (double)(hi[i] - lo[i]);
    rows_out[i] = vals[i];
    if (labels_out) labels_out[i] = labelled ? labels_all[vals[i]] : 0.0f;  // the label's own bits (-0.0, NaN payloads)
    if (weight_out) {
      float w = 1.0f;
      if (strategy == DAE_TRIPLET_BATCH_ALL) w = (float)(2.0 * (n - 1.0) * ((double)B - n) + T - n * (n - 1.0));
      if (strategy == DAE_TRIPLET_BATCH_HARD) w = 0.0f;  // filled by dae_triplet_batch_hard
      weight_out[i] = w;
    }
  }
  if (tid < DAE_STAT_SLOTS) {
    double v = 0.0;
    if (tid == DAE_STAT_SUM_W) v = (strategy == DAE_TRIPLET_BATCH_ALL) ? 3.0 * NV : (strategy == DAE_TRIPLET_NONE ? (double)B : 0.0);
    if (tid == DAE_STAT_N_VALID) v = (strategy == DAE_TRIPLET_BATCH_ALL) ? NV : 0.0;
    stats[tid] = v;
  }
}

// B > kMaxB (up to DAE_MAX_BLOCKED_BATCH): the same outputs from one CTA that sorts inside the caller's buffers -- labels_out holds
// the keys (label_key bits) until the segments are known, rows_out the row ids.  The network is the bitonic sort whose every
// compare-exchange puts the smaller (key, row) pair at the lower index (the first step of each merge compares mirrored positions),
// so the power-of-two padding needs no storage: a virtual (largest key, largest row) at an index >= B never moves.  Partner
// distances below kMaxB run on aligned kMaxB-element blocks staged in shared memory; only the longer ones (6 stages at B = 32768)
// go through global memory.  Rows end in the order batch_prepare_kernel produces.

// one global compare-exchange stage: pair t's lower index a (bit log2(j) clear), partner a + j, or its mirror a ^ (2j - 1) (flip)
__device__ void prepare_global_stage(uint32_t* keys, int32_t* vals, int B, int P, int j, bool flip) {
  for (int t = threadIdx.x; t < P / 2; t += blockDim.x) {
    const int a = 2 * t - (t & (j - 1));
    const int b = flip ? (a ^ (2 * j - 1)) : a + j;
    if (b < B) {
      const uint32_t ka = keys[a], kb = keys[b];
      const int va = vals[a], vb = vals[b];
      if (pair_greater(ka, va, kb, vb)) { keys[a] = kb; keys[b] = ka; vals[a] = vb; vals[b] = va; }
    }
  }
  __syncthreads();
}

// the stages of merge size k with partner distances j < kMaxB, on each aligned kMaxB block in shared memory (k <= kMaxB: the whole
// merge, flip step included)
__device__ void prepare_local_stages(uint32_t* keys, int32_t* vals, int B, int k, uint32_t* sk, int* sv) {
  for (int b0 = 0; b0 < B; b0 += kMaxB) {
    for (int t = threadIdx.x; t < kMaxB; t += blockDim.x) {
      const bool ok = b0 + t < B;
      sk[t] = ok ? keys[b0 + t] : kNanKey;
      sv[t] = ok ? vals[b0 + t] : 0x7fffffff;
    }
    __syncthreads();
    // k <= kMaxB: the whole merges of sizes 2 .. k; k > kMaxB: the steps j = kMaxB/2 .. 1 of merge k
    for (int kk = (k <= kMaxB) ? 2 : k; kk <= k; kk <<= 1) {
      for (int j = (kk <= kMaxB) ? kk >> 1 : kMaxB >> 1; j > 0; j >>= 1) {
        const bool flip = (kk <= kMaxB) && j == (kk >> 1);
        for (int t = threadIdx.x; t < kMaxB / 2; t += blockDim.x) {
          const int a = 2 * t - (t & (j - 1));
          const int b = flip ? (a ^ (2 * j - 1)) : a + j;
          const uint32_t ka = sk[a], kb = sk[b];
          const int va = sv[a], vb = sv[b];
          if (pair_greater(ka, va, kb, vb)) { sk[a] = kb; sk[b] = ka; sv[a] = vb; sv[b] = va; }
        }
        __syncthreads();
      }
    }
    for (int t = threadIdx.x; t < kMaxB && b0 + t < B; t += blockDim.x) { keys[b0 + t] = sk[t]; vals[b0 + t] = sv[t]; }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(1024) batch_prepare_large_kernel(
    const int32_t* __restrict__ perm, int64_t offset, const int64_t* __restrict__ ctl, int B, const float* __restrict__ labels_all,
    int strategy, int32_t* rows_out, float* labels_out, int32_t* seg_lo, int32_t* seg_hi, float* __restrict__ weight_out,
    double* __restrict__ stats, int64_t n_perm) {
  if (ctl) offset += ctl[0];
  if (n_perm > 0 && offset + B > n_perm) return;
  __shared__ uint32_t sk[kMaxB];
  __shared__ int sv[kMaxB];
  __shared__ double red[32];
  const int tid = threadIdx.x, nt = blockDim.x;
  uint32_t* keys = reinterpret_cast<uint32_t*>(labels_out);
  int32_t* vals = rows_out;
  for (int i = tid; i < B; i += nt) {
    const int r = perm ? perm[offset + i] : (int)(offset + i);
    vals[i] = r;
    keys[i] = label_key(labels_all[r]);
  }
  __syncthreads();
  int P = 1;
  while (P < B) P <<= 1;
  prepare_local_stages(keys, vals, B, kMaxB, sk, sv);            // every aligned kMaxB block sorted
  for (int k = 2 * kMaxB; k <= P; k <<= 1) {
    prepare_global_stage(keys, vals, B, P, k >> 1, true);
    for (int j = k >> 2; j >= kMaxB; j >>= 1) prepare_global_stage(keys, vals, B, P, j, false);
    prepare_local_stages(keys, vals, B, k, sk, sv);
  }
  for (int i = tid; i < B; i += nt) class_segment(keys, B, i, seg_lo, seg_hi);
  __syncthreads();
  for (int i = tid; i < B; i += nt) labels_out[i] = labels_all[vals[i]];  // keys -> the labels' own bits (-0.0, NaN payloads)
  double t_part = 0.0, nv_part = 0.0;
  for (int i = tid; i < B; i += nt) {
    const double n = (double)(seg_hi[i] - seg_lo[i]);
    t_part += n - 1.0;
    nv_part += (n - 1.0) * ((double)B - n);
  }
  const double T = block_sum(t_part, red);
  const double NV = block_sum(nv_part, red);
  if (weight_out) {
    for (int i = tid; i < B; i += nt) {
      const double n = (double)(seg_hi[i] - seg_lo[i]);
      weight_out[i] = (strategy == DAE_TRIPLET_BATCH_ALL) ? (float)(2.0 * (n - 1.0) * ((double)B - n) + T - n * (n - 1.0)) : 0.0f;
    }
  }
  if (tid < DAE_STAT_SLOTS) {
    double v = 0.0;
    if (tid == DAE_STAT_SUM_W) v = (strategy == DAE_TRIPLET_BATCH_ALL) ? 3.0 * NV : 0.0;
    if (tid == DAE_STAT_N_VALID) v = (strategy == DAE_TRIPLET_BATCH_ALL) ? NV : 0.0;
    stats[tid] = v;
  }
}

// strategy none: keep the permutation order, w = 1, one segment; any B.
__global__ void batch_rows_kernel(const int32_t* __restrict__ perm, int64_t offset, const int64_t* __restrict__ ctl, int B,
                                  int32_t* __restrict__ rows_out, float* __restrict__ labels_out, int32_t* __restrict__ seg_lo,
                                  int32_t* __restrict__ seg_hi, float* __restrict__ weight_out, double* __restrict__ stats) {
  if (ctl) offset += ctl[0];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) {
    rows_out[i] = perm ? perm[offset + i] : (int)(offset + i);
    if (labels_out) labels_out[i] = 0.0f;
    if (seg_lo) seg_lo[i] = 0;
    if (seg_hi) seg_hi[i] = B;
    if (weight_out) weight_out[i] = 1.0f;
  }
  if (i < DAE_STAT_SLOTS) stats[i] = (i == DAE_STAT_SUM_W) ? (double)B : 0.0;
}

// staged batch (prepared on a side branch during the previous step) -> the live per-batch buffers
__global__ void batch_commit_kernel(int B, const int32_t* __restrict__ rows_s, const float* __restrict__ labels_s,
                                    const int32_t* __restrict__ seg_lo_s, const int32_t* __restrict__ seg_hi_s,
                                    const float* __restrict__ weight_s, const double* __restrict__ stats_s, int32_t* __restrict__ rows,
                                    float* __restrict__ labels_b, int32_t* __restrict__ seg_lo, int32_t* __restrict__ seg_hi,
                                    float* __restrict__ weight, double* __restrict__ stats) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) { rows[i] = rows_s[i]; labels_b[i] = labels_s[i]; seg_lo[i] = seg_lo_s[i]; seg_hi[i] = seg_hi_s[i]; weight[i] = weight_s[i]; }
  if (i < DAE_STAT_SLOTS) stats[i] = stats_s[i];
}

// explicit (org, pos, neg) triplets: the three row blocks of the stacked [org; pos; neg] matrix for batch perm[offset : offset+B]
// (autoencoder/utils.py:73-91 gen_batches_triplet); each of the three reconstruction terms is a mean over B rows.
__global__ void batch_rows_explicit_kernel(const int32_t* __restrict__ perm, int64_t offset, const int64_t* __restrict__ ctl, int B,
                                           int64_t n_each, int32_t* __restrict__ rows_out, double* __restrict__ stats) {
  if (ctl) offset += ctl[0];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) {
    const int64_t r = perm ? (int64_t)perm[offset + i] : offset + i;
    rows_out[i] = (int32_t)r;
    rows_out[B + i] = (int32_t)(r + n_each);
    rows_out[2 * B + i] = (int32_t)(r + 2 * n_each);
  }
  if (i < DAE_STAT_SLOTS) stats[i] = (i == DAE_STAT_SUM_W) ? (double)B : 0.0;
}

__global__ void step_advance_kernel(int64_t* ctl, int64_t row_stride) {
  ctl[0] += row_stride;  // batch cursor into the epoch permutation
  ctl[1] += 1;           // row of the per-epoch stats log
  ctl[2] += 1;           // optimizer step (Adam bias correction)
}

}  // namespace dae

extern "C" int dae_step_advance(int64_t* ctl, int64_t row_stride, void* stream) {
  DAE_REQUIRE(ctl, "dae_step_advance: null ctl");
  dae::step_advance_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(ctl, row_stride);
  DAE_CHECK_LAUNCH("dae_step_advance");
  return DAE_OK;
}

namespace dae {
// dae_batch_prepare(_blocked) / dae_batch_prepare_next(_blocked): the same kernels under two batch caps, DAE_MAX_TRIPLET_BATCH for the
// engines that hold B x B mining buffers and DAE_MAX_BLOCKED_BATCH for the block-mined ones.
static const char* const kCapWhy[2] = {"the cap of the B x B mining buffers", "the cap of block-mined batches"};

static int batch_prepare(const char* fn, int blocked, const int32_t* perm, int64_t offset, const int64_t* ctl, int32_t B,
                         const float* labels_all, int32_t strategy, int32_t* rows_out, float* labels_out, int32_t* seg_lo,
                         int32_t* seg_hi, float* weight_out, double* stats, void* stream) {
  DAE_REQUIRE(B >= 1 && rows_out && stats, "%s: bad B or null output", fn);
  if (strategy == DAE_TRIPLET_NONE) {
    batch_rows_kernel<<<(B + 255) / 256, 256, 0, (cudaStream_t)stream>>>(perm, offset, ctl, B, rows_out, labels_out, seg_lo, seg_hi,
                                                                         weight_out, stats);
    DAE_CHECK_LAUNCH("dae_batch_prepare(none)");
    return DAE_OK;
  }
  const int cap = blocked ? DAE_MAX_BLOCKED_BATCH : DAE_MAX_TRIPLET_BATCH;
  DAE_REQUIRE(B <= cap, "%s: triplet strategies need B <= %d rows, %s (got %d)", fn, cap, kCapWhy[blocked], B);
  DAE_REQUIRE(seg_lo && seg_hi, "%s: null segment outputs", fn);
  DAE_REQUIRE(strategy == DAE_TRIPLET_NONE || labels_all, "%s: labels required for triplet strategies", fn);
  if (B > kMaxB) {
    DAE_REQUIRE(labels_out, "%s: B > %d needs labels_out (the batch is sorted inside it)", fn, kMaxB);
    batch_prepare_large_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(perm, offset, ctl, B, labels_all, strategy, rows_out, labels_out,
                                                                     seg_lo, seg_hi, weight_out, stats, 0);
  } else {
    batch_prepare_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(perm, offset, ctl, B, labels_all, strategy, rows_out, labels_out, seg_lo,
                                                               seg_hi, weight_out, stats, 0);
  }
  DAE_CHECK_LAUNCH(fn);
  return DAE_OK;
}

static int batch_prepare_next(const char* fn, int blocked, const int32_t* perm, int64_t n_perm, int64_t stride, const int64_t* ctl,
                              int32_t B, const float* labels_all, int32_t strategy, int32_t* rows_s, float* labels_s, int32_t* seg_lo_s,
                              int32_t* seg_hi_s, float* weight_s, double* stats_s, void* stream) {
  DAE_REQUIRE(ctl && n_perm > 0 && B >= 1 && rows_s && seg_lo_s && seg_hi_s && stats_s && labels_all, "%s: bad arguments", fn);
  const int cap = blocked ? DAE_MAX_BLOCKED_BATCH : DAE_MAX_TRIPLET_BATCH;
  DAE_REQUIRE(B <= cap, "%s: triplet strategies need B <= %d rows, %s (got %d)", fn, cap, kCapWhy[blocked], B);
  DAE_REQUIRE(strategy == DAE_TRIPLET_BATCH_ALL || strategy == DAE_TRIPLET_BATCH_HARD, "%s: triplet strategies only", fn);
  if (B > kMaxB) {
    DAE_REQUIRE(labels_s, "%s: B > %d needs labels_s (the batch is sorted inside it)", fn, kMaxB);
    batch_prepare_large_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(perm, stride, ctl, B, labels_all, strategy, rows_s, labels_s,
                                                                     seg_lo_s, seg_hi_s, weight_s, stats_s, n_perm);
  } else {
    batch_prepare_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(perm, stride, ctl, B, labels_all, strategy, rows_s, labels_s, seg_lo_s,
                                                               seg_hi_s, weight_s, stats_s, n_perm);
  }
  DAE_CHECK_LAUNCH(fn);
  return DAE_OK;
}
}  // namespace dae

extern "C" int dae_batch_prepare(const int32_t* perm, int64_t offset, const int64_t* ctl, int32_t B, const float* labels_all,
                                 int32_t strategy, int32_t* rows_out, float* labels_out, int32_t* seg_lo,
                                 int32_t* seg_hi, float* weight_out, double* stats, void* stream) {
  return dae::batch_prepare("dae_batch_prepare", 0, perm, offset, ctl, B, labels_all, strategy, rows_out, labels_out, seg_lo, seg_hi,
                            weight_out, stats, stream);
}

extern "C" int dae_batch_prepare_blocked(const int32_t* perm, int64_t offset, const int64_t* ctl, int32_t B, const float* labels_all,
                                         int32_t strategy, int32_t* rows_out, float* labels_out, int32_t* seg_lo,
                                         int32_t* seg_hi, float* weight_out, double* stats, void* stream) {
  return dae::batch_prepare("dae_batch_prepare_blocked", 1, perm, offset, ctl, B, labels_all, strategy, rows_out, labels_out, seg_lo,
                            seg_hi, weight_out, stats, stream);
}

extern "C" int dae_batch_prepare_next(const int32_t* perm, int64_t n_perm, int64_t stride, const int64_t* ctl, int32_t B,
                                      const float* labels_all, int32_t strategy, int32_t* rows_s, float* labels_s, int32_t* seg_lo_s,
                                      int32_t* seg_hi_s, float* weight_s, double* stats_s, void* stream) {
  return dae::batch_prepare_next("dae_batch_prepare_next", 0, perm, n_perm, stride, ctl, B, labels_all, strategy, rows_s, labels_s,
                                 seg_lo_s, seg_hi_s, weight_s, stats_s, stream);
}

extern "C" int dae_batch_prepare_next_blocked(const int32_t* perm, int64_t n_perm, int64_t stride, const int64_t* ctl, int32_t B,
                                              const float* labels_all, int32_t strategy, int32_t* rows_s, float* labels_s,
                                              int32_t* seg_lo_s, int32_t* seg_hi_s, float* weight_s, double* stats_s, void* stream) {
  return dae::batch_prepare_next("dae_batch_prepare_next_blocked", 1, perm, n_perm, stride, ctl, B, labels_all, strategy, rows_s,
                                 labels_s, seg_lo_s, seg_hi_s, weight_s, stats_s, stream);
}

extern "C" int dae_batch_commit(int32_t B, const int32_t* rows_s, const float* labels_s, const int32_t* seg_lo_s, const int32_t* seg_hi_s,
                                const float* weight_s, const double* stats_s, int32_t* rows, float* labels_b, int32_t* seg_lo,
                                int32_t* seg_hi, float* weight, double* stats, void* stream) {
  DAE_REQUIRE(B >= 1 && rows_s && labels_s && seg_lo_s && seg_hi_s && weight_s && stats_s && rows && labels_b && seg_lo && seg_hi && weight && stats,
              "dae_batch_commit: null pointer");
  dae::batch_commit_kernel<<<(B + 255) / 256, 256, 0, (cudaStream_t)stream>>>(B, rows_s, labels_s, seg_lo_s, seg_hi_s, weight_s, stats_s, rows,
                                                                           labels_b, seg_lo, seg_hi, weight, stats);
  DAE_CHECK_LAUNCH("dae_batch_commit");
  return DAE_OK;
}

extern "C" int dae_batch_prepare_explicit(const int32_t* perm, int64_t offset, const int64_t* ctl, int32_t B, int64_t n_each,
                                          int32_t* rows_out, double* stats, void* stream) {
  DAE_REQUIRE(B >= 1 && n_each >= 1 && rows_out && stats, "dae_batch_prepare_explicit: bad arguments");
  // the neg block's row ids r + 2 n_each (r < n_each) must fit in int32
  DAE_REQUIRE(n_each <= INT32_MAX / 3, "dae_batch_prepare_explicit: n_each = %lld rows per block: the row ids of [org; pos; neg] "
              "overflow int32 above %d", (long long)n_each, INT32_MAX / 3);
  dae::batch_rows_explicit_kernel<<<(B + 255) / 256, 256, 0, (cudaStream_t)stream>>>(perm, offset, ctl, B, n_each, rows_out, stats);
  DAE_CHECK_LAUNCH("dae_batch_prepare_explicit");
  return DAE_OK;
}
