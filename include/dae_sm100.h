/*
 * dae_sm100.h -- C ABI of libdae_sm100.so: the sm_90a (H100) kernels behind
 * DenoisingAutoencoder.fit / transform (DAE-with-triplet-loss training hot path).
 *
 * The reference (louislung/DAE_RNN_News_Recommendation) has NO FFI: its arithmetic is a
 * TensorFlow-1.12 graph run by `tf.Session.run` (autoencoder/autoencoder.py:233,241).  Each entry
 * point below replaces the TF ops cited next to it; INTEGRATION.md shows the ctypes stub a
 * maintainer of the reference would add.  All citations are relative to the reference root.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; sizes are element counts
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous on that stream
 *   - return value: 0 = ok, <0 = DAE_ERR_*; dae_last_error() gives the message (thread local)
 *   - the library owns no persistent device memory; the caller (Python/torch) owns every buffer
 *   - CSR: indptr int64[N+1], indices int32[nnz] (sorted inside a row), values float32[nnz]
 *   - parameters: ONE flat fp32 buffer theta = [ W (F x H row-major) | bh (H) | bv (F) ]
 *     gradients / optimizer slots use the same flat layout
 *   - activations: 0 = identity ('none'), 1 = sigmoid, 2 = tanh      (autoencoder.py:380-387,402-409)
 *   - losses: 0 = cross_entropy, 1 = mean_squared, 2 = cosine_proximity (triplet_loss_utils.py:268-273)
 *   - strategies: 0 = none, 1 = batch_all, 2 = batch_hard            (autoencoder.py:70)
 *   - optimizers: 0 = gradient_descent, 1 = ada_grad, 2 = momentum, 3 = adam (autoencoder.py:451-472)
 */
#ifndef DAE_SM100_H
#define DAE_SM100_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DAE_OK 0
#define DAE_ERR_BAD_ARG (-1)
#define DAE_ERR_CUDA (-2)
#define DAE_ERR_UNSUPPORTED (-3)

#define DAE_ACT_NONE 0
#define DAE_ACT_SIGMOID 1
#define DAE_ACT_TANH 2

#define DAE_LOSS_CE 0
#define DAE_LOSS_MSE 1
#define DAE_LOSS_COSINE 2

#define DAE_TRIPLET_NONE 0
#define DAE_TRIPLET_BATCH_ALL 1
#define DAE_TRIPLET_BATCH_HARD 2
/* largest batch of the batch_all / batch_hard strategies: S, G and G's bf16 hi/lo copy take ~13 GB at 32768 rows */
#define DAE_MAX_TRIPLET_BATCH 32768
/* Largest batch of a block-mined engine (dae_batch_prepare_blocked, dae_triplet_*_rows): the one-CTA sort and dZ's B x Fp x 4 bytes
 * bound it, not S -- the mining holds R anchor rows of S / G at a time. */
#define DAE_MAX_BLOCKED_BATCH 262144

#define DAE_OPT_SGD 0
#define DAE_OPT_ADAGRAD 1
#define DAE_OPT_MOMENTUM 2
#define DAE_OPT_ADAM 3

/* per-step scalar slots written by the kernels (float64 each), see dae_step_finalize */
#define DAE_STAT_COST 0
#define DAE_STAT_AE_LOSS 1
#define DAE_STAT_TRIPLET_LOSS 2
#define DAE_STAT_FRACTION 3
#define DAE_STAT_NUM 4
#define DAE_STAT_SUM_W 5
#define DAE_STAT_N_VALID 6
#define DAE_STAT_SUM_LW 7
#define DAE_STAT_TRIPLET_SUM 8
#define DAE_STAT_N_ACTIVE 9
#define DAE_STAT_SLOTS 16

int dae_version(void);
/* copies the calling thread's last error message into buf (NUL terminated); returns its length */
int dae_last_error(char* buf, size_t len);

/* ---- batching -------------------------------------------------------------------------------
 * Replaces utils.gen_batches' per-batch fancy indexing + get_sparse_ind_val_shape
 * (autoencoder/utils.py:53-66,162-180) and the label-only parts of batch_all
 * (triplet_loss_utils.py:47-76,110-111,129): takes rows perm[offset : offset+B] of the epoch's
 * permutation, orders them by label (the loss is invariant to the order of rows in a batch),
 * and emits for each batch row its dataset row id, label, class segment [seg_lo, seg_hi) and -
 * for batch_all - the closed-form data weight w_i and N_valid.  strategy none: order kept, w = 1.
 * One CTA.  Triplet strategies: B <= DAE_MAX_TRIPLET_BATCH; up to 4096 rows the batch is sorted in shared memory, above that
 * inside labels_out / rows_out (labels_out must then be non-NULL).  The order is ascending (label, row id) either way.
 * stats: float64[DAE_STAT_SLOTS], zeroed here, SUM_W / N_VALID filled.
 * ctl (optional, device int64[4]): per-step cursors kept in device memory so that a captured CUDA graph of the
 * step can be replayed without host-side argument changes -- ctl[0] is added to `offset`, ctl[1] is the row of the
 * stats log dae_step_finalize writes, ctl[2] the 1-based optimizer step; dae_step_advance moves all three.
 */
int dae_step_advance(int64_t* ctl, int64_t row_stride, void* stream);
int dae_batch_prepare(const int32_t* perm, int64_t offset, const int64_t* ctl, int32_t B, const float* labels_all,
                      int32_t strategy, int32_t* rows_out, float* labels_out, int32_t* seg_lo,
                      int32_t* seg_hi, float* weight_out, double* stats, void* stream);
/* The one-CTA sort is 20 us of pure latency, so a graph-replayed step prepares the NEXT batch (cursor ctl[0] + stride) on a side
 * branch into staging buffers (*_s) while the current step computes -- nothing is written when that batch would run past
 * n_perm -- and the next step starts with dae_batch_commit, a copy of the staged batch into the live buffers. */
int dae_batch_prepare_next(const int32_t* perm, int64_t n_perm, int64_t stride, const int64_t* ctl, int32_t B,
                           const float* labels_all, int32_t strategy, int32_t* rows_s, float* labels_s,
                           int32_t* seg_lo_s, int32_t* seg_hi_s, float* weight_s, double* stats_s, void* stream);
/* dae_batch_prepare / dae_batch_prepare_next with the cap DAE_MAX_BLOCKED_BATCH instead of DAE_MAX_TRIPLET_BATCH: same kernels, same
 * outputs.  For the engines that mine one block of anchor rows at a time (dae_triplet_batch_all_rows / _hard_rows). */
int dae_batch_prepare_blocked(const int32_t* perm, int64_t offset, const int64_t* ctl, int32_t B, const float* labels_all,
                              int32_t strategy, int32_t* rows_out, float* labels_out, int32_t* seg_lo,
                              int32_t* seg_hi, float* weight_out, double* stats, void* stream);
int dae_batch_prepare_next_blocked(const int32_t* perm, int64_t n_perm, int64_t stride, const int64_t* ctl, int32_t B,
                                   const float* labels_all, int32_t strategy, int32_t* rows_s, float* labels_s,
                                   int32_t* seg_lo_s, int32_t* seg_hi_s, float* weight_s, double* stats_s, void* stream);
int dae_batch_commit(int32_t B, const int32_t* rows_s, const float* labels_s, const int32_t* seg_lo_s,
                     const int32_t* seg_hi_s, const float* weight_s, const double* stats_s, int32_t* rows,
                     float* labels_b, int32_t* seg_lo, int32_t* seg_hi, float* weight, double* stats, void* stream);
/* explicit (org, pos, neg) triplets (autoencoder/utils.py:73-91, autoencoder_triplet.py:106-147): rows_out[3B] = the batch's
 * rows in the three blocks of the stacked [org; pos; neg] matrix (n_each rows per block); stats zeroed, SUM_W = B. */
int dae_batch_prepare_explicit(const int32_t* perm, int64_t offset, const int64_t* ctl, int32_t B, int64_t n_each,
                               int32_t* rows_out, double* stats, void* stream);

/* ---- K1: CSR x dense encode ---------------------------------------------------------------------
 * E[r,:] = f( in_scale * X[rows[r],:] . W + bh ) - f(bh)      (autoencoder.py:377,389; transform :494-497;
 * in_scale folds utils.decay_noise, utils.py:147-159).  rows == NULL means rows[r] = r.
 * E is written fp32 with leading dimension ldE.  Entries whose value is exactly 0 (masked) are skipped.
 * col_count (optional, int32[F]): zeroed, then receives the number of kept entries per feature column of the batch --
 * the bucket sizes dae_encode_csr_bwd_gather needs.
 * e_hi / e_lo (optional, bf16 [n_rows x ld_split]): columns [0, H) of the bf16 hi/lo operand copy of E for the tensor-core
 * GEMMs (the caller keeps the padding columns zero and the all-ones column set).
 */
int dae_encode_csr_fwd(const int64_t* indptr, const int32_t* indices, const float* values,
                       const int32_t* rows, int32_t n_rows, int32_t F, int32_t H, float in_scale,
                       const float* W, const float* bh, int32_t enc_act, float* E, int64_t ldE,
                       int32_t* col_count, void* e_hi, void* e_lo, int64_t ld_split, void* stream);

/* ---- K5: encode backward -------------------------------------------------------------------------
 * dA = dE * f'(A);  dbh = sum_i dA_i - f'(bh) * sum_i dE_i;  dW[c,:] += v * dA[r,:] for every stored
 * (r,c,v) of the corrupted batch (autodiff of autoencoder.py:389).  dE is overwritten with dA.
 * dW is accumulated with fp32 atomics on top of whatever the decode backward wrote.
 * dE_add (optional, same layout as dE): a second contribution to dL/dE, added before f' is applied -- the triplet term
 * alpha (G + G^T) E, computed on the mining branch of the step, meets the decode term here instead of in a GEMM of its own.
 * dbh_zeroed != 0: the caller has already zeroed dbh (it zeroes the whole flat gradient buffer), skip the memset node.
 */
int dae_encode_csr_bwd(const int64_t* indptr, const int32_t* indices, const float* values,
                       const int32_t* rows, int32_t n_rows, int32_t F, int32_t H, float in_scale,
                       const float* E, const float* bh, int32_t enc_act, float* dE, const float* dE_add,
                       int64_t ldE, float* dW, float* dbh, int32_t dbh_zeroed, void* stream);

/* Same result with ~6x fewer atomics on dW: the batch's kept entries are bucketed by feature column (col_count from the
 * forward call; col_start int32[F+1], col_cursor int32[F], ent_col/ent_row int32[cap], ent_val f32[cap] are
 * caller-provided scratch, cap >= kept entries of the batch); CTAs then walk fixed-size chunks of the bucketed entry
 * list, accumulate v * dA[r,:] in registers per column run and issue one vector red.global.add per (chunk, column) run.
 * Supports H <= 1024 (H % 4 == 0) / 512 (H % 2 == 0) / 256; larger H: use dae_encode_csr_bwd.
 */
/* exclusive scan of the per-column counts into col_start[F+1] / col_cursor[F]; dae_encode_csr_bwd_gather runs it itself unless
 * it is called with col_count == NULL (then the scan must already have been issued, e.g. on a parallel stream) */
int dae_col_scan(const int32_t* col_count, int32_t F, int32_t* col_start, int32_t* col_cursor, void* stream);
int dae_encode_csr_bwd_gather(const int64_t* indptr, const int32_t* indices, const float* values,
                              const int32_t* rows, int32_t n_rows, int32_t F, int32_t H, float in_scale,
                              const float* E, const float* bh, int32_t enc_act, float* dE, const float* dE_add,
                              int64_t ldE, float* dW, float* dbh, int32_t dbh_zeroed, const int32_t* col_count,
                              int32_t* col_start, int32_t* col_cursor, int32_t* ent_col, int32_t* ent_row,
                              float* ent_val, void* stream);

/* transform-sized K1 (many rows, one launch): persistent CTAs stage the K most frequent rows of W (hot_cols[K], 2 kB each at
 * H = 500) in shared memory with 1-D bulk-TMA copies and serve the entries of those columns from there; the cold tail gathers from
 * L2 as in dae_encode_csr_fwd.  hot_slot[F] = index of the column in hot_cols, or -1.  K * H * 4 <= 200 KB, H % 4 == 0.
 * groups = 4 or 8 row groups of 128 threads per CTA; the number of CTAs per SM follows from the size of the staged set.
 * Same results as dae_encode_csr_fwd up to fp32 summation order inside a row (identical: entries are added in CSR order). */
int dae_encode_csr_fwd_hot(const int64_t* indptr, const int32_t* indices, const float* values, int32_t n_rows,
                           int32_t F, int32_t H, float in_scale, const float* W, const float* bh, int32_t enc_act,
                           float* E, int64_t ldE, const int32_t* hot_cols, const int32_t* hot_slot, int32_t K,
                           int32_t groups, void* stream);

/* ---- fp32 reference GEMM (CUDA cores) ----------------------------------------------------------
 * C[m,n] = alpha * sum_k A[m*sam + k*sak] * B[n*sbn + k*sbk] + beta * C[m,n]; generic strides.
 * The v1 / validation path for the dense contractions (autoencoder.py:411 and its autodiff,
 * triplet_loss_utils.py:93,219); the production path is dae_gemm_bf16x3 / dae_decode_fused_bf16x3.
 */
int dae_sgemm(int32_t M, int32_t N, int32_t K, float alpha, const float* A, int64_t sam, int64_t sak,
              const float* B, int64_t sbn, int64_t sbk, float beta, float* C, int64_t ldc, void* stream);

/* ---- tensor-core (wgmma) path for the dense contractions (K2/K3, Gram matrix) ---------------------
 * fp32-accurate GEMM on the Hopper tensor cores: each fp32 operand is carried as bf16 hi + bf16 lo
 * (dae_split_bf16) and D = A_hi.B_hi + A_lo.B_hi + A_hi.B_lo is accumulated in fp32 registers.
 * TMA-fed (128B swizzle), persistent, warp specialised; operands are read K-major or MN-major straight
 * from row-major arrays (majorness flags), so dZ^T / E^T / W^T are never materialised.
 *
 * dae_split_bf16: hi/lo [rows x ld_dst] <- src [rows x cols] * scale, zero padded; column `ones_col`
 *   (if >= 0) is set to 1.0 -- the [E | 1] trick that makes dW = dZ^T.[E | 1] also deliver dbv.
 * dae_sym_split_bf16: hi/lo <- alpha * (G + G^T)   (dE_tri = alpha (G + G^T) E).
 * dae_gemm_bf16x3: C[m,n] (+)= alpha * sum_k A(m,k) B(n,k).
 *   a_mn_major = 0: A stored [M x lda] (K contiguous); 1: A stored [K x lda] (M contiguous).  Same for B/N.
 *   columns n < n_store go to C; column special_col (if special_out != NULL) goes to special_out[m].
 *   k_splits > 1 (uniform split-K), k_splits < 0 (stream-K: the tile x k-block units are shared evenly by the SMs, chosen
 *   automatically when the 128x128 tiling does not fill whole waves) or accumulate != 0: fp32 atomics into C (C is zeroed
 *   first unless accumulate).
 * dae_decode_fused_bf16x3: Z = E.W^T with the decode-loss epilogue fused (D = g(Z+bv), CE/MSE row loss
 *   against the clean CSR rows, dZ written directly as bf16 hi/lo [B x ld_dz]); row_loss_part is the
 *   [B] row-loss vector (zeroed here, accumulated with fp32 atomics, one add per half tile).  Replaces autoencoder.py:411 +
 *   triplet_loss_utils.py:262-275 and their autodiff without materialising Z, D or dense X.
  *   tile_ptr is int32 scratch [Brows x (2*ceil(F/128) + 1)] (per-row CSR offsets of every 64-column part, filled here).
 */
int dae_split_bf16(const float* src, int32_t rows, int32_t cols, int64_t ld_src, void* hi, void* lo,
                   int64_t ld_dst, int32_t ones_col, float scale, void* stream);
int dae_sym_split_bf16(const float* G, int32_t B, int64_t ldg, float alpha, void* hi, void* lo, int64_t ld,
                       void* stream);
int dae_gemm_bf16x3(int32_t M, int32_t N, int32_t K, float alpha, const void* a_hi, const void* a_lo,
                    int64_t lda, int32_t a_mn_major, const void* b_hi, const void* b_lo, int64_t ldb,
                    int32_t b_mn_major, float* C, int64_t ldc, int32_t n_store, int32_t special_col,
                    float* special_out, int32_t k_splits, int32_t accumulate, void* stream);
/* C[m,n] (+)= alpha * sum_k (G[m,k] + G[k,m]) * B[k,n] for a square G [M x M] (bf16 hi/lo, row-major) and B stored [M x ldb] row-major:
 * dE2 = alpha (G + G^T) E of the triplet backward in ONE launch -- the k loop runs over G's columns and then over G's rows (the same
 * array through an M-contiguous tensor map), so G + G^T is never formed.  Stream-K with fp32 atomics; C is zeroed first unless accumulate. */
int dae_gemm_sym_bf16x3(int32_t M, int32_t N, float alpha, const void* g_hi, const void* g_lo, int64_t ldg,
                        const void* b_hi, const void* b_lo, int64_t ldb, float* C, int64_t ldc, int32_t accumulate,
                        void* stream);
/* Tile engine selection of dae_gemm_bf16x3 (test hook).  pair_mode: 1 = CTA pairs (a two-CTA cluster works on two
 * adjacent 128-row tiles and each CTA multicasts half of the shared B tile into both) whenever possible (not the fused decode);
 * -1 (default) or 0 = never (slower on the H100 at the BASELINE shapes).  lean: 0 (default) = 128x128 / 128x64 tiles chosen by shape;
 * 1 = dae_gemm_bf16x3 on 128x64 tiles with 2-stage rings (~130 KB of shared memory per CTA). */
int dae_gemm_config(int32_t pair_mode, int32_t lean);
/* The part of the fused decode that needs only the batch's row ids: zero row_loss_part and fill tile_ptr.  dae_decode_fused_bf16x3
 * runs it in line unless it is called with prepared != 0 (a graph-replayed step issues it on a parallel branch, next to K1). */
int dae_decode_prepare(int32_t Brows, int32_t F, const int64_t* indptr, const int32_t* indices, const int32_t* rows,
                       float* row_loss_part, int32_t* tile_ptr, void* stream);
int dae_decode_fused_bf16x3(int32_t Brows, int32_t F, int32_t K, const void* e_hi, const void* e_lo,
                            int64_t lde, const void* w_hi, const void* w_lo, int64_t ldw,
                            const int64_t* indptr, const int32_t* indices, const float* values,
                            const int32_t* rows, const float* bv, int32_t dec_act, int32_t loss_func,
                            const float* weight, const double* stats, void* dz_hi, void* dz_lo,
                            int64_t ld_dz, float* row_loss_part, int32_t* tile_ptr, int32_t prepared, void* stream);
/* out[i] = sum_p parts[p * n + i] (deterministic reduction of the per-tile row-loss partials) */
int dae_reduce_parts(const float* parts, int32_t n_parts, int32_t n, float* out, void* stream);

/* ---- decode loss + dZ (elementwise part of K2) ------------------------------------------------------
 * In place on Z (B x F, leading dim ldz), where Z = E.W^T (no bias yet):
 *   D = g(Z + bv); row loss l_i per triplet_loss_utils.py:268-273 against the CLEAN batch rows (CSR,
 *   densified on the fly); dZ = (w_i / (sum_w + 1e-16)) * dl_i/dD * g'(Z)   (autodiff of :269-275, :411)
 * Z is overwritten with dZ; row_loss[B] receives l_i.  weight == NULL means w = 1 (strategy none);
 * sum_w is read from stats[DAE_STAT_SUM_W].
 */
int dae_decode_loss_bwd(const int64_t* indptr, const int32_t* indices, const float* values,
                        const int32_t* rows, int32_t n_rows, int32_t F, const float* bv, int32_t dec_act,
                        int32_t loss_func, const float* weight, const double* stats, float* Z, int64_t ldz,
                        float* row_loss, void* stream);

/* column sums: out[f] = sum_r M[r*ld + f]  (dbv = sum_i dZ_i) */
int dae_colsum(const float* M, int32_t n_rows, int32_t n_cols, int64_t ld, float* out, void* stream);

/* ---- K4: triplet mining -------------------------------------------------------------------------
 * batch_all (triplet_loss_utils.py:79-131, pos_triplets_only=False as called at autoencoder.py:430):
 *   rows must be label sorted (dae_batch_prepare). S = E.E^T is an input (B x B, ld lds).
 *   Writes G (B x B): dL_tri/dS, accumulates loss sum / positive count into stats.
 *   pos_only != 0 (pos_triplets_only=True, :118-120; never used by the model): the loss sum covers positive triplets
 *   only and G receives raw COUNTS of positive triplets (G[i,j] = -#k, G[i,k] = +#j) from which the caller derives the weights.
 *   g_hi / g_lo (optional, bf16 [B x ld_split]): G also leaves as the hi / lo operand pair dae_gemm_sym_bf16x3 reads.
 *   B <= DAE_MAX_TRIPLET_BATCH.  Up to 4096 rows one CTA per anchor keeps the whole row in shared memory (~52 B bytes); above,
 *   a tiled sweep streams the anchor's positives / negatives through fixed-size chunks (47 KB of shared memory at any B).
 * batch_hard (triplet_loss_utils.py:202-259): also writes the data weight (w) and sum_w.
 */
int dae_triplet_batch_all(const float* S, int64_t lds, int32_t B, const int32_t* seg_lo, const int32_t* seg_hi,
                          float* G, int64_t ldg, double* stats, int32_t pos_only, void* g_hi, void* g_lo,
                          int64_t ld_split, void* stream);
/* Sweep selection of dae_triplet_batch_all (test hook): force_tiled != 0 runs the tiled sweep at every B; 0 (default) only above
 * 4096 rows. */
int dae_triplet_config(int32_t force_tiled);
int dae_triplet_batch_hard(const float* S, int64_t lds, int32_t B, const float* labels, float* G, int64_t ldg,
                           float* weight, double* stats, void* stream);
/* Block mining (batches up to DAE_MAX_BLOCKED_BATCH without any B x B buffer): the anchors row0 .. row0 + n_rows - 1 of a batch of B
 * rows.  Row r of S_blk / G_blk (and of g_hi / g_lo) belongs to anchor row0 + r; segments and labels are indexed by the anchor.
 * dae_triplet_batch_all_rows: the tiled sweep of dae_triplet_batch_all on those anchors (same chunks, order and fp64 flushes, so
 *   the same G rows bit for bit as the tiled sweep on the whole matrix).
 * dae_triplet_batch_hard_rows: the per-row batch_hard of dae_triplet_batch_hard on those anchors.  G_blk is written UNSCALED (the
 *   1/(sum c + eps) factor is known only after the last block) and `weight` is accumulated, not cleared: zero it once per batch.
 * dae_triplet_batch_hard_finish, after the last block: stats[SUM_W] = sum of weight, and dE2 [B x H, ld] *= 1/(N_ACTIVE + eps)
 *   (dE2 == NULL: forward only). */
int dae_triplet_batch_all_rows(const float* S_blk, int64_t lds, int32_t row0, int32_t n_rows, int32_t B, const int32_t* seg_lo,
                               const int32_t* seg_hi, float* G_blk, int64_t ldg, double* stats, int32_t pos_only, void* g_hi,
                               void* g_lo, int64_t ld_split, void* stream);
int dae_triplet_batch_hard_rows(const float* S_blk, int64_t lds, int32_t row0, int32_t n_rows, int32_t B, const float* labels,
                                float* G_blk, int64_t ldg, float* weight, double* stats, void* stream);
int dae_triplet_batch_hard_finish(const float* weight, int32_t B, double* stats, float* dE2, int32_t H, int64_t ld, void* stream);
/* explicit triplets (autoencoder_triplet.py:308-311): loss = mean softplus(e.en - e.ep); ACCUMULATES alpha * dloss
 * into dE/dEp/dEn (on top of the reconstruction gradient) and the loss sum into stats[DAE_STAT_TRIPLET_SUM]. */
int dae_triplet_explicit(const float* E, const float* Ep, const float* En, int32_t B, int32_t H, int64_t ld,
                         float alpha, float* dE, float* dEp, float* dEn, double* stats, void* stream);

/* ---- step epilogue ---------------------------------------------------------------------------------
 * Reduces row_loss -- or, if parts != NULL, the [n_parts x B] per-tile partials of dae_decode_fused_bf16x3 -- (x weight)
 * deterministically and fills COST / AE_LOSS / TRIPLET_LOSS / FRACTION / NUM
 * of `stats` (autoencoder.py:438,441; triplet_loss_utils.py:127,131,257,259,275); then copies the
 * DAE_STAT_SLOTS doubles to stats_log (one row of the per-epoch log) if non-NULL.
 */
int dae_step_finalize(const float* row_loss, const float* parts, int32_t n_parts, const float* weight, int32_t B,
                      int32_t strategy, float alpha, double* stats, double* stats_log, const int64_t* ctl, void* stream);

/* ---- K6: optimizer ------------------------------------------------------------------------------------
 * theta <- update(theta, grad * grad_scale) over the flat buffer (autoencoder.py:451-472; TF-1.12 rules:
 * SGD; Adagrad accum(0)=0.1, no eps; Momentum accum=mu*accum+g, theta-=lr*accum; Adam b1 .9 b2 .999 eps 1e-8
 * with lr_t = lr*sqrt(1-b2^t)/(1-b1^t), t = step (1-based)).
 * If w_hi/w_lo are non-NULL the updated W (first F*H entries) is also written as the bf16 hi/lo pair [F x ld_split]
 * consumed by the tensor-core GEMMs (fuses dae_split_bf16 of W into the update).
 */
int dae_optimizer_step(float* theta, const float* grad, float* slot1, float* slot2, int64_t n, int32_t opt,
                       float lr, float momentum, float grad_scale, int32_t step, const int64_t* ctl, void* w_hi,
                       void* w_lo, int32_t F, int32_t H, int64_t ld_split, void* stream);

/* ---- corruption -----------------------------------------------------------------------------------------
 * values_out[p] = keep[p] ? values[p] : 0 where keep is a host-generated byte mask (bit-parity mode with
 * np.random.rand(nnz) >= v, utils.py:111) -- or, if keep == NULL, a Philox4x32-10 draw keyed by
 * (seed, epoch, p):  u >= corr_frac  (device mode; same distribution, different stream).
 */
int dae_mask_values(const float* values, const uint8_t* keep, int64_t nnz, float corr_frac, uint64_t seed,
                    uint64_t epoch, float* values_out, void* stream);

/* Salt-and-pepper noise (utils.salt_and_pepper_noise, utils.py:118-144) of the clean CSR rows [row0, row0 + n), appended to an
 * output CSR.  Row r draws v columns with replacement; draw j sets its column to hi (coin 1) or lo (coin 0), the last draw of a
 * column decides, a column that ends at 0 is not stored, and untouched entries keep their clean value (explicit zeros too).  The
 * input must be canonical (sorted, unique columns per row); so is the output.
 *   draws == NULL: Philox4x32-10, key (seed lo, seed hi), counter (j / 2, r, epoch lo, epoch hi) with r the GLOBAL row; an even j
 *     takes the output words (c0, c1), an odd j (c2, c3): column = floor(c_a * F / 2^32), coin = (c_b >= 2^31).
 *   draws != NULL: n * v host draws (row-major), column | coin << 31 (utils.salt_and_pepper_draws: the reference's stream).
 * The call writes indptr_out[row0 + 1 .. row0 + n], starting from indptr_out[row0] as the device holds it when the call runs (0 for
 * the first call, or what the previous call on the stream wrote), so calls over consecutive row ranges form one stacked CSR.  If the
 * total would exceed cap, no entry is written, rows row0 .. row0 + n - 1 are left empty and *overflow is set to 1 (never cleared).
 * Sizes: F in [1, 2^30), v in [0, 2^30).  ws: dae_salt_pepper_workspace(n) bytes, reused by every call on the stream.
 */
int dae_salt_pepper_csr(const int64_t* indptr, const int32_t* indices, const float* values, int64_t row0, int64_t n, int32_t F,
                        int64_t v, float lo, float hi, const uint32_t* draws, uint64_t seed, uint64_t epoch, int64_t* indptr_out,
                        int32_t* indices_out, float* values_out, int64_t cap, int32_t* overflow, void* ws, size_t ws_bytes,
                        void* stream);
int dae_salt_pepper_workspace(int64_t n, size_t* bytes);

/* ---- "next" row (SURVEY 8f rank 1): pairwise similarity of embeddings + nearest-article lookup -----------------
 * Replaces helpers.pairwise_similarity (helpers.py:11-50: sklearn cosine_similarity / linear_kernel, optional normalize,
 * zeroed diagonal) and the nanargmax lookup of main_autoencoder.py:352-353.  sim = normalize(E).normalize(E)^T runs on
 * dae_gemm_bf16x3; these are the two kernels around it.
 * dae_rownorm_split_bf16: rows scaled by 1/||x||_2 (norm_kind 2), 1/||x||_1 (1), 1/max|x| (3) or 1 (0), written as bf16 hi/lo
 *   [rows x ld_dst] (columns [cols, ld_dst) = 0) and/or as fp32 x_out.  A row whose fp32 norm is 0 (all zeros, or a squared norm
 *   that underflows) is left untouched, like sklearn; a row whose norm overflows fp32 (for l2: max |x| above ~1.8e19) comes out
 *   as zeros.
 * dae_row_argmax: per row the arg-max / max of S over the non-NaN entries, skipping column row + diag_offset (optionally zeroing
 *   it in place).  The first maximum wins (np.argmax); the skipped diagonal never wins, even when every other entry is negative.
 *   A row without a candidate (cols = 1 with the diagonal, or every other entry NaN) gets index -1 and value -inf.
 */
int dae_rownorm_split_bf16(const float* X, int32_t rows, int32_t cols, int64_t ld, int32_t norm_kind, void* hi, void* lo,
                           int64_t ld_dst, float* x_out, int64_t ld_out, void* stream);
int dae_row_argmax(float* S, int32_t rows, int32_t cols, int64_t ld, int64_t diag_offset, int32_t zero_diag,
                   int32_t* idx_out, float* val_out, void* stream);

/* ---- k most similar articles without the similarity matrix ---------------------------------------------------------
 * dae_similarity_topk_bf16x3: S = Q.C^T (Q [n_query x dim], C [n_corpus x dim], both as bf16 hi/lo pairs with row strides ldq /
 *   ldc, e.g. from dae_rownorm_split_bf16) on the tensor cores, bf16x3 as dae_gemm_bf16x3, with a k-best selection fused into the
 *   epilogue: S never leaves the SM.  Row i of idx_out / val_out [n_query x k] (int32 / fp32, row stride k) lists the k corpus
 *   rows of highest score in strictly decreasing (score, -index) order -- among equal scores the lower index first, the rule of
 *   dae_row_argmax -- padded with -1 / -inf when a row has fewer than k candidates.  exclude != 0: column i + diag_offset is not
 *   a candidate of row i (the self match when Q is C or a row window of it).  1 <= k <= 32; ldq, ldc >= dim and multiples of 8;
 *   operands 16-byte aligned.  Each CTA sweeps a contiguous range of column tiles of a 128-row block; `splits` (> 0) sets the
 *   number of ranges, 0 picks the fewest that fill the SMs.  The scores do not depend on it (no split over dim), so neither
 *   does the output.  workspace: at least dae_similarity_topk_workspace bytes (same n_query, n_corpus, k, splits), 16-byte aligned.
 * dae_similarity_topk_workspace: *bytes = the workspace size of that call (2 * splits partial lists of k per query row).
 */
int dae_similarity_topk_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo,
                               int64_t ldq, const void* c_hi, const void* c_lo, int64_t ldc, int32_t k,
                               int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace,
                               int64_t workspace_bytes, int32_t* idx_out, float* val_out, void* stream);
int dae_similarity_topk_workspace(int32_t n_query, int32_t n_corpus, int32_t k, int32_t splits, int64_t* bytes);

/* ---- k most similar articles of sparse (bag-of-words) vectors ------------------------------------------------------
 * dae_csr_similarity_topk: the same selection as dae_similarity_topk_bf16x3 for S[q, c] = sum_f Q[q, f] C[c, f] of two CSR
 *   matrices (indptr int64, indices int32 sorted inside a row, values fp32; q_features == c_features), on the CUDA cores and
 *   without forming S.  Every corpus row is a candidate, a row sharing no column with q included (score 0), except column
 *   q + diag_offset when `exclude` is set; order (score desc, index asc); padding -1 / -inf.  Each score accumulates in fp32 from
 *   0, one term per shared column in increasing column order, each term the product rounded to fp32 and then added (no FMA), so
 *   the output does not depend on `splits` (> 0: the number of corpus parts, 0: automatic) and a float32 host loop over the
 *   columns reproduces it exactly.  1 <= k <= 32; corpus nnz < 2^31; workspace 16-byte aligned, at least
 *   dae_csr_similarity_topk_workspace bytes for the same n_query, n_corpus, c_nnz, features, k and splits.
 * dae_csr_similarity_topk_workspace: *bytes = that workspace: the corpus postings (8 B per entry), their bucket offsets
 *   ((n_corpus / 2048 + 1) x features int32) and, when the corpus is split, the partial lists (8 B per entry).
 */
int dae_csr_similarity_topk(const int64_t* q_indptr, const int32_t* q_indices, const float* q_values, int32_t n_query,
                            int64_t q_nnz, int32_t q_features, const int64_t* c_indptr, const int32_t* c_indices,
                            const float* c_values, int32_t n_corpus, int64_t c_nnz, int32_t c_features, int32_t k,
                            int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace, int64_t workspace_bytes,
                            int32_t* idx_out, float* val_out, void* stream);
int dae_csr_similarity_topk_workspace(int32_t n_query, int32_t n_corpus, int64_t corpus_nnz, int32_t n_features, int32_t k,
                                      int32_t splits, int64_t* bytes);

/* ---- k best unread articles: top-k with per-query exclusion lists ---------------------------------------------------
 * dae_similarity_topk_excl_bf16x3 / dae_csr_similarity_topk_excl: dae_similarity_topk_bf16x3 / dae_csr_similarity_topk with the
 *   same arguments, workspace (the same size queries) and contract, plus an exclusion list per query row: the device CSR structure
 *   ex_indptr int64 [n_query + 1], ex_indices int32 [ex_nnz] (no values).  Row i lists the corpus rows that are never candidates of
 *   query i (e.g. the articles a user has read).  The caller guarantees ex_indptr[0] = 0, ex_indptr[n_query] = ex_nnz, and every
 *   row sorted, without duplicates, inside [0, n_corpus): the kernels do not check the list contents.  `exclude` / diag_offset
 *   still leave out column i + diag_offset as well.  Order (score desc, index asc), padding -1 / -inf when fewer than k
 *   candidates remain, independent of `splits`; with every list empty the output equals the plain call's bit for bit.
 *   ex_indptr 8-byte and ex_indices 4-byte aligned; ex_indices may be NULL when ex_nnz = 0.
 */
int dae_similarity_topk_excl_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo,
                                    int64_t ldq, const void* c_hi, const void* c_lo, int64_t ldc, int32_t k,
                                    int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace,
                                    int64_t workspace_bytes, int32_t* idx_out, float* val_out, const int64_t* ex_indptr,
                                    const int32_t* ex_indices, int64_t ex_nnz, void* stream);
int dae_csr_similarity_topk_excl(const int64_t* q_indptr, const int32_t* q_indices, const float* q_values, int32_t n_query,
                                 int64_t q_nnz, int32_t q_features, const int64_t* c_indptr, const int32_t* c_indices,
                                 const float* c_values, int32_t n_corpus, int64_t c_nnz, int32_t c_features, int32_t k,
                                 int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace, int64_t workspace_bytes,
                                 int32_t* idx_out, float* val_out, const int64_t* ex_indptr, const int32_t* ex_indices,
                                 int64_t ex_nnz, void* stream);

/* ---- at most one article per story: top-k over near-duplicate groups ------------------------------------------------
 * dae_similarity_topk_groups_bf16x3 / dae_csr_similarity_topk_groups: the *_excl exports with the same arguments, workspace (the
 *   plain *_workspace queries) and exclusion lists, plus groups int32 [n_corpus]: one label >= 0 per corpus row, rows with equal
 *   labels forming one group (helpers.duplicate_groups' output fits as is).  For each query row the candidates are those of the
 *   *_excl call; each group is represented by its candidate that comes first by (score desc, index asc), and the k best
 *   representatives are returned in that order, padded with -1 / -inf.  Scores are the plain calls' bits; the result does not
 *   depend on `splits`.  ex_indptr may be NULL (no lists; ex_nnz must then be 0).  groups 4-byte aligned.  The kernels do not
 *   check the label values: the caller guarantees 0 <= groups[c].  With groups[c] = c the output equals the *_excl call's bit for
 *   bit (the plain call's without lists).
 */
int dae_similarity_topk_groups_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo,
                                      int64_t ldq, const void* c_hi, const void* c_lo, int64_t ldc, int32_t k,
                                      int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace,
                                      int64_t workspace_bytes, int32_t* idx_out, float* val_out, const int64_t* ex_indptr,
                                      const int32_t* ex_indices, int64_t ex_nnz, const int32_t* groups, void* stream);
int dae_csr_similarity_topk_groups(const int64_t* q_indptr, const int32_t* q_indices, const float* q_values, int32_t n_query,
                                   int64_t q_nnz, int32_t q_features, const int64_t* c_indptr, const int32_t* c_indices,
                                   const float* c_values, int32_t n_corpus, int64_t c_nnz, int32_t c_features, int32_t k,
                                   int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace, int64_t workspace_bytes,
                                   int32_t* idx_out, float* val_out, const int64_t* ex_indptr, const int32_t* ex_indices,
                                   int64_t ex_nnz, const int32_t* groups, void* stream);

/* ---- "next" row (SURVEY 8f rank 2): related-vs-unrelated AUROC of a pairwise similarity matrix ---------------------
 * Replaces the numeric part of helpers.visualize_pairwise_similarity (helpers.py:88-100).
 * dae_pair_partition: for every pair i > j of the strict lower triangle with labels[i] >= 0 and labels[j] >= 0
 *   (-1 = missing, helpers.py:91) append S[i, j] to `related` if labels[i] == labels[j] (helpers.py:92-95) else to
 *   `unrelated` (helpers.py:96-97).  cursors[0..1] are device counters the caller zeroes; on return they hold the
 *   group sizes.  Order inside a group is unspecified.  Capacity: R = sum_c n_c(n_c-1)/2, U = M(M-1)/2 - R floats.
 * dae_auroc_count: *twice_u += sum_q 2*#{t < q} + #{t == q} (query_is_positive = 1: queries are the related scores,
 *   sorted_targets the ascending unrelated scores) or sum_q 2*#{t > q} + #{t == q} (0: roles swapped).  Then
 *   AUROC = twice_u / (2 R U) -- the area sklearn's roc_curve + auc (helpers.py:99-100) return, ties included.
 */
int dae_pair_partition(const float* S, int64_t lds, int32_t n, const int32_t* labels, float* related, float* unrelated,
                       uint64_t* cursors, void* stream);
int dae_auroc_count(const float* queries, int64_t n_queries, const float* sorted_targets, int64_t n_targets,
                    int32_t query_is_positive, uint64_t* twice_u, void* stream);

/* ---- related-vs-unrelated AUROC without the similarity matrix: pair histograms ------------------------------------
 * The same pairs as dae_pair_partition -- S[i, j] with i > j (i the row / first operand), both labels >= 0; related when the
 * labels are equal -- of a set against itself, counted on a grid instead of sorted, so that memory stays O(bins) at any n.
 * Grid: `bins` bins (a power of two, 2^10 .. 2^24) over [-M, M] (`range` = M, a power of two in [2^-64, 2^64]; 1 for cosine, for
 *   the linear kernel the smallest power of two >= (1 - 1e-6) max_i ||x_i||^2).  A score s goes to bin
 *   b = clamp(floor(fl32(s + M) * bins / (2M)), 0, bins - 1): bins / (2M) is a power of two, so the only rounding is the fp32
 *   add and a float32 host expression gives the same bin.  The map is monotone in s; scores outside [-M, M] land in the end bins.
 * Output, ACCUMULATED into caller-zeroed buffers: hist uint64 [2 x bins] (row 0 related, row 1 unrelated: exact counts, so
 *   independent of atomic order and launch shape) and sums fp64 [2] (the fp32 scores of each group summed in fp64, for the mean).
 *   The AUROC on the grid, twice_u = sum_b n_r[b] (2 sum_{b' < b} n_u[b'] + n_u[b]), differs from the exact AUROC of the same
 *   fp32 scores by at most sum_b n_r[b] n_u[b] / (2 R U); helpers.auroc_from_histograms computes both on the host.
 * Every argument is checked before any CUDA call; n >= 2.
 * dae_similarity_pair_hist_bf16x3: S = X.X^T of dense rows (bf16 hi / lo pair [n x ldx], ldx >= dim and a multiple of 8, 16-byte
 *   aligned, e.g. from dae_rownorm_split_bf16) on the tensor cores, bf16x3 as dae_similarity_topk_bf16x3; only the tiles on and
 *   below the diagonal are computed and S never leaves the SM.
 * dae_csr_similarity_pair_hist: S of one CSR matrix (the layout of dae_csr_similarity_topk, nnz < 2^31) with the scores of
 *   dae_csr_similarity_topk, bit for bit: fp32 from 0, one rounded product per shared column in increasing column order, no FMA.
 *   workspace: 16-byte aligned, at least dae_csr_similarity_pair_hist_workspace bytes (the postings and their bucket offsets).
 */
int dae_similarity_pair_hist_bf16x3(int32_t n, int32_t dim, const void* x_hi, const void* x_lo, int64_t ldx,
                                    const int32_t* labels, float range, int32_t bins, uint64_t* hist, double* sums,
                                    void* stream);
int dae_csr_similarity_pair_hist(const int64_t* indptr, const int32_t* indices, const float* values, int32_t n, int64_t nnz,
                                 int32_t n_features, const int32_t* labels, float range, int32_t bins, void* workspace,
                                 int64_t workspace_bytes, uint64_t* hist, double* sums, void* stream);
int dae_csr_similarity_pair_hist_workspace(int32_t n, int64_t nnz, int32_t n_features, int64_t* bytes);

/* ---- near-duplicate articles: every pair at or above a similarity threshold, without the similarity matrix --------
 * Pairs: self mode (self != 0, the corpus arguments are the query arguments: same pointers and sizes) lists the pairs (i, j) with
 *   i > j and S[i, j] >= threshold, where S[i, j] is computed with i as the query (first operand) row -- the convention of
 *   dae_similarity_pair_hist_bf16x3; S[j, i] is not evaluated and need not have the same bits.  Corpus mode (self = 0) lists every
 *   (i, j), i < n_query, j < n_corpus, with S[i, j] >= threshold.
 * Threshold: compared as s >= threshold in fp32 (the caller converts it to float once); a NaN score never qualifies.
 * Output: *count, a uint64 the caller zeroes, is ACCUMULATED by the exact number of qualifying pairs.  The first `capacity` of them
 *   (in unspecified order: atomic slot reservation) are written as i_out[s], j_out[s] (int32) and s_out[s] (fp32, the score) for
 *   s < capacity; nothing is written at or past capacity, so a count above capacity means the call must be repeated with at
 *   least count slots (and a zeroed counter).  capacity = 0 only counts (the outputs may then be null).
 * Every argument is checked before any CUDA call.
 * dae_similarity_pairs_bf16x3: dense rows as bf16 hi / lo pairs (as dae_similarity_topk_bf16x3: ldq, ldc >= dim and multiples of
 *   8, operands 16-byte aligned); the tiles, operand ring and k16 order of dae_similarity_topk_bf16x3, so each score has the bits
 *   top-k reports for the same (i, j).  Self mode computes only the tiles on and below the diagonal.  threshold finite.
 * dae_csr_similarity_pairs: CSR rows (the layout of dae_csr_similarity_topk, corpus nnz < 2^31) with its scores, bit for bit:
 *   fp32 from 0, one rounded product per shared column in increasing column order, no FMA.  threshold finite and > 0: a pair
 *   sharing no column scores exactly 0 and is never listed.  workspace: 16-byte aligned, at least
 *   dae_csr_similarity_pairs_workspace bytes (the corpus postings and their bucket offsets).
 */
int dae_similarity_pairs_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo, int64_t ldq,
                                const void* c_hi, const void* c_lo, int64_t ldc, int32_t self, float threshold, uint64_t* count,
                                int64_t capacity, int32_t* i_out, int32_t* j_out, float* s_out, void* stream);
int dae_csr_similarity_pairs(const int64_t* q_indptr, const int32_t* q_indices, const float* q_values, int32_t n_query,
                             int64_t q_nnz, int32_t q_features, const int64_t* c_indptr, const int32_t* c_indices,
                             const float* c_values, int32_t n_corpus, int64_t c_nnz, int32_t c_features, int32_t self,
                             float threshold, void* workspace, int64_t workspace_bytes, uint64_t* count, int64_t capacity,
                             int32_t* i_out, int32_t* j_out, float* s_out, void* stream);
int dae_csr_similarity_pairs_workspace(int32_t n_query, int32_t n_corpus, int64_t corpus_nnz, int32_t n_features, int64_t* bytes);
/* dae_pairs_sort: the canonical order of n pairs.  keys[t] = i * n_corpus + j (unique, below 2^key_bits) are sorted ascending with
 *   s[t] as the payload on a double-buffered radix sort: keys_alt and s_alt (n entries each, distinct from keys and s) are the
 *   alternate buffers, and the workspace (at least dae_pairs_sort_workspace bytes) does not grow with n beyond the sort's tile
 *   bookkeeping.  On return *which (host int32) = 0 when the sorted keys and scores are in keys / s, 1 when in keys_alt / s_alt; the
 *   other key buffer holds the decoded pairs as int32: i in its first n entries, j in the next n.  n < 2^31.
 */
int dae_pairs_sort(int64_t n, int32_t n_corpus, int32_t key_bits, uint64_t* keys, uint64_t* keys_alt, float* s, float* s_alt,
                   void* workspace, int64_t workspace_bytes, int32_t* which, void* stream);
int dae_pairs_sort_workspace(int64_t n, int32_t key_bits, int64_t* bytes);

/* ---- deterministic training step (DESIGN 4.7) ----------------------------------------------------------------------------
 * Variants of the step's kernels in which no floating-point sum depends on timing: with the same inputs, build and GPU model they
 * give the same bits on every run.  Each takes caller-owned workspace; the *_workspace / *_parts queries size it.
 *
 * dae_gemm_bf16x3_det / dae_gemm_sym_bf16x3_det: dae_gemm_bf16x3 / dae_gemm_sym_bf16x3 with the same schedule and main loop.  A
 *   stream-K segment that covers a whole tile stores it (adds it when accumulate != 0: it is the element's only writer); a segment
 *   that covers part of a tile stores it to its CTA's workspace slot, and a fixup kernel adds each split tile's slots in k order and
 *   stores (adds) the sum once.  k_splits: 1 or -1 (stream-K where dae_gemm_bf16x3 would use it).  workspace: at least
 *   dae_gemm_det_workspace bytes (2 slots of 128 x 128 fp32 per SM).  Concurrent calls need separate workspaces.
 * dae_decode_fused_bf16x3_det: dae_decode_fused_bf16x3, but row_loss_parts is [n_parts x Brows] (n_parts from
 *   dae_decode_loss_parts: two per 128-column tile) and every (half tile, row) partial is stored, not added; dae_step_finalize
 *   (parts, n_parts) or dae_reduce_parts sums them in part order.
 * dae_encode_csr_bwd_det: dA = dE * f'(A) in place of dE (dE_add added first, as in dae_encode_csr_bwd_gather) and dbh STORED (the
 *   sums of 4-row CTAs, added in order in groups of 32, then the groups in order).  The sparse dW = X_c^T . dA stays in the workspace: the batch's kept entries are
 *   bucketed by column in batch-row order (a stable counting sort), summed per column in that order in chunks of fixed entry
 *   positions, and dae_encode_sparse_dw_add later adds them onto dW (F x H, e.g. the dense dW stored by dae_gemm_bf16x3_det).
 *   col_count: the per-column counts dae_encode_csr_fwd wrote for this batch.  cap_nnz: at least the batch's stored entries; the
 *   same value goes to the workspace query and to dae_encode_sparse_dw_add.  Rows must be canonical (no repeated column).  Any H up
 *   to 12800.
 * dae_triplet_*_det: the mining kernels with the triplet loss of anchor (explicit: row) a stored to loss_slots[a] (fp64, one per
 *   anchor of the batch; batch_hard stores 0 for inactive anchors) instead of added to stats; dae_triplet_loss_sum then adds the n
 *   slots to stats[DAE_STAT_TRIPLET_SUM] in a fixed order.  The integer-valued statistics (NUM, N_ACTIVE, batch_hard's weights)
 *   keep their atomics: their sums are exact in any order.
 */
int dae_gemm_det_workspace(int64_t* bytes);
int dae_gemm_bf16x3_det(int32_t M, int32_t N, int32_t K, float alpha, const void* a_hi, const void* a_lo, int64_t lda,
                        int32_t a_mn_major, const void* b_hi, const void* b_lo, int64_t ldb, int32_t b_mn_major, float* C,
                        int64_t ldc, int32_t n_store, int32_t special_col, float* special_out, int32_t k_splits,
                        int32_t accumulate, void* workspace, int64_t workspace_bytes, void* stream);
int dae_gemm_sym_bf16x3_det(int32_t M, int32_t N, float alpha, const void* g_hi, const void* g_lo, int64_t ldg, const void* b_hi,
                            const void* b_lo, int64_t ldb, float* C, int64_t ldc, int32_t accumulate, void* workspace,
                            int64_t workspace_bytes, void* stream);
int dae_decode_loss_parts(int32_t F, int32_t* n_parts);
int dae_decode_fused_bf16x3_det(int32_t Brows, int32_t F, int32_t K, const void* e_hi, const void* e_lo,
                                int64_t lde, const void* w_hi, const void* w_lo, int64_t ldw,
                                const int64_t* indptr, const int32_t* indices, const float* values,
                                const int32_t* rows, const float* bv, int32_t dec_act, int32_t loss_func,
                                const float* weight, const double* stats, void* dz_hi, void* dz_lo,
                                int64_t ld_dz, float* row_loss_parts, int32_t* tile_ptr, int32_t prepared, void* stream);
int dae_encode_csr_bwd_det_workspace(int32_t n_rows, int32_t F, int32_t H, int64_t cap_nnz, int64_t* bytes);
int dae_encode_csr_bwd_det(const int64_t* indptr, const int32_t* indices, const float* values, const int32_t* rows,
                           int32_t n_rows, int32_t F, int32_t H, float in_scale, const float* E, const float* bh,
                           int32_t enc_act, float* dE, const float* dE_add, int64_t ldE, float* dbh, const int32_t* col_count,
                           int64_t cap_nnz, void* workspace, int64_t workspace_bytes, void* stream);
int dae_encode_sparse_dw_add(int32_t n_rows, int32_t F, int32_t H, int64_t cap_nnz, const void* workspace, int64_t workspace_bytes,
                             float* dW, void* stream);
int dae_triplet_batch_all_det(const float* S, int64_t lds, int32_t B, const int32_t* seg_lo, const int32_t* seg_hi,
                              float* G, int64_t ldg, double* stats, int32_t pos_only, void* g_hi, void* g_lo,
                              int64_t ld_split, double* loss_slots, void* stream);
int dae_triplet_batch_hard_det(const float* S, int64_t lds, int32_t B, const float* labels, float* G, int64_t ldg,
                               float* weight, double* stats, double* loss_slots, void* stream);
int dae_triplet_batch_all_rows_det(const float* S_blk, int64_t lds, int32_t row0, int32_t n_rows, int32_t B, const int32_t* seg_lo,
                                   const int32_t* seg_hi, float* G_blk, int64_t ldg, double* stats, int32_t pos_only, void* g_hi,
                                   void* g_lo, int64_t ld_split, double* loss_slots, void* stream);
int dae_triplet_batch_hard_rows_det(const float* S_blk, int64_t lds, int32_t row0, int32_t n_rows, int32_t B, const float* labels,
                                    float* G_blk, int64_t ldg, float* weight, double* stats, double* loss_slots, void* stream);
int dae_triplet_explicit_det(const float* E, const float* Ep, const float* En, int32_t B, int32_t H, int64_t ld,
                             float alpha, float* dE, float* dEp, float* dEn, double* stats, double* loss_slots, void* stream);
int dae_triplet_loss_sum(const double* loss_slots, int32_t n, double* stats, void* stream);

/* ---- GRU user encoder over reading sequences (DESIGN 4.10) -----------------------------------------------------------------
 * A batch of users is ordered by length, descending (PackedSequence layout): at step t the users still reading are rows [0, n_t)
 * and their positions are rows off_t + i of every packed [positions x ...] buffer.  Gates follow torch.nn.GRU (order r, z, n):
 * r = s(xr + hr), z = s(xz + hz), n = tanh(xn + r hn), h = (1 - z) n + z h_prev, with XP = [X | 1].[W_ih | b_ih]^T and
 * HP = [h_prev | 1].[W_hh | b_hh]^T computed by dae_gemm_bf16x3.
 * dae_gather_split_bf16: hi / lo [n_rows x ld_dst] <- rows rows[r] of src (columns [0, cols)), column ones_col (if >= 0) = 1,
 *   the other columns 0: the packed [X | 1] operand of a batch.
 * dae_gru_cell_fwd: one step for rows [0, n) from XP (ld_xp >= 3H) and HP (ld_hp >= 3H).  h_prev NULL: h_prev = 0; h_out may equal
 *   h_prev.  Rows i < n_split of h also go to h_hi / h_lo [.. x ld_split] (the next step's GEMM operand) when h_hi is non-NULL;
 *   gates (optional, ld_gates >= 4H) <- [r | z | n | hn], what dae_gru_cell_bwd needs.
 * dae_gru_cell_bwd: one step backward for rows [0, n): dh = carry + dh_in (dh_in optional).  Writes dXP = [dr^, dz^, dn^] and
 *   dHP = [dr^, dz^, r dn^] as bf16 hi / lo rows (ld_g >= 3H) and carry <- dh z, onto which the caller accumulates dHP . W_hh.
 * dae_seq_negatives: neg[p] = (pos[p] + 1 + floor(u (n_items - 1))) mod n_items, u = c / 2^32 where c is the first word of
 *   Philox4x32-10 with key seed and counter (p, batch, epoch lo, epoch hi): uniform over the other articles, never pos[p].
 *   pos[p] < 0: neg[p] = -1.  The counter's first word is p mod 2^32, so draws repeat beyond 2^32 positions in one call.
 * dae_seq_rank_loss: one warp per position p with pos[p] >= 0: x = h_p . e(neg[p]) - h_p . e(pos[p]); *loss_sum += softplus(x)
 *   (fp64 atomics); dh_p = scale s(x) (e(neg) - e(pos)).  Positions with pos[p] < 0 get dh_p = 0.
 */
int dae_gather_split_bf16(const float* src, int64_t ld_src, const int32_t* rows, int32_t n_rows, int32_t cols, void* hi, void* lo,
                          int64_t ld_dst, int32_t ones_col, void* stream);
int dae_gru_cell_fwd(int32_t n, int32_t H, const float* xp, int64_t ld_xp, const float* hp, int64_t ld_hp, const float* h_prev,
                     int64_t ld_hprev, float* h_out, int64_t ld_h, int32_t n_split, void* h_hi, void* h_lo, int64_t ld_split,
                     float* gates, int64_t ld_gates, void* stream);
int dae_gru_cell_bwd(int32_t n, int32_t H, const float* dh_in, int64_t ld_dh_in, float* carry, int64_t ld_carry, const float* gates,
                     int64_t ld_gates, const float* h_prev, int64_t ld_hprev, void* dxp_hi, void* dxp_lo, void* dhp_hi, void* dhp_lo,
                     int64_t ld_g, void* stream);
int dae_seq_negatives(const int32_t* pos, int64_t n_pos, int32_t n_items, uint64_t seed, uint64_t epoch, uint64_t batch, int32_t* neg,
                      void* stream);
int dae_seq_rank_loss(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int32_t* pos, const int32_t* neg,
                      int64_t n_pos, float scale, float* dh, int64_t ld_dh, double* loss_sum, void* stream);

/* ---- data-parallel exchange step (SURVEY 8e): in-switch all-reduce of the flat gradient buffer -------------------
 * The reference is single-process; row-sharded training adds ONE sum over ranks of [dW | dbh | dbv] between the
 * gradient kernels and dae_optimizer_step.  Default transport: ncclAllReduce.  dae_allreduce_multimem is the
 * in-graph alternative: `multicast_grad` is the NVSwitch multicast address bound to every rank's gradient buffer
 * (symmetric memory, identical offset on every rank, n floats, 16-byte aligned); `peer_flags` is a DEVICE array of
 * `world` pointers to each rank's flag words (2 * n_blocks * world zero-initialised uint32, peer-mapped); `epochs` is
 * this rank's own uint32[n_blocks] (zero-initialised, ordinary device memory): the per-CTA exchange counter the
 * flags carry, advanced by the kernel itself so that it stays in step with CUDA-graph replays.  Every rank calls it
 * with the same n and n_blocks on its step stream, the same number of times; on return (stream order) every rank's
 * buffer holds the sum.  Rank r reduces float4 packets [r*ceil(n4/P), ...) with multimem.ld_reduce and writes them
 * back with multimem.st; CTA-level flag barriers (one remote store per peer to arrive, local polling to wait) open and
 * close the exchange and trap after 5 s instead of hanging a replica.
 */
int dae_allreduce_multimem(float* multicast_grad, void* const* peer_flags, uint32_t* epochs, int32_t rank,
                           int32_t world, int64_t n, int32_t n_blocks, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DAE_SM100_H */
