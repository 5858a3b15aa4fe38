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
 * Classes are those of the reference's tf.equal: -0.0 and +0.0 are one class (ordered as one key, by row id); a NaN label equals
 * nothing, so each NaN row is a class of one, [seg_lo, seg_hi) = [i, i + 1), and the NaN rows come last in row-id order.
 * labels_out holds labels_all[rows_out] with their own bits.
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
 * rows in the three blocks of the stacked [org; pos; neg] matrix (n_each rows per block, n_each <= (2^31 - 1) / 3 so that every
 * row id fits in int32); stats zeroed, SUM_W = B. */
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
 *   columns n < n_store go to C; column special_col (if special_out != NULL) goes to special_out[m].  n_store <= 0 or > N means
 *   N.  Rejected before any device work: ldc < n_store, and special_out != NULL unless n_store <= special_col < N (so the
 *   special column never aliases a stored one).  The same rules hold for dae_gemm_bf16x3_det.
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
 *   matrices (indptr int64, indices int32 strictly increasing inside a row, values fp32; q_features == c_features), on the CUDA
 *   cores and without forming S.  A column may appear only once in a row, in Q and in C: the kernels bucket the corpus entries by
 *   (2048-row range, column) and add a bucket's entries into distinct accumulators at once, so a repeated column would race
 *   (scipy's sum_duplicates() / sort_indices() give the required form; helpers canonicalise every matrix they upload).  Every
 *   corpus row is a candidate, a row sharing no column with q included (score 0), except column q + diag_offset when `exclude`
 *   is set; order (score desc, index asc); padding -1 / -inf.  A NaN or -inf score is never a candidate, so a row whose every
 *   candidate scores NaN or -inf (a stored 0 times inf gives NaN) is all padding; +inf is listed.  Each score accumulates in fp32
 *   from 0, one term per shared column in increasing column order, each term the product rounded to fp32 and then added (no FMA), so
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

/* ---- long top-k lists: k up to 1024 on the tensor cores, in three stages (DESIGN 4.14) ------------------------------
 * The stages give, per query row, exactly what dae_similarity_topk_groups_bf16x3 / _excl / the plain call would give for the same
 * arguments if they accepted k: order (score desc, index asc), -0.0 equal to +0.0, padding -1 / -inf, no NaN, the same exclusion
 * and group semantics, independent of `splits`, every score the bits those calls report for that (i, j).  1 <= k <= 1024.
 * dae_similarity_topk_bound_bf16x3: the arguments of dae_similarity_topk_groups_bf16x3 (groups may be NULL: no groups;
 *   ex_indptr may be NULL when ex_nnz = 0) with a bound workspace of at least dae_similarity_topk_bound_workspace bytes (16-byte
 *   aligned, same n_query, n_corpus, k, splits).  Writes tau [n_query] (fp32, 4-byte aligned): a lower bound on row i's k-th best
 *   answer score (-FLT_MAX when it has fewer than k answers).  `splits` sets the least number of corpus parts; the call uses at
 *   least ceil(k / 32) of them.
 * dae_similarity_topk_collect_bf16x3: every candidate (i, j) of the same rows (no self match with `exclude`, nothing listed in
 *   ex_indptr / ex_indices) with S[i, j] >= max(tau[i], -FLT_MAX): so never -inf or NaN.  The count protocol of
 *   dae_similarity_pairs_bf16x3 (*count caller-zeroed and accumulated, the first `capacity` written to i_out / j_out / s_out),
 *   plus row_count [n_query] (uint32, caller-zeroed, accumulated): the candidates of each row.  Every tile of S is computed.
 * dae_similarity_topk_select: n_pairs candidates sorted by (i, j) (dae_pairs_sort's output; i in [0, n_query)) -> idx_out /
 *   val_out [n_query x k], the k best of each row by (score desc, j asc); with groups (int32 [n_corpus] labels >= 0, or NULL) each
 *   group contributes its first candidate in that order only.  Any number of candidates per row.
 * Every argument is checked before any CUDA call.
 */
int dae_similarity_topk_bound_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo,
                                     int64_t ldq, const void* c_hi, const void* c_lo, int64_t ldc, int32_t k,
                                     int64_t diag_offset, int32_t exclude, int32_t splits, void* workspace,
                                     int64_t workspace_bytes, const int64_t* ex_indptr, const int32_t* ex_indices,
                                     int64_t ex_nnz, const int32_t* groups, float* tau, void* stream);
int dae_similarity_topk_bound_workspace(int32_t n_query, int32_t n_corpus, int32_t k, int32_t splits, int64_t* bytes);
int dae_similarity_topk_collect_bf16x3(int32_t n_query, int32_t n_corpus, int32_t dim, const void* q_hi, const void* q_lo,
                                       int64_t ldq, const void* c_hi, const void* c_lo, int64_t ldc, int64_t diag_offset,
                                       int32_t exclude, const float* tau, const int64_t* ex_indptr, const int32_t* ex_indices,
                                       int64_t ex_nnz, uint64_t* count, uint32_t* row_count, int64_t capacity, int32_t* i_out,
                                       int32_t* j_out, float* s_out, void* stream);
int dae_similarity_topk_select(int32_t n_query, int64_t n_pairs, const int32_t* i_sorted, const int32_t* j_sorted,
                               const float* s_sorted, int32_t k, const int32_t* groups, int32_t* idx_out, float* val_out,
                               void* stream);

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
 * NaN scores (a row holding NaN or inf): a NaN score is counted in bin 0 of its group, and that group's sums entry becomes NaN.
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

/* ---- LSTM user encoder over reading sequences (DESIGN 4.15) ----------------------------------------------------------------
 * The packed layout and the GEMMs are the GRU's above; the cell is torch.nn.LSTM's (gate order i, f, g, o) with XP and HP 4H wide:
 * i = s(xi + hi), f = s(xf + hf), g = tanh(xg + hg), o = s(xo + ho), c_t = f c_{t-1} + i g, h_t = o tanh(c_t).
 * dae_lstm_cell_fwd: one step for rows [0, n) from XP (ld_xp >= 4H), HP (ld_hp >= 4H) and c_prev (NULL: c_{t-1} = 0).  Writes c_out
 *   and h_out (fp32); c_out may equal c_prev (then ld_c == ld_cprev).  h_{t-1} is not read (it enters through HP), so h_out may be
 *   the buffer the step's GEMM operand came from.  Rows i < n_split of h also go to h_hi / h_lo [.. x ld_split] (the next step's
 *   GEMM operand) when h_hi is non-NULL; gates (optional, ld_gates >= 4H) <- [i | f | g | o], what dae_lstm_cell_bwd needs with
 *   c_t and c_{t-1}.
 * dae_lstm_cell_bwd: one step backward for rows [0, n): dh = carry_h + dh_in (dh_in optional), dc = carry_c + dh o (1 - tanh^2 c_t)
 *   with c = c_t and c_prev = c_{t-1} (NULL: 0).  Writes dA = [di, df, dg, do] (the pre-activation gradient, which is both dXP and
 *   dHP) as bf16 hi / lo rows (ld_da >= 4H) and carry_c <- dc f.  carry_h is read only: the caller then STORES
 *   dh_{t-1}[0, n) = dA . W_hh over it (there is no direct h -> h term).  Rows [n_t, n_{t-1}) of both carries must be zero when
 *   step t - 1 starts: those users' last read is at t - 1.
 */
int dae_lstm_cell_fwd(int32_t n, int32_t H, const float* xp, int64_t ld_xp, const float* hp, int64_t ld_hp, const float* c_prev,
                      int64_t ld_cprev, float* c_out, int64_t ld_c, float* h_out, int64_t ld_h, int32_t n_split, void* h_hi, void* h_lo,
                      int64_t ld_split, float* gates, int64_t ld_gates, void* stream);
int dae_lstm_cell_bwd(int32_t n, int32_t H, const float* dh_in, int64_t ld_dh_in, const float* carry_h, int64_t ld_carry_h,
                      float* carry_c, int64_t ld_carry_c, const float* gates, int64_t ld_gates, const float* c, int64_t ld_c,
                      const float* c_prev, int64_t ld_cprev, void* da_hi, void* da_lo, int64_t ld_da, void* stream);

/* ---- long-term user vectors (LSTUR-ini, DESIGN 4.18) -------------------------------------------------------------------------
 * dae_rows_optimizer_step: the row-sparse (lazy) optimizer step of a table [rows x ld] (columns [0, cols) used).  For each i < n
 *   with rows[i] >= 0, row rows[i] of table, slot1 and slot2 (laid out as the table) is updated from grad row i ([n x ld_grad]) by
 *   dae_optimizer_step's rules (grad_scale 1); rows not listed and their slots are not touched.  counts (int32, one per table row;
 *   required for adam, optional otherwise) is incremented for each updated row, and Adam's bias correction uses the incremented
 *   count as its step.  The listed rows must be distinct (no atomics; the result is deterministic).
 */
int dae_rows_optimizer_step(float* table, int64_t ld, int32_t cols, const int32_t* rows, int32_t n, const float* grad, int64_t ld_grad,
                            float* slot1, float* slot2, int32_t* counts, int32_t opt, float lr, float momentum, void* stream);

/* ---- attention user encoder over reading sequences (DESIGN 4.17) -----------------------------------------------------------
 * NRMS's user encoder made causal, in the packed layout above: batch user i (of B) has lens[i] reads (int32, device), read t at
 * position off[t] + i (off: int64 [T + 1], device; lens[i] <= T <= 1024 must hold, the kernels trust it).  H = heads x d with head
 * dim d <= 128.  The projections QKV = [X | 1].[W_in | b_in]^T, M = [O | 1].[W_out | b_out]^T and Z = [M | 1].[W_a | b_a]^T are
 * dae_gemm_bf16x3 calls.  Every output element is written by one thread in a fixed order: the same bits on every run.
 * dae_seq_attention_fwd: per (user, head), with q, k, v the head's columns [h d, (h + 1) d) of QKV's thirds (ld_qkv >= 3H),
 *   O_t = sum_{s <= t} softmax_s(q_t . k_s / sqrt(d)) v_s.  Writes O (fp32, columns [0, H)), its bf16 hi / lo split (columns
 *   [0, H) of o_hi / o_lo [.. x ld_split]; the caller keeps column H at 1 for the bias) and lse[p * ld_lse + h], the log-sum-exp
 *   of row p's scaled scores.
 * dae_seq_attention_bwd: from QKV, O, lse and dO (ld_do >= H) writes dQKV = [dQ | dK | dV] as bf16 hi / lo rows (columns [0, 3H),
 *   ld_dqkv >= 3H), the operand of [dW_in | db_in] = dQKV^T.[X | 1].  The probabilities are recomputed from lse.
 * dae_seq_pool_fwd: a_s = q . tanh(Z_s) (Z: ld_z >= A, q: [A]) -> score[p], the prefix log-sum-exp lse_t = log sum_{s <= t} e^{a_s}
 *   -> plse[p], and u_t = sum_{s <= t} e^{a_s - lse_t} M_s -> u (ld_u >= H).
 * dae_seq_pool_bwd: from dU (du), u, M, Z, q, score and plse writes dM (fp32, ld_dm >= H; the value path sum_{t >= s} w_ts dU_t),
 *   dZ = da q (1 - tanh^2 Z) as bf16 hi / lo (columns [0, A), ld_dz >= A) with da_s = sum_{t >= s} w_ts dU_t . (M_s - u_t), and
 *   dq[k] = sum_s da_s tanh Z_s[k] (fp32 [A], stored; a fixed-order sum over users).  workspace: B x A floats.  The scorer path
 *   of dM is the caller's GEMM dM += dZ.W_a.
 */
int dae_seq_attention_fwd(int32_t B, int32_t T, const int64_t* off, const int32_t* lens, int32_t H, int32_t heads, const float* qkv,
                          int64_t ld_qkv, float* o, int64_t ld_o, void* o_hi, void* o_lo, int64_t ld_split, float* lse, int64_t ld_lse,
                          void* stream);
int dae_seq_attention_bwd(int32_t B, int32_t T, const int64_t* off, const int32_t* lens, int32_t H, int32_t heads, const float* qkv,
                          int64_t ld_qkv, const float* o, int64_t ld_o, const float* lse, int64_t ld_lse, const float* dout, int64_t ld_do,
                          void* dqkv_hi, void* dqkv_lo, int64_t ld_dqkv, void* stream);
int dae_seq_pool_fwd(int32_t B, int32_t T, const int64_t* off, const int32_t* lens, int32_t H, int32_t A, const float* z, int64_t ld_z,
                     const float* q, const float* m, int64_t ld_m, float* u, int64_t ld_u, float* score, float* plse, void* stream);
int dae_seq_pool_bwd(int32_t B, int32_t T, const int64_t* off, const int32_t* lens, int32_t H, int32_t A, const float* du, int64_t ld_du,
                     const float* u, int64_t ld_u, const float* m, int64_t ld_m, const float* z, int64_t ld_z, const float* q,
                     const float* score, const float* plse, float* dm, int64_t ld_dm, void* dz_hi, void* dz_lo, int64_t ld_dz, float* dq,
                     void* workspace, void* stream);

/* ---- impression logs (DESIGN 4.13) ------------------------------------------------------------------------------------------
 * An impression is a list of shown articles items[indptr[i] .. indptr[i + 1]) (rows of emb) with clicked[k] != 0 where the article
 * was clicked; C and N are its clicked and not-clicked articles.  One warp per row of work; lists of any length are walked in
 * chunks of per-warp shared memory.
 * dae_impression_rank_loss: the impression loss of a packed GRU batch.  The impressions of packed position p are
 *   [pos_indptr[p], pos_indptr[p + 1]) (ids into imp_indptr); with s_j = h_p . e(items[j]), impression q adds
 *   l_q = 1 / (|C| |N|) sum_{c, n} softplus(s_n - s_c) to *loss_sum (fp64 atomics) and scale / (|C| |N|) sum_j w_j e(items[j])
 *   to dh_p, where w_n = sum_c s(s_n - s_c) and w_c = -sum_n s(s_n - s_c).  Impressions with |C| = 0 or |N| = 0 add nothing.
 *   EVERY row p < n_pos of dh is written (zero without impressions), in a fixed order per row: no atomics on dh.
 * dae_impression_softmax_loss (DESIGN 4.16): the sampled-softmax impression loss of a packed batch, arguments as
 *   dae_impression_rank_loss's plus imp_ids (int64 [pos_indptr[n_pos]]: impression q's global id, < 2^32), K in [0, 32], seed,
 *   epoch and workspace (8 bytes per shown article: imp_indptr[pos_indptr[n_pos]] x 8 bytes, any contents).  For each click c of
 *   a usable impression, r its ordinal among the impression's clicks: S_c = N when K = 0 or K >= |N|, else K distinct non-clicks
 *   by Floyd's algorithm over the ordinals into N in item order (d = 0 .. K - 1: j = |N| - K + d, t = floor(u_d (j + 1) / 2^32);
 *   j if t is already chosen, else t), u_d = word d & 3 of Philox4x32-10, key (seed lo, seed hi), counter (imp_ids[q] lo,
 *   r, epoch lo, d >> 2).  *loss_sum += l_c = log(e^{s_c} + sum_{n in S_c} e^{s_n}) - s_c (max subtracted, fp64 atomics) and
 *   dh_p += scale sum_c sum_{j in {c} + S_c} (p_cj - [j = c]) e(items[j]), p_cj the softmax weight.  Every row p < n_pos of dh
 *   is written (zero without impressions), in a fixed order per row: no atomics on dh.
 * dae_impression_metrics: one query row q_i (ld_q) per impression.  scores[k] (fp32, every k < indptr[n_imp]) = q_i . e(items[k]),
 *   or with cosine = 1 that over |q_i| |e(items[k])| (0 when either is zero).  The dot products and squared norms are fp32 sums:
 *   with every |x| <= 2^63 / sqrt(H) they stay below 2^126 and every score is finite (impression_metrics rejects larger
 *   entries); beyond that a score may be inf or NaN.  A cosine operand whose fp32 squared norm underflows to 0 (every |x| <=
 *   2^-75) counts as zero and scores 0; a subnormal squared norm gives a finite score without fp32's relative accuracy.
 *   metrics[i] (fp64 [n_imp x 4]) = AUC, MRR, nDCG@5,
 *   nDCG@10 of those scores: rank_j = #{k: s_k > s_j} + #{k before j: s_k = s_j}; AUC = (#{s_c > s_n} + #{s_c = s_n} / 2) /
 *   (|C| |N|); MRR = mean over C of 1 / (rank + 1); nDCG@K = sum_{c: rank < K} 1 / log2(rank + 2) over its value for the first
 *   min(|C|, K) ranks.  |C| = 0 or |N| = 0: four NaNs.
 */
int dae_impression_rank_loss(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int64_t* pos_indptr,
                             int64_t n_pos, const int64_t* imp_indptr, const int32_t* items, const uint8_t* clicked, float scale,
                             float* dh, int64_t ld_dh, double* loss_sum, void* stream);
int dae_impression_softmax_loss(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int64_t* pos_indptr,
                                int64_t n_pos, const int64_t* imp_indptr, const int32_t* items, const uint8_t* clicked,
                                const int64_t* imp_ids, int32_t K, uint64_t seed, uint64_t epoch, float scale, float* dh, int64_t ld_dh,
                                double* loss_sum, void* workspace, void* stream);
int dae_impression_metrics(const float* q, int64_t ld_q, const float* emb, int64_t ld_emb, int32_t H, int32_t cosine,
                           const int64_t* indptr, const int32_t* items, const uint8_t* clicked, int64_t n_imp, float* scores,
                           double* metrics, void* stream);

/* ---- article encoder fine-tuned through the user encoders' losses (DESIGN 4.19) -----------------------------------------
 * dae_encode_csr_fwd_groups: dae_encode_csr_fwd with the thread groups per row given (groups = 1 or 4) instead of chosen from
 *   n_rows.  A row's output bits depend on the group count, the row and the parameters only, so with the count pinned a row is
 *   bit-identical whether it is encoded alone, within a subset (rows) or within the whole set.
 * dae_seq_rank_loss_grad, dae_impression_rank_loss_grad, dae_impression_softmax_loss_grad: the losses above with the same
 *   arguments and the same dh, bit for bit, plus the gradient with respect to the scored rows of emb: each scored candidate j of
 *   position p adds g_j h_p to demb row items[j] (fp32 atomics, so the sums' order depends on the schedule), where g_j is the
 *   coefficient of e_j in dh_p.  demb [rows of emb x ld_demb] is accumulated onto, never cleared.
 * dae_touch_compact: the compact table of the ids a batch touches.  ids [n] (n < 2^31) are row ids in [0, N) of a table of N rows,
 *   < 0 for none.  tag (uint64 [N], zero before the first call) keeps per id the last call's stamp; stamp > 0 must grow from call to
 *   call on the same tag, so tag is never cleared.  slot_of (int32 [N]) is scratch.  Out: T distinct ids in rows[0, T) in the order
 *   of their first occurrence in ids, slots[i] = the slot of ids[i] in rows (-1 where ids[i] < 0) and ws[0] = T; ws holds
 *   dae_touch_compact_workspace(n) int32 words.
 * dae_rows_scatter_add: dst[idx[p], 0:cols] += src[p, 0:cols] for p < n with idx[p] >= 0 (fp32 atomics).
 */
int dae_encode_csr_fwd_groups(const int64_t* indptr, const int32_t* indices, const float* values, const int32_t* rows, int32_t n_rows,
                              int32_t F, int32_t H, float in_scale, const float* W, const float* bh, int32_t enc_act, float* E, int64_t ldE,
                              int32_t* col_count, void* e_hi, void* e_lo, int64_t ld_split, int32_t groups, void* stream);
int dae_seq_rank_loss_grad(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int32_t* pos,
                           const int32_t* neg, int64_t n_pos, float scale, float* dh, int64_t ld_dh, double* loss_sum, float* demb,
                           int64_t ld_demb, void* stream);
int dae_impression_rank_loss_grad(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int64_t* pos_indptr,
                                  int64_t n_pos, const int64_t* imp_indptr, const int32_t* items, const uint8_t* clicked, float scale,
                                  float* dh, int64_t ld_dh, double* loss_sum, float* demb, int64_t ld_demb, void* stream);
int dae_impression_softmax_loss_grad(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H,
                                     const int64_t* pos_indptr, int64_t n_pos, const int64_t* imp_indptr, const int32_t* items,
                                     const uint8_t* clicked, const int64_t* imp_ids, int32_t K, uint64_t seed, uint64_t epoch, float scale,
                                     float* dh, int64_t ld_dh, double* loss_sum, void* workspace, float* demb, int64_t ld_demb,
                                     void* stream);
int dae_touch_compact_workspace(int64_t n, int64_t* count);
int dae_touch_compact(const int32_t* ids, int64_t n, uint32_t stamp, void* tag, int32_t* slot_of, int32_t* rows, int32_t* slots,
                      int32_t* ws, void* stream);
int dae_rows_scatter_add(const float* src, int64_t ld_src, const int32_t* idx, int64_t n, int32_t cols, float* dst, int64_t ld_dst,
                         void* stream);

/* ---- deterministic user-encoder training (DESIGN 4.21) -----------------------------------------------------------------------
 * With the same inputs, build and GPU model these give the same bits on every run.
 * dae_seq_rank_loss_det, dae_impression_rank_loss_det, dae_impression_softmax_loss_det: the losses above with the same arguments and
 *   the same dh, bit for bit, but loss_slots (fp64 [n_pos], 8-byte aligned) in place of loss_sum: position p's loss term is STORED
 *   to loss_slots[p] (0 for a position without a term); nothing is added anywhere.  For the impression losses the slot is the
 *   warp's butterfly sum of its lanes' terms for that position.
 * dae_*_loss_grad_det: the same, and in place of demb the article gradient as triples (t_slot, t_row, t_coef: int32, int32, fp32)
 *   meaning "add t_coef * h[t_row] to row t_slot", each at an index fixed by the data layout: the rank loss writes 2 n_pos triples,
 *   2p = (neg[p], p, +g) and 2p + 1 = (pos[p], p, -g); the impression losses write one triple per shown article k at index k of
 *   items (imp_indptr[pos_indptr[n_pos]] triples), with g its coefficient in dh_p.  t_slot = -1 marks a triple that adds nothing.
 * dae_loss_slots_sum: *out += sum of loss_slots[0, n) in a fixed order: 256 partials, partial t the sum of slots t, t + 256, ... in
 *   index order from +0, then the partials in order from +0, then that total added to *out.
 * dae_ordered_rows: dst[t, 0:cols] for every t < n_slots, STORED: the terms whose slot is t, taken in term order, as
 *   acc = acc + c * src_row (fp32, +0 first, each product and sum rounded on its own).  Term i < n_a is the triple (a_slot[i],
 *   a_row[i], a_coef[i]) over rows of src_a; term n_a + p is (b_slot[p], p, 1) over rows of src_b.  Slots must be < n_slots; a
 *   slot < 0 adds nothing; a slot without terms gets a zero row.  workspace (256-byte aligned): dae_ordered_rows_workspace bytes,
 *   16 bytes per term (the sort's keys and values, double-buffered) plus cub's radix-sort scratch.
 */
int dae_seq_rank_loss_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int32_t* pos,
                          const int32_t* neg, int64_t n_pos, float scale, float* dh, int64_t ld_dh, double* loss_slots, void* stream);
int dae_seq_rank_loss_grad_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int32_t* pos,
                               const int32_t* neg, int64_t n_pos, float scale, float* dh, int64_t ld_dh, double* loss_slots,
                               int32_t* t_slot, int32_t* t_row, float* t_coef, void* stream);
int dae_impression_rank_loss_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H, const int64_t* pos_indptr,
                                 int64_t n_pos, const int64_t* imp_indptr, const int32_t* items, const uint8_t* clicked, float scale,
                                 float* dh, int64_t ld_dh, double* loss_slots, void* stream);
int dae_impression_rank_loss_grad_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H,
                                      const int64_t* pos_indptr, int64_t n_pos, const int64_t* imp_indptr, const int32_t* items,
                                      const uint8_t* clicked, float scale, float* dh, int64_t ld_dh, double* loss_slots, int32_t* t_slot,
                                      int32_t* t_row, float* t_coef, void* stream);
int dae_impression_softmax_loss_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H,
                                    const int64_t* pos_indptr, int64_t n_pos, const int64_t* imp_indptr, const int32_t* items,
                                    const uint8_t* clicked, const int64_t* imp_ids, int32_t K, uint64_t seed, uint64_t epoch, float scale,
                                    float* dh, int64_t ld_dh, double* loss_slots, void* workspace, void* stream);
int dae_impression_softmax_loss_grad_det(const float* h, int64_t ld_h, const float* emb, int64_t ld_emb, int32_t H,
                                         const int64_t* pos_indptr, int64_t n_pos, const int64_t* imp_indptr, const int32_t* items,
                                         const uint8_t* clicked, const int64_t* imp_ids, int32_t K, uint64_t seed, uint64_t epoch,
                                         float scale, float* dh, int64_t ld_dh, double* loss_slots, void* workspace, int32_t* t_slot,
                                         int32_t* t_row, float* t_coef, void* stream);
int dae_loss_slots_sum(const double* loss_slots, int64_t n, double* out, void* stream);
int dae_ordered_rows_workspace(int64_t n_a, int64_t n_b, int32_t n_slots, int64_t* bytes);
int dae_ordered_rows(const int32_t* a_slot, const int32_t* a_row, const float* a_coef, int64_t n_a, const float* src_a, int64_t ld_a,
                     const int32_t* b_slot, int64_t n_b, const float* src_b, int64_t ld_b, int32_t n_slots, int32_t cols, float* dst,
                     int64_t ld_dst, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- bag-of-words user profiles and their impression metrics (DESIGN 4.20) --------------------------------------------------
 * The history W [n_users x n_articles] and the articles X [n_articles x n_features] are CSR matrices: indptr int64, indices int32
 * strictly increasing inside a row (sorted, no duplicates), values fp32; the kernels do not check the contents.  The profiles
 * P = W.X are the CSR matrix whose row u holds the union of the stored columns of every row of X that row u of W stores (explicit
 * zero weights and explicit zero entries included).  Memory is O(nnz(P)): never n_users x n_features.  1 <= n_features <= 2^24.
 * dae_csr_profiles_count: p_indptr (int64 [n_users + 1]) = the complete row pointers of P: p_indptr[0] = 0 and p_indptr[u + 1] -
 *   p_indptr[u] = the column count of row u.  One pass over every user; w_indices / x_indices may be NULL when W / X store nothing.
 * dae_csr_profiles: rows [first_user, first_user + n_fill) of P (n_fill >= 1), with p_indptr from dae_csr_profiles_count.  Entry t
 *   of row u goes to p_indices / p_values[p_indptr[u] - p_indptr[first_user] + t], the columns increasing within the row, so a
 *   caller can fill and use P a range of users at a time.  P[u, f] accumulates in fp32 from +0, one term per entry of row u of W
 *   in increasing article order, each term __fmul_rn(w, x) added with __fadd_rn (no FMA): the values do not depend on the launch
 *   shape or the range, and a float32 host loop reproduces them bit for bit.  normalise = 1 then divides each row by its L2 norm:
 *   n^2 = the fp32 sum of the rounded squares in increasing column order, v = __fdiv_rn(v, __fsqrt_rn(n^2)); a row with n^2 = 0 is
 *   left as it is.  Any user may read any number of articles.
 * dae_csr_impression_metrics: dae_impression_metrics for CSR query rows (q_indptr [n_imp + 1], row i the query of impression i)
 *   against the articles' CSR X (x_indptr [n_articles + 1], items in [0, n_articles)), columns < n_features in both.  scores[k] =
 *   q_i . x(items[k]): the fp32 sum from +0 of the rounded products over the shared columns in increasing column order, the score
 *   dae_csr_similarity_topk gives the same pair, bit for bit.  cosine = 1: dot / (sqrt(qq) sqrt(ee)), qq and ee the fp32 sums of
 *   the rounded squares of the rows in increasing column order, every operation IEEE-rounded; 0 when qq or ee is 0.  metrics as in
 *   dae_impression_metrics (the same device code).  q / x indices and values may be NULL when the matrix stores nothing.
 */
int dae_csr_profiles_count(const int64_t* w_indptr, const int32_t* w_indices, int32_t n_users, int32_t n_articles,
                           const int64_t* x_indptr, const int32_t* x_indices, int32_t n_features, int64_t* p_indptr, void* stream);
int dae_csr_profiles(const int64_t* w_indptr, const int32_t* w_indices, const float* w_values, int32_t n_users, int32_t n_articles,
                     const int64_t* x_indptr, const int32_t* x_indices, const float* x_values, int32_t n_features,
                     const int64_t* p_indptr, int32_t first_user, int32_t n_fill, int32_t normalise, int32_t* p_indices,
                     float* p_values, void* stream);
int dae_csr_impression_metrics(const int64_t* q_indptr, const int32_t* q_indices, const float* q_values, const int64_t* x_indptr,
                               const int32_t* x_indices, const float* x_values, int32_t n_articles, int32_t n_features, int32_t cosine,
                               const int64_t* indptr, const int32_t* items, const uint8_t* clicked, int64_t n_imp, float* scores,
                               double* metrics, void* stream);

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
