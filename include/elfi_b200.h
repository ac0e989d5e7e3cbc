/*
 * elfi_b200.h -- C ABI of libelfi_b200.so: the H100 (sm_90a) implementation of ELFI's
 * data-parallel sampler / BOLFI hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  ELFI is pure Python: the binding a
 * maintainer adds on the reference side is a ctypes stub (see INTEGRATION.md) called from
 * the node operations that `elfi.executor.Executor._run` invokes (elfi/executor.py:143-159)
 * and from the sampler bookkeeping in elfi/methods/inference/samplers.py.
 *
 * Conventions
 *   - every function returns 0 on success, <0 on error (ELFI_B200_ERR_*); the message for
 *     the calling host thread is available from elfi_b200_last_error();
 *   - all array arguments are caller-allocated DEVICE pointers unless the name ends in
 *     `_host`; matrices are row-major with a leading dimension given in ELEMENTS;
 *   - sizes are int64_t; `stream` is a cudaStream_t passed as void* (NULL = legacy default
 *     stream); kernels are asynchronous on that stream;
 *   - the context owns only scratch memory; it never takes ownership of caller buffers;
 *   - one context per device; a context may be used by one host thread and one stream at a
 *     time (its scratch arena is ordered by that stream; growing it synchronises the device).
 */
#ifndef ELFI_B200_H
#define ELFI_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ELFI_B200_VERSION 101

#define ELFI_B200_OK 0
#define ELFI_B200_ERR_ARG (-1)     /* invalid argument (shape, alignment, NULL) */
#define ELFI_B200_ERR_CUDA (-2)    /* a CUDA runtime / driver call failed */
#define ELFI_B200_ERR_NOMEM (-3)   /* scratch allocation failed */
#define ELFI_B200_ERR_UNSUPPORTED (-4)

#define ELFI_B200_MAX_NESTED 32    /* max nested distance columns K */

typedef struct elfi_b200_ctx elfi_b200_ctx;

/* ---- context ------------------------------------------------------------------------ */

int elfi_b200_version(void);
const char* elfi_b200_last_error(void);

/* Creates the context of CUDA device `device` (must be compute capability 9.0). */
int elfi_b200_ctx_create(int device, elfi_b200_ctx** out);
int elfi_b200_ctx_destroy(elfi_b200_ctx* ctx);
/* Number of SMs of the context's device (grid sizing is a multiple of this). */
int elfi_b200_ctx_sm_count(const elfi_b200_ctx* ctx);

/* ---- distance + acceptance ------------------------------------------------------------
 * Replaces, for the Euclidean family, the body of
 *   elfi/model/utils.py:37-52        distance_as_discrepancy  (column_stack + dist + flatten)
 *   elfi/model/elfi_model.py:1037    Distance -> scipy.spatial.distance.cdist(X, obs, 'euclidean')
 *   elfi/model/elfi_model.py:1135-1151  AdaptiveDistance.nested_distance (K weighted columns)
 * and the acceptance test of
 *   elfi/methods/inference/samplers.py:223-225   accepted = all_k(d[:, k] <= thr[k])
 *
 *   d[i, k] = sqrt( sum_j  W[k, j] * (S[i, j] - obs[j])^2 ),   j = 0 .. D-1 strictly in order,
 * every multiply and add rounded separately in fp64 (SciPy's order: bit-identical results).
 *
 *   S        (B, D) row-major, leading dimension ldS (elements)
 *   obs      (D)
 *   W        (K, D) row-major weights (cdist's `w`, i.e. 1/scale^2), or NULL = unweighted
 *            (K must then be 1; a row of ones is bit-identical to the unweighted form)
 *   K        number of nested distance columns, 1 <= K <= ELFI_B200_MAX_NESTED
 *   thr_host HOST pointer to K thresholds, or NULL = no acceptance test
 *   d_out    (B, K) row-major distances
 *   acc_idx  int32[B] ascending indices of accepted rows, or NULL (requires thr_host)
 *   n_acc    device int64[1] number of accepted rows (written when thr_host != NULL), or NULL
 */
int elfi_b200_dist_euclid_thr_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B,
                                  int64_t D, const double* obs, const double* W, int64_t K,
                                  const double* thr_host, double* d_out, int32_t* acc_idx,
                                  int64_t* n_acc, void* stream);

/* Same with the K thresholds in DEVICE memory (thr_dev, not NULL): a threshold that was itself
 * computed on the device -- the weighted quantile of the previous population
 * (samplers.py:542-549), the running n-th best distance of the buffer (samplers.py:243) -- feeds
 * the next distance call without a host round trip. */
int elfi_b200_dist_euclid_thr_dev_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B,
                                      int64_t D, const double* obs, const double* W, int64_t K,
                                      const double* thr_dev, double* d_out, int32_t* acc_idx,
                                      int64_t* n_acc, void* stream);

/* Distances + acceptance AND the per-column moments of the same batch from ONE read of S:
 * AdaptiveDistance evaluates its K nested columns (elfi_model.py:1135-1151) and then feeds the
 * batch to add_data (elfi_model.py:1104-1125); the reference reads S K + 1 times for that.
 * moments (2, D) device: row 0 = column means of the batch, row 1 = M2 = sum_i (x_ij - mean_j)^2
 * (what elfi_b200_colmoments_f64 returns; Chan-merged into (n, mean, M2) by the caller).
 * Accuracy of the moments (the distances stay bit-identical): as elfi_b200_colmoments_f64, with
 * the fused kernel's summation depth h = 8 rows per lane + 2 shuffle levels + ceil(B / 32 / nwarps)
 * tiles per warp + ceil(nwarps / 32) + 31 in the flush, nwarps = 8 or 12 per SM in use.
 * Thresholds: thr_host or thr_dev (at most one non-NULL; both NULL = no acceptance test).
 * W may be NULL only when the stand-alone moments pass is acceptable (the fused kernel is the
 * weighted / nested row stream; pass a row of ones for plain Euclidean distances). */
int elfi_b200_dist_euclid_mom_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B,
                                  int64_t D, const double* obs, const double* W, int64_t K,
                                  const double* thr_host, const double* thr_dev, double* d_out,
                                  int32_t* acc_idx, int64_t* n_acc, double* moments, void* stream);

/* Other cdist metrics that elfi.Distance forwards to SciPy (elfi/model/elfi_model.py:1016-1037):
 *   SQEUCLIDEAN  sum_j (S_ij - obs_j)^2          CITYBLOCK  sum_j |S_ij - obs_j|
 *   CHEBYSHEV    max_j |S_ij - obs_j|            MINKOWSKI  (sum_j |S_ij - obs_j|^pexp)^(1/pexp)
 * accumulated left to right in fp64 like SciPy does (the first three are bit-identical to cdist,
 * Minkowski to the accuracy of pow).  Unweighted, one distance column; otherwise the arguments and
 * the acceptance outputs are those of elfi_b200_dist_euclid_thr_f64 (d_out has B entries). */
#define ELFI_B200_METRIC_SQEUCLIDEAN 1
#define ELFI_B200_METRIC_CITYBLOCK 2
#define ELFI_B200_METRIC_CHEBYSHEV 3
#define ELFI_B200_METRIC_MINKOWSKI 4
int elfi_b200_dist_metric_thr_f64(elfi_b200_ctx* ctx, int32_t metric, double pexp, const double* S,
                                  int64_t ldS, int64_t B, int64_t D, const double* obs,
                                  const double* thr_host, double* d_out, int32_t* acc_idx,
                                  int64_t* n_acc, void* stream);

/* cdist(S, obs, 'seuclidean', V=V) (elfi/model/elfi_model.py:1016-1037 with the V keyword of the
 * Distance docstring, elfi_model.py:996-1003): d_i = sqrt(sum_j (S_ij - obs_j)^2 / V_j) in the
 * summation order of SciPy's compiled loop -- two running sums over the even and the odd columns of
 * the first D - D%2 columns, their sum, then the last term when D is odd -- with an IEEE division
 * per term, so the result is bit-identical to cdist.  V (D) device, strictly positive.  Other
 * arguments and the acceptance outputs as for elfi_b200_dist_metric_thr_f64. */
int elfi_b200_dist_seuclidean_thr_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B,
                                      int64_t D, const double* obs, const double* V,
                                      const double* thr_host, double* d_out, int32_t* acc_idx,
                                      int64_t* n_acc, void* stream);

/* cdist(S, obs, 'mahalanobis', VI=VI) (elfi/model/elfi_model.py:1016-1037 with the VI keyword of
 * the Distance docstring): with u = S_i - obs,
 *   t_r = TS_c(VI[r, c] * u_c)  over ROW r of VI,   q = TS_r(u_r * t_r),   d_i = sqrt(q),
 * TS being the summation order of SciPy's compiled loop that elfi_b200_dist_seuclidean_thr_f64
 * follows (two running sums over the even and the odd positions of the first D - D%2 terms, their
 * sum, then the last term when D is odd), every product and sum rounded on its own: bit-identical
 * to cdist for any VI, symmetric or not.  Non-finite inputs propagate; a VI that makes q < 0 gives
 * NaN, which no threshold accepts.  VI (D, D) row-major device.  1 <= D <=
 * ELFI_B200_MAHALANOBIS_D_MAX: each thread of a 128-thread CTA keeps its row of u in shared memory
 * next to a tile of 8 rows of VI.  Other arguments, the scratch use (the acceptance mask) and the
 * acceptance outputs as for elfi_b200_dist_metric_thr_f64. */
#define ELFI_B200_MAHALANOBIS_D_MAX 192
int elfi_b200_dist_mahalanobis_thr_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B,
                                       int64_t D, const double* obs, const double* VI,
                                       const double* thr_host, double* d_out, int32_t* acc_idx,
                                       int64_t* n_acc, void* stream);

/* ---- summary statistics ----------------------------------------------------------------
 * Row-wise summaries with NumPy's pairwise summation order (bit-identical results).
 *
 * elfi_b200_summary_autocov_f64 replaces elfi/examples/ma2.py:40-59 (autocov):
 *   out[i*ld_out + l] = mean_j( X[i, j+lag_l] * X[i, j] ),  j = 0 .. n-lag_l-1
 * for every lag in lags_host (HOST int32 array, 1 <= lag < n).  All lags of a call are
 * evaluated from one pass over X where possible (lags {1,2} fused), and written straight
 * into the column-stacked (B, nlags) summary matrix that the distance kernel consumes
 * (this is the np.column_stack of elfi/model/utils.py:39, done for free).
 *
 * elfi_b200_summary_meanvar_f64 replaces elfi/examples/gauss.py:142-173 (ss_mean, ss_var):
 *   out[i*ld_out + col_mean] = np.mean(X[i]),  out[i*ld_out + col_var] = np.var(X[i])
 * (either column index may be -1 to skip that statistic).
 */
int elfi_b200_summary_autocov_f64(elfi_b200_ctx* ctx, const double* X, int64_t ldX, int64_t B,
                                  int64_t n, const int32_t* lags_host, int64_t nlags, double* out,
                                  int64_t ld_out, void* stream);
int elfi_b200_summary_meanvar_f64(elfi_b200_ctx* ctx, const double* X, int64_t ldX, int64_t B,
                                  int64_t n, double* out, int64_t ld_out, int32_t col_mean,
                                  int32_t col_var, void* stream);

/* ---- ordering primitives ---------------------------------------------------------------
 * elfi_b200_sort_pairs_f64: stable ascending argsort of n fp64 keys (NaN last).  Replaces
 * np.argsort in Rejection._merge_batch (elfi/methods/inference/samplers.py:232-237) and in
 * weighted_sample_quantile (elfi/methods/utils.py:397).  keys_sorted and perm may each be
 * NULL.  (NumPy's default argsort is unstable; the two agree whenever keys are distinct.)
 *
 * elfi_b200_gather_rows_f64: dst[i, 0:width] = src[idx[i], 0:width] -- the fancy-index
 * permutation `v[:] = v[sort_mask]` / `batch[node][accepted]` (samplers.py:228-237).
 *
 * elfi_b200_accept_append_f64: `v[-num_accepted:] = batch[node][accepted]` for every output node
 * (samplers.py:228-230) with the counts read ON THE DEVICE, so a threshold-mode batch needs no
 * host round trip between the distance kernel and the merge: rows acc_idx[0 .. *n_acc) (acc_idx
 * == NULL: rows 0 .. *n_acc) of n_src <= 8 source arrays (src_host[k] = device pointer of a
 * (B, width_host[k]) array with leading dimension ld_src_host[k]; the three descriptor arrays
 * themselves are HOST arrays) are written side by side behind row *count of the packed candidate
 * buffer dst (capacity rows; NULL when capacity is 0); *count += rows appended; rows that do not
 * fit are dropped and counted in *dropped (may be NULL).  n_acc, count, dropped are DEVICE int64.
 * ld_dst >= the total width; columns beyond it are left untouched.  max_rows bounds
 * *n_acc (sizes the launch).  The best n rows are taken once, when the population is extracted
 * (sort_pairs on the distance column + gather_rows) -- the same rows the reference's per-batch
 * argsort over n + batch_size rows leaves in its buffer (samplers.py:232-237).
 */
int elfi_b200_sort_pairs_f64(elfi_b200_ctx* ctx, const double* keys, int64_t n,
                             double* keys_sorted, int32_t* perm, void* stream);
int elfi_b200_gather_rows_f64(elfi_b200_ctx* ctx, const double* src, int64_t ld_src,
                              const int32_t* idx, int64_t n, int64_t width, double* dst,
                              int64_t ld_dst, void* stream);
int elfi_b200_accept_append_f64(elfi_b200_ctx* ctx, const int32_t* acc_idx, const int64_t* n_acc,
                                int64_t max_rows, int64_t n_src, const double* const* src_host,
                                const int64_t* ld_src_host, const int64_t* width_host, double* dst,
                                int64_t ld_dst, int64_t capacity, int64_t* count, int64_t* dropped,
                                void* stream);
/* One batch of a threshold-mode rejection round in one call (Rejection.update ->
 * _merge_batch, samplers.py:140-230): elfi_b200_dist_euclid_thr[_dev]_f64 followed by
 * elfi_b200_accept_append_f64 of the rows [d (K columns) | extra sources] -- four launches, no
 * synchronisation, one host -> library transition.  Exactly one of thr_host / thr_dev is given. */
int elfi_b200_rejection_batch_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B,
                                  int64_t D, const double* obs, const double* W, int64_t K,
                                  const double* thr_host, const double* thr_dev, double* d_out,
                                  int32_t* acc_idx, int64_t* n_acc, int64_t n_extra,
                                  const double* const* extra_host, const int64_t* ld_extra_host,
                                  const int64_t* width_extra_host, double* dst, int64_t ld_dst,
                                  int64_t capacity, int64_t* count, int64_t* dropped, void* stream);

/* elfi_b200_topn_merge_f64: Rejection._merge_batch (samplers.py:226-237) in one call.  The
 * reference appends the accepted rows of a batch behind its best-n buffers, argsorts the distance
 * column over n + batch rows and permutes every output; here the virtual concatenation
 *     [A (nA rows of the current best-n) ; B[mapB] (nB accepted rows of the batch, mapB NULL = 0..nB-1)]
 * is ranked by its keys (keysA / keysB: the LAST distance column, addressed with a leading
 * dimension so that a column of a (rows, K) matrix can be passed in place; stable, NaN last) and
 * the n_keep smallest rows of each of the n_out outputs are gathered from their two sources:
 *     dst_host[k] (n_keep, width_host[k]) <- rows of A_host[k] (nA, width) / B_host[k] (batch, width).
 * The seven descriptor arrays are HOST arrays of length n_out; destinations must not alias sources.
 * merge_keys + 8-bit radix passes + one gather per output on `stream`, no synchronisation. */
int elfi_b200_topn_merge_f64(elfi_b200_ctx* ctx, const double* keysA, int64_t ld_keysA, int64_t nA,
                             const double* keysB, int64_t ld_keysB, const int32_t* mapB, int64_t nB,
                             int64_t n_keep, int64_t n_out, const double* const* A_host,
                             const int64_t* ldA_host, const double* const* B_host,
                             const int64_t* ldB_host, const int64_t* width_host,
                             double* const* dst_host, const int64_t* ld_dst_host, void* stream);

/* elfi_b200_topn_merge_seg_f64: R independent elfi_b200_topn_merge_f64 calls in one (the lock-step
 * Rejection repetitions of elfi_b200.Testbench).  Segment r = 0 .. R-1 ranks its virtual
 * concatenation [A_r (nA rows); B_r (nB rows)] by keys keysA + r seg_keysA (leading dimension
 * ld_keysA) and keysB + r seg_keysB, and gathers its n_keep smallest rows of each output k into
 * dst_host[k] + r seg_dst_host[k]; sources are A_host[k] + r segA_host[k] and
 * B_host[k] + r segB_host[k].  Segment strides and leading dimensions count doubles.  Each
 * segment's result is bit-identical to elfi_b200_topn_merge_f64 (mapB = NULL) on that segment:
 * stable, NaN last.  The 8 key passes run over all R (nA + nB) keys at once, then one more stable
 * 8-bit pass per byte of R - 1 sorts by segment.  Limits: R >= 1, R (nA + nB) < 2^31.  The ten
 * descriptor arrays are HOST arrays of length n_out; destinations must not alias sources.
 * Asynchronous on `stream`, deterministic. */
int elfi_b200_topn_merge_seg_f64(elfi_b200_ctx* ctx, int64_t R, const double* keysA,
                                 int64_t ld_keysA, int64_t seg_keysA, int64_t nA,
                                 const double* keysB, int64_t ld_keysB, int64_t seg_keysB,
                                 int64_t nB, int64_t n_keep, int64_t n_out,
                                 const double* const* A_host, const int64_t* ldA_host,
                                 const int64_t* segA_host, const double* const* B_host,
                                 const int64_t* ldB_host, const int64_t* segB_host,
                                 const int64_t* width_host, double* const* dst_host,
                                 const int64_t* ld_dst_host, const int64_t* seg_dst_host,
                                 void* stream);

/* elfi_b200_wquantile_f64: weighted_sample_quantile (elfi/methods/utils.py:379-411).
 *   x (n), w (n) or NULL (equal weights), 0 <= alpha <= 1.
 *   out[0] = alpha-quantile (an element of x), out[1] = its rank in sorted order (as double).
 * np.sum (pairwise) and np.cumsum (sequential) are reproduced in the reference's order, so
 * the selected element is identical even when alpha falls exactly on a cumulative weight
 * (equal weights + round alpha, the normal case in SMC round 0).  A parallel scan with a rigorous
 * error bound answers first; the sequential kernel only runs when alpha is within that bound of a
 * cumulative weight.  With w == NULL the position follows in closed form from n and alpha (the
 * sequential sum of n copies of 1/n is an arithmetic progression per binade) and nothing is
 * scanned.  The call synchronises `stream` unless w == NULL. */
int elfi_b200_wquantile_f64(elfi_b200_ctx* ctx, const double* x, const double* w, int64_t n,
                            double alpha, double* out, void* stream);

/* ---- SMC population arithmetic ---------------------------------------------------------
 * elfi_b200_colmoments_f64: per-column mean and M2 = sum_i (x_ij - mean_j)^2 of one (B, D)
 * batch: out[0:D] = mean, out[D:2D] = M2.  The host merges batches with Chan's formula,
 * which is algebraically AdaptiveDistance.add_data (elfi/model/elfi_model.py:1104-1125);
 * parity is tolerance-level (the reference itself only promises np.std agreement,
 * tests/unit/test_elfi_model.py:185-253).
 *   Accuracy: the sums run over d_i = x_ij - x_0j (shift = first row), so with u = 2^-53,
 *   gamma_k = k u / (1 - k u) and summation depth h = ceil(R / 8) + 7 + ceil(B / R), where
 *   R = max(64, ceil(B / ceil(8 sm_count / ceil(D / 32)))) rows go to one block:
 *     |M2^ - M2|     <= 4 gamma_{h+3} sum_i d_i^2 <= 4 gamma_{h+3} (B + 1) M2,
 *     |mean^ - mean| <= u |mean| + gamma_{h+2} sum_i |d_i| / B.
 *   sum_i d_i^2 <= (B + 1) M2 because x_0 is one of the data: the cancellation is bounded
 *   whatever the offset of the column.  A constant column gives M2 = 0.0 exactly.  The derivation
 *   and the checks are in tests/rowstream_cases.py.
 *
 * elfi_b200_weighted_stats_f64: weighted_var and its ingredients (elfi/methods/utils.py:108-139):
 *   stats = [V1 = sum w, V2 = sum w^2, xbar_0..p-1 = np.average(x, weights=w),
 *            s2_0..p-1 = sum w (x - xbar)^2 / (V1 - V2/V1)],   w == NULL means all ones.
 *   With fewer than two nonzero weights (N = 1 included) the denominator is exactly zero and s2
 *   is non-finite (SMC then falls back to the unit covariance), even where the rounded
 *   V2 / V1 would miss V1 by an ulp.
 *
 * elfi_b200_gm_logpdf_f64: GMDistribution.logpdf (elfi/methods/utils.py:146-197) --
 *   logq[i] = log sum_j (w_j / sum w) N(x_i; means_j, Sigma), plain sum of densities as in the
 *   reference (no log-sum-exp shift), Sigma shared.  Linv_host = inverse of the lower Cholesky
 *   factor of Sigma (HOST, p x p row-major), logdet = log det Sigma.  p <= 16.
 *   Tolerance: <= 1e-8 relative on q (range-reduced exp with a degree-6 minimax polynomial, max
 *   term error 1.9e-9; fp64 accumulation).
 * elfi_b200_gm_logpdf_mixed_f64: the same density with 2^f taken from the special-function unit in
 *   fp32 (range reduction and accumulation stay fp64): fewer fp64 instructions per term, term
 *   error <= 2.5e-7 (ex2.approx.f32's 2 ulp, 2^-22 relative just above 1.0, plus the fp32
 *   rounding of the fraction, ln 2 * 2^-26) -- used where parity with the reference is
 *   statistical anyway (throughput mode: device RNG), 40x inside the 1e-5 tolerance on SMC weights.
 *   Both: terms (w_j / sum w) exp(-maha_ij / 2) below 2^-1020 are flushed to zero, and logq[i]
 *   = -inf where all of them are; the reference underflows only below 2^-1074, with the
 *   normaliser inside the exp, so in a narrow band of far-out points the two differ.
 *
 * elfi_b200_smc_weights_f64: w_i = exp(logprior_i - logq_i) (samplers.py:514).
 */
int elfi_b200_colmoments_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B, int64_t D,
                             double* out, void* stream);
int elfi_b200_weighted_stats_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, const double* w,
                                 int64_t N, int64_t p, double* stats, void* stream);
int elfi_b200_gm_logpdf_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t N,
                            const double* means, int64_t ldm, const double* w, int64_t M, int64_t p,
                            const double* Linv_host, double logdet, double* logq, void* stream);
int elfi_b200_gm_logpdf_mixed_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t N,
                                  const double* means, int64_t ldm, const double* w, int64_t M,
                                  int64_t p, const double* Linv_host, double logdet, double* logq,
                                  void* stream);
int elfi_b200_smc_weights_f64(elfi_b200_ctx* ctx, const double* logprior, const double* logq,
                              int64_t n, double* w, void* stream);

/* ---- BOLFI Gaussian-process surrogate (fp64) -------------------------------------------------
 * RBF + bias kernel k(a, b) = kernel_var * exp(-|a-b|^2 / (2 lengthscale^2)) + bias_var, Gaussian
 * noise.  These replace the GPy calls behind elfi/methods/bo/gpy_regression.py:
 *   update()/_init_gp() (242-315): Gram + Cholesky of Ky = K + noise_var I  -> elfi_b200_gp_fit_f64
 *   predict()/predict_mean() (98-163), incl. the cached-RBF restatement (127-140)
 *                                                                   -> elfi_b200_gp_predict_f64
 *   predictive_gradients() (186-223, restatement 206-218)           -> elfi_b200_gp_predict_grad_f64
 * and LCBSC.evaluate / evaluate_gradient (elfi/methods/bo/acquisition.py:262-301)
 *                                                                   -> `acq` outputs / elfi_b200_lcbsc_f64
 *
 * Factor storage (caller-allocated, n_pad x n_pad row-major, n_pad = elfi_b200_gp_padded_size(n)):
 *   L lower Cholesky factor (padded with the identity), W = L^-1, U = W^T;  alpha = Ky^-1 y (n).
 * As in LAPACK's potrf, only the lower triangle of L[0:n, 0:n] is the factor: its strict upper
 * triangle is workspace and holds unspecified values.  The padding rows and columns of L, W and U
 * hold the identity (exact zeros off the diagonal), and W (U) has exact zeros above (below) the
 * diagonal.  noise_var must already include any jitter (GPy adds 1e-8).  info (device int32) is
 * 0 on success or 1 + the index of the first non-positive (or NaN) pivot; L, W, U and alpha are
 * then unspecified.
 * gp_predict: mean/var/acq may each be NULL; var = k** - |W k|^2 + noise_add; acq = mean -
 * sqrt(beta * (noiseless var)).  Queries are processed in chunks through context scratch.
 */
int64_t elfi_b200_gp_padded_size(int64_t n);
int elfi_b200_gp_fit_f64(elfi_b200_ctx* ctx, const double* X, int64_t ldX, const double* y,
                         int64_t n, int64_t p, double kernel_var, double lengthscale,
                         double bias_var, double noise_var, double* L, double* W, double* U,
                         int64_t n_pad, double* alpha, int32_t* info, void* stream);
int elfi_b200_gp_predict_f64(elfi_b200_ctx* ctx, const double* Xq, int64_t ldq, int64_t m,
                             const double* X, int64_t ldX, int64_t n, int64_t p, const double* W,
                             int64_t n_pad, const double* alpha, double kernel_var,
                             double lengthscale, double bias_var, double noise_add, double beta,
                             double* mean, double* var, double* acq, void* stream);
int elfi_b200_gp_predict_grad_f64(elfi_b200_ctx* ctx, const double* Xq, int64_t ldq, int64_t m,
                                  const double* X, int64_t ldX, int64_t n, int64_t p,
                                  const double* W, const double* U, int64_t n_pad,
                                  const double* alpha, double kernel_var, double lengthscale,
                                  double bias_var, double* mean, double* var, double* grad_mean,
                                  double* grad_var, void* stream);
int elfi_b200_lcbsc_f64(elfi_b200_ctx* ctx, const double* mean, const double* var,
                        const double* grad_mean, const double* grad_var, int64_t m, int64_t p,
                        double beta, double* acq, double* grad_acq, void* stream);

/* Posterior cross-covariance of the GP between two sets of points, as ExpIntVar needs it
 * (elfi/methods/bo/acquisition.py:776-821; the reference re-factorises Ky on every evaluation,
 * :807).  With W from gp_fit, cov(x_a, x_b) = k(x_a, x_b) - (W k_a) . (W k_b):
 *   gp_whiten:    T[q, 0:n] = W k_q,  k_q[j] = k(Xq[q], X[j])  (RBF + bias);  T is (m, ldT), ldT >= n
 *   gp_cross_cov: cov[b * ma + a] = k(Xa[a], Xb[b]) - Ta[a, :] . Tb[b, :]     (mb x ma, row-major) */
int elfi_b200_gp_whiten_f64(elfi_b200_ctx* ctx, const double* Xq, int64_t ldq, int64_t m,
                            const double* X, int64_t ldX, int64_t n, int64_t p, const double* W,
                            int64_t n_pad, double kernel_var, double lengthscale, double bias_var,
                            double* T, int64_t ldT, void* stream);
/* out[q, 0:n] = W^T T[q, 0:n] (U = W^T from gp_fit): with T = gp_whiten(X_new) these are the rows
 * T W that a rank-b update of the factor (b new evidence points appended, no refit) needs. */
int elfi_b200_gp_apply_wt_f64(elfi_b200_ctx* ctx, const double* T, int64_t ldT, int64_t m,
                              const double* U, int64_t n_pad, int64_t n, double* out, int64_t ldo,
                              void* stream);
int elfi_b200_gp_cross_cov_f64(elfi_b200_ctx* ctx, const double* Xa, int64_t lda, int64_t ma,
                               const double* Ta, int64_t ldTa, const double* Xb, int64_t ldb,
                               int64_t mb, const double* Tb, int64_t ldTb, int64_t n, int64_t p,
                               double kernel_var, double lengthscale, double bias_var, double* cov,
                               void* stream);

/* Measures the sustained fp64 throughput of this device: tflops_host[0] = DFMA (vector pipe),
 * tflops_host[1] = DMMA (mma.sync m8n8k4.f64).  Roofline denominators for the compute-bound
 * kernels (mixture density, GP products); blocks the host for a few milliseconds. */
int elfi_b200_probe_fp64_f64(elfi_b200_ctx* ctx, double* tflops_host);

/* ---- throughput mode: device-side generation (SURVEY.md section 8f, N2) --------------------
 * Counter-based Philox4x32-10 streams keyed by (seed, offset + row): statistically equivalent to,
 * not bit-identical with, the reference's host RandomState.  `offset` = global index of the first
 * row of this call (e.g. batch_index * batch_size), so that any row sharding yields the same
 * particles.
 *   elfi_b200_prior_ma2_f64     CustomPrior1 / CustomPrior2 draws (elfi/examples/ma2.py:96-186);
 *                               mode 0 = (t1, t2) jointly, 1 = t1 only, 2 = t2 given the t1 passed in
 *   elfi_b200_logprior_ma2_f64  their joint log density (what ModelPrior.logpdf returns for MA2)
 *   elfi_b200_sim_ma2_f64       MA2 simulator (ma2.py:11-37); writes X (B, n_obs) and/or, fused,
 *                               the lag-1 / lag-2 autocovariances S (B, 2) (ma2.py:40-59, NumPy
 *                               pairwise order) so that X never has to touch HBM
 *   elfi_b200_gm_cdf_f64        inclusive running sum of the (unnormalised) component weights, the
 *                               table np.random.choice(p=weights) builds on every call
 *                               (utils.py:239); one per population, reused by every batch of it.
 *                               Nondecreasing whatever the weights (>= 0), so a zero-weight
 *                               component is never drawn; deterministic
 *   elfi_b200_gm_rvs_cdf_f64    GMDistribution.rvs (elfi/methods/utils.py:200-261) with that table
 *                               (`cumw`, device, N): component by weight, + MVN(0, Sigma) with
 *                               Sigma = L L^T (Lchol_host, p <= 16), redrawn until inside the
 *                               support (0 = none, 1 = MA2 prior support (p = 2), 2 = box:
 *                               box_host = [lo_0..lo_{p-1}, hi_0..hi_{p-1}], 3 = prior: box_host =
 *                               the 5p-word prior table of elfi_b200_prior_logpdf_f64, a draw is
 *                               kept iff its joint log density is finite; 4 = the same with the
 *                               7p-word table of conditional priors).  At most 1000 draws per row:
 *                               when all of them fall outside the support, the 1000th draw is
 *                               returned as it is (outside the support).  For p <= 4 with supports
 *                               0-2 the streams are those of earlier versions; support 3 uses the
 *                               same blocks, and z_4 .. z_15 come from a stream of their own
 */
int elfi_b200_prior_ma2_f64(elfi_b200_ctx* ctx, int64_t B, uint64_t seed, uint64_t offset,
                            int32_t mode, double* t1, double* t2, void* stream);
int elfi_b200_logprior_ma2_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B,
                               double* out, void* stream);
int elfi_b200_sim_ma2_f64(elfi_b200_ctx* ctx, const double* t1, const double* t2, int64_t B,
                          int64_t n_obs, uint64_t seed, uint64_t offset, double* X, int64_t ldX,
                          double* S, int64_t ldS, void* stream);
int elfi_b200_gm_cdf_f64(elfi_b200_ctx* ctx, const double* weights, int64_t N, double* cumw,
                         void* stream);
int elfi_b200_gm_rvs_cdf_f64(elfi_b200_ctx* ctx, const double* means, int64_t ldm, const double* cumw,
                             int64_t N, int64_t p, const double* Lchol_host, int64_t B, uint64_t seed,
                             uint64_t offset, int32_t support, const double* box_host, double* out,
                             int64_t ldo, void* stream);

/* Stock scipy.stats priors (uniform, norm, truncnorm, expon, gamma, beta) on the device: the
 * throughput-mode fast path of ModelPrior for independent priors with constant parameters.
 * A parameter is five doubles [kind, p0, p1, p2, p3] with scipy's positional parameters, loc and
 * scale filled in: 0 uniform (loc, scale), 1 norm (loc, scale), 2 truncnorm (a, b, loc, scale),
 * 3 expon (loc, scale), 4 gamma (a, loc, scale), 5 beta (a, b, loc, scale); unused words ignored.
 * Invalid parameters (scale <= 0, truncnorm a >= b, gamma a <= 0, beta a or b <= 0, an unknown
 * kind, non-finite values) return ELFI_B200_ERR_ARG with a message naming the parameter index.
 *   elfi_b200_prior_rvs_f64     B draws of ONE parameter (spec_host: 5 words) into out (B,);
 *                               row i is a pure function of (seed, offset + i).  Uniform, norm,
 *                               truncnorm (inverse CDF, mirrored in the upper tail) and expon take
 *                               one Philox block per row; gamma and beta use Marsaglia-Tsang
 *                               (stream layout in elfi_b200/csrc/prior.cu) with at most 64 trials
 *                               per gamma component.  If all 64 are rejected (probability below
 *                               1e-80 for every valid shape) the component's value is
 *                               d = a - 1/3 (a >= 1) or a + 2/3 (a < 1), a point of the support
 *   elfi_b200_prior_logpdf_f64  joint log density of p <= ELFI_B200_MAX_PRIOR_PARAMS independent
 *                               parameters at the rows of x (B, p; leading dimension ldx): the sum,
 *                               left to right, of scipy.stats.<kind>.logpdf, -inf outside the
 *                               closed support and scipy's values on its edges (spec_host: 5p
 *                               words)
 *
 * Conditional loc / scale (a hierarchical prior such as t2 ~ U(t1, t1 + 10)): the 7-word form
 * [kind, p0, p1, p2, p3, loc_src, scale_src] takes the loc and / or the scale of a parameter from
 * column loc_src / scale_src of the same row (-1: the constant word; j: column j, 0 <= j < p, not
 * the parameter itself).  A sourced word among the first five is a placeholder and is not
 * validated; shape parameters are always constants; a bad source returns ELFI_B200_ERR_ARG.  Per
 * row, as SciPy 1.18.1:
 *   logpdf: a scale that is not > 0, or NaN, gives NaN; a NaN loc gives NaN; an infinite scale
 *           gives -inf for uniform (y = 0 and -log(inf)).  A sourced scale takes its log on the
 *           device, a constant one keeps the host's; with every source -1 the result is the bits
 *           of the 5-word table.
 *   rvs:    a scale of 0 gives loc; a NaN loc gives NaN; a scale < 0 or NaN gives NaN (where
 *           SciPy raises).
 *   elfi_b200_prior_rvs_cond_f64     prior_rvs with per-row loc and / or scale: `loc`, `scale` are
 *                                    device (B,) vectors or NULL (then spec_host's word is used);
 *                                    out[i] = fma(scale_i, y_i, loc_i) with y_i the standard draw
 *                                    of the same stream as elfi_b200_prior_rvs_f64 (which computes
 *                                    fma(scale, y_i, loc)); with both NULL the two are the same bits
 *   elfi_b200_prior_logpdf_cond_f64  prior_logpdf with the 7p-word table
 *   elfi_b200_gm_rvs_cdf_f64 with support = 4: box_host is the 7p-word table; the draws use the
 *                                    blocks of support 3, so with every source -1 they are its bits
 */
#define ELFI_B200_MAX_PRIOR_PARAMS 16       /* parameters p of one prior table */
#define ELFI_B200_PRIOR_SPEC_WORDS 5        /* [kind, p0, p1, p2, p3] per parameter */
#define ELFI_B200_PRIOR_COND_SPEC_WORDS 7   /* [kind, p0, p1, p2, p3, loc_src, scale_src] */
int elfi_b200_prior_rvs_f64(elfi_b200_ctx* ctx, const double* spec_host, int64_t B, uint64_t seed,
                            uint64_t offset, double* out, void* stream);
int elfi_b200_prior_logpdf_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B, int64_t p,
                               const double* spec_host, double* out, void* stream);
int elfi_b200_prior_rvs_cond_f64(elfi_b200_ctx* ctx, const double* spec_host, int64_t B,
                                 uint64_t seed, uint64_t offset, const double* loc,
                                 const double* scale, double* out, void* stream);
int elfi_b200_prior_logpdf_cond_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B,
                                    int64_t p, const double* spec_host, double* out, void* stream);

/* Gaussian noise model of elfi/examples/gauss.py (1-d case): priors mu ~ U(prm[0], prm[0]+prm[1]),
 * sigma ~ truncnorm(prm[2], prm[3]) (gauss.py:118-126); simulator y = mu + sigma z (gauss.py:11-35)
 * with np.mean / np.var summaries (gauss.py:142-173, pairwise order) fused in the same kernel
 * (S (B, 2) = [mean, var]); Y (B, n_obs) is written only when requested. */
int elfi_b200_prior_gauss_f64(elfi_b200_ctx* ctx, int64_t B, uint64_t seed, uint64_t offset,
                              const double* prm_host, double* mu, double* sigma, void* stream);
int elfi_b200_logprior_gauss_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B,
                                 const double* prm_host, double* out, void* stream);
int elfi_b200_sim_gauss_f64(elfi_b200_ctx* ctx, const double* mu, const double* sigma, int64_t B,
                            int64_t n_obs, uint64_t seed, uint64_t offset, double* Y, int64_t ldY,
                            double* S, int64_t ldS, void* stream);

/* g-and-k model of elfi/examples/gnk.py (throughput mode, statistical parity).
 * sim_gnk: Y[i, j] = A_i + B_i (1 + c (1 - exp(-g_i z)) / (1 + exp(-g_i z))) (1 + z^2)^k_i z with
 * z = z_ij ~ N(0, 1) from the Philox stream (seed, offset + i, j) (gnk.py:11-68); Y is (B, n_obs)
 * with leading dimension ldY.  The order-statistic summary is elfi_b200_rowsort_f64 on Y.
 * logprior_box: sum of independent uniform log densities, box_host = [lo (p), width (p)], p <= 8
 * (the priors A, B, g, k ~ uniform(0, 10) of gnk.py:99-103); -inf outside. */
int elfi_b200_sim_gnk_f64(elfi_b200_ctx* ctx, const double* A, const double* Bs, const double* g,
                          const double* k, double c, int64_t B, int64_t n_obs, uint64_t seed,
                          uint64_t offset, double* Y, int64_t ldY, void* stream);
int elfi_b200_logprior_box_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t B, int64_t p,
                               const double* box_host, double* out, void* stream);

/* Robust and octile g-and-k summaries (elfi/examples/gnk.py:164-248), bit for bit.
 * kind 0 = ss_robust: [L2, ss_B, ss_g, ss_k] per dimension; kind 1 = ss_octile: [E1 .. E7].
 * The output row is laid out as the reference's np.hstack: value j of dimension a at
 * out[i * ld_out + j * d + a].  picks_host = lo[7], hi[7], t[7] (doubles) of
 * np.percentile(.., [12.5, 25, .., 87.5], method='linear') for the series length (ops.gnk_picks):
 * value = t >= 0.5 ? b - (b - a)(1 - t) : a + (b - a) t with a, b the sorted elements lo, hi.
 * NaN rules as NumPy's: a NaN in a series makes all its octiles NaN; an infinity at a picked
 * position with t = 0 gives NaN through (inf - a) * 0; ss_B = 0 becomes eps.
 * gnk_summaries: series (i, a) of a data matrix is X[i * ld_row + j * ld_obs + a], j < n,
 *   1 <= n <= ELFI_B200_GNK_SERIES_MAX, d in {1, 2}.
 * sim_gnk_summaries: the summaries of the rows elfi_b200_sim_gnk_f64 would simulate, without
 *   writing them (1 <= n_obs <= ELFI_B200_GNK_FUSED_MAX); equal to sim_gnk followed by
 *   gnk_summaries.
 * sim_bignk: bivariate g-and-k (elfi/examples/bignk.py:12-108).  P[i * ldP + 0..8] = A1, A2, B1, B2,
 *   g1, g2, k1, k2, rho.  Observation j of row i: Philox block (seed, offset + i, j) gives n0, n1;
 *   z1 = n0, z2 = rho n0 + sqrt(1 - rho^2) n1, y_a = the g-and-k quantile of (A_a, B_a, g_a, k_a, c)
 *   at z_a.  |rho| > 1 or NaN gives NaN rows.  Y (B, n_obs, 2) with leading dimension ldY (may be
 *   NULL); S (B, 2 * width) fused summaries of kind `kind` (may be NULL, needs
 *   n_obs <= ELFI_B200_GNK_FUSED_MAX).
 * euclidean_multiss (gnk.py:115-142) on (B, K, 1) summaries stored as (B, K) with leading dimension
 *   ldS, K <= 128, obs (K) on the device: out[i] = sqrt(sum_j (S[i, j] - obs[j])^2), summed in
 *   NumPy's pairwise order. */
#define ELFI_B200_GNK_SERIES_MAX 2048   /* series length of gnk_summaries: the shared-memory sort */
#define ELFI_B200_GNK_FUSED_MAX 512     /* n_obs of the fused summaries: 32 lanes x 16 keys */
int elfi_b200_gnk_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_row, int64_t ld_obs,
                                int64_t B, int64_t n, int64_t d, int32_t kind,
                                const double* picks_host, double* out, int64_t ld_out, void* stream);
int elfi_b200_sim_gnk_summaries_f64(elfi_b200_ctx* ctx, const double* A, const double* Bs,
                                    const double* g, const double* k, double c, int64_t B,
                                    int64_t n_obs, uint64_t seed, uint64_t offset, int32_t kind,
                                    const double* picks_host, double* out, int64_t ld_out,
                                    void* stream);
int elfi_b200_sim_bignk_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, double c, int64_t B,
                            int64_t n_obs, uint64_t seed, uint64_t offset, double* Y, int64_t ldY,
                            int32_t kind, const double* picks_host, double* S, int64_t ldS,
                            void* stream);
int elfi_b200_euclidean_multiss_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B,
                                    int64_t K, const double* obs, double* out, void* stream);

/* Ricker model of elfi/examples/ricker.py (throughput mode, statistical parity); stream layout,
 * algorithms and limits in elfi_b200/csrc/ricker.cu and poisson.cuh.
 * poisson: out[i] ~ Poisson(lam[i]) (device vectors of n doubles), a pure function of
 *   (seed, offset + i).  Inversion for lam < 10, PTRS (Hoermann 1993) with a cancellation-free
 *   log-pmf test above.  lam == 0 gives 0; lam < 0, NaN or lam > ELFI_B200_POISSON_LAM_MAX
 *   (NumPy's limit, where NumPy raises) give NaN.  PTRS takes at most 32 trials (each rejected
 *   with probability below 0.12); if all 32 are rejected the draw is floor(lam).  The inversion
 *   search stops at 64.  Counts are doubles.
 * sim_ricker: one row per parameter row P[i * ldP + ..]: n_params 3 = (r, sigma, phi), the
 *   stochastic model N_t = N_{t-1} exp((r - N_{t-1}) + sigma e_t) from N_{-1} = stock_init and
 *   Y_t ~ Poisson(phi N_t), t < n_obs; n_params 1 = (r), the deterministic model Y_0 = stock_init,
 *   Y_t = Y_{t-1} exp(r - Y_{t-1}) (N = Y).  1 <= n_obs <= ELFI_B200_RICKER_NOBS_MAX.
 *   Y (B, n_obs; ldY), N (B, n_obs; ldN) and S (B, 3; ldS) may each be NULL.
 *   S = [np.mean(Y), np.var(Y), number of zeros of Y] per row, computed in the simulator without
 *   writing Y (needs n_obs <=
 *   ELFI_B200_RICKER_FUSED_MAX); equal bit for bit to summary_meanvar and count_zeros of Y.
 * count_zeros: out[i * ld_out] = the number of entries of row i of X (B, n; ldX) equal to 0, as a
 *   double (num_zeros of ricker.py).
 * chi_squared (ricker.py:147-161) on summaries S (B, K; ldS), K <= 128, obs (K) on the device:
 *   out[i] = sum_j (S[i, j] - obs[j])^2 / obs[j] summed in NumPy's pairwise order; obs[j] = 0
 *   gives NumPy's inf / NaN terms. */
#define ELFI_B200_POISSON_LAM_MAX 9.223372006484771e18   /* NumPy's POISSON_LAM_MAX */
#define ELFI_B200_RICKER_NOBS_MAX 16777216   /* 2^24: t << 8 fits the 32-bit block word */
#define ELFI_B200_RICKER_FUSED_MAX 128       /* fused summaries: one leaf of NumPy's pairwise sum */
int elfi_b200_poisson_f64(elfi_b200_ctx* ctx, const double* lam, int64_t n, uint64_t seed,
                          uint64_t offset, double* out, void* stream);
int elfi_b200_sim_ricker_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t n_params,
                             int64_t B, int64_t n_obs, double stock_init, uint64_t seed,
                             uint64_t offset, double* Y, int64_t ldY, double* N, int64_t ldN,
                             double* S, int64_t ldS, void* stream);
int elfi_b200_count_zeros_f64(elfi_b200_ctx* ctx, const double* X, int64_t ldX, int64_t B, int64_t n,
                              double* out, int64_t ld_out, void* stream);
int elfi_b200_chi_squared_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B, int64_t K,
                              const double* obs, double* out, void* stream);

/* The 13 Ricker statistics of Wood (2010, Nature 466:1102) in this project's reading (ss_wood of
 * elfi_b200/examples/ricker.py defines them in NumPy); layout in elfi_b200/csrc/ricker_wood.cu.
 * Row i of Y (B, n; ldY >= n), ELFI_B200_RICKER_WOOD_NOBS_MIN <= n <=
 * ELFI_B200_RICKER_WOOD_NOBS_MAX, gives out[i * ld_out + 0..12] (ld_out >=
 * ELFI_B200_RICKER_WOOD_WIDTH):
 *   0 mean; 1 number of zeros; 2..7 autocovariances sum_t (y_t - m)(y_{t+k} - m) / n, k = 0..5;
 *   8..10 P e, e the sorted differences y_{t+1} - y_t and P (3 x (n-1), row-major, on the device)
 *   the pseudo-inverse of [o, o^2, o^3] for the sorted observed differences o;
 *   11..12 the minimum-norm least-squares (a1, a2) of y_{t+1}^0.3 = a1 y_t^0.3 + a2 y_t^0.6.
 * Rank rule of (a1, a2), with N the distinct nonzero values among y_0 .. y_{n-2}: N empty gives
 * (0, 0); N = {k} gives s (k^0.3, k^0.6) / (k^0.6 + k^1.2), s the mean of y_{t+1}^0.3 over the t
 * with y_t = k; otherwise the normal equations of the two columns.
 * Accuracy against the host definition on the same row:
 *   * columns 0..7 are bit-identical for every n (NumPy's pairwise summation order, also above
 *     128 terms);
 *   * column 8 + j is within 2 (n-1) 2^-53 sum_t |P_jt e_t|;
 *   * the branch of the rank rule is the same, and on rows of full column rank (a1, a2) is within
 *     1e3 2^-53 cond([u v])^2 relative (u, v the two regressor columns).
 * A row with a non-finite value gives 13 NaN.  Results are bit-identical across calls and do not
 * depend on B or on the other rows; B = 0 is a no-op. */
#define ELFI_B200_RICKER_WOOD_NOBS_MIN 7
#define ELFI_B200_RICKER_WOOD_NOBS_MAX 2048   /* the shared-memory sort of the differences */
#define ELFI_B200_RICKER_WOOD_WIDTH 13
int elfi_b200_ricker_wood_f64(elfi_b200_ctx* ctx, const double* Y, int64_t ldY, int64_t B, int64_t n,
                              const double* P, double* out, int64_t ld_out, void* stream);

/* Lorenz forecast model of elfi/examples/lorenz.py (throughput mode, statistical parity); stream
 * layout, lane layout and arithmetic in elfi_b200/csrc/lorenz.cu and lorenz.cuh.
 * sim_lorenz: row i has parameters (theta1, theta2) = P[i * ldP], P[i * ldP + 1] (ldP >= 2) and
 *   starts from init (n_obs doubles on the device); for s = 1 .. n_timestep - 1 it draws e (n_obs
 *   normals, a pure function of (seed, offset + i, s, k): Box-Muller normal (k & 1) of Philox block
 *   (s << 6) | (k >> 1)), sets eta = phi * eta + e * s_phi and takes one RK4 step of length dt.
 *   s_phi = sqrt(1 - phi^2) and dt = total_duration / n_timestep are computed by the caller
 *   (phi > 1 gives NaN rows, as in the reference).
 *   ELFI_B200_LORENZ_NOBS_MIN <= n_obs <= ELFI_B200_LORENZ_NOBS_MAX, 2 <= n_timestep <=
 *   ELFI_B200_LORENZ_T_MAX.
 *   X (B, n_timestep, n_obs), C-contiguous, may be NULL; S (B, 6; ldS >= 6) may be NULL and needs
 *   n_timestep * n_obs <= ELFI_B200_LORENZ_SUMM_MAX_TERMS.  With S and without X the summaries are
 *   computed in the simulator from a per-warp scratch slab (up to 512 MiB of the context's scratch,
 *   independent of B); with both, X is written and summarised.  Either way S equals
 *   lorenz_summaries of X bit for bit.
 * lorenz_summaries: S[i * ldS + 0..5] = [Mean, Var, Autocov, Cov, CrosscovPrev, CrosscovNext]
 *   (lorenz.py:231-320) of the row X[i * ld_row + t * ld_t + k * ld_k] (n_timestep, n_obs), bit for
 *   bit NumPy's on a C-contiguous array; ELFI_B200_LORENZ_SUMM_NOBS_MIN <= n_obs <=
 *   ELFI_B200_LORENZ_NOBS_MAX (with one variable NumPy sums over time pairwise), n_timestep >= 2,
 *   n_timestep * n_obs <= ELFI_B200_LORENZ_SUMM_MAX_TERMS.  NaN and inf propagate as in NumPy. */
#define ELFI_B200_LORENZ_NOBS_MIN 4             /* variables of the ring of sim_lorenz */
#define ELFI_B200_LORENZ_NOBS_MAX 128
#define ELFI_B200_LORENZ_SUMM_NOBS_MIN 2
#define ELFI_B200_LORENZ_T_MAX 67108864         /* 2^26: s << 6 fits the 32-bit block word */
#define ELFI_B200_LORENZ_SUMM_MAX_TERMS 30728   /* (120 << 8) + 8, what PairwiseLeaves<8> sums */
int elfi_b200_sim_lorenz_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                             int64_t n_obs, int64_t n_timestep, const double* init, double f,
                             double phi, double s_phi, double dt, uint64_t seed, uint64_t offset,
                             double* X, double* S, int64_t ldS, void* stream);
int elfi_b200_lorenz_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_row,
                                   int64_t ld_t, int64_t ld_k, int64_t B, int64_t n_timestep,
                                   int64_t n_obs, double* S, int64_t ldS, void* stream);

/* Toad movement model of elfi/examples/toad.py (throughput mode, statistical parity); stream
 * layout, thread layout and arithmetic in elfi_b200/csrc/toad.cu and toad.cuh.
 * sim_toad: row i has parameters (alpha, gamma, p0) = P[i * ldP + 0..2] (ldP >= 3).  Every toad
 *   starts at 0; on day d >= 1 toad k returns (its uniform < p0) to its position of day j, j
 *   uniform in [0, d), or steps from day d - 1 by gamma times a symmetric alpha-stable variate
 *   (SciPy's levy_stable, S1, beta = 0).  The draws of (d, k) are a pure function of
 *   (seed, offset + i, d, k): Philox blocks (c << 1) | 0 and (c << 1) | 1 with c = d * n_toads + k.
 *   alpha outside (0, 2] or gamma < 0 or NaN (where the reference raises) give a row of NaN.
 *   n_toads >= 1, n_days >= 1, n_days * n_toads <= ELFI_B200_TOAD_CELLS_MAX.
 *   X (B, n_days, n_toads), C-contiguous, may be NULL.  S (B, n_lags * (n_p + 1); ldS) may be NULL;
 *   it holds toad_summaries of each lag lags[l] (host array, 1 <= lags[l] < n_days,
 *   n_lags <= ELFI_B200_TOAD_LAGS_MAX) in columns l * (n_p + 1) .. and needs
 *   n_toads * (n_days - 1) <= ELFI_B200_TOAD_DISP_MAX and 1 <= n_p <= ELFI_B200_TOAD_NP_MAX (p a
 *   host array).  With S and without X the row is simulated into shared memory and summarised
 *   there; with both, X is written and summarised.  Either way S equals toad_summaries of X bit for
 *   bit.
 * toad_summaries: S[i * ldS + 0 .. n_p] = compute_summaries(X, lag, p, thd) (toad.py:73-132) of the
 *   row X[d * ld_day + k * ld_toad + i * ld_row] (n_days, n_toads): the number of |displacements|
 *   < thd, the median of the others (NaN dropped) and the n_p - 1 logs of the gaps between their p
 *   quantiles floored at exp(-20), through nan_to_num(nan=inf); bit for bit NumPy's except for
 *   the logs, which use the device's log.  1 <= lag < n_days,
 *   n_toads * (n_days - lag) <= ELFI_B200_TOAD_DISP_MAX, 1 <= n_p <= ELFI_B200_TOAD_NP_MAX levels
 *   in [0, 1] (host array p). */
#define ELFI_B200_TOAD_CELLS_MAX 2147483648LL   /* 2^31 n_days * n_toads: (cell << 1) | h < 2^32 */
#define ELFI_B200_TOAD_DISP_MAX 4096   /* displacements of one lag, sorted per CTA */
#define ELFI_B200_TOAD_LAGS_MAX 8      /* lags of the fused summaries */
#define ELFI_B200_TOAD_NP_MAX 32       /* quantile levels */
int elfi_b200_sim_toad_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                           int64_t n_toads, int64_t n_days, uint64_t seed, uint64_t offset,
                           double* X, int64_t n_lags, const int64_t* lags, int64_t n_p,
                           const double* p, double thd, double* S, int64_t ldS, void* stream);
int elfi_b200_toad_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_day,
                                 int64_t ld_toad, int64_t ld_row, int64_t n_days, int64_t n_toads,
                                 int64_t B, int64_t lag, int64_t n_p, const double* p, double thd,
                                 double* S, int64_t ldS, void* stream);

/* Stochastic Lotka-Volterra model of elfi/examples/lotka_volterra.py (throughput mode, statistical
 * parity); stream layout, lane layout and arithmetic in elfi_b200/csrc/lotka_volterra.cu and
 * lotka_volterra.cuh.
 * sim_lotka_volterra: row i has parameters (r1, r2, r3, prey0, predator0, sigma) = P[i * ldP +
 *   0..5] (ldP >= 6) and starts from (floor(prey0), floor(predator0)); Gillespie's direct method
 *   runs it to time_end (finite, > 0).  X[i * 2 n_obs + 2 j + s] (B, n_obs, 2) is the count of
 *   species s (0 prey, 1 predators) at t_out[j] (device array of n_obs <= ELFI_B200_LV_NOBS_MAX
 *   times, t_out[0] = 0, t_out[n_obs - 1] = time_end; np.linspace), interpolated linearly between
 *   the events around it, plus sigma times a standard normal for j >= 1, truncated toward zero as
 *   int32 (NaN or out of range: -2^31).  n_events[i] (int64) is the number of events row i ran.
 *   Event k draws Philox block k, observation j block j, of (seed, offset + i): a pure function of
 *   the row, whatever the launch.  A row still short of time_end after max_events (1 ..
 *   ELFI_B200_LV_MAX_EVENTS_LIMIT) events gets NaN observations and n_events = max_events; a
 *   negative or NaN rate or sigma, initial counts outside [0, 2^31) or a negative or NaN total
 *   hazard (where the reference raises) give NaN observations.  The kernel is persistent: its lanes
 *   take new rows as theirs finish.
 * lv_summaries: S[i * ldS + 0..8] = prey_mean, pred_mean, prey_log_var, pred_log_var,
 *   prey_autocorr_1, pred_autocorr_1, prey_autocorr_2, pred_autocorr_2, crosscorr
 *   (lotka_volterra.py:206-277) of the row X[i * ld_row + j * ld_obs + s * ld_species]
 *   (n_obs, 2), ELFI_B200_LV_SUMM_NOBS_MIN <= n_obs <= ELFI_B200_LV_SUMM_NOBS_MAX,
 *   ldS >= ELFI_B200_LV_NSUMM; bit for bit NumPy's except for log(var + 1), which
 *   uses the device's log. */
#define ELFI_B200_LV_NOBS_MAX 1024       /* observation times staged in shared memory */
#define ELFI_B200_LV_SUMM_NOBS_MIN 3     /* the lag-2 autocorrelation needs one product */
#define ELFI_B200_LV_SUMM_NOBS_MAX 128   /* one leaf of NumPy's pairwise sum */
#define ELFI_B200_LV_NSUMM 9
#define ELFI_B200_LV_MAX_EVENTS_LIMIT 4294967295LL   /* 2^32 - 1: the event is one Philox word */
int elfi_b200_sim_lotka_volterra_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                                     const double* t_out, int64_t n_obs, double time_end,
                                     int64_t max_events, uint64_t seed, uint64_t offset,
                                     double* X, int64_t* n_events, void* stream);
int elfi_b200_lv_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_row, int64_t ld_obs,
                               int64_t ld_species, int64_t B, int64_t n_obs, double* S,
                               int64_t ldS, void* stream);

/* Birth-death-mutation (BDM) model of elfi/examples/bdm.py, whose reference simulator is the
 * executable elfi/examples/cpp/bdm.cpp with --mode 1 (throughput mode, statistical parity); law,
 * stream layout, lane layout and arithmetic in elfi_b200/csrc/bdm.cu and bdm.cuh.
 * sim_bdm: row i has rates (alpha, delta, tau) = P[i * ldP + 0..2] (ldP >= 3) and population bound
 *   N (1 <= N <= ELFI_B200_BDM_N_MAX, B <= ELFI_B200_BDM_BATCH_MAX).  X[i * ldX + j] (int16, ldX >=
 *   N) is the size of cluster j when the population first exceeds N (that birth undone) or dies
 *   out; S[i * ldS + 0..1] (ldS >= 2) are T1 = count(c > 0) / sum(c) (NaN for an extinct row) and
 *   T2 = 1 - sum_j (c_j / n_t2)^2 in NumPy's pairwise order; either of X and S may be NULL.
 *   n_events[i] (int64) is the number of events row i ran.  Event k draws Philox block k of (seed,
 *   offset + i): a pure function of the row, whatever the launch.  A rate that is negative, NaN or
 *   infinite, or a total rate of 0 or
 *   +inf, gives counts of -1, NaN summaries and n_events = -1; a row still running after
 *   max_events (1 .. ELFI_B200_BDM_MAX_EVENTS_LIMIT) events gives counts of -1, NaN summaries and
 *   n_events = max_events.  The kernel is persistent: its lanes take new rows as theirs finish.
 * bdm_summaries: S[i * ldS + 0..1] = T1, T2 (with n) of the row X[i * ld_row + j * ld_col]
 *   (int16, 1 <= N <= ELFI_B200_BDM_N_MAX), bit for bit NumPy's and sim_bdm's; a row with a
 *   negative count gets NaN summaries. */
#define ELFI_B200_BDM_N_MAX 1024   /* a count stays below N + 2 <= 2^16 (uint16 in shared memory) */
#define ELFI_B200_BDM_NSUMM 2      /* T1, T2 */
#define ELFI_B200_BDM_BATCH_MAX 2147483647   /* 2^31 - 1 */
#define ELFI_B200_BDM_MAX_EVENTS_LIMIT 4294967295LL  /* 2^32 - 1: the event is one Philox word */
int elfi_b200_sim_bdm_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B, int64_t N,
                          double n_t2, int64_t max_events, uint64_t seed, uint64_t offset,
                          int16_t* X, int64_t ldX, double* S, int64_t ldS, int64_t* n_events,
                          void* stream);
int elfi_b200_bdm_summaries_f64(elfi_b200_ctx* ctx, const int16_t* X, int64_t ld_row,
                                int64_t ld_col, int64_t B, int64_t N, double n, double* S,
                                int64_t ldS, void* stream);

/* Day care model of elfi/examples/daycare.py (throughput mode, statistical parity); law, stream
 * layout, lane layout and arithmetic in elfi_b200/csrc/daycare.cu and daycare.cuh.
 * sim_daycare: row i has parameters (t1, t2, t3) = P[i * ldP + 0..2] (ldP >= 3); each of its n_dcc
 *   (<= ELFI_B200_DC_DCC_MAX) DCCs of n_ind (2 .. ELFI_B200_DC_IND_MAX) children and n_strains
 *   (<= ELFI_B200_DC_STRAINS_MAX) strains, community
 *   frequencies freq (device, n_strains), runs Gillespie's direct method, and every DCC of the row
 *   takes as many transitions K[i] (int64) as the one that needs most to pass time_end (finite,
 *   > 0).  Transition k of DCC c draws Philox block k of (seed, offset + i) salted with c: a pure
 *   function of the row, whatever the launch.  S (or NULL; ldS >= 4 n_dcc) gets the summaries
 *   S[i * ldS + j * n_dcc + c], j = Shannon, n_strains, prevalence, multi, of the first n_obs
 *   (1 .. n_ind) children; X (or NULL) gets their states X[((i * n_dcc + c) * n_obs + o) *
 *   n_strains + s] as 0 / 1.  t1, t2 or t3 negative, NaN or infinite, time_end n_ind n_strains
 *   max(1, max(1, t3) (t1 + 1e-9 + t2 max(freq))) >= 2^32 - 1, or freq negative or not finite:
 *   NaN summaries, zero data, K = -1.  B <= ELFI_B200_DC_BATCH_MAX.
 * daycare_summaries: S[i * ldS + j * n_dcc + c] as above from X[i * ld_b + c * ld_c + o * ld_i +
 *   s * ld_s] (uint8, nonzero = carrier;
 *   n_strains <= ELFI_B200_DC_SUMM_STRAINS_MAX); bit for bit NumPy's except for the log
 *   in Shannon, which uses the device's log.
 * daycare_distance: d[i] (daycare.py:278-312) of the n_ss summaries S[i * ldS + k * n_dcc + c]
 *   (n_ss * n_dcc <= ELFI_B200_DC_DIST_TERMS_MAX) against the observed maxima obs_max (n_ss, 0
 *   replaced by 1) and the sorted observed values divided by them y (n_ss, n_dcc), both device; bit
 *   for bit NumPy's, including its summation order for B == 1 and B > 1. */
#define ELFI_B200_DC_DCC_MAX 32             /* one lane per DCC */
#define ELFI_B200_DC_IND_MAX 64             /* num_s * 64 stays within int64 for n_strains <= 40 */
#define ELFI_B200_DC_STRAINS_MAX 40         /* lcm(1 .. 40) = 5.3e15 < 2^53 */
#define ELFI_B200_DC_SUMM_STRAINS_MAX 64    /* one 64-bit strain mask per child */
#define ELFI_B200_DC_NSUMM 4                /* Shannon, n_strains, prevalence, multi */
#define ELFI_B200_DC_DIST_TERMS_MAX 128     /* n_ss * n_dcc of the distance: one pairwise leaf */
#define ELFI_B200_DC_BATCH_MAX 2147483647   /* 2^31 - 1: one CTA per row */
int elfi_b200_sim_daycare_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                              int64_t n_dcc, int64_t n_ind, int64_t n_strains,
                              const double* freq, int64_t n_obs, double time_end, uint64_t seed,
                              uint64_t offset, double* S, int64_t ldS, uint8_t* X, int64_t* K,
                              void* stream);
int elfi_b200_daycare_summaries_f64(elfi_b200_ctx* ctx, const uint8_t* X, int64_t ld_b,
                                    int64_t ld_c, int64_t ld_i, int64_t ld_s, int64_t B,
                                    int64_t n_dcc, int64_t n_obs, int64_t n_strains, double* S,
                                    int64_t ldS, void* stream);
int elfi_b200_daycare_distance_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t B,
                                   int64_t n_ss, int64_t n_dcc, const double* obs_max,
                                   const double* y, double* d, void* stream);

/* ARCH(1) model of elfi/examples/arch.py (throughput mode, statistical parity); stream layout,
 * thread layout and arithmetic in elfi_b200/csrc/arch.cu and arch.cuh.
 * Both take ELFI_B200_ARCH_NOBS_MIN <= n_obs (n) <= ELFI_B200_ARCH_NOBS_MAX and
 * 1 <= n_lags <= min(ELFI_B200_ARCH_LAGS_MAX, n - 1); the summaries are
 * S[i * ldS + k], k < 2 + L + L(L-1)/2 (ldS at least that): MU, VAR (ddof = 1), AC_1 .. AC_L, then
 * PW_i_j = AC_i * AC_j in itertools.combinations order, bit for bit NumPy's.
 * sim_arch: row i has parameters (t1, t2) = P[i * ldP + 0..1] (ldP >= 2) and observations
 *   Y[i * ldY + 0 .. n_obs - 1] (y_1 .. y_n of the reference).  Block m of (seed, offset + i) gives
 *   the normals z_{2m}, z_{2m+1}, z_0 = e_0, z_k = xi_k: a pure function of the row, whatever the
 *   launch.  Y and S may each be NULL; S is computed from the row without writing Y.
 * arch_summaries: the summaries of the row X[i * ld_b + j * ld_j], j < n, any strides. */
#define ELFI_B200_ARCH_NOBS_MIN 2
#define ELFI_B200_ARCH_NOBS_MAX 128   /* one leaf of NumPy's pairwise sum per reduction */
#define ELFI_B200_ARCH_LAGS_MAX 8
int elfi_b200_sim_arch_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                           int64_t n_obs, int64_t n_lags, uint64_t seed, uint64_t offset,
                           double* Y, int64_t ldY, double* S, int64_t ldS, void* stream);
int elfi_b200_arch_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_b, int64_t ld_j,
                                 int64_t B, int64_t n, int64_t n_lags, double* S, int64_t ldS,
                                 void* stream);

/* AR(1) model of elfi/examples/ar1.py (throughput mode, statistical parity) with the Euclidean
 * distance to an observed series fused; stream layout, thread layout and arithmetic in
 * elfi_b200/csrc/ar1.cu and ar1.cuh.  Row i has parameter phi[i] and series
 * x_t = phi x_{t-1} + w_t (x_0 = 0), X[i * ldX + t - 1] for t = 1 .. n_obs (ldX >= n_obs; X may be
 * NULL).  Block m of (seed, offset + i) gives the innovations w_{2m+1}, w_{2m+2}: a pure function
 * of the row, whatever the launch.  0 <= B <= ELFI_B200_AR1_BATCH_MAX,
 * 1 <= n_obs <= ELFI_B200_AR1_NOBS_MAX.
 * With obs (n_obs doubles) the row's distance d_out[i] = sqrt(sum_t (x_t - obs_t)^2), t ascending,
 * one rounding per operation: bit for bit elfi_b200_dist_euclid_thr_f64 of the written series
 * (K = 1, no weights), computed without writing X.  With a threshold (one double, thr_host on the
 * host or thr_dev on the device, not both) rows with d <= threshold are accepted; acc_idx
 * (B int32, may be NULL) gets their indices ascending and n_acc (one int64 on the device, may be
 * NULL) their number, the contract of the distance entry points above.  Without obs, d_out,
 * thresholds, acc_idx and n_acc must be NULL. */
#define ELFI_B200_AR1_NOBS_MAX 16777216     /* 2^24 */
#define ELFI_B200_AR1_BATCH_MAX 2147483647  /* 2^31 - 1: accepted rows are int32 indices */
int elfi_b200_sim_ar1_f64(elfi_b200_ctx* ctx, const double* phi, int64_t B, int64_t n_obs,
                          uint64_t seed, uint64_t offset, double* X, int64_t ldX,
                          const double* obs, const double* thr_host, const double* thr_dev,
                          double* d_out, int32_t* acc_idx, int64_t* n_acc, void* stream);

/* n-D Gaussian mean model of elfi/examples/gauss.py (nd_mean=True); stream layout, thread layout
 * and arithmetic in elfi_b200/csrc/gauss_nd.cu and gauss_nd.cuh.  Every sum below starts from 0.0,
 * as NumPy's reductions do, and every operation is rounded on its own.
 * gauss_nd_summaries: the (n, D) block of row b is X[b * ld_b + t * ld_t + j * ld_j], any strides;
 *   out[b * ld_out + j] = np.mean(y, axis=1)[b, j] and out[b * ld_out + D + j] =
 *   np.var(y, axis=1)[b, j] (ld_out >= 2 D), bit for bit NumPy's on the C-contiguous (B, n, D)
 *   array: for D = 1 the sum over t is NumPy's pairwise sum, for D >= 2 a left fold
 *   t = 0 .. n - 1; var = sum_t (y - m) * (y - m) / n in the same order, m = sum / n.
 *   1 <= n <= ELFI_B200_GAUSS_ND_SUMM_NOBS_MAX, D >= 1, B * D < 2^62.
 * gauss_nd_distance: d[b] = sqrt(sum_j (S[b * ld_b + j * ld_j] - obs[j])^2), the sum in NumPy's
 *   pairwise order (np.sum(..., axis=1) of a contiguous (B, D) array), bit for bit the reference's
 *   euclidean_multidim.  1 <= D <= ELFI_B200_GAUSS_ND_SUMM_NOBS_MAX.
 * sim_gauss_nd (throughput mode, statistical parity): row i has the means
 *   mu[i * ld_b + j * ld_j], j < D (1 <= D <= ELFI_B200_GAUSS_ND_D_MAX), and observations
 *   y[t, j] = (sum_k z[t, k] A[k, j]) + mu_j, t < n_obs (1 <= n_obs <= ELFI_B200_GAUSS_ND_NOBS_MAX),
 *   with A_host the D x D row-major factor sqrt(s)[:, None] * vh of the covariance (NumPy's
 *   multivariate_normal), on the host.  The sum over k runs in ascending order as
 *   z_0 A_0j, then fma(z_k, A_kj, s) (FMA is used).  z[t, k] is normal q = t D + k of the row:
 *   block q / 2 of (seed, offset + i) gives normals 2 (q / 2) and 2 (q / 2) + 1, so the row is a
 *   pure function of (seed, offset + i), whatever the launch.  Y[i * ldY + t D + j] (ldY >= n_obs D)
 *   and S[i * ldS + 0 .. 2 D - 1] (ldS >= 2 D) may each be NULL, not both; S is computed without
 *   writing Y and is bit for bit gauss_nd_summaries of the written Y. */
#define ELFI_B200_GAUSS_ND_D_MAX 16                  /* the device priors take 16 parameters */
#define ELFI_B200_GAUSS_ND_NOBS_MAX 7688             /* D = 1: a pairwise sum of depth 6 */
#define ELFI_B200_GAUSS_ND_SUMM_NOBS_MAX 16777216    /* 2^24 */
int elfi_b200_gauss_nd_summaries_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_b,
                                     int64_t ld_t, int64_t ld_j, int64_t B, int64_t n, int64_t D,
                                     double* out, int64_t ld_out, void* stream);
int elfi_b200_gauss_nd_distance_f64(elfi_b200_ctx* ctx, const double* S, int64_t ld_b,
                                    int64_t ld_j, int64_t B, int64_t D, const double* obs,
                                    double* d, void* stream);
int elfi_b200_sim_gauss_nd_f64(elfi_b200_ctx* ctx, const double* mu, int64_t ld_b, int64_t ld_j,
                               int64_t B, int64_t D, const double* A_host, int64_t n_obs,
                               uint64_t seed, uint64_t offset, double* Y, int64_t ldY, double* S,
                               int64_t ldS, void* stream);

/* M/G/1 queue of elfi/examples/mg1.py (throughput mode, statistical parity); stream layout, thread
 * layout and arithmetic in elfi_b200/csrc/mg1.cu and mg1.cuh.  Rows where the reference's NumPy
 * raises (1/t3 with its sign bit set, t2 - t1 not finite) give NaN data and NaN quantiles.
 * sim_mg1: row i has parameters (t1, t2, t3) = P[i * ldP + 0..2] (ldP >= 3) and inter-departure
 *   times Y[i * ldY + j], j < n_obs (ELFI_B200_MG1_NOBS_MIN <= n_obs <= ELFI_B200_MG1_NOBS_MAX);
 *   S[i * ldS + k] = np.quantile(y_i, q[k]) (method 'linear'; 1 <= nq <= ELFI_B200_MG1_NQ_MAX,
 *   q_host on the host, each in [0, 1]) is computed in the same kernel.  Y or S may be NULL; row i
 *   is a pure function of (seed, offset + i).
 * row_quantiles: S[b * ldS + k] = np.quantile(X[b, :], q[k]) of the row X[b * ld_b + j * ld_j],
 *   j < n (ELFI_B200_MG1_NOBS_MIN <= n <= ELFI_B200_MG1_NOBS_MAX), any strides; a row with a NaN
 *   has every quantile NaN.  Bit for bit
 *   NumPy's, and the quantiles sim_mg1 fuses are the bits of row_quantiles of its data. */
#define ELFI_B200_MG1_NOBS_MIN 2
#define ELFI_B200_MG1_NOBS_MAX 512   /* one warp sorts a row in registers (32 lanes x 16 keys) */
#define ELFI_B200_MG1_NQ_MAX 32      /* one quantile per lane */
int elfi_b200_sim_mg1_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                          int64_t n_obs, int64_t nq, const double* q_host, uint64_t seed,
                          uint64_t offset, double* Y, int64_t ldY, double* S, int64_t ldS,
                          void* stream);
int elfi_b200_row_quantiles_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_b, int64_t ld_j,
                                int64_t B, int64_t n, int64_t nq, const double* q_host, double* S,
                                int64_t ldS, void* stream);

/* Alpha-stable stochastic volatility model of elfi/examples/stochastic_volatility_model.py
 * (throughput mode, statistical parity); stream layout, thread layout and arithmetic in
 * elfi_b200/csrc/svm.cu, svm.cuh and stable.cuh.
 * sim_svm: row i has parameters (alpha, beta, kappa, eta, mu, phi, sigma) = P[i * ldP + 0..6]
 *   (ldP >= 7) and observations Y[i * ldY + j], j < n_obs (2 <= n_obs <= 512): an AR(1)
 *   log-volatility x_j (stationary start) times levy_stable(alpha, beta, loc=eta, scale=kappa)
 *   shocks in the S0 parameterization.  S[i * ldS + 0..1] (ldS >= 2) = (kurt, skew) of the row's
 *   np.quantile at 0.05, 0.25, 0.5, 0.75, 0.95, computed in the same kernel, bit for bit the
 *   row_quantiles of its data followed by the reference's subtractions and division.  Rows where
 *   the reference raises (0 < alpha <= 2, -1 <= beta <= 1, kappa >= 0, sigma >= 0 violated, NaN
 *   included, or phi = NaN) give NaN data and NaN summaries.  Y or S may be NULL; row i is a pure
 *   function of (seed, offset + i). */
int elfi_b200_sim_svm_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                          int64_t n_obs, uint64_t seed, uint64_t offset, double* Y, int64_t ldY,
                          double* S, int64_t ldS, void* stream);

/* Scratch assay model of elfi/examples/scratch_assay.py (throughput mode, exact replay of its
 * streams); law, stream layout and warp layout in elfi_b200/csrc/scratch_assay.cuh and
 * scratch_assay.cu.
 * sim_scratch_assay: row i has parameters (pm, pp) = P[i * ldP + 0..1] (ldP >= 2) and starts from
 *   the lattice init[r * ncols + c] (device, nrows * ncols <= ELFI_B200_SA_SITES_MAX bytes, nonzero
 *   = a cell).  It runs num_iter (<= ELFI_B200_SA_ITER_MAX) iterations of motility then
 *   proliferation and observes the lattice every obs_interval (>= 1) iterations: num_obs = num_iter
 *   / obs_interval frames after the initial one.  S[i * ldS + k] (ldS >= num_obs + 1) gets the
 *   mismatches between frames k and k + 1, k < num_obs, then S[i * ldS + num_obs] the cells of the
 *   last frame; X gets the frames X[((i * nrows + r) * ncols + c) * (num_obs + 1) + k] as 0 / 1.  S
 *   and X may each be NULL; S is computed without writing X.  Row i is a pure function of (seed,
 *   offset + i); B <= ELFI_B200_SA_BATCH_MAX.
 * scratch_assay_summaries: the same summaries S[i * ldS + k], k < n_frames (ldS >= n_frames), of
 *   the frames X[i * ld_b + r * ld_r + c * ld_c + k * ld_k] (uint8, nonzero = a cell), any
 *   strides: n_frames - 1 mismatches, then the cells of the last frame. */
#define ELFI_B200_SA_SITES_MAX 4096         /* lattice sites: list entries fit uint16 */
#define ELFI_B200_SA_ITER_MAX 2147483647    /* 2^31 - 1: iteration counters of the Philox streams */
#define ELFI_B200_SA_BATCH_MAX 2147483647   /* 2^31 - 1: one warp per row */
int elfi_b200_sim_scratch_assay_f64(elfi_b200_ctx* ctx, const double* P, int64_t ldP, int64_t B,
                                    const uint8_t* init, int64_t nrows, int64_t ncols,
                                    int64_t num_iter, int64_t obs_interval, uint64_t seed,
                                    uint64_t offset, double* S, int64_t ldS, uint8_t* X,
                                    void* stream);
int elfi_b200_scratch_assay_summaries_f64(elfi_b200_ctx* ctx, const uint8_t* X, int64_t ld_b,
                                          int64_t ld_r, int64_t ld_c, int64_t ld_k, int64_t B,
                                          int64_t nrows, int64_t ncols, int64_t n_frames,
                                          double* S, int64_t ldS, void* stream);

/* ---- Bayesian synthetic likelihood (elfi/methods/bsl/pdf_methods.py) ---------------------------
 * elfi_b200_synlik_f64: the Gaussian synthetic log-likelihood of the observed summaries y (d) under
 * each of G groups of n simulated summary rows, S[g * ld_group + i * ld_row + j], i < n, j < d
 * (ld_row >= d; groups may be gapped or interleaved).  Per group: mu the column means, Sigma the
 * covariance with divisor n - 1.
 *   W (d x d row-major, device) or NULL: whitening; W mu, W Sigma W^T and W y replace mu, Sigma, y.
 *   estimator 0, standard: ll = -(d log 2 pi + log det Sigma_l + m) / 2, m = (y - mu)^T Sigma_l^-1
 *     (y - mu), with Warton shrinkage Sigma_l = (1 - l) Sigma + l diag(Sigma_jj + 1e-5) for each
 *     of the K penalties l in [0, 1] (penalties_host, HOST), or Sigma itself when K = 0.
 *   estimator 1, unbiased (Ghurye and Olkin 1969): ll = -d log(2 pi) / 2 + A + B + C with
 *     A = log c(d, n - 2) - log c(d, n - 1) - d log(1 - 1/n) / 2,
 *     B = -(n - d - 2)(log(n - 1) + log det Sigma) / 2,
 *     C = (n - d - 3) log|det Psi| / 2, Psi = (n - 1) Sigma - (y - mu)(y - mu)^T / (1 - 1/n),
 *     log|det Psi| = d log(n - 1) + log det Sigma + log|1 - n m / (n - 1)^2| (determinant lemma).
 *     W must be NULL and K = 0.
 * loglik[g * max(K, 1) + k] (device) gets group g's value at penalty k.  A group gives -inf when
 * any of its n x d values is not finite (or its column sum overflows), or when a Cholesky pivot of
 * Sigma_l is not finite or L_jj^2 <= 1e6 * DBL_EPSILON * max_i Sigma_l,ii.  SciPy instead tests the
 * eigenvalues against 1e6 eps lambda_max and gives up near cond(Sigma) ~ 4.5e9; near that boundary
 * the two tests can disagree (by a factor that depends on d), and one may return a finite value
 * where the other returns -inf.  Limits: 1 <= d <= ELFI_B200_SYNLIK_D_MAX, n >= 2, G <= 2^22, K <=
 * 65535.  Results are bit-identical across calls, and a group's value does not depend on G, K or
 * the other groups.  Asynchronous on `stream`; uses the context's scratch (about G d^2 doubles,
 * more with whitening or when few groups split their rows over several CTAs). */
#define ELFI_B200_SYNLIK_D_MAX 160   /* Sigma, its factor and y in one CTA's shared memory */
int elfi_b200_synlik_f64(elfi_b200_ctx* ctx, const double* S, int64_t ld_row, int64_t ld_group,
                         int64_t G, int64_t n, int64_t d, const double* y, const double* W,
                         int32_t estimator, const double* penalties_host, int64_t K,
                         double* loglik, void* stream);

/* elfi_b200_synlik_obs_f64: elfi_b200_synlik_f64 with an observation per group: group g's
 * observed summaries are Y[g * ld_y + j], j < d (device), and ld_y = 0 gives every group the one
 * row Y.  ld_y must be 0 or at least d.  Every promise of elfi_b200_synlik_f64 holds per group:
 * the -inf rules, whitening (W y_g replaces y), the Warton penalties, the unbiased estimator,
 * bit-identity across calls, and independence of a group's value from G, K and the other groups
 * and their observations.  So group g gives the bits of elfi_b200_synlik_f64 on group g alone with
 * y = Y + g * ld_y, and a Testbench's repetitions, each with its own observation, share one call.
 * Same limits, scratch and stream behaviour. */
int elfi_b200_synlik_obs_f64(elfi_b200_ctx* ctx, const double* S, int64_t ld_row,
                             int64_t ld_group, int64_t G, int64_t n, int64_t d, const double* Y,
                             int64_t ld_y, const double* W, int32_t estimator,
                             const double* penalties_host, int64_t K, double* loglik,
                             void* stream);

/* elfi_b200_bsl_mh_step_f64: iteration t of C lock-step BSL Metropolis-Hastings chains in
 * throughput mode (elfi/methods/inference/bsl.py), for p <= 16 parameters.  Device arrays:
 * loglik (C) the synthetic log-likelihoods of the round (elfi_b200_synlik_f64 with G = C), prop
 * (C x p) and prop_lp (C) the pending proposals and their joint prior log densities, chains
 * (C x n_samples x p), logpost (C x n_samples), n_acc (C, int64), rows (column-major C b x p:
 * column j at rows + j * ld_rows).  Host: spec_host the 7p-word prior table of
 * elfi_b200_prior_logpdf_cond_f64, chol_host the (p x p, row-major) lower Cholesky factor L of the
 * proposal covariance, bounds_host NULL or (p x 2) [lower, upper] per parameter.
 *   t = 0: chain c takes prop[c] as its state, logpost[c, 0] = loglik[c] + prop_lp[c].
 *   t >= 1: a proposal with a finite log prior is accepted iff u < min(1, exp(clip(r, -700, 700)))
 *     with r = (J(prop) - J(state)) + (loglik[c] + prop_lp[c] - logpost[c, t - 1]), where J is the
 *     log Jacobian of the back transform evaluated at the parameters themselves (the reference's
 *     rule; 0 without bounds), summed left to right, and clip maps NaN to -700.  Otherwise, or for
 *     a non-finite prop_lp, row t and logpost[c, t] copy row t - 1.  n_acc[c] += 1 for an
 *     accepted step (t = 0 included) with t >= burn_in.
 *   t + 1 < n_samples: the proposal of iteration t + 1 is written to prop[c] and its prior log
 *     density (conditional sources included) to prop_lp[c]: theta~ = logit(state) per parameter,
 *     log((x - a) / (b - x)), log(1 / (b - x)), log(x - a) or x by which bounds are finite;
 *     y_a = theta~_a + sum_{k <= a} L[a, k] z_k accumulated in order of k; the back transform of y.
 *     Rows [c b, (c + 1) b) of every column get the proposal, or the new state when the proposal's
 *     log prior is not finite.
 * Random stream: Philox4x32-10 keyed by seed; u = u01(x, y) of counter (t, c, 0, 0x4253434c), and
 * z_2k, z_2k+1 the two Box-Muller normals of counter (t + 1, c, 1 + k, 0x4253434c), so that no
 * value depends on C or on the other chains.  Limits: 1 <= C <= ELFI_B200_BSL_MAX_CHAINS,
 * 1 <= p <= 16, b >= 1, C b < 2^31, ld_rows >= C b, 0 <= t < n_samples < 2^32.  Asynchronous on
 * `stream`, bit-identical across calls. */
#define ELFI_B200_BSL_MAX_CHAINS 4194304   /* 2^22 */
int elfi_b200_bsl_mh_step_f64(elfi_b200_ctx* ctx, int64_t C, int64_t p, int64_t t,
                              int64_t n_samples, int64_t burn_in, int64_t b, uint64_t seed,
                              const double* spec_host, const double* chol_host,
                              const double* bounds_host, const double* loglik, double* prop,
                              double* prop_lp, double* chains, double* logpost, int64_t* n_acc,
                              double* rows, int64_t ld_rows, void* stream);

/* elfi_b200_bsl_mh_step_keyed_f64: elfi_b200_bsl_mh_step_f64 with a Philox key and a lane per
 * chain slot: keys (C, uint64) and lanes (C, uint32), device, both required.  Slot c draws its
 * uniform from counter (t, lanes[c], 0, 0x4253434c) and its proposal normals from
 * (t + 1, lanes[c], 1 + k, 0x4253434c) of Philox4x32-10 keyed by keys[c]; everything else is the
 * contract above.  elfi_b200_bsl_mh_step_f64 is the case keys[c] = seed, lanes[c] = c, so slot c
 * of a keyed call gives the bits of an unkeyed call in which the same chain sits at slot lanes[c]
 * under seed keys[c]: the chains of several samplers, each with its own seed, step in one launch. */
int elfi_b200_bsl_mh_step_keyed_f64(elfi_b200_ctx* ctx, int64_t C, int64_t p, int64_t t,
                                    int64_t n_samples, int64_t burn_in, int64_t b,
                                    const uint64_t* keys, const uint32_t* lanes,
                                    const double* spec_host, const double* chol_host,
                                    const double* bounds_host, const double* loglik, double* prop,
                                    double* prop_lp, double* chains, double* logpost,
                                    int64_t* n_acc, double* rows, int64_t ld_rows, void* stream);

/* ---- regression adjustment (elfi/methods/post_processing.py: LinearAdjustment) ------------------
 * The local-linear adjustment of Beaumont et al. (2002) on N rows of q summaries
 * S[i * ldS + j] (ldS >= q), the observed summaries obs (q) and p parameters T[i * ldT + k]
 * (ldT >= p); all device.  The regressors are x_i = S_i - obs.
 * elfi_b200_regadj_mask_f64: flags[i] (device, N bytes) = 1 when every S[i, j] - obs[j] is finite,
 *   else 0 (a non-finite obs drops every row); counts (device, p + 1 int64) = [the flagged rows,
 *   then per parameter k the flagged rows whose T[i, k] is not finite].
 * A group is the parameter columns cols_host[0 .. pg - 1] (HOST int32, each in [0, p)) and the rows
 *   with flags[i] != 0 and, when sel >= 0, T[i, sel] finite.  d = q + pg.
 * elfi_b200_regadj_moments_f64: mom (device, 1 + d + d * d doubles) = [n_g, the means m of
 *   [x | T_g] over the group's rows, the full symmetric d x d sum over those rows of
 *   ([x | T_g] - m)([x | T_g] - m)^T, row-major].  Two passes, means first.  Rows are split into
 *   chunks whose length depends on N and d only; each chunk sum starts from zero and the chunk sums
 *   are added left to right, so the result is bit-identical across calls and GPUs.  n_g = 0
 *   leaves NaN means and zero moments.
 * elfi_b200_regadj_adjust_f64: for each group row i in row order and each k < pg,
 *   out[k * ld_out + pos] = T[i, cols_host[k]] - sum_j (S[i, j] - obs[j]) coef[j * pg + k]
 *   (coef device, q x pg row-major).  dense = 1 states that every row is in the group (n_g = N):
 *   pos = i, with no compaction; dense = 0 gives pos = the rank of i among the group's rows.
 *   ld_out >= N when dense.
 * Limits: q, p >= 1, q + p <= ELFI_B200_REGADJ_D_MAX, 1 <= N <= ELFI_B200_REGADJ_N_MAX,
 * 1 <= pg <= p, -1 <= sel < p.  Asynchronous on `stream`; moments use about min(N / 256, 2048) *
 * 64^2 doubles of the context's scratch, adjust
 * N / 2048 int64. */
#define ELFI_B200_REGADJ_D_MAX 256   /* q + p: a group's mean and tile rows in shared memory */
#define ELFI_B200_REGADJ_N_MAX 2147483647   /* 2^31 - 1: int32 row ranks in the compaction */
int elfi_b200_regadj_mask_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t N,
                              int64_t q, const double* obs, const double* T, int64_t ldT, int64_t p,
                              uint8_t* flags, int64_t* counts, void* stream);
int elfi_b200_regadj_moments_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t N,
                                 int64_t q, const double* obs, const double* T, int64_t ldT,
                                 int64_t p, const uint8_t* flags, const int32_t* cols_host,
                                 int64_t pg, int64_t sel, double* mom, void* stream);
int elfi_b200_regadj_adjust_f64(elfi_b200_ctx* ctx, const double* S, int64_t ldS, int64_t N,
                                int64_t q, const double* obs, const double* T, int64_t ldT,
                                int64_t p, const uint8_t* flags, const int32_t* cols_host,
                                int64_t pg, int64_t sel, int32_t dense, const double* coef,
                                double* out, int64_t ld_out, void* stream);

/* ---- BOLFIRE ratio-estimation classifier (elfi/methods/classifier.py: LogisticRegression) ------
 * elfi_b200_logreg_fit_f64: sklearn's StandardScaler then penalised logistic regression with
 * liblinear's primal and intercept_scaling = 1, on the n rows X[i * ld_row + j], j < d (device,
 * ld_row >= d) with labels y[i] (device, each +1 or -1).
 *   Standardisation: mean_j and var_j over all n rows (ddof 0; var_j = (S2 - S1^2 / n) / n with
 *     S1, S2 the sums of x - mean_j and (x - mean_j)^2), scale_j = sqrt(var_j), or 1 when the column
 *     is constant by sklearn's rule var_j <= n eps var_j + (n mean_j eps)^2.  x~_ij =
 *     (x_ij - mean_j) / scale_j, and every row gets a trailing 1 (the intercept, penalised too).
 *   Objective, penalty 0 (L1): F(w) = sum_j |w_j| + C sum_i log(1 + exp(-y_i w . x~_i));
 *              penalty 1 (L2): F(w) = |w|^2 / 2 + C sum_i log(1 + exp(-y_i w . x~_i)).
 *   Solved to convergence (proximal Newton, liblinear's newGLMNET without its tolerance): stops
 *     when the infinity norm of the minimum-norm subgradient is <= 1e-10 C n (for L1, g_j +
 *     sign(w_j) where w_j != 0 and max(|g_j| - 1, 0) where w_j = 0), or after max_iter Newton steps,
 *     or when a step gives no decrease; the last two return the last iterate with status 0.
 *   fit (device, ELFI_B200_LOGREG_BLOCK(d) doubles): [0] intercept_, [1] Newton steps taken
 *     (n_iter_), [2] status (1 converged, 0 not converged, -1 labels not all +-1 or one class only,
 *     -2 a non-finite value in X or a variance that overflows), [3] F at the returned weights,
 *     [4] the subgradient norm there, [5..7] 0, then mean_ (d), scale_ (d), coef_ (d).  A negative
 *     status leaves NaN in every other value.
 * elfi_b200_logreg_predict_f64: out[i] (device, i < m) = log(p / (1 - p)) of row Xq[i * ld_row + j]
 *   with v = sum_j coef_j (x_j - mean_j) / scale_j + intercept_, p = 1 / (1 + exp(-v)), then
 *   p = max(p, class_min): the reference's log-likelihood ratio (p = 1 gives +inf).  A row with a
 *   non-finite value, or a fit with a negative status, gives NaN.
 * Limits: 1 <= d <= ELFI_B200_LOGREG_D_MAX, 2 <= n < 2^31, C > 0.  One CTA per fit; reductions in a
 * fixed order, no atomics: repeated calls are bit-identical.  Asynchronous on `stream`; the fit
 * uses 4 n doubles of the context's scratch. */
#define ELFI_B200_LOGREG_D_MAX 160   /* H and the row tiles in one CTA's shared memory */
#define ELFI_B200_LOGREG_HEAD 8      /* header doubles of a fit block */
#define ELFI_B200_LOGREG_BLOCK(d) (ELFI_B200_LOGREG_HEAD + 3 * (d))
int elfi_b200_logreg_fit_f64(elfi_b200_ctx* ctx, const double* X, int64_t ld_row, int64_t n,
                             int64_t d, const double* y, int32_t penalty, double C,
                             int64_t max_iter, double* fit, void* stream);
int elfi_b200_logreg_predict_f64(elfi_b200_ctx* ctx, const double* fit, int64_t d,
                                 const double* Xq, int64_t ld_row, int64_t m, double class_min,
                                 double* out, void* stream);

/* ---- KLIEP density-ratio estimation (AdaptiveThresholdSMC) -------------------------------------
 * DensityRatioEstimation.fit + max_ratio (elfi/methods/density_ratio_estimation.py:71-207):
 * basis centres = first n_basis rows of x, A = RBF(x, centres), b = weighted RBF mean over y,
 * <= max_iter projected-gradient steps with a convergence check every conv_check_interval
 * steps.  wx (unnormalised, as the reference passes it) and wy may be NULL (ones).
 * alpha_out: device (n_basis);  result_host[0] = max_i r(x_i), result_host[1] = steps taken.
 * Blocks until done (the convergence test needs the host). */
int elfi_b200_kliep_fit_f64(elfi_b200_ctx* ctx, const double* x, int64_t ldx, int64_t Nx,
                            const double* y, int64_t ldy, int64_t Ny, int64_t p, const double* wx,
                            const double* wy, double sigma, int64_t n_basis, double epsilon,
                            int64_t max_iter, double abs_tol, int64_t conv_check_interval,
                            double* alpha_out, double* result_host);

/* elfi_b200_rowsort_f64: out[i, :] = np.sort(X[i, :]) (ascending, NaN last), 1 <= n <= 2048.
 * Order-statistic summaries such as the g-and-k model's (elfi/examples/gnk.py:145-161; the
 * 2-d form np.sort(y[:, :, 0], axis=1) that an (B, n_obs) summary matrix needs, SURVEY 8d #5). */
int elfi_b200_rowsort_f64(elfi_b200_ctx* ctx, const double* X, int64_t ldX, int64_t B, int64_t n,
                          double* out, int64_t ld_out, void* stream);

/* ---- summary-statistic selection (TwoStageSelection, elfi/methods/diagnostics.py) -------------
 * elfi_b200_subset_distance_f64: the distance of every candidate combination of summaries, from
 * one read of each row (diagnostics.py:172-212 runs one rejection sampler per combination).
 *   S       (B, W) row-major resident summary columns, leading dimension ldS >= W; a candidate
 *           summary is a column range [col, col + width) of it.
 *   obs     (W) the observed summaries in the same columns.
 *   ranges  device int32 (n_ranges, 2) rows (col, width), width >= 1, col + width <= W;
 *   comb    device int32 (C + 1) offsets: combination c is the ordered list of ranges
 *           comb[c] .. comb[c + 1] - 1 (at least one).
 *   d_out   (C, ld_out) row-major, ld_out >= B: d_out[c, i] = cdist(X_c[i], obs_c, metric), where
 *           X_c and obs_c are the concatenations of combination c's ranges in list order.
 * metric is ELFI_B200_METRIC_EUCLIDEAN, _SQEUCLIDEAN, _CITYBLOCK or _CHEBYSHEV; the terms are
 * accumulated left to right over the concatenated columns with one rounding per multiply and add,
 * the arithmetic of elfi_b200_dist_metric_thr_f64, so every value is bit-identical to SciPy's cdist
 * on the concatenation, NaN and +-inf included (a NaN term makes the sums NaN; 'chebyshev' skips
 * it, as SciPy does).  Limits: 1 <= W <= ELFI_B200_SUBSET_MAX_WIDTH,
 * 1 <= C <= ELFI_B200_SUBSET_MAX_COMBINATIONS, 0 <= B < 2^31.  One CTA stages 32
 * rows in shared memory (32 (W + 1) doubles) and its warps take the combinations in turn, so each
 * row is read from HBM once for all C.  No scratch, no atomics: repeated calls give the same bits.
 * Asynchronous on `stream`. */
#define ELFI_B200_METRIC_EUCLIDEAN 0
#define ELFI_B200_SUBSET_MAX_WIDTH 512
#define ELFI_B200_SUBSET_MAX_COMBINATIONS 16777215   /* 2^24 - 1 */

int elfi_b200_subset_distance_f64(elfi_b200_ctx* ctx, int32_t metric, const double* S, int64_t ldS,
                                  int64_t B, int64_t W, const double* obs, const int32_t* ranges,
                                  const int32_t* comb, int64_t C, double* d_out, int64_t ld_out,
                                  void* stream);

/* elfi_b200_dist_seg_f64: R segments of B rows of S (leading dimension ldS), segment r against
 * observed row r of obs (R rows, leading dimension ld_obs): d_out[r B + i] = cdist(S[r B + i],
 * obs[r], metric).  metric is ELFI_B200_METRIC_EUCLIDEAN, _SQEUCLIDEAN, _CITYBLOCK, _CHEBYSHEV or
 * _MINKOWSKI (pexp); each segment is bit-identical to elfi_b200_dist_euclid_thr_f64 (unweighted)
 * or elfi_b200_dist_metric_thr_f64 on that segment.  No thresholds.  Limits: R >= 1, D >= 1,
 * R B < 2^31.  The row-stream kernel keeps all R observed rows in shared memory; when D < 16,
 * S is not TMA-addressable, or R ceil(D / 16) 16 doubles do not fit beside a two-slot ring (about
 * R ceil(D / 16) 16 <= 20000 on an H100), a thread per row reads them from global memory instead,
 * with the same arithmetic.  Asynchronous on `stream`. */
int elfi_b200_dist_seg_f64(elfi_b200_ctx* ctx, int32_t metric, double pexp, const double* S,
                           int64_t ldS, int64_t R, int64_t B, int64_t D, const double* obs,
                           int64_t ld_obs, double* d_out, void* stream);

/* elfi_b200_knn_entropy_f64: the nearest-neighbour part of the minimum-entropy criterion
 * (diagnostics.py:214-253) for C point sets of n points in q dimensions at once.
 *   X       (C * n, q) row-major, leading dimension ldX >= q: set c is rows c n .. c n + n - 1.
 *   R       (C, n): R[c, i] = the k-th smallest Euclidean distance from point i of set c to the
 *           points of set c, the point itself included -- cKDTree(X_c).query(X_c[i], k)[0][-1]: the
 *           self-distance is 0, so k = 1 gives 0; a duplicate gives 0; k > n gives +inf.  Squared
 *           distances are summed over the q coordinates in order with one rounding per multiply
 *           and add, then the root is taken (cKDTree agrees to a few ulps).  Coordinates must be
 *           finite.
 *   logsum  (C): logsum[c] = sum_i log(R[c, i]) added in a fixed order (each of 256 threads sums
 *           i = t, t + 256, ... in turn, then a fixed pairwise tree), so identical sets give
 *           identical bits; a zero R gives -inf, an infinite one +inf.
 * The host forms the entropy log(pi^(q/2) / Gamma(q/2 + 1)) - digamma(k) + log(n) + q / n logsum.
 * Limits: 1 <= q <= ELFI_B200_KNN_MAX_Q, 1 <= k <= ELFI_B200_KNN_MAX_K, 
 * 1 <= n <= ELFI_B200_KNN_MAX_N, 1 <= C <= ELFI_B200_KNN_MAX_SETS.  Brute force: a CTA of 128
 * query points streams the set through shared memory in tiles of 256 points, and each thread keeps
 * its k smallest squared distances in registers (a sorted insertion).  Two launches, no scratch,
 * no atomics.  Asynchronous on `stream`. */
#define ELFI_B200_KNN_MAX_Q 16
#define ELFI_B200_KNN_MAX_K 32
#define ELFI_B200_KNN_MAX_N 1048576    /* 2^20 */
#define ELFI_B200_KNN_MAX_SETS 65535   /* 2^16 - 1 */
int elfi_b200_knn_entropy_f64(elfi_b200_ctx* ctx, const double* X, int64_t ldX, int64_t C,
                              int64_t n, int64_t q, int64_t k, double* R, double* logsum,
                              void* stream);

/* elfi_b200_mrsse_f64: the mean root sum of squared errors of diagnostics.py:255-289 for C sets.
 *   T       (C * n, q) row-major, leading dimension ldT >= q: set c is rows c n .. c n + n - 1.
 *   P       (m, q) row-major, leading dimension ldP >= q: the m 'closest' parameter vectors.
 *   out     (C): out[c] = sum_j sqrt(sum_{i,l} (T_c[i, l] - P[j, l])^2) / m, j = 0 .. m - 1 -- the
 *           Frobenius norm of the (n, q) difference per closest vector.  Each sum of squares is
 *           taken in a fixed order (256 threads over the n q entries, then a fixed tree) and the
 *           roots are added in order of j, so repeated calls give the same bits; NumPy's norm sums
 *           in another order, so the two agree to rounding.  NaN and inf propagate.
 * Limits: 1 <= q <= ELFI_B200_KNN_MAX_Q, 1 <= n q < 2^31, 1 <= m < 2^31, 1 <= C < 2^31.  One CTA
 * per set, one launch, no scratch, no atomics.  Asynchronous on `stream`. */
int elfi_b200_mrsse_f64(elfi_b200_ctx* ctx, const double* T, int64_t ldT, int64_t C, int64_t n,
                        int64_t q, const double* P, int64_t ldP, int64_t m, double* out,
                        void* stream);

/* ---- robust optimisation Monte Carlo (ROMC, elfi/methods/inference/romc.py) ----------------
 * P optimisation problems with 1 <= p <= ELFI_B200_ROMC_MAX_P parameters advance in lock-step:
 * every call consumes the objective value of the point each problem proposed last call and writes
 * the next point.
 * The host evaluates all P points of a call as one batch, so the stream row of problem i stays i.
 * Products, sums and quotients that must match NumPy use round-to-nearest intrinsics (no FMA).
 * One thread per problem (or per point), no scratch, no atomics.  Asynchronous on `stream`. */
#define ELFI_B200_ROMC_MAX_P 16
#define ELFI_B200_ROMC_NM_INTS 8   /* ints of Nelder-Mead state per problem */
#define ELFI_B200_ROMC_NM_DONE 6   /* istate[i, 0] of a finished problem */
/* doubles of Nelder-Mead state per problem: the simplex (p + 1, p), fsim (p + 1), xbar, the
 * reflected point and the trial point (p each), f at the reflection and f_min */
#define ELFI_B200_ROMC_NM_DOUBLES(p) (((p) + 1) * ((p) + 1) + 3 * (p) + 2)

/* elfi_b200_romc_nm_init_f64: scipy's initial simplex around each x0 row (x0, then x0 with
 * coordinate k scaled by 1 + 0.05, or set to 0.00025 when it is 0) and fsim = +inf.
 *   x0       (P, p), leading dimension ld_x0 >= p.
 *   state    (P, ELFI_B200_ROMC_NM_DOUBLES(p)) and istate (P, ELFI_B200_ROMC_NM_INTS), written.
 *   theta    (P, p), leading dimension ld_theta: the first point of every problem (x0). */
int elfi_b200_romc_nm_init_f64(elfi_b200_ctx* ctx, int64_t P, int64_t p, const double* x0,
                               int64_t ld_x0, double* state, int32_t* istate, double* theta,
                               int64_t ld_theta, void* stream);

/* elfi_b200_romc_nm_step_f64: one step of scipy 1.18's _minimize_neldermead (adaptive=False,
 * bounds=None) per problem.  fvals (P) holds f at the points of the previous call; each running
 * problem advances to the next point it needs and writes it to row i of theta.  The reflection,
 * expansion, outside and inside contractions and the shrink use scipy's expressions in scipy's
 * order (xbar = the first p vertices added row after row, divided by p); a shrink proposes its p
 * vertices in p calls.  The convergence test (xatol, fatol), the maxiter / maxfev stops and an
 * evaluation refused at maxfev (the iteration is not counted) are scipy's.  Vertices are ordered
 * by a stable sort, NaN last: np.argsort's order whenever fsim has no ties, and for p <= 2; with
 * ties at p >= 3 NumPy's order depends on the CPU's SIMD sort (DESIGN.md section 7, "ROMC").
 * A finished problem keeps x_min in its theta row and ignores its value from then on:
 *   istate[i, 0] = ELFI_B200_ROMC_NM_DONE, istate[i, 1] = nit, istate[i, 2] = nfev, istate[i, 4] =
 *   scipy's warnflag (0 success, 1 maxfev, 2 maxiter); the first p doubles of state row i are x_min
 *   and double ELFI_B200_ROMC_NM_DOUBLES(p) - 1 is f_min = np.min(fsim) (NaN when any vertex is
 *   NaN).
 * Limits: 0 <= P < 2^31, 1 <= maxiter, maxfev < 2^30. */
int elfi_b200_romc_nm_step_f64(elfi_b200_ctx* ctx, int64_t P, int64_t p, double* state,
                               int32_t* istate, const double* fvals, double* theta,
                               int64_t ld_theta, int64_t maxiter, int64_t maxfev, double xatol,
                               double fatol, void* stream);

/* elfi_b200_romc_line_search_f64: romc.py line_search for the 2p (direction, side) pairs of every
 * problem with active[i] != 0.  Pair dp = 2 d + s searches from x_min[i] along -v (s = 0) or +v
 * (s = 1), v = column d of rot[i] (P, p, p row-major): while f(th) < eps and rep <= rep_lim,
 * th += eta v and offset += eta; then one step back, and eta halves, K times or until rep_lim is
 * exceeded; an offset <= 0 becomes the last eta.
 *   init != 0: th = x_min for every pair; fvals is not read.
 *   fvals    (2p, P): f at the points of the previous call; theta (2p, P, p): the next points.
 *   state    (2p P, p + 2) doubles and istate (2p P, 4) ints.
 *   limits   (P, p, 2): limits[i, d, 0] = -offset of side 0, limits[i, d, 1] = offset of side 1,
 *            written when the pair finishes; istate[t, 2] != 0 marks a finished pair t = dp P + i.
 * Limits: 2 p P < 2^31, 1 <= K < 2^30, 0 <= rep_lim < 2^30, finite eta > 0. */
int elfi_b200_romc_line_search_f64(elfi_b200_ctx* ctx, int32_t init, int64_t P, int64_t p,
                                   const double* x_min, const double* rot, const int32_t* active,
                                   double* state, int32_t* istate, const double* fvals,
                                   double* theta, double eps, int64_t K, double eta,
                                   int64_t rep_lim, double* limits, void* stream);

/* elfi_b200_romc_box_sample_f64: n2 uniform points in each of R rotated boxes.
 *   center (R, p), rot and rot_inv (R, p, p), limits (R, p, 2) [lo, hi], volume (R).
 *   pts (R, n2, p): point j of box r is center + rot (lo + (hi - lo) u), u_d the 53-bit (0, 1]
 *            uniform of Philox4x32-10 keyed by seed at counter (j, r, d / 2, 0x524f4d43), words
 *            (x, y) for even d and (z, w) for odd d; the product is summed over d in order.
 *   q (R, n2): 1 / volume[r] when rot_inv (x - center) lies within [lo, hi] (NDimBoundingBox.
 *            contains), else 0.
 *   surr (R, n2), optional (then coef (R, 1 + p + p (p + 1) / 2) is read): the region's local
 *            quadratic at the point, coefficients in PolynomialFeatures(degree=2) order (1, x_i,
 *            then x_i x_j for i <= j), summed in that order. */
int elfi_b200_romc_box_sample_f64(elfi_b200_ctx* ctx, int64_t R, int64_t p, int64_t n2,
                                  const double* center, const double* rot, const double* rot_inv,
                                  const double* limits, const double* volume, uint64_t seed,
                                  const double* coef, double* pts, double* q, double* surr,
                                  void* stream);

/* elfi_b200_romc_weights_f64: RomcPosterior.sample's weights, w = (dist < eps) prior / q, or 0
 * when q <= 0; all arrays (n). */
int elfi_b200_romc_weights_f64(elfi_b200_ctx* ctx, int64_t n, const double* dist,
                               const double* prior, const double* q, double eps, double* w,
                               void* stream);

/* elfi_b200_romc_posterior_unnorm_f64: RomcPosterior's unnormalised density at M points theta
 * (M, p; leading dimension ld_theta): out[m] = prior[m] * count[m], where with fitted local
 * models (fvals NULL) count[m] = #{k : region k contains theta_m and its quadratic <= eps}, and
 * without them (fvals (M, R), leading dimension ld_f) count[m] = #{k : fvals[m, k] <= eps}, as the
 * reference counts objectives without a surrogate.  center, rot_inv, limits and coef as above.
 * Limits: M < 2^40, R < 2^31. */
int elfi_b200_romc_posterior_unnorm_f64(elfi_b200_ctx* ctx, int64_t M, int64_t R, int64_t p,
                                        const double* theta, int64_t ld_theta,
                                        const double* center, const double* rot_inv,
                                        const double* limits, const double* coef,
                                        const double* fvals, int64_t ld_f, double eps,
                                        const double* prior, double* out, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* ELFI_B200_H */
