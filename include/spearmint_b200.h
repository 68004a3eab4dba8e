/*
 * spearmint_b200.h -- C ABI of the H100-native (sm_90a) GP-EI hot path (libspearmint_b200.so).
 *
 * Drop-in boundary: the reference (JasperSnoek/spearmint) is pure Python and binds nothing
 * native on this path, so the "FFI" a maintainer would add is a ctypes binding inside a
 * chooser plugin (see INTEGRATION.md).  Every entry point below replaces a span of the
 * reference's numpy/scipy code; the span is cited as file:line relative to
 * /root/reference/spearmint/spearmint  (GP = gp.py, OPT = chooser/GPEIOptChooser.py,
 * PSEC = chooser/GPEIperSecChooser.py).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch / C++ types.
 *   - every function returns int: 0 ok; <0 bad argument (-(position)); >0 LAPACK-style info
 *     (SMK_ERR_NOT_PD: a pivot was not positive, details in the info[] array);
 *     SMK_ERR_CUDA (1000+cudaError) if a launch failed.
 *   - device functions never allocate and never synchronise the stream; the caller passes
 *     workspaces sized by the *_bytes() queries.  `stream` is a cudaStream_t cast to void*.
 *   - T suffix _f32 / _f64: element type of every floating-point buffer of that call.
 *   - matrices are row-major.  Npad = smk_npad(N) (N rounded up to a multiple of 128); factor
 *     storage is [S][Npad][Npad] with the identity on the padding diagonal.
 *   - `kind`: 0 SE (GP:87-93, ignores ls), 1 ARDSE (GP:95-100), 2 Matern32 (GP:107-113),
 *     3 Matern52 (GP:120-127).
 *   - per-sample hyper-parameters are device arrays: inv_ls[S][D] (=1/ls), amp2[S], noise[S],
 *     mean[S]  -- one row per slice-sampled draw (the reference's hyper_samples list, OPT:628).
 */
#ifndef SPEARMINT_B200_H
#define SPEARMINT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SMK_OK 0
#define SMK_ERR_NOT_PD 1
#define SMK_ERR_CUDA 1000

enum { SMK_SE = 0, SMK_ARDSE = 1, SMK_MATERN32 = 2, SMK_MATERN52 = 3 };

/* ---- library info ------------------------------------------------------------------- */
int smk_version(void);
int smk_npad(int N);                       /* N rounded up to the factor block size (128)   */
int smk_block(int elem_bytes);             /* diagonal-block size NB: 128 for f32, 64 for f64 */
long long smk_launch_count(void);          /* kernels launched by this library so far        */
const char* smk_last_error(void);          /* text of the last SMK_ERR_CUDA                  */
/* measurement aid: when enabled, CUDA events are recorded on the launch stream around the heavy kernels
 * ("predict_tc_kernel", "kxt_kernel", "trtri", "predict_kernel"); smk_timing_ms sums spans by name substring. */
void smk_timing_enable(int on);
double smk_timing_ms(const char* name_substr, int* count);

/* ---- (1) covariance build: gp.dist2 + kernel + chooser.cov  (GP:34-54, GP:87-127, OPT:207-212)
 * out[s][i][j] = amp2[s] * k_kind((X[i]-Y[j]) * inv_ls[s])  (+ diag below when Y == NULL)
 * Y == NULL (self case): out is [S][ld][ld], ld >= N; diagonal gets amp2*1e-6 + diag_add[s]
 *   (OPT:209-210 jitter plus the caller's noise*I, OPT:539), rows/cols N..ld-1 get the identity.
 * Y != NULL (cross case): out is [S][N][ld], ld >= M, no diagonal term.
 * diag_add may be NULL (treated as 0).                                                         */
int smk_cov_build_f32(int kind, int N, int M, int D, int S, const float* X, const float* Y,
                      const float* inv_ls, const float* amp2, const float* diag_add,
                      float* out, int ld, void* stream);
int smk_cov_build_f64(int kind, int N, int M, int D, int S, const double* X, const double* Y,
                      const double* inv_ls, const double* amp2, const double* diag_add,
                      double* out, int ld, void* stream);
/* Self case for a consumer that reads the lower triangle only (the Cholesky inside every slice-sampler log-probability,
 * OPT:637, 659, 690): 32 x 32 tiles strictly above the diagonal are skipped and left as they were.                  */
int smk_cov_build_lower_f32(int kind, int N, int D, int S, const float* X, const float* inv_ls, const float* amp2,
                            const float* diag_add, float* out, int ld, void* stream);
int smk_cov_build_lower_f64(int kind, int N, int D, int S, const double* X, const double* inv_ls, const double* amp2,
                            const double* diag_add, double* out, int ld, void* stream);

/* ---- (2) batched lower Cholesky: spla.cholesky(., lower=True)  (OPT:540, 567, 585)
 * A: [S][Npad][Npad] in/out: only the lower triangle is read, and it is overwritten with L.  On
 * return the strict upper triangle is unspecified: the trailing updates rewrite the upper half
 * of the diagonal tiles they touch (and the tensor-core variant below also the block right of
 * the diagonal in every block-column pair).  winv: [S][Npad/NB][NB][NB] receives the inverses of the
 * diagonal blocks of L (used by every triangular solve below).  info[s] = 0, or 1+index of
 * the first non-positive pivot (the reference raises LinAlgError there, SURVEY 8b).           */
int smk_potrf_lower_batched_f32(int Npad, int S, float* A, float* winv, int* info, void* stream);
int smk_potrf_lower_batched_f64(int Npad, int S, double* A, double* winv, int* info, void* stream);

/* ---- (3) alpha = K^-1 (y - mean), log-determinant, quadratic form
 *          spla.cho_solve((L,True), vals-mean)  (OPT:543, 603);  logprob pieces (OPT:637-640)
 * y: [N] shared by all samples when y_stride == 0, else y + s*y_stride... with F right-hand sides
 *    laid out y[f*ldy + n] (F columns, each contiguous), ldy >= N.
 * alpha: [S][F][Npad] (padding zero).  sum_log_diag[s] = sum_i log L_ii;  quad[s][f] = r' K^-1 r.
 * mean[s] is subtracted from every rhs (may be NULL).  alpha / sum_log_diag / quad may be NULL.
 * N < Npad solves against the leading N x N block of the factor: only rows < N of L and winv are read, so rows >= N
 * of a joint factor may hold anything, NaN included (both entries).
 * One CTA per (sample, group of right-hand sides) holds that group in shared memory, one launch; where it does not fit
 * (Npad > 14080, float32 and float64) the call runs smk_chol_solve_gm_* instead, with its contract.
 * smk_chol_solve_gm_*: the same solve with the right-hand sides in global memory, at any Npad.  alpha is its working
 *   vector and must not be NULL (-11).  About 2 * ceil(N / NB) launches on `stream`.                                */
int smk_chol_solve_f32(int N, int Npad, int S, int F, const float* L, const float* winv,
                       const float* y, long long y_stride, int ldy, const float* mean,
                       float* alpha, float* sum_log_diag, float* quad, void* stream);
int smk_chol_solve_f64(int N, int Npad, int S, int F, const double* L, const double* winv,
                       const double* y, long long y_stride, int ldy, const double* mean,
                       double* alpha, double* sum_log_diag, double* quad, void* stream);
int smk_chol_solve_gm_f32(int N, int Npad, int S, int F, const float* L, const float* winv,
                          const float* y, long long y_stride, int ldy, const float* mean,
                          float* alpha, float* sum_log_diag, float* quad, void* stream);
int smk_chol_solve_gm_f64(int N, int Npad, int S, int F, const double* L, const double* winv,
                          const double* y, long long y_stride, int ldy, const double* mean,
                          double* alpha, double* sum_log_diag, double* quad, void* stream);

/* ---- (3b) GP log marginal likelihood by augmentation (slice-sampler logprob, OPT:637-640, 659-661, 690-692)
 * smk_loglik_set_rhs_*: A[s][N][0:N] = y - mean[s], A[s][N][N] = 1e30 in covariance storage with Npad > N, BEFORE
 * smk_potrf_lower_batched_*; the factorisation then leaves L^-1 (y - mean) in row N.
 * smk_loglik_finish_*: sum_log_diag[s] = sum_{i<N} log L_ii;  quad[s] = |L[N][0:N]|^2 = (y-mean)' K^-1 (y-mean).   */
int smk_loglik_set_rhs_f32(int N, int Npad, int S, const float* y, const float* mean, float* A, void* stream);
int smk_loglik_set_rhs_f64(int N, int Npad, int S, const double* y, const double* mean, double* A, void* stream);
int smk_loglik_finish_f32(int N, int Npad, int S, const float* L, float* sum_log_diag, float* quad, void* stream);
int smk_loglik_finish_f64(int N, int Npad, int S, const double* L, double* sum_log_diag, double* quad, void* stream);

/* ---- (3c) float64 Cholesky of the log-likelihood path (the spla.cholesky inside every slice-sampler logprob,
 * OPT:637, 659, 690): NB = 128 right-looking with one step of look-ahead on two internal streams, diagonal blocks on one
 * SM (warp-synchronous), panel and trailing update on the fp64 tensor path (mma.sync.m8n8k4.f64).  A: [S][Npad][Npad]
 * (lower triangle in/out, Npad % 128 == 0), info[S] as in (2).  use_graph != 0: the launch sequence is captured into a
 * CUDA graph per (A, workspace, info, Npad, S) on first use and replayed afterwards.  Only L is produced.          */
size_t smk_potrf_loglik_workspace_bytes(int Npad, int S);
int smk_potrf_loglik_f64(int Npad, int S, double* A, void* workspace, size_t workspace_bytes, int* info, int use_graph,
                         void* stream);

/* ---- (3d) the whole log-likelihood of a small GP in one launch, one CTA per item: (3) cov_build_lower, (3b)
 * set_rhs, (3c) and (3b) finish fused, the augmented (N+1) x (N+1) lower triangle packed in shared memory.
 * X: [N][D]; per item b: inv_ls[b][D], amp2[b], noise[b], mean[b]; y: [N].  Writes sum_log_diag[b], quad[b] as (3b)
 * and info[b] as (2) (then sum_log_diag[b] = quad[b] = NaN).  N <= SMK_LOGLIK_SMALL_MAX_N: the largest N whose packed
 * triangle (plus 272 doubles of scratch) fits in the 227 KB of shared memory an H100 block can opt into.  Per-item
 * results are bitwise independent of B and of the item's position.  Never allocates, never synchronises; a bad argument
 * #k returns -k.                                                                                                      */
#define SMK_LOGLIK_SMALL_MAX_N 238
int smk_loglik_small_f64(int kind, int N, int D, int B, const double* X, const double* inv_ls, const double* amp2,
                         const double* noise, const double* mean, const double* y, double* sum_log_diag, double* quad,
                         int* info, void* stream);

/* ---- (4) fused predict: cross-covariance tiles generated on the fly -> blocked triangular
 *          solve against L -> predictive mean and variance.  beta and Kx never reach HBM as
 *          N x M matrices.            (OPT:535 cand_cross, OPT:544 beta, OPT:547-548 func_m/func_v)
 * X: [N][D] observed (or observed+pending) inputs, C: [M][D] candidates.
 * mu[s][j]  = C-cov(X, C_j)' alpha[s] + mean[s];   var[s][j] = amp2[s](1+1e-6) - |L^-1 Kx_j|^2
 * mu, var: [S][ldm].  workspace: smk_predict_workspace_bytes(...) bytes.                        */
size_t smk_predict_workspace_bytes(int elem_bytes, int Npad);
int smk_predict_f32(int kind, int N, int Npad, int M, int D, int S, const float* X, const float* C,
                    const float* inv_ls, const float* amp2, const float* mean, const float* L,
                    const float* winv, const float* alpha, float* mu, float* var, int ldm,
                    void* workspace, size_t workspace_bytes, void* stream);
int smk_predict_f64(int kind, int N, int Npad, int M, int D, int S, const double* X, const double* C,
                    const double* inv_ls, const double* amp2, const double* mean, const double* L,
                    const double* winv, const double* alpha, double* mu, double* var, int ldm,
                    void* workspace, size_t workspace_bytes, void* stream);
/* (4-mma) smk_predict_f64 on the fp64 tensor cores (mma.sync.m8n8k4.f64): same arguments, outputs, error codes and
 * workspace (smk_predict_workspace_bytes(8, Npad)).  The off-diagonal update and the diagonal-block solve of every row
 * block run on DMMA, the cross-covariance on DFMA; results differ from smk_predict_f64 only by summation order.   */
int smk_predict_mma_f64(int kind, int N, int Npad, int M, int D, int S, const double* X, const double* C,
                        const double* inv_ls, const double* amp2, const double* mean, const double* L,
                        const double* winv, const double* alpha, double* mu, double* var, int ldm,
                        void* workspace, size_t workspace_bytes, void* stream);

/* ---- (4-tc) fused predict on the tensor cores (wgmma + TMA, register accumulators; float32 in/out, 3 x FP16 split products
 *      with exact power-of-two operand scaling, fp32 accumulation)
 * Same outputs as smk_predict_f32 (OPT:536, 544, 547-548).  Steps, so that the factor-only part is done once:
 *   smk_trtri_split_f32 : Linv = L^-1 (explicit inverse of the blocked factor) as a tf32 hi / lo pair of float arrays,
 *                         each [S][Np][Np] with Np = smk_tc_np(N) (N rounded up to 256), zero above the diagonal.
 *   smk_linv_pack_f16   : the GEMM operand copy of Linv: per-sample scale 2^linv_exp[s] (largest |entry| -> [2^14, 2^15))
 *                         and the round-to-nearest fp16 (hi, lo) pair, each [S][Np][Np] halves.
 *                         linv_exp: [2*S] ints (first S: exponents, rest scratch).
 *   smk_predict_tc_f32  : cross-covariance (candidate-major, fp16 hi/lo) -> D = Kxt * Linv^T on wgmma -> var, mu.
 *                         var can come out NEGATIVE for a candidate on or next to an observation when the noise is
 *                         small: beta is formed with the explicit float32 inverse, and |beta|^2 can exceed amp2 (1 + 1e-6)
 *                         by the inverse's error (measured down to -2.9e-4 amp2 at noise 1e-4, N <= 2560).
 *                         smk_ei_sweep_* take EI = max(best - mu, 0) wherever var <= 0.
 * alpha: [S][Npad_alpha] (first right-hand side).  dbg_beta (tests only, may be NULL): [S][Mc][Np] dump of
 * beta^T, Mc = the candidates of one chunk (ceil128(M) when all fit in one).  Every chunk writes its rows from row 0
 * of the dump, so after a call of several chunks it holds the last chunk only.
 * z (may be NULL): [S][Np], z = Linv (y - mean) -- the `tmp` output of smk_linv_alpha_f32.  With z the predictive mean is
 *   reduced in the GEMM epilogue (mu - mean = alpha . kx = z . beta) and the generator needs no alpha; then chunk 0 of the
 *   cross-covariance can be generated AHEAD of this call, while K is still being factored:
 *   smk_predict_tc_pregen_f32 (same workspace, same shapes; runs on an internal stream forked from `stream`), followed by
 *   smk_predict_tc_f32(..., z, pregenerated = 1).  pregenerated = 1 without a matching pre-generation returns -21.     */
int smk_tc_np(int N);
size_t smk_trtri_workspace_bytes(int Np, int S);
int smk_trtri_split_f32(int Npad, int Np, int S, const float* L, const float* winv, float* linv_hi,
                        float* linv_lo, void* workspace, size_t workspace_bytes, void* stream);
/* Tensor-core variants of the N^3 steps (float32, 3xTF32; the same outputs, and for the factorisation the same contract
 * as (2): only the lower triangle of A is read, the strict upper triangle is unspecified on return):
 *   smk_potrf_lower_batched_tc_f32 : left-looking blocked Cholesky, the rank-(jb*128) update of every block-column pair
 *       runs on wgmma (workspace: 2*S*Npad*Npad floats for the tf32 hi/lo copies of the finished panels).
 *   smk_trtri_split_tc_f32 : L^-1 by row blocks, X[K,:] = -(W_KK L[K,:]) X on wgmma; writes linv_hi/linv_lo like
 *       smk_trtri_split_f32 (workspace: smk_trtri_tc_workspace_bytes).                                          */
int smk_potrf_lower_batched_tc_f32(int Npad, int S, float* A, float* winv, int* info, void* workspace,
                                   size_t workspace_bytes, void* stream);
size_t smk_trtri_tc_workspace_bytes(int Npad, int Np, int S);
int smk_trtri_split_tc_f32(int Npad, int Np, int S, const float* L, const float* winv, float* linv_hi,
                           float* linv_lo, void* workspace, size_t workspace_bytes, void* stream);
/* Both of the above in one call, pipelined: the inverse runs one block step behind the factorisation on an internal second
 * stream (row block K of L^-1 only needs block column K of L to be final), ordered behind `stream` on entry and joined
 * back into it on return.  winv receives the full diagonal-block inverses as usual.  potrf_ws: 2*S*Npad*Npad floats;
 * trtri_ws: smk_trtri_tc_workspace_bytes -- two distinct buffers, both live until the call's work has completed.   */
int smk_potrf_trtri_tc_f32(int Npad, int Np, int S, float* A, float* winv, int* info, void* potrf_ws,
                           size_t potrf_ws_bytes, float* linv_hi, float* linv_lo, void* trtri_ws,
                           size_t trtri_ws_bytes, void* stream);
/* alpha[s] = K_s^-1 (y - mean[s]) from the explicit inverse (two parallel mat-vecs; OPT:543); tmp: [S][Np] floats. */
int smk_linv_alpha_f32(int N, int Np, int S, const float* linv_hi, const float* linv_lo, const float* y,
                       const float* mean, float* alpha, int ld_alpha, float* tmp, void* stream);
/* Accuracy guard of the tensor-core path (csrc/guard.cu): g[s] = estimated RELATIVE error of the predictive variance of a
 * candidate sitting on an observed point, measured by pushing 4 columns of K = L L^T (rows[]: the caller's incumbents) through the explicit inverse
 * (float64 accumulation):  | |Linv (L v)|^2 - |v|^2 | / (noise + 1e-6 amp2),  v = a row of L.  The caller routes the
 * batch to smk_predict_f32 (blocked substitution) when it exceeds its threshold.                                   */
size_t smk_tc_guard_workspace_bytes(int Np, int S);
int smk_tc_guard_f32(int N, int Npad, int Np, int S, const float* L, const float* linv_hi, const float* linv_lo,
                     const float* amp2, const float* noise, const int* rows /* [4] probe rows (device) */, float* g,
                     void* workspace, size_t workspace_bytes, void* stream);
size_t smk_predict_tc_workspace_bytes(int Np, int M, int S, int F);
/* F > 1 with alpha_f [S][F][Npad_alpha] and mu_f [S][F][ldm] non-NULL: additionally the fantasy means
 * mu_f[s][f][j] = cov(X, C_j)' alpha_f[s][f] + mean[s]  (OPT:609) as a second wgmma GEMM on the same Kxt chunk. */
/* The cross-covariance operand generator on its own (cov(comp, cand), OPT:536, and the mean OPT:544), one chunk:
 * k_h16 / k_l16: [S][ceil128(M)][Np] halves = amp2 k(X_n, C_c) * 2^ea as an fp16 (hi, lo) pair, ea = 15 - ceil(log2(
 * amp2 (1 + 1e-6) 1.00001));  mu: [S][ldm].  impl 0: SIMT kernel (any D, S); impl 1: tensor-core kernel
 * (q = (x - c)^2 once per pair, contraction over dimensions for all samples on wgmma; D <= 32, S <= 64, else -1).  */
size_t smk_kxt_pack_workspace_bytes(int Np, int M, int S);
/* debug only: clock64() stamps of the first 64 tiles of CTA 0 of the last impl-1 launch made with SMK_KXT_TIMELINE=1
 * ([tile][8]: production start / end, issuer arrives / operands+accumulator ready / committed, epilogue waits / accumulator
 * ready / drained); out: host memory. */
int smk_debug_kxt_tc_timeline(long long* out, int n);
int smk_kxt_pack_f16(int impl, int kind, int N, int Np, int M, int D, int S, const float* X, const float* C,
                     const float* inv_ls, const float* amp2, const float* mean, const float* alpha, int Npad_alpha,
                     void* k_h16, void* k_l16, float* mu, int ldm, void* workspace, size_t workspace_bytes, void* stream);
int smk_linv_pack_f16(int Np, int S, const float* linv_hi, const float* linv_lo, void* linv_h16, void* linv_l16,
                      int* linv_exp, void* stream);
int smk_predict_tc_f32(int kind, int N, int Np, int M, int D, int S, const float* X, const float* C,
                       const float* inv_ls, const float* amp2, const float* mean, const void* linv_h16,
                       const void* linv_l16, const int* linv_exp, const float* alpha, int Npad_alpha, float* mu,
                       float* var, int ldm, void* workspace, size_t workspace_bytes, float* dbg_beta, int F,
                       const float* alpha_f, float* mu_f, const float* z, int pregenerated, void* stream);
int smk_predict_tc_pregen_f32(int kind, int N, int Np, int M, int D, int S, const float* X, const float* C,
                              const float* inv_ls, const float* amp2, void* workspace, size_t workspace_bytes, int F,
                              void* stream);

/* ---- (4b) cross mean only: mu[s][f][j] = cov(X, C_j)' alpha[s][f] + mean[s]
 *          time-GP mean of EI-per-second (PSEC:442-459) and fantasy means (OPT:609).
 * alpha: [S][F][Npad]; mu: [S][F][ldm].                                                         */
int smk_cross_mean_f32(int kind, int N, int Npad, int M, int D, int S, int F, const float* X,
                       const float* C, const float* inv_ls, const float* amp2, const float* mean,
                       const float* alpha, float* mu, int ldm, void* stream);
int smk_cross_mean_f64(int kind, int N, int Npad, int M, int D, int S, int F, const double* X,
                       const double* C, const double* inv_ls, const double* amp2, const double* mean,
                       const double* alpha, double* mu, int ldm, void* stream);

/* ---- (5) EI sweep: the acquisition scan over candidates  (OPT:551-555; pending OPT:613-619;
 *          per-second PSEC:490-491, 548)
 * mu: [S][F][ldm], var: [S][ldm], best: [S][F] (the caller fills min(vals) or the per-fantasy
 * bests, OPT:532 / OPT:597).  EI is evaluated in double, averaged over the F fantasies.
 * log_time (optional, [S][ldm]): EI is divided by exp(log_time) (PSEC:459, 490).
 * ei (optional): [S][ldm] per-sample EI;  ei_sum (optional): [ldm] += sum over s (caller zeroes).
 * ei and ei_sum are DOUBLE for both variants: late in a run max EI can be < 1e-38 and float storage would flush
 * every candidate to zero (the reference ranks those tail values in float64).                              */
int smk_ei_sweep_f32(int M, int S, int F, const float* mu, const float* var, int ldm,
                     const float* best, const float* log_time, double* ei, double* ei_sum,
                     unsigned long long* ei_max, void* stream);
int smk_ei_sweep_f64(int M, int S, int F, const double* mu, const double* var, int ldm,
                     const double* best, const double* log_time, double* ei, double* ei_sum,
                     unsigned long long* ei_max, void* stream);
/* ei_max (optional, [S]): receives the bit pattern of max_j EI[s][j] as a double (the engine's accuracy guard compares it
 * with the error bound of the explicit-inverse path).  smk_ei_colsum: ei_sum[j] += sum_s ei[s][j].                    */
int smk_ei_colsum(int M, int S, const double* ei, int ldm, double* ei_sum, void* stream);

/* ---- (5b) constrained EI (CONS = chooser/GPConstrainedEIChooser.py)
 * smk_constraint_prob: p[s][j] = Phi(gain[s] * m[s][j]),  m[s][j] = amp2[s] k_s(X, C_j)' t_alpha[s]   (CONS:819-842)
 *   X [N][D] every complete input (violations included), C [M][D], inv_ls/amp2 of the constraint GP (element type T);
 *   t_alpha [S][Npad] = K_c^-1 ff, gain [S], p [S][ldm] and the optional m_out [S][ldm] are DOUBLE for both variants,
 *   and so is the arithmetic (K_c^-1 ff has large entries of both signs: float32 kernel values lose m); Phi is
 *   evaluated with an erfc tail.  The variants differ only in the element type of X, C, inv_ls and amp2.
 * smk_ei_sweep_weighted: the contract of smk_ei_sweep without log_time, each per-sample EI (mean over the F fantasies)
 *   multiplied by w[s][j] (double [S][ldm]: the p of smk_constraint_prob)  (CONS:878, 940).                          */
/* smk_loglik_set_rhs_batched: smk_loglik_set_rhs with one right-hand side per batch item, y [S][ldy], and no mean
 *   subtracted: the joint [amp2, ff] slice move of the classification GP moves ff with every proposal (CONS:1169-1190).
 * smk_lower_matvec_f64: out = L z for the lower factor L [Npad][Npad] of smk_potrf_lower_batched_f64 (one matrix): the
 *   direction of an elliptical-slice step (CONS:1241).                                                             */
int smk_loglik_set_rhs_batched_f32(int N, int Npad, int S, const float* y, int ldy, float* A, void* stream);
int smk_loglik_set_rhs_batched_f64(int N, int Npad, int S, const double* y, int ldy, double* A, void* stream);
int smk_lower_matvec_f64(int N, int Npad, const double* L, const double* z, double* out, void* stream);
int smk_constraint_prob_f32(int kind, int N, int Npad, int M, int D, int S, const float* X, const float* C,
                            const float* inv_ls, const float* amp2, const double* t_alpha, const double* gain,
                            double* p_out, double* m_out, int ldm, void* stream);
int smk_constraint_prob_f64(int kind, int N, int Npad, int M, int D, int S, const double* X, const double* C,
                            const double* inv_ls, const double* amp2, const double* t_alpha, const double* gain,
                            double* p_out, double* m_out, int ldm, void* stream);
int smk_ei_sweep_weighted_f32(int M, int S, int F, const float* mu, const float* var, int ldm, const float* best,
                              const double* w, double* ei, double* ei_sum, unsigned long long* ei_max, void* stream);
int smk_ei_sweep_weighted_f64(int M, int S, int F, const double* mu, const double* var, int ldm, const double* best,
                              const double* w, double* ei, double* ei_sum, unsigned long long* ei_max, void* stream);

/* ---- (5c) random forest (RF = chooser/RandomForestEIChooser.py)
 * smk_forest_fit_f64: grows T regression trees as scikit-learn 1.9's RandomForestRegressor does (RF:64, 72):
 *   DepthFirstTreeBuilder + BestSplitter + MSE, min_samples_leaf 1, min_weight_leaf 0, on X [N][D] (float32, the
 *   conversion sklearn applies), y [N], bootstrap counts w [T][N] as sample weights and the splitter's rand_r state per
 *   tree, rand_r_state [T] -- both drawn on the host from numpy's RNG.  max_depth: INT32_MAX for none;
 *   min_samples_split >= 2.  Node arrays [T][ldn], ldn >= 2N-1, in sklearn's layout and node order: feature (-2 at a
 *   leaf), threshold (-2.0 at a leaf), left / right (-1 at a leaf), n_node_samples, value (sum_total / weighted n);
 *   node_count [T].  One CTA per tree; D is bounded by the per-tree feature arrays in shared memory (32 D bytes, -2
 *   beyond the opt-in limit).  workspace: smk_forest_workspace_bytes(N, D, T).
 * smk_forest_predict_ei_f64: for each candidate C [M][D] (float32), mean = (sum of the T leaf values in tree order)/T,
 *   var = sum_t (leaf_t - mean)^2 / (T-1) (NaN for T = 1, as np.var(ddof=1)), and
 *   ei = s (u Phi(u) + phi(u)), s = sqrt(var) + 1e-4, u = (best - mean)/s  (RF:16-26, 80-85).  mean, var and ei are
 *   optional outputs [M] (NULL: not written).                                                                       */
size_t smk_forest_workspace_bytes(int N, int D, int T);
int smk_forest_fit_f64(int N, int D, int T, const float* X, const double* y, const double* w,
                       const uint32_t* rand_r_state, int max_features, int max_depth, int min_samples_split, int ldn,
                       int* feature, double* threshold, int* left, int* right, int* n_node_samples, double* value,
                       int* node_count, void* workspace, size_t workspace_bytes, void* stream);
int smk_forest_predict_ei_f64(int M, int D, int T, int ldn, const float* C, const int* feature, const double* threshold,
                              const int* left, const int* right, const double* value, double best, double* mean,
                              double* var, double* ei, void* stream);

/* ---- (6) selection: argsort(mean)[-k:] and argmax(mean)   (OPT:270-271, OPT:294)
 * score: [M].  idx_out[k]: indices of the k largest scores in ASCENDING score order (so
 * idx_out[k-1] is the argmax; ties resolved towards the lower index, numpy's first-max rule).
 * NaN scores are never selected: with fewer than k non-NaN scores the first slots get index -1 and value -inf.
 * k <= 256 and k <= M (else -2).  workspace: smk_topk_workspace_bytes(M, k) (else -6).              */
size_t smk_topk_workspace_bytes(int M, int k);
int smk_topk_f32(int M, int k, const float* score, int* idx_out, float* val_out,
                 void* workspace, size_t workspace_bytes, void* stream);
int smk_topk_f64(int M, int k, const double* score, int* idx_out, double* val_out,
                 void* workspace, size_t workspace_bytes, void* stream);

/* ---- (7) whole path with HOST buffers: GPEIOptChooser.ei_over_hypers, no pending (OPT:331-341)
 * Copies inputs host->device, runs (1)-(5) for all S samples on the current device, copies the
 * (S x M) EI matrix back (row s = sample s).  hypers as host arrays ls[S][D], amp2, noise, mean.
 * Returns SMK_ERR_NOT_PD if any factorisation failed (info_out[S] optional).                      */
int smk_ei_over_hypers_host_f32(int kind, int N, int M, int D, int S, const double* comp,
                                const double* cand, const double* vals, const double* ls,
                                const double* amp2, const double* noise, const double* mean,
                                double* ei_out, int* info_out);

/* ---- (8) EI value + input-gradient terms at Q query points with cached factors
 *          GPEIOptChooser.grad_optimize_ei (OPT:391-525), gp.grad_dist2 / grad_<kernel> (GP:56-85, 102-132)
 * alpha: [S][F][Npad] (K^-1 (y_f - mean));  gamma: [S][Q][Npad] (K^-1 kx_q, from smk_chol_solve with the
 * cross-covariance columns as right-hand sides);  xq: [Q][D] query points.
 * out: [S][Q][F+1][D+1]:  out[f][d] = sum_n alpha_f[n] gk[n][d];  out[f][D] = kx' alpha_f;
 *                         out[F][d] = sum_n gamma[n] gk[n][d];     out[F][D] = kx' K^-1 kx,
 * with gk[n][d] = dk/dr2 * (2/ls_d) (X[n][d] - xq[d]) / ls_d  (correlation gradient, no amp2 -- the
 * reference applies 0.5*amp2 afterwards, OPT:437).  kind SMK_SE is rejected like the reference (no gp.grad_SE): -1.
 * Any F >= 1 (the fantasy rows are staged 64 at a time); -4 also when D is too large for the shared-memory staging
 * (D > 324 in float64, D > 712 in float32).  Each output element is summed over n = 0 .. N-1 in order, so row f of
 * an F-fantasy call equals row f of any call with more fantasies bit for bit.                                     */
int smk_ei_grad_terms_f32(int kind, int N, int Npad, int D, int S, int Q, int F, const float* X, const float* xq,
                          const float* inv_ls, const float* amp2, const float* alpha, const float* gamma,
                          float* out, void* stream);
int smk_ei_grad_terms_f64(int kind, int N, int Npad, int D, int S, int Q, int F, const double* X, const double* xq,
                          const double* inv_ls, const double* amp2, const double* alpha, const double* gamma,
                          double* out, void* stream);

/* ---- (8b) ML-II: the traces of GP.optimize_hypers' grad_nlogprob (GP:238-264) at one hyper-parameter setting per sample
 * alpha: [S][lda] = K^-1 (y - mean);  Kinv: [S][N][ldk] = K^-1 (smk_chol_solve with the identity as right-hand sides).
 * out: [S][D+2] doubles:  out[0] = sum_ij J_ij (corr_ij + 1e-6 delta_ij),  out[1] = tr J,
 *                         out[2+d] = sum_ij J_ji gcorr_ij^d X[i][d],   J = alpha alpha' - K^-1  (GP:246).
 * Host side: grad = [0.5 out[0] amp2, 0.5 out[1] noise, -amp2 out[2+d]] and grad_nlogprob = -grad -- including the
 * reference's length-scale expression (GP:258-259), which is not the true derivative and is reproduced as is.        */
int smk_mll_grad_terms_f32(int kind, int N, int D, int S, const float* X, const float* inv_ls, const float* alpha, int lda,
                           const float* Kinv, int ldk, double* out, void* stream);
int smk_mll_grad_terms_f64(int kind, int N, int D, int S, const double* X, const double* inv_ls, const double* alpha, int lda,
                           const double* Kinv, int ldk, double* out, void* stream);

/* ---- (9) Sobol candidate grid on the device: sobol_lib.i4_sobol_generate (spearmint/spearmint/sobol_lib.py:125-156,
 *          called by ExperimentGrid GRID:192-196 and spearmint-lite LITE:171-173)
 * out[j][d], j < n, d < D (row-major [n][D], i.e. the TRANSPOSE of the reference's (D, n) return value -- the layout
 * its callers use): point of Gray-code seed max(skip + j - 1, 0).  V: device copy of the direction numbers [D][30]
 * (spearmint_b200/data/sobol_v_1111x30.npy, frozen from the reference's Joe-Kuo table by tools/make_sobol_table.py).
 * Returns -3 past the reference's 2^30 point limit.                                                               */
int smk_sobol_generate_f32(int D, long long n, long long skip, const uint32_t* V, float* out, void* stream);
int smk_sobol_generate_f64(int D, long long n, long long skip, const uint32_t* V, double* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SPEARMINT_B200_H */
