// api.cu -- extern "C" surface of libspearmint_b200.so (see include/spearmint_b200.h).
#include <cuda_fp16.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <vector>

#include "../../include/spearmint_b200.h"
#include "common.cuh"

namespace smk {

static std::atomic<long long> g_launches{0};
static char g_err[512] = "";

void count_launch(int n) { g_launches += n; }
long long launch_count() { return g_launches.load(); }

// ---- optional kernel timing: (name, start, stop) event triples recorded around selected launches
struct TimedSpan { const char* name; cudaEvent_t e0, e1; };
static std::vector<TimedSpan> g_spans;
static int g_timing = 0;
static cudaEvent_t g_open = nullptr;

void timing_begin(const char* name, cudaStream_t st) {
  if (!g_timing) return;
  TimedSpan t;
  t.name = name;
  cudaEventCreate(&t.e0);
  cudaEventCreate(&t.e1);
  cudaEventRecord(t.e0, st);
  g_spans.push_back(t);
}
void timing_end(cudaStream_t st) {
  if (!g_timing || g_spans.empty()) return;
  cudaEventRecord(g_spans.back().e1, st);
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) return SMK_OK;
  snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
  return SMK_ERR_CUDA + (int)e;
}

// implemented in the other translation units
template <typename T>
int cov_build(int, int, int, int, int, const T*, const T*, const T*, const T*, const T*, T*, int, cudaStream_t, int lower = 0);
template <typename T>
int potrf_lower_batched(int, int, T*, T*, int*, cudaStream_t);
template <typename T>
int chol_solve(int, int, int, int, const T*, const T*, const T*, long long, int, const T*, T*, T*, T*, cudaStream_t);
template <typename T>
int chol_solve_gm(int, int, int, int, const T*, const T*, const T*, long long, int, const T*, T*, T*, T*, cudaStream_t);
template <typename T>
int loglik_set_rhs(int, int, int, const T*, const T*, T*, cudaStream_t);
template <typename T>
int loglik_finish(int, int, int, const T*, T*, T*, cudaStream_t);
template <typename T>
int predict(int, int, int, int, int, int, const T*, const T*, const T*, const T*, const T*, const T*, const T*,
            const T*, T*, T*, int, void*, size_t, cudaStream_t);
template <typename T>
int cross_mean(int, int, int, int, int, int, int, const T*, const T*, const T*, const T*, const T*, const T*, T*,
               int, cudaStream_t);
template <typename T>
int ei_sweep(int, int, int, const T*, const T*, int, const T*, const T*, double*, double*, unsigned long long*, cudaStream_t);
int ei_colsum(int, int, const double*, int, double*, cudaStream_t);
template <typename T>
int ei_sweep_weighted(int, int, int, const T*, const T*, int, const T*, const double*, double*, double*,
                      unsigned long long*, cudaStream_t);
template <typename T>
int loglik_set_rhs_batched(int, int, int, const T*, int, T*, cudaStream_t);
int lower_matvec(int, int, const double*, const double*, double*, cudaStream_t);
template <typename T>
int constraint_prob(int, int, int, int, int, int, const T*, const T*, const T*, const T*, const double*, const double*,
                    double*, double*, int, cudaStream_t);
template <typename T>
int topk(int, int, const T*, int*, T*, void*, size_t, cudaStream_t);
template <typename T>
int ei_grad_terms(int, int, int, int, int, int, int, const T*, const T*, const T*, const T*, const T*, const T*, T*,
                  cudaStream_t);
template <typename T>
int mll_grad_terms(int, int, int, int, const T*, const T*, const T*, int, const T*, int, double*, cudaStream_t);
size_t topk_workspace_bytes(int, int);
int tc_np(int);
size_t trtri_workspace_bytes(int, int);
int trtri_split(int, int, int, const float*, const float*, float*, float*, void*, size_t, cudaStream_t);
size_t predict_tc_workspace_bytes(int, int, int, int);
int potrf_lower_batched_tc(int, int, float*, float*, int*, float*, float*, cudaStream_t, cudaEvent_t* blk_done = nullptr);
int potrf_trtri_tc(int, int, int, float*, float*, int*, float*, float*, float*, float*, void*, size_t, cudaStream_t);
size_t trtri_tc_workspace_bytes(int, int, int);
int trtri_split_tc(int, int, int, const float*, const float*, float*, float*, void*, size_t, cudaStream_t);
int linv_alpha(int, int, int, const float*, const float*, const float*, const float*, float*, int, float*, cudaStream_t);
int linv_pack_f16(int, int, const float*, const float*, __half*, __half*, int*, cudaStream_t);
size_t kxt_pack_workspace_bytes(int, int, int);
int kxt_tc_timeline(long long*, int);
int kxt_pack(int, int, int, int, int, int, int, const float*, const float*, const float*, const float*, const float*,
             const float*, int, __half*, __half*, float*, int, void*, size_t, cudaStream_t);
int predict_tc(int, int, int, int, int, int, const float*, const float*, const float*, const float*, const float*,
               const __half*, const __half*, const int*, const float*, int, float*, float*, int, void*, size_t, float*,
               int, const float*, float*, const float*, int, cudaStream_t);
int predict_tc_pregen(int, int, int, int, int, int, const float*, const float*, const float*, const float*, void*, size_t,
                      int, cudaStream_t);
size_t predict_workspace_bytes_any(int, int);
size_t potrf_ll_workspace_bytes(int, int);
template <typename T>
int sobol_generate(int, long, long, const uint32_t*, T*, cudaStream_t);
size_t tc_guard_workspace_bytes(int, int);
int tc_guard(int, int, int, int, const float*, const float*, const float*, const float*, const float*, const int*, float*, void*,
             size_t, cudaStream_t);
int potrf_ll_f64(int, int, double*, double*, int*, int, cudaStream_t);
size_t forest_workspace_bytes(int, int, int);
int forest_fit(int, int, int, const float*, const double*, const double*, const uint32_t*, int, int, int, int, int*,
               double*, int*, int*, int*, double*, int*, void*, size_t, cudaStream_t);
int forest_predict_ei(int, int, int, int, const float*, const int*, const double*, const int*, const int*, const double*,
                      double, double*, double*, double*, cudaStream_t);

}  // namespace smk

using namespace smk;
#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" {

int smk_version(void) { return 100; }
int smk_npad(int N) { return ((N + kNpadMult - 1) / kNpadMult) * kNpadMult; }
int smk_block(int elem_bytes) { return elem_bytes == 8 ? Cfg<double>::NB : Cfg<float>::NB; }
long long smk_launch_count(void) { return g_launches.load(); }
const char* smk_last_error(void) { return g_err; }

void smk_timing_enable(int on) {
  g_timing = on;
  for (auto& t : g_spans) { cudaEventDestroy(t.e0); cudaEventDestroy(t.e1); }
  g_spans.clear();
}
/* Sum of the recorded durations (ms) of every span whose name contains `substr`, and their count.
 * Synchronises on the recorded events; spans stay recorded until smk_timing_enable() is called again. */
double smk_timing_ms(const char* substr, int* count) {
  double tot = 0.0;
  int n = 0;
  for (auto& t : g_spans) {
    if (substr && !strstr(t.name, substr)) continue;
    cudaEventSynchronize(t.e1);
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, t.e0, t.e1) == cudaSuccess) { tot += ms; ++n; }
  }
  if (count) *count = n;
  return tot;
}

int smk_cov_build_f32(int kind, int N, int M, int D, int S, const float* X, const float* Y, const float* inv_ls,
                      const float* amp2, const float* diag_add, float* out, int ld, void* stream) {
  return cov_build<float>(kind, N, M, D, S, X, Y, inv_ls, amp2, diag_add, out, ld, ST(stream));
}
int smk_cov_build_f64(int kind, int N, int M, int D, int S, const double* X, const double* Y, const double* inv_ls,
                      const double* amp2, const double* diag_add, double* out, int ld, void* stream) {
  return cov_build<double>(kind, N, M, D, S, X, Y, inv_ls, amp2, diag_add, out, ld, ST(stream));
}
int smk_cov_build_lower_f32(int kind, int N, int D, int S, const float* X, const float* inv_ls, const float* amp2,
                            const float* diag_add, float* out, int ld, void* stream) {
  return cov_build<float>(kind, N, N, D, S, X, nullptr, inv_ls, amp2, diag_add, out, ld, ST(stream), 1);
}
int smk_cov_build_lower_f64(int kind, int N, int D, int S, const double* X, const double* inv_ls, const double* amp2,
                            const double* diag_add, double* out, int ld, void* stream) {
  return cov_build<double>(kind, N, N, D, S, X, nullptr, inv_ls, amp2, diag_add, out, ld, ST(stream), 1);
}

int smk_potrf_lower_batched_f32(int Npad, int S, float* A, float* winv, int* info, void* stream) {
  return potrf_lower_batched<float>(Npad, S, A, winv, info, ST(stream));
}
int smk_potrf_lower_batched_f64(int Npad, int S, double* A, double* winv, int* info, void* stream) {
  return potrf_lower_batched<double>(Npad, S, A, winv, info, ST(stream));
}

size_t smk_potrf_loglik_workspace_bytes(int Npad, int S) { return potrf_ll_workspace_bytes(Npad, S); }
int smk_potrf_loglik_f64(int Npad, int S, double* A, void* workspace, size_t workspace_bytes, int* info, int use_graph,
                         void* stream) {
  if (!workspace || workspace_bytes < potrf_ll_workspace_bytes(Npad, S)) return -4;
  return potrf_ll_f64(Npad, S, A, reinterpret_cast<double*>(workspace), info, use_graph, ST(stream));
}

int smk_chol_solve_f32(int N, int Npad, int S, int F, const float* L, const float* winv, const float* y,
                       long long y_stride, int ldy, const float* mean, float* alpha, float* sum_log_diag,
                       float* quad, void* stream) {
  return chol_solve<float>(N, Npad, S, F, L, winv, y, y_stride, ldy, mean, alpha, sum_log_diag, quad, ST(stream));
}
int smk_chol_solve_f64(int N, int Npad, int S, int F, const double* L, const double* winv, const double* y,
                       long long y_stride, int ldy, const double* mean, double* alpha, double* sum_log_diag,
                       double* quad, void* stream) {
  return chol_solve<double>(N, Npad, S, F, L, winv, y, y_stride, ldy, mean, alpha, sum_log_diag, quad, ST(stream));
}
int smk_chol_solve_gm_f32(int N, int Npad, int S, int F, const float* L, const float* winv, const float* y,
                          long long y_stride, int ldy, const float* mean, float* alpha, float* sum_log_diag,
                          float* quad, void* stream) {
  return chol_solve_gm<float>(N, Npad, S, F, L, winv, y, y_stride, ldy, mean, alpha, sum_log_diag, quad, ST(stream));
}
int smk_chol_solve_gm_f64(int N, int Npad, int S, int F, const double* L, const double* winv, const double* y,
                          long long y_stride, int ldy, const double* mean, double* alpha, double* sum_log_diag,
                          double* quad, void* stream) {
  return chol_solve_gm<double>(N, Npad, S, F, L, winv, y, y_stride, ldy, mean, alpha, sum_log_diag, quad, ST(stream));
}

int smk_loglik_set_rhs_f32(int N, int Npad, int S, const float* y, const float* mean, float* A, void* stream) {
  return loglik_set_rhs<float>(N, Npad, S, y, mean, A, ST(stream));
}
int smk_loglik_set_rhs_f64(int N, int Npad, int S, const double* y, const double* mean, double* A, void* stream) {
  return loglik_set_rhs<double>(N, Npad, S, y, mean, A, ST(stream));
}
int smk_loglik_finish_f32(int N, int Npad, int S, const float* L, float* sld, float* quad, void* stream) {
  return loglik_finish<float>(N, Npad, S, L, sld, quad, ST(stream));
}
int smk_loglik_finish_f64(int N, int Npad, int S, const double* L, double* sld, double* quad, void* stream) {
  return loglik_finish<double>(N, Npad, S, L, sld, quad, ST(stream));
}

size_t smk_predict_workspace_bytes(int elem_bytes, int Npad) { return predict_workspace_bytes_any(elem_bytes, Npad); }

int smk_predict_f32(int kind, int N, int Npad, int M, int D, int S, const float* X, const float* C,
                    const float* inv_ls, const float* amp2, const float* mean, const float* L, const float* winv,
                    const float* alpha, float* mu, float* var, int ldm, void* workspace, size_t workspace_bytes,
                    void* stream) {
  return predict<float>(kind, N, Npad, M, D, S, X, C, inv_ls, amp2, mean, L, winv, alpha, mu, var, ldm, workspace,
                        workspace_bytes, ST(stream));
}
int smk_predict_f64(int kind, int N, int Npad, int M, int D, int S, const double* X, const double* C,
                    const double* inv_ls, const double* amp2, const double* mean, const double* L,
                    const double* winv, const double* alpha, double* mu, double* var, int ldm, void* workspace,
                    size_t workspace_bytes, void* stream) {
  return predict<double>(kind, N, Npad, M, D, S, X, C, inv_ls, amp2, mean, L, winv, alpha, mu, var, ldm, workspace,
                         workspace_bytes, ST(stream));
}

int smk_tc_np(int N) { return tc_np(N); }
size_t smk_trtri_workspace_bytes(int Np, int S) { return trtri_workspace_bytes(Np, S); }
int smk_trtri_split_f32(int Npad, int Np, int S, const float* L, const float* winv, float* linv_hi, float* linv_lo,
                        void* workspace, size_t workspace_bytes, void* stream) {
  return trtri_split(Npad, Np, S, L, winv, linv_hi, linv_lo, workspace, workspace_bytes, ST(stream));
}
size_t smk_predict_tc_workspace_bytes(int Np, int M, int S, int F) { return predict_tc_workspace_bytes(Np, M, S, F); }
int smk_potrf_lower_batched_tc_f32(int Npad, int S, float* A, float* winv, int* info, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  if (!workspace || workspace_bytes < 2 * (size_t)S * Npad * Npad * sizeof(float)) return -6;
  float* lhi = reinterpret_cast<float*>(workspace);
  return potrf_lower_batched_tc(Npad, S, A, winv, info, lhi, lhi + (size_t)S * Npad * Npad, ST(stream));
}
size_t smk_trtri_tc_workspace_bytes(int Npad, int Np, int S) { return trtri_tc_workspace_bytes(Npad, Np, S); }
int smk_trtri_split_tc_f32(int Npad, int Np, int S, const float* L, const float* winv, float* linv_hi, float* linv_lo,
                           void* workspace, size_t workspace_bytes, void* stream) {
  return trtri_split_tc(Npad, Np, S, L, winv, linv_hi, linv_lo, workspace, workspace_bytes, ST(stream));
}
int smk_potrf_trtri_tc_f32(int Npad, int Np, int S, float* A, float* winv, int* info, void* potrf_ws, size_t potrf_ws_bytes,
                           float* linv_hi, float* linv_lo, void* trtri_ws, size_t trtri_ws_bytes, void* stream) {
  if (!potrf_ws || potrf_ws_bytes < 2 * (size_t)S * Npad * Npad * sizeof(float)) return -8;
  float* lhi = reinterpret_cast<float*>(potrf_ws);
  return potrf_trtri_tc(Npad, Np, S, A, winv, info, lhi, lhi + (size_t)S * Npad * Npad, linv_hi, linv_lo, trtri_ws,
                        trtri_ws_bytes, ST(stream));
}
int smk_linv_alpha_f32(int N, int Np, int S, const float* linv_hi, const float* linv_lo, const float* y,
                       const float* mean, float* alpha, int ld_alpha, float* tmp, void* stream) {
  return linv_alpha(N, Np, S, linv_hi, linv_lo, y, mean, alpha, ld_alpha, tmp, ST(stream));
}
int smk_sobol_generate_f32(int D, long long n, long long skip, const uint32_t* V, float* out, void* stream) {
  return sobol_generate<float>(D, (long)n, (long)skip, V, out, ST(stream));
}
int smk_sobol_generate_f64(int D, long long n, long long skip, const uint32_t* V, double* out, void* stream) {
  return sobol_generate<double>(D, (long)n, (long)skip, V, out, ST(stream));
}
size_t smk_tc_guard_workspace_bytes(int Np, int S) { return tc_guard_workspace_bytes(Np, S); }
int smk_tc_guard_f32(int N, int Npad, int Np, int S, const float* L, const float* linv_hi, const float* linv_lo,
                     const float* amp2, const float* noise, const int* rows, float* g, void* workspace, size_t workspace_bytes,
                     void* stream) {
  return tc_guard(N, Npad, Np, S, L, linv_hi, linv_lo, amp2, noise, rows, g, workspace, workspace_bytes, ST(stream));
}
int smk_debug_kxt_tc_timeline(long long* out, int n) { return kxt_tc_timeline(out, n); }
size_t smk_kxt_pack_workspace_bytes(int Np, int M, int S) { return kxt_pack_workspace_bytes(Np, M, S); }
int smk_kxt_pack_f16(int impl, int kind, int N, int Np, int M, int D, int S, const float* X, const float* C,
                     const float* inv_ls, const float* amp2, const float* mean, const float* alpha, int Npad_alpha,
                     void* k_h16, void* k_l16, float* mu, int ldm, void* workspace, size_t workspace_bytes, void* stream) {
  return kxt_pack(impl, kind, N, Np, M, D, S, X, C, inv_ls, amp2, mean, alpha, Npad_alpha,
                  reinterpret_cast<__half*>(k_h16), reinterpret_cast<__half*>(k_l16), mu, ldm, workspace, workspace_bytes,
                  ST(stream));
}
int smk_linv_pack_f16(int Np, int S, const float* linv_hi, const float* linv_lo, void* linv_h16, void* linv_l16,
                      int* linv_exp, void* stream) {
  return linv_pack_f16(Np, S, linv_hi, linv_lo, reinterpret_cast<__half*>(linv_h16), reinterpret_cast<__half*>(linv_l16),
                       linv_exp, ST(stream));
}
int smk_predict_tc_f32(int kind, int N, int Np, int M, int D, int S, const float* X, const float* C,
                       const float* inv_ls, const float* amp2, const float* mean, const void* linv_h16,
                       const void* linv_l16, const int* linv_exp, const float* alpha, int Npad_alpha, float* mu,
                       float* var, int ldm, void* workspace, size_t workspace_bytes, float* dbg_beta, int F,
                       const float* alpha_f, float* mu_f, const float* z, int pregenerated, void* stream) {
  return predict_tc(kind, N, Np, M, D, S, X, C, inv_ls, amp2, mean, reinterpret_cast<const __half*>(linv_h16),
                    reinterpret_cast<const __half*>(linv_l16), linv_exp, alpha, Npad_alpha, mu, var, ldm, workspace,
                    workspace_bytes, dbg_beta, F, alpha_f, mu_f, z, pregenerated, ST(stream));
}
int smk_predict_tc_pregen_f32(int kind, int N, int Np, int M, int D, int S, const float* X, const float* C,
                              const float* inv_ls, const float* amp2, void* workspace, size_t workspace_bytes, int F,
                              void* stream) {
  return predict_tc_pregen(kind, N, Np, M, D, S, X, C, inv_ls, amp2, workspace, workspace_bytes, F, ST(stream));
}

int smk_cross_mean_f32(int kind, int N, int Npad, int M, int D, int S, int F, const float* X, const float* C,
                       const float* inv_ls, const float* amp2, const float* mean, const float* alpha, float* mu,
                       int ldm, void* stream) {
  return cross_mean<float>(kind, N, Npad, M, D, S, F, X, C, inv_ls, amp2, mean, alpha, mu, ldm, ST(stream));
}
int smk_cross_mean_f64(int kind, int N, int Npad, int M, int D, int S, int F, const double* X, const double* C,
                       const double* inv_ls, const double* amp2, const double* mean, const double* alpha,
                       double* mu, int ldm, void* stream) {
  return cross_mean<double>(kind, N, Npad, M, D, S, F, X, C, inv_ls, amp2, mean, alpha, mu, ldm, ST(stream));
}

int smk_ei_sweep_f32(int M, int S, int F, const float* mu, const float* var, int ldm, const float* best,
                     const float* log_time, double* ei, double* ei_sum, unsigned long long* ei_max, void* stream) {
  return ei_sweep<float>(M, S, F, mu, var, ldm, best, log_time, ei, ei_sum, ei_max, ST(stream));
}
int smk_ei_sweep_f64(int M, int S, int F, const double* mu, const double* var, int ldm, const double* best,
                     const double* log_time, double* ei, double* ei_sum, unsigned long long* ei_max, void* stream) {
  return ei_sweep<double>(M, S, F, mu, var, ldm, best, log_time, ei, ei_sum, ei_max, ST(stream));
}
int smk_ei_colsum(int M, int S, const double* ei, int ldm, double* ei_sum, void* stream) {
  return ei_colsum(M, S, ei, ldm, ei_sum, ST(stream));
}
int smk_ei_sweep_weighted_f32(int M, int S, int F, const float* mu, const float* var, int ldm, const float* best,
                              const double* w, double* ei, double* ei_sum, unsigned long long* ei_max, void* stream) {
  return ei_sweep_weighted<float>(M, S, F, mu, var, ldm, best, w, ei, ei_sum, ei_max, ST(stream));
}
int smk_ei_sweep_weighted_f64(int M, int S, int F, const double* mu, const double* var, int ldm, const double* best,
                              const double* w, double* ei, double* ei_sum, unsigned long long* ei_max, void* stream) {
  return ei_sweep_weighted<double>(M, S, F, mu, var, ldm, best, w, ei, ei_sum, ei_max, ST(stream));
}

int smk_loglik_set_rhs_batched_f32(int N, int Npad, int S, const float* y, int ldy, float* A, void* stream) {
  return loglik_set_rhs_batched<float>(N, Npad, S, y, ldy, A, ST(stream));
}
int smk_loglik_set_rhs_batched_f64(int N, int Npad, int S, const double* y, int ldy, double* A, void* stream) {
  return loglik_set_rhs_batched<double>(N, Npad, S, y, ldy, A, ST(stream));
}
int smk_lower_matvec_f64(int N, int Npad, const double* L, const double* z, double* out, void* stream) {
  return lower_matvec(N, Npad, L, z, out, ST(stream));
}

int smk_constraint_prob_f32(int kind, int N, int Npad, int M, int D, int S, const float* X, const float* C,
                            const float* inv_ls, const float* amp2, const double* t_alpha, const double* gain,
                            double* p_out, double* m_out, int ldm, void* stream) {
  return constraint_prob<float>(kind, N, Npad, M, D, S, X, C, inv_ls, amp2, t_alpha, gain, p_out, m_out, ldm,
                                ST(stream));
}
int smk_constraint_prob_f64(int kind, int N, int Npad, int M, int D, int S, const double* X, const double* C,
                            const double* inv_ls, const double* amp2, const double* t_alpha, const double* gain,
                            double* p_out, double* m_out, int ldm, void* stream) {
  return constraint_prob<double>(kind, N, Npad, M, D, S, X, C, inv_ls, amp2, t_alpha, gain, p_out, m_out, ldm,
                                 ST(stream));
}

size_t smk_forest_workspace_bytes(int N, int D, int T) { return forest_workspace_bytes(N, D, T); }
int smk_forest_fit_f64(int N, int D, int T, const float* X, const double* y, const double* w,
                       const uint32_t* rand_r_state, int max_features, int max_depth, int min_samples_split, int ldn,
                       int* feature, double* threshold, int* left, int* right, int* n_node_samples, double* value,
                       int* node_count, void* workspace, size_t workspace_bytes, void* stream) {
  return forest_fit(N, D, T, X, y, w, rand_r_state, max_features, max_depth, min_samples_split, ldn, feature, threshold,
                    left, right, n_node_samples, value, node_count, workspace, workspace_bytes, ST(stream));
}
int smk_forest_predict_ei_f64(int M, int D, int T, int ldn, const float* C, const int* feature, const double* threshold,
                              const int* left, const int* right, const double* value, double best, double* mean,
                              double* var, double* ei, void* stream) {
  return forest_predict_ei(M, D, T, ldn, C, feature, threshold, left, right, value, best, mean, var, ei, ST(stream));
}

size_t smk_topk_workspace_bytes(int M, int k) { return topk_workspace_bytes(M, k); }
int smk_topk_f32(int M, int k, const float* score, int* idx_out, float* val_out, void* workspace,
                 size_t workspace_bytes, void* stream) {
  return topk<float>(M, k, score, idx_out, val_out, workspace, workspace_bytes, ST(stream));
}
int smk_topk_f64(int M, int k, const double* score, int* idx_out, double* val_out, void* workspace,
                 size_t workspace_bytes, void* stream) {
  return topk<double>(M, k, score, idx_out, val_out, workspace, workspace_bytes, ST(stream));
}

int smk_ei_grad_terms_f32(int kind, int N, int Npad, int D, int S, int Q, int F, const float* X, const float* xq,
                          const float* inv_ls, const float* amp2, const float* alpha, const float* gamma,
                          float* out, void* stream) {
  if (kind == SMK_SE) return -1;
  return ei_grad_terms<float>(kind, N, Npad, D, S, Q, F, X, xq, inv_ls, amp2, alpha, gamma, out, ST(stream));
}
int smk_ei_grad_terms_f64(int kind, int N, int Npad, int D, int S, int Q, int F, const double* X, const double* xq,
                          const double* inv_ls, const double* amp2, const double* alpha, const double* gamma,
                          double* out, void* stream) {
  if (kind == SMK_SE) return -1;
  return ei_grad_terms<double>(kind, N, Npad, D, S, Q, F, X, xq, inv_ls, amp2, alpha, gamma, out, ST(stream));
}

int smk_mll_grad_terms_f32(int kind, int N, int D, int S, const float* X, const float* inv_ls, const float* alpha, int lda,
                           const float* Kinv, int ldk, double* out, void* stream) {
  return mll_grad_terms<float>(kind, N, D, S, X, inv_ls, alpha, lda, Kinv, ldk, out, ST(stream));
}
int smk_mll_grad_terms_f64(int kind, int N, int D, int S, const double* X, const double* inv_ls, const double* alpha, int lda,
                           const double* Kinv, int ldk, double* out, void* stream) {
  return mll_grad_terms<double>(kind, N, D, S, X, inv_ls, alpha, lda, Kinv, ldk, out, ST(stream));
}

// -------------------------------------------------------------------------------------------------
// Host-buffer pipeline: the call a non-Python host (or a ctypes stub) makes for ei_over_hypers.
// Device buffers are cached between calls (grow-only) so steady-state calls do no cudaMalloc.
// -------------------------------------------------------------------------------------------------
namespace {
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  void* get(size_t bytes) {
    if (bytes > cap) {
      if (p) cudaFree(p);
      p = nullptr;
      cap = 0;
      if (cudaMalloc(&p, bytes) != cudaSuccess) return nullptr;
      cap = bytes;
    }
    return p;
  }
};
DevBuf g_in, g_fac, g_winv, g_alpha, g_mv, g_ws, g_ei, g_linv, g_ws2, g_l16;
std::vector<float> g_host;
}  // namespace

int smk_ei_over_hypers_host_f32(int kind, int N, int M, int D, int S, const double* comp, const double* cand,
                                const double* vals, const double* ls, const double* amp2, const double* noise,
                                const double* mean, double* ei_out, int* info_out) {
  if (kind < 0 || kind > 3) return -1;
  if (N <= 0) return -2;
  if (M <= 0) return -3;
  if (D <= 0) return -4;
  if (S <= 0) return -5;
  if (!comp || !cand || !vals || !ls || !amp2 || !noise || !mean || !ei_out) return -6;
  const int Npad = smk_npad(N), NB = Cfg<float>::NB, ldm = ((M + 127) / 128) * 128, Np = smk_tc_np(N);
  cudaStream_t st = 0;
  // ---- pack all small inputs into one pinned-size host block: X | C | y | inv_ls | amp2 | noise | mean | best
  const size_t nX = (size_t)N * D, nC = (size_t)M * D, nH = (size_t)S * D;
  const size_t tot = nX + nC + N + nH + 4 * (size_t)S;
  g_host.resize(tot);
  float* h = g_host.data();
  float *hX = h, *hC = hX + nX, *hy = hC + nC, *hil = hy + N, *ha = hil + nH, *hn = ha + S, *hm = hn + S,
        *hb = hm + S;
  for (size_t i = 0; i < nX; ++i) hX[i] = (float)comp[i];
  for (size_t i = 0; i < nC; ++i) hC[i] = (float)cand[i];
  double best = vals[0];
  for (int i = 0; i < N; ++i) { hy[i] = (float)vals[i]; if (vals[i] < best) best = vals[i]; }
  for (size_t i = 0; i < nH; ++i) hil[i] = (kind == SMK_SE) ? 1.0f : (float)(1.0 / ls[i]);
  for (int s = 0; s < S; ++s) { ha[s] = (float)amp2[s]; hn[s] = (float)noise[s]; hm[s] = (float)mean[s]; hb[s] = (float)best; }

  float* d = (float*)g_in.get(tot * sizeof(float));
  float* fac = (float*)g_fac.get((size_t)S * Npad * Npad * sizeof(float));
  float* winv = (float*)g_winv.get((size_t)S * Npad * NB * sizeof(float));
  float* alpha = (float*)g_alpha.get((size_t)S * Npad * sizeof(float));
  float* mv = (float*)g_mv.get(2 * (size_t)S * ldm * sizeof(float));
  double* ei = (double*)g_ei.get((size_t)S * ldm * sizeof(double) + S * sizeof(int));
  const size_t wsb = smk_predict_tc_workspace_bytes(Np, M, S, 1);
  void* ws = g_ws.get(wsb);
  const size_t ws2b = smk_trtri_workspace_bytes(Np, S) + (size_t)S * Np * sizeof(float);
  void* ws2 = g_ws2.get(ws2b);
  float* linv = (float*)g_linv.get(2 * (size_t)S * Np * Np * sizeof(float));
  unsigned char* l16 = (unsigned char*)g_l16.get(2 * (size_t)S * Np * Np * sizeof(__half) + 2 * (size_t)S * sizeof(int));
  if (!d || !fac || !winv || !alpha || !mv || !ei || !ws || !ws2 || !linv || !l16) {
    snprintf(g_err, sizeof(g_err), "cudaMalloc failed");
    return SMK_ERR_CUDA;
  }
  int* info = reinterpret_cast<int*>(ei + (size_t)S * ldm);
  cudaMemcpyAsync(d, h, tot * sizeof(float), cudaMemcpyHostToDevice, st);
  float *dX = d, *dC = dX + nX, *dy = dC + nC, *dil = dy + N, *da = dil + nH, *dn = da + S, *dm = dn + S,
        *db = dm + S;
  int rc;
  if ((rc = smk_cov_build_f32(kind, N, N, D, S, dX, nullptr, dil, da, dn, fac, Npad, st))) return rc;
  if ((rc = smk_potrf_lower_batched_f32(Npad, S, fac, winv, info, st))) return rc;
  // Factors of fewer than SMK_TC_MIN_N (default 2048) observations take the blocked-substitution chain (3-8x more accurate
  // on the smooth, ill-conditioned problems small N goes with; DESIGN.md section 6), larger ones the tensor-core chain:
  // explicit inverse (split), alpha by two mat-vecs, fp16 operand pack, wgmma 3xFP16 predict.
  int tc_min_n = 2048;
  { const char* e = getenv("SMK_TC_MIN_N"); if (e && e[0]) tc_min_n = atoi(e); }
  if (N < tc_min_n) {
    const size_t pwb = smk_predict_workspace_bytes(4, Npad);
    void* pws = g_ws.get(pwb > wsb ? pwb : wsb);
    if (!pws) { snprintf(g_err, sizeof(g_err), "cudaMalloc failed"); return SMK_ERR_CUDA; }
    if ((rc = smk_chol_solve_f32(N, Npad, S, 1, fac, winv, dy, 0, N, dm, alpha, nullptr, nullptr, st))) return rc;
    if ((rc = smk_predict_f32(kind, N, Npad, M, D, S, dX, dC, dil, da, dm, fac, winv, alpha, mv, mv + (size_t)S * ldm, ldm,
                              pws, pwb, st)))
      return rc;
  } else {
    float* lhi = linv;
    float* llo = linv + (size_t)S * Np * Np;
    float* tmp = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(ws2) + smk_trtri_workspace_bytes(Np, S));
    if ((rc = smk_trtri_split_f32(Npad, Np, S, fac, winv, lhi, llo, ws2, smk_trtri_workspace_bytes(Np, S), st))) return rc;
    if ((rc = smk_linv_alpha_f32(N, Np, S, lhi, llo, dy, dm, alpha, Npad, tmp, st))) return rc;
    void* lh16 = l16;
    void* ll16 = l16 + (size_t)S * Np * Np * sizeof(__half);
    int* lexp = reinterpret_cast<int*>(l16 + 2 * (size_t)S * Np * Np * sizeof(__half));
    if ((rc = smk_linv_pack_f16(Np, S, lhi, llo, lh16, ll16, lexp, st))) return rc;
    if ((rc = smk_predict_tc_f32(kind, N, Np, M, D, S, dX, dC, dil, da, dm, lh16, ll16, lexp, alpha, Npad, mv,
                                 mv + (size_t)S * ldm, ldm, ws, wsb, nullptr, 1, nullptr, nullptr, tmp, 0, st)))
      return rc;
  }
  if ((rc = smk_ei_sweep_f32(M, S, 1, mv, mv + (size_t)S * ldm, ldm, db, nullptr, ei, nullptr, nullptr, st))) return rc;
  std::vector<double> hout((size_t)S * ldm);
  std::vector<int> hinfo(S);
  cudaMemcpyAsync(hout.data(), ei, hout.size() * sizeof(double), cudaMemcpyDeviceToHost, st);
  cudaMemcpyAsync(hinfo.data(), info, S * sizeof(int), cudaMemcpyDeviceToHost, st);
  cudaError_t e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    snprintf(g_err, sizeof(g_err), "ei_over_hypers_host: %s", cudaGetErrorString(e));
    return SMK_ERR_CUDA + (int)e;
  }
  int bad = 0;
  for (int s = 0; s < S; ++s) {
    if (info_out) info_out[s] = hinfo[s];
    if (hinfo[s]) bad = 1;
    for (int j = 0; j < M; ++j) ei_out[(size_t)s * M + j] = hout[(size_t)s * ldm + j];
  }
  return bad ? SMK_ERR_NOT_PD : SMK_OK;
}

}  // extern "C"
