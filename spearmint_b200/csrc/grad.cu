// grad.cu -- EI value + input-gradient terms at a few query points with CACHED factors.
//
// Reference: GPEIOptChooser.grad_optimize_ei (OPT:391-525) rebuilds K and re-factors it on every L-BFGS
// function evaluation (OPT:397-402; ~160 evaluations x S Choleskys per next()).  Here the S factors are
// computed once; one evaluation is  cov_build(cross, N x Q) -> chol_solve (gamma = K^-1 kx) -> this kernel.
// It also retires the reference's only native snippet, the weave loop of grad_dist2 (GP:69-79): the
// N x M x D gradient tensor is never materialised, it is contracted on the fly.
//
// For sample s and query point q this kernel forms the small product  OUT = A * T  with
//     A[f][n] = alpha[s][f][n]  (f < F),   A[F][n] = gamma[s][q][n]
//     T[n][d] = gk[n][d]        (d < D),   T[n][D] = kx[n] = amp2 * k(r2_n)
//     gk[n][d] = dk/dr2(r2_n) * (2 * inv_ls_d) * (X[n][d] - x_q[d]) * inv_ls_d        (GP:56-85, GP:102-132)
// so that (host side, float64):
//     OUT[f][D]  = kx' alpha_f           -> func_m - mean            (OPT:417, 508)
//     OUT[f][d]  = grad_xp_m[f][d]                                    (OPT:433, 516)
//     OUT[F][d]  = -0.5 * grad_xp_v[d]                                (OPT:434-435, 517-518)
//     OUT[F][D]  = kx' K^-1 kx = sum(beta^2)                          (OPT:418, 509)
#include "common.cuh"

namespace smk {

template <typename T>
__device__ __forceinline__ T dk_dr2(int kind, T r2) {
  if (kind <= 1) return T(-0.5) * smk_exp(T(-0.5) * r2);                              // GP:102-105
  T r = smk_sqrt(r2);
  if (kind == 2) return T(-1.5) * smk_exp(-T(1.7320508075688772) * r);                // GP:115-118
  T a = T(2.23606797749979) * r;
  return T(-5.0 / 6.0) * smk_exp(-a) * (T(1) + a);                                    // GP:129-132
}

constexpr int kGC = 64;  // rows of X per staged chunk
constexpr int kFR = 64;  // rows of A (fantasies + the gamma row) staged at a time: shared memory does not grow with F

// Rows of A one pass of pairs reads.
__host__ __device__ __forceinline__ int ei_grad_rows(int F) { return F + 1 < kFR ? F + 1 : kFR; }

template <typename T>
__global__ void __launch_bounds__(256) ei_grad_terms_kernel(int kind, int N, int Npad, int D, int Q, int F,
                                                             const T* __restrict__ X, const T* __restrict__ xq,
                                                             const T* __restrict__ inv_ls,
                                                             const T* __restrict__ amp2,
                                                             const T* __restrict__ alpha,
                                                             const T* __restrict__ gamma, T* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int D1 = D + 1, F1 = F + 1;
  T* Tt = reinterpret_cast<T*>(smem_raw);   // [kGC][D1]
  T* At = Tt + kGC * D1;                    // [ei_grad_rows(F)][kGC]: rows f0 .. f0 + nf - 1 of A
  T* xs = At + ei_grad_rows(F) * kGC;       // [D] scaled query point
  T* il = xs + D;                           // [D]
  const int q = blockIdx.x, s = blockIdx.y, tid = threadIdx.x;
  for (int d = tid; d < D; d += 256) {
    T sc = inv_ls[(long)s * D + d];
    il[d] = sc;
    xs[d] = xq[(long)q * D + d] * sc;
  }
  __syncthreads();
  const T a2 = amp2[s];
  const T* al = alpha + (long)s * F * Npad;
  const T* ga = gamma + ((long)s * Q + q) * Npad;
  T* o = out + ((long)s * Q + q) * F1 * D1;
  const int npairs = F1 * D1;
  constexpr int R = 8;
  // pairs (f, d), p = f D1 + d, in passes of up to 256 R; a pass of at most (kFR - 1) D1 + 1 pairs reads at most kFR
  // rows of A.  Each output element is one pass's sum over n = 0 .. N-1 in order, whatever the pass boundaries.
  const int P = F1 <= kFR ? 256 * R : min(256 * R, (kFR - 1) * D1);

  for (int p0 = 0; p0 < npairs; p0 += P) {
    const int p1 = min(npairs, p0 + P);
    const int f0 = p0 / D1, nf = (p1 - 1) / D1 - f0 + 1;
    T acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = T(0);
    for (int n0 = 0; n0 < N; n0 += kGC) {
      __syncthreads();
      // stage T chunk: one thread per row computes r2 and the kernel derivatives, then all fill columns
      for (int i = tid; i < kGC; i += 256) {
        int n = n0 + i;
        T r2 = T(0);
        if (n < N)
          for (int d = 0; d < D; ++d) {
            T df = X[(long)n * D + d] * il[d] - xs[d];
            r2 = fma(df, df, r2);
          }
        T kv = (n < N) ? a2 * kernel_of_r2<T>(kind, r2) : T(0);
        T w = (n < N) ? dk_dr2<T>(kind, r2) : T(0);
        Tt[i * D1 + D] = kv;
        // park w in the first column slot temporarily (overwritten below after the barrier)
        At[i] = w;
      }
      __syncthreads();
      for (int e = tid; e < kGC * D; e += 256) {
        int i = e / D, d = e % D, n = n0 + i;
        T w = At[i];
        T g = (n < N) ? w * (T(2) * il[d]) * (X[(long)n * D + d] * il[d] - xs[d]) : T(0);
        Tt[i * D1 + d] = g;
      }
      __syncthreads();
      for (int e = tid; e < nf * kGC; e += 256) {
        int f = f0 + e / kGC, i = e % kGC, n = n0 + i;
        At[e] = (n < N) ? (f < F ? al[(long)f * Npad + n] : ga[n]) : T(0);
      }
      __syncthreads();
#pragma unroll
      for (int r = 0; r < R; ++r) {
        int p = p0 + r * 256 + tid;
        if (p < p1) {
          int f = p / D1 - f0, d = p % D1;
          T a = acc[r];
          for (int i = 0; i < kGC; ++i) a = fma(At[f * kGC + i], Tt[i * D1 + d], a);
          acc[r] = a;
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      int p = p0 + r * 256 + tid;
      if (p < p1) o[p] = acc[r];
    }
  }
}

template <typename T>
int ei_grad_terms(int kind, int N, int Npad, int D, int S, int Q, int F, const T* X, const T* xq, const T* inv_ls,
                  const T* amp2, const T* alpha, const T* gamma, T* out, cudaStream_t st) {
  if (kind < 0 || kind > 3) return -1;
  if (N <= 0 || Npad < N) return -2;
  if (D <= 0) return -4;
  if (S <= 0) return -5;
  if (Q <= 0) return -6;
  if (F <= 0) return -7;
  if (!X || !xq || !inv_ls || !amp2 || !alpha || !gamma || !out) return -8;
  // F adds at most kFR rows; D alone can exceed the budget (D > 324 in float64, D > 712 in float32)
  const size_t dsm = sizeof(T) * ((size_t)kGC * (D + 1) + (size_t)ei_grad_rows(F) * kGC + 2 * (size_t)D);
  if (dsm > 200 * 1024) return -4;
  static size_t attr_set = 48 * 1024;
  if (dsm > attr_set) {
    cudaFuncSetAttribute(ei_grad_terms_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsm);
    attr_set = dsm;
  }
  ei_grad_terms_kernel<T><<<dim3(Q, S), 256, dsm, st>>>(kind, N, Npad, D, Q, F, X, xq, inv_ls, amp2, alpha, gamma, out);
  count_launch();
  return check_launch("ei_grad_terms");
}

template int ei_grad_terms<float>(int, int, int, int, int, int, int, const float*, const float*, const float*,
                                  const float*, const float*, const float*, float*, cudaStream_t);
template int ei_grad_terms<double>(int, int, int, int, int, int, int, const double*, const double*, const double*,
                                   const double*, const double*, const double*, double*, cudaStream_t);


// ---------------------------------------------------------------------------------------------------------------
// ML-II (GP.optimize_hypers, GP:181-292): the traces of grad_nlogprob (GP:238-264) for one setting of the hyper-parameters.
// With  J = alpha alpha' - K^-1  (GP:246, "jacobian"), alpha = K^-1 (y - mean):
//     out[0]     = sum_ij J_ij (corr_ij + 1e-6 delta_ij)                    -> grad[0] = 0.5 * out[0] * amp2      (GP:251)
//     out[1]     = sum_i  J_ii                                              -> grad[1] = 0.5 * out[1] * noise     (GP:254)
//     out[2 + d] = sum_ij J_ji gcorr_ij^d X[i][d]                           -> grad[2 + d] = -amp2 * out[2 + d]   (GP:258-259)
// where gcorr_ij^d = dk/dr2(r2_ij) * (2 / ls_d) (X[i][d] - X[j][d]) / ls_d is the reference's grad_<kernel>(ls, comp)[i][j][d]
// (GP:56-85, 102-132); the reference's exp(ls_d) factors cancel.  That last expression is what the reference hands to
// L-BFGS-B as the length-scale gradient -- it is not the derivative of the likelihood, and it is reproduced as is.
// The N x N x D gradient tensor of the reference is never materialised.  One thread per (i, j) pair, dimensions in chunks
// of 8 accumulators, warp + atomic reduction (double atomics: the result is summed in a run-dependent order, ~1e-15).
constexpr int kMllDC = 8;

template <typename T>
__global__ void __launch_bounds__(256) mll_grad_terms_kernel(int kind, int N, int D, const T* __restrict__ X,
                                                              const T* __restrict__ inv_ls, const T* __restrict__ alpha,
                                                              int lda, const T* __restrict__ Kinv, int ldk,
                                                              double* __restrict__ out) {
  const int s = blockIdx.z;
  const int i = blockIdx.y * 16 + (threadIdx.x >> 4), j = blockIdx.x * 16 + (threadIdx.x & 15);
  const bool act = i < N && j < N;
  const T* il = inv_ls + (long)s * D;
  const T* xi = X + (long)(act ? i : 0) * D;
  const T* xj = X + (long)(act ? j : 0) * D;
  double* o = out + (long)s * (D + 2);
  T r2 = T(0);
  for (int d = 0; d < D; ++d) { const T df = (xi[d] - xj[d]) * il[d]; r2 = fma(df, df, r2); }
  // J_ji: row j of K^-1 (chol_solve column layout [f][n]) -- symmetric up to rounding
  const T Jv = act ? alpha[(long)s * lda + i] * alpha[(long)s * lda + j] - Kinv[((long)s * N + j) * ldk + i] : T(0);
  const T w = act ? Jv * dk_dr2<T>(kind, r2) * T(2) : T(0);
  double t0 = act ? (double)(Jv * (kernel_of_r2<T>(kind, r2) + ((i == j) ? T(1e-6) : T(0)))) : 0.0;
  double t1 = (act && i == j) ? (double)Jv : 0.0;
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) { t0 += __shfl_xor_sync(0xffffffffu, t0, o2); t1 += __shfl_xor_sync(0xffffffffu, t1, o2); }
  if (lane == 0) { atomicAdd(&o[0], t0); atomicAdd(&o[1], t1); }
  for (int d0 = 0; d0 < D; d0 += kMllDC) {
    double acc[kMllDC];
#pragma unroll
    for (int q = 0; q < kMllDC; ++q) {
      const int d = d0 + q;
      acc[q] = (d < D) ? (double)(w * (xi[d] - xj[d]) * il[d] * il[d] * xi[d]) : 0.0;
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o2);
    }
    if (lane == 0)
#pragma unroll
      for (int q = 0; q < kMllDC; ++q)
        if (d0 + q < D) atomicAdd(&o[2 + d0 + q], acc[q]);
  }
}

template <typename T>
int mll_grad_terms(int kind, int N, int D, int S, const T* X, const T* inv_ls, const T* alpha, int lda, const T* Kinv,
                   int ldk, double* out, cudaStream_t st) {
  if (kind < 0 || kind > 3) return -1;
  if (N <= 0) return -2;
  if (D <= 0) return -3;
  if (S <= 0) return -4;
  if (!X || !inv_ls || !alpha || !Kinv || !out) return -5;
  if (lda < N || ldk < N) return -8;
  cudaMemsetAsync(out, 0, sizeof(double) * S * (D + 2), st);
  mll_grad_terms_kernel<T><<<dim3((N + 15) / 16, (N + 15) / 16, S), 256, 0, st>>>(kind, N, D, X, inv_ls, alpha, lda, Kinv, ldk, out);
  count_launch();
  return check_launch("mll_grad_terms");
}
template int mll_grad_terms<float>(int, int, int, int, const float*, const float*, const float*, int, const float*, int,
                                   double*, cudaStream_t);
template int mll_grad_terms<double>(int, int, int, int, const double*, const double*, const double*, int, const double*, int,
                                    double*, cudaStream_t);

}  // namespace smk
