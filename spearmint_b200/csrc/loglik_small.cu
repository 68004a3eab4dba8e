// loglik_small.cu -- the slice-sampler log-likelihood of a small GP in ONE launch: one CTA per hyper-parameter setting
// builds the augmented covariance (solve.cu: loglik_set_rhs)
//     [ amp2 (k + 1e-6 I) + noise I   .    ]
//     [ (y - mean)'                   1e30 ]
// as a packed lower triangle in shared memory, factors it in place (right-looking, one column per step) and reduces
//     sum_log_diag = sum_{i<N} log L_ii,   quad = |L[N][0:N]|^2 = (y - mean)' K^-1 (y - mean).
// This is the contract of cov_build_lower -> loglik_set_rhs -> potrf_loglik_f64 -> loglik_finish, which costs four
// launches (and a graph replay) for microseconds of flops at the sizes most experiments run at.
//
// Every CTA reads only its own item's hyper-parameters and runs the same instruction sequence whatever B is, so an
// item's results are bitwise independent of the batch size and of its position in the batch (the lockstep chains of
// chains.py rely on this).
#include "../../include/spearmint_b200.h"
#include "common.cuh"

namespace smk {

namespace small {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxN = SMK_LOGLIK_SMALL_MAX_N;
constexpr int kRed = 32;                                   // reduction scratch (doubles)
constexpr int kColPad = kMaxN + 2;                         // scaled column j, contiguous (n = N + 1 entries)
constexpr size_t kOptinBytes = 227 * 1024;                 // shared memory an H100 block can opt into

__host__ __device__ constexpr int tri(int n) { return n * (n + 1) / 2; }
__host__ __device__ constexpr size_t smem_bytes(int n) { return (size_t)(tri(n) + kColPad + kRed) * sizeof(double); }
static_assert(smem_bytes(kMaxN + 1) <= kOptinBytes, "SMK_LOGLIK_SMALL_MAX_N does not fit in shared memory");
static_assert(smem_bytes(kMaxN + 2) > kOptinBytes, "SMK_LOGLIK_SMALL_MAX_N is not the largest size that fits");

__device__ __forceinline__ int at(int i, int k) { return tri(i) + k; }      // (i, k), k <= i, of the packed triangle

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The same order of additions in every CTA: per-thread strided partial sums, warp butterflies, then warp 0 adds the
// eight warp totals in warp order.
__device__ double cta_sum(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double t = 0.0;
  if (threadIdx.x == 0)
    for (int w = 0; w < kWarps; ++w) t += red[w];
  return t;                                                 // valid in thread 0
}

__global__ void __launch_bounds__(kThreads) loglik_small_kernel(int kind, int N, int D, const double* __restrict__ X,
                                                                 const double* __restrict__ inv_ls,
                                                                 const double* __restrict__ amp2,
                                                                 const double* __restrict__ noise,
                                                                 const double* __restrict__ mean,
                                                                 const double* __restrict__ y, double* __restrict__ sld,
                                                                 double* __restrict__ quad, int* __restrict__ info) {
  extern __shared__ __align__(16) double sm[];
  const int b = blockIdx.x, n = N + 1;
  double* A = sm;                                           // packed lower triangle, tri(n) entries
  double* col = sm + tri(n);                                // scaled column of the current step
  double* red = col + kColPad;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double* ils = inv_ls + (long)b * D;
  const double a2 = amp2[b], dg = a2 * 1e-6 + noise[b], mu = mean[b];

  // covariance rows 0..N-1 (lower triangle), the same scaled direct differences as cov_build
  for (int i = warp; i < N; i += kWarps) {
    const double* xi = X + (long)i * D;
    for (int k = lane; k <= i; k += 32) {
      const double* xk = X + (long)k * D;
      double r2 = 0.0;
      for (int d = 0; d < D; ++d) {
        const double sc = ils[d];
        const double df = __dmul_rn(xi[d], sc) - __dmul_rn(xk[d], sc);     // both products rounded, as staged there
        r2 = fma(df, df, r2);
      }
      double v = a2 * kernel_of_r2<double>(kind, r2);
      if (k == i) v += dg;
      A[at(i, k)] = v;
    }
  }
  for (int k = threadIdx.x; k <= N; k += kThreads) A[at(N, k)] = (k < N) ? y[k] - mu : 1e30;   // augmented row
  __syncthreads();

  // right-looking Cholesky of columns 0..N-1; row N undergoes the forward substitution L^-1 (y - mean)
  int bad = 0;
  for (int j = 0; j < N; ++j) {
    const double p = A[at(j, j)];
    if (!(p > 0.0)) { bad = j + 1; break; }                 // uniform: every thread read the same pivot
    const double d = sqrt(p);
    for (int i = j + 1 + threadIdx.x; i < n; i += kThreads) {
      const double l = A[at(i, j)] / d;
      A[at(i, j)] = l;
      col[i] = l;
    }
    __syncthreads();
    if (threadIdx.x == 0) A[at(j, j)] = d;
    for (int i = j + 1 + warp; i < n; i += kWarps) {
      const double li = col[i];
      double* Ai = A + tri(i);
      for (int k = j + 1 + lane; k <= i; k += 32) Ai[k] = fma(-li, col[k], Ai[k]);
    }
    __syncthreads();
  }

  double s = 0.0, q = 0.0;
  if (!bad) {
    for (int k = threadIdx.x; k < N; k += kThreads) {
      s += log(A[at(k, k)]);
      const double v = A[at(N, k)];
      q = fma(v, v, q);
    }
  }
  s = cta_sum(s, red);
  q = cta_sum(q, red);
  if (threadIdx.x == 0) {
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    sld[b] = bad ? nan : s;
    quad[b] = bad ? nan : q;
    info[b] = bad;
  }
}

}  // namespace small

int loglik_small_f64(int kind, int N, int D, int B, const double* X, const double* inv_ls, const double* amp2,
                     const double* noise, const double* mean, const double* y, double* sld, double* quad, int* info,
                     cudaStream_t st) {
  if (kind < 0 || kind > 3) return -1;
  if (N <= 0 || N > small::kMaxN) return -2;
  if (D <= 0) return -3;
  if (B <= 0) return -4;
  const void* ptrs[] = {X, inv_ls, amp2, noise, mean, y, sld, quad, info};
  for (int a = 0; a < 9; ++a)
    if (!ptrs[a]) return -(5 + a);
  const size_t bytes = small::smem_bytes(N + 1);
  static bool attr_set = false;                             // host-side attribute, set once (no synchronisation)
  if (!attr_set) {
    cudaFuncSetAttribute(small::loglik_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)small::smem_bytes(small::kMaxN + 1));
    attr_set = true;
  }
  small::loglik_small_kernel<<<B, small::kThreads, bytes, st>>>(kind, N, D, X, inv_ls, amp2, noise, mean, y, sld, quad,
                                                                info);
  count_launch();
  return check_launch("loglik_small");
}

}  // namespace smk
