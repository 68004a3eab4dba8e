// guard.cu -- accuracy guard of the tensor-core predict path.
//
// The tensor-core predict forms beta = Linv * kx with an EXPLICIT float32 inverse of the Cholesky factor.  That is not
// backward stable: the variance  amp2 (1 + 1e-6) - |beta|^2  of a candidate close to the data carries an error of about
// eps32 * ||K||_2 * |K^-1 kx|^2, which for smooth low-dimensional problems (D = 8, N = 512: ||K|| ~ 340, noise 1e-3)
// is percents of the variance itself -- above the stated 5e-3 EI tolerance -- while the blocked substitution of the
// SIMT predict kernel stays within it (tools/tc_error_probe.py).
//
// The guard measures exactly that error, on the device, before any candidate is touched.  For a few observed points
// x_i (the caller passes the incumbents -- the lowest observed values, where EI concentrates and where the chooser's own
// jitter cloud sits) the cross-covariance vector is a column of K = L L^T, so with v = row i of L:  L^-1 (K e_i) = v
// EXACTLY, and
//     | |Linv (L v)|^2 - |v|^2 | / (noise + 1e-6 amp2)
// is the relative variance error the explicit inverse causes for a candidate sitting on x_i (two triangular mat-vecs
// per probe, float64 accumulation so that the check itself adds nothing).  The second error source of the path -- the
// truncating float32 accumulation inside the tensor cores, which is systematic along the rows of L^-1 -- is estimated from
// the running sums of the same products (guard_bv_kernel); g is the sum of both.  The engine reads max g once per
// factor batch (it synchronises there anyway for the not-positive-definite check) and routes the batch to the
// substitution-based float32 kernel when g exceeds its threshold.
#include "common.cuh"

namespace smk {

constexpr int kGuardQ = 4;     // probe rows, chosen by the caller: the observed points where EI matters (the incumbents)

// p[s][q][j] = sum_{k <= min(j, i_q)} L[j][k] L[i_q][k]     (column i_q of L L^T); one warp per row j
__global__ void __launch_bounds__(256) guard_lv_kernel(int N, int Npad, int Np, const float* __restrict__ L,
                                                        const int* __restrict__ rows, double* __restrict__ p) {
  const int s = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int j = blockIdx.x * 8 + warp;
  if (j >= N) return;
  const float* Ls = L + (long)s * Npad * Npad;
  const float* lj = Ls + (long)j * Npad;
  double acc[kGuardQ];
#pragma unroll
  for (int q = 0; q < kGuardQ; ++q) acc[q] = 0.0;
  for (int k = lane; k <= j; k += 32) {
    const double x = (double)lj[k];
#pragma unroll
    for (int q = 0; q < kGuardQ; ++q) {
      const int i = rows[q];
      if (k <= i) acc[q] = fma(x, (double)Ls[(long)i * Npad + k], acc[q]);
    }
  }
#pragma unroll
  for (int q = 0; q < kGuardQ; ++q) {
    double a = acc[q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) p[((long)s * kGuardQ + q) * Np + j] = a;
  }
}

// acc[s][q]      += sum over this block's rows r of b_r^2,           b_r = sum_{j <= r} Linv[r][j] p[q][j]
// acc[s][Q + q]  += sum over this block's rows r of 2 b_r t_r,       t_r = the accumulation bias of the tensor-core GEMM:
//   the tensor core accumulates in float32 with truncation; along a row of L^-1 the running sum is negative almost to the end (the
//   off-diagonal entries of the inverse of a positive matrix are mostly negative, the diagonal -- the LAST term -- is large
//   and positive), so every one of the 3 MMAs per 16 observations loses about half an ulp of the running sum in the same
//   direction:  t_r = -3 * 2^-24 * sum over 16-wide steps of the running sum  (tools/tc_error_probe.py measures it).
__global__ void __launch_bounds__(256) guard_bv_kernel(int N, int Np, const float* __restrict__ hi, const float* __restrict__ lo,
                                                        const double* __restrict__ p, double* __restrict__ acc) {
  const int s = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 8 + warp;
  if (r >= N) return;
  const long base = ((long)s * Np + r) * Np;
  const double* ps = p + (long)s * kGuardQ * Np;
  double carry[kGuardQ], run[kGuardQ];
#pragma unroll
  for (int q = 0; q < kGuardQ; ++q) { carry[q] = 0.0; run[q] = 0.0; }
  for (int j0 = 0; j0 <= r; j0 += 32) {
    const int j = j0 + lane;
    const double x = (j <= r) ? (double)hi[base + j] + (double)lo[base + j] : 0.0;
#pragma unroll
    for (int q = 0; q < kGuardQ; ++q) {
      double v = (j <= r) ? x * ps[(long)q * Np + j] : 0.0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {                 // inclusive warp scan
        const double u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
      }
      const double p15 = carry[q] + __shfl_sync(0xffffffffu, v, 15), p31 = carry[q] + __shfl_sync(0xffffffffu, v, 31);
      run[q] += p15 + ((j0 + 16 <= r) ? p31 : 0.0);     // running sum after each 16-wide MMA step of this row
      carry[q] = p31;
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < kGuardQ; ++q) {
      const double b = carry[q], t = -3.0 * 5.9604644775390625e-08 * run[q];
      atomicAdd(&acc[s * 2 * kGuardQ + q], b * b);
      atomicAdd(&acc[s * 2 * kGuardQ + kGuardQ + q], 2.0 * b * t);
    }
  }
}

// g[s] = max_q ( 0.5 | acc[s][q] - |row i_q of L|^2 |  +  | acc[s][Q + q] | ) / (noise + 1e-6 amp2)
// (the inconsistency of the explicit inverse enters with the factor 1/2 that it shows against measured EI errors: the
// probe sits ON an observed point, the candidates that matter sit next to one)
__global__ void __launch_bounds__(256) guard_finish_kernel(int N, int Npad, const float* __restrict__ L,
                                                            const int* __restrict__ rows, const double* __restrict__ acc,
                                                            const float* __restrict__ amp2,
                                                            const float* __restrict__ noise, float* __restrict__ g) {
  __shared__ double red[8];
  const int s = blockIdx.x, tid = threadIdx.x;
  const float* Ls = L + (long)s * Npad * Npad;
  double worst = 0.0;
  for (int q = 0; q < kGuardQ; ++q) {
    const int i = rows[q];
    double a = 0.0;
    for (int k = tid; k <= i; k += 256) { const double x = (double)Ls[(long)i * Npad + k]; a = fma(x, x, a); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    __syncthreads();
    if ((tid & 31) == 0) red[tid >> 5] = a;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];
    worst = fmax(worst, 0.5 * fabs(acc[s * 2 * kGuardQ + q] - t) + fabs(acc[s * 2 * kGuardQ + kGuardQ + q]));
  }
  if (tid == 0) {
    g[s] = (float)(worst / ((double)noise[s] + 1e-6 * (double)amp2[s]));
  }
}

size_t tc_guard_workspace_bytes(int Np, int S) { return sizeof(double) * ((size_t)S * kGuardQ * Np + (size_t)S * 2 * kGuardQ); }

int tc_guard(int N, int Npad, int Np, int S, const float* L, const float* linv_hi, const float* linv_lo, const float* amp2,
             const float* noise, const int* rows, float* g, void* ws, size_t ws_bytes, cudaStream_t st) {
  if (N <= 0 || Npad < N || Np < N) return -1;
  if (S <= 0) return -4;
  if (!L || !linv_hi || !linv_lo || !amp2 || !noise || !rows || !g) return -5;
  if (!ws || ws_bytes < tc_guard_workspace_bytes(Np, S)) return -11;
  double* p = reinterpret_cast<double*>(ws);
  double* acc = p + (size_t)S * kGuardQ * Np;
  cudaMemsetAsync(acc, 0, sizeof(double) * S * 2 * kGuardQ, st);
  guard_lv_kernel<<<dim3((N + 7) / 8, S), 256, 0, st>>>(N, Npad, Np, L, rows, p);
  guard_bv_kernel<<<dim3((N + 7) / 8, S), 256, 0, st>>>(N, Np, linv_hi, linv_lo, p, acc);
  guard_finish_kernel<<<S, 256, 0, st>>>(N, Npad, L, rows, acc, amp2, noise, g);
  count_launch(3);
  return check_launch("tc_guard");
}

}  // namespace smk
