// constraint.cu -- probability of feasibility at the candidate grid (CONS = chooser/GPConstrainedEIChooser.py).
//
// Reference span replaced (per hyper-sample, CONS:819-842):
//   cand_constraint_cross = self.cov(constraint_amp2, constraint_ls, compfull, cand)     (N x M, float64)
//   func_constraint_m     = np.dot(cand_constraint_cross.T, t_alpha)                     t_alpha = K_c^-1 ff
//   func_constraint_m     = sps.norm.cdf(constraint_gain * func_constraint_m)
// One block owns 128 candidates of one sample and walks the observations in tiles of 64, 8 candidates x 4 observations
// per thread (the register tiling of the SIMT cross-covariance generator), but it reduces k . t_alpha instead of storing
// k: nothing N x M-sized is written, 8 bytes leave per (candidate, sample).  Two blocks share an SM (128 registers, a
// small spill in the kernel-value epilogue), so one block's staging and barriers overlap the other's float64 arithmetic:
// at the headline shape this took 176-188 ms against 280 ms for 8 x 8 micro-tiles at one block per SM (H100, 400 W).
// The kernel function is a template argument: no branch on it in the unrolled epilogue (fewer registers, less spill).
//
// Precision: K_c = amp2 (k + 1e-6 I) + 1e-3 I is a classification GP's covariance; K_c^-1 ff has entries of both signs
// that are orders of magnitude larger than the mean they sum to (sum |t_alpha| ~ 1e4 - 1e5 against |m| ~ 3 for SE at
// N=300), and Phi is steep in its tail.  So t_alpha stays float64, and the scaling, the distances, the kernel values and
// the contraction are evaluated in float64 for both element types: with float32 arithmetic the latent mean of an SE
// classification GP was off by 3e-4 - 6e-4 of max|m| on the H100, with float32 INPUTS and float64 arithmetic by 3e-5
// (numpy emulation of the same case).  The float32 variant differs from the float64 one only in what it reads.  p is
// written in double with an erfc tail, so a candidate deep in the infeasible region keeps a ranking value.
#include "common.cuh"

namespace smk {

constexpr int kProbTN = 4;   // observations per thread (x 8 candidates)

template <typename T, int KIND>
__global__ void __launch_bounds__(256, 2) constraint_prob_kernel(int N, int Npad, int M, int D,
                                                              const T* __restrict__ X, const T* __restrict__ Cc,
                                                              const T* __restrict__ inv_ls, const T* __restrict__ amp2,
                                                              const double* __restrict__ t_alpha,
                                                              const double* __restrict__ gain, double* __restrict__ p,
                                                              double* __restrict__ m_out, int ldm) {
  constexpr int BT = 128, TN = kProbTN, BN = 16 * TN, KD = 8;
  __shared__ __align__(16) double cs[KD][BT + kPad];      // scaled candidates [d][c]
  __shared__ __align__(16) double xs[KD][BN + kPad];      // scaled observations [d][n]
  __shared__ double ts[BN];                   // t_alpha of the current observation tile (zero past N)
  __shared__ double red[16][BT];              // epilogue: per-thread row partials
  const int s = blockIdx.y, c0 = blockIdx.x * BT;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const T* ils = inv_ls + (long)s * D;   // scaling, distances and kernel values in double, whatever T is
  const double* ta = t_alpha + (long)s * Npad;
  double mdot[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) mdot[r] = 0.0;

  for (int n0 = 0; n0 < N; n0 += BN) {
    double acc[8][TN];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int c = 0; c < TN; ++c) acc[r][c] = 0.0;
    __syncthreads();
    if (tid < BN) ts[tid] = (n0 + tid < N) ? ta[n0 + tid] : 0.0;
    for (int d0 = 0; d0 < D; d0 += KD) {
      __syncthreads();
      for (int e = tid; e < BT * KD; e += 256) {
        const int row = e / KD, dd = e % KD, d = d0 + dd;
        const int gc = min(c0 + row, M - 1);
        cs[dd][row] = (d < D) ? (double)Cc[(long)gc * D + d] * (double)ils[d] : 0.0;
      }
      for (int e = tid; e < BN * KD; e += 256) {
        const int row = e / KD, dd = e % KD, d = d0 + dd, n = n0 + row;
        xs[dd][row] = (d < D && n < N) ? (double)X[(long)n * D + d] * (double)ils[d] : 0.0;
      }
      __syncthreads();
      const int dmax = min(KD, D - d0);
      for (int dd = 0; dd < dmax; ++dd) {
        double a[8], b[TN];
#pragma unroll
        for (int g = 0; g < 2; ++g) {
          const V4<double> u = ld4(&cs[dd][g * 64 + ty * 4]);
#pragma unroll
          for (int e = 0; e < 4; ++e) a[g * 4 + e] = u.v[e];
        }
#pragma unroll
        for (int g = 0; g < TN / 4; ++g) {
          const V4<double> v = ld4(&xs[dd][g * 64 + tx * 4]);
#pragma unroll
          for (int e = 0; e < 4; ++e) b[g * 4 + e] = v.v[e];
        }
#pragma unroll
        for (int r = 0; r < 8; ++r)
#pragma unroll
          for (int c = 0; c < TN; ++c) {
            const double df = a[r] - b[c];
            acc[r][c] = fma(df, df, acc[r][c]);
          }
      }
    }
    double tv[TN];
#pragma unroll
    for (int c = 0; c < TN; ++c) tv[c] = ts[tile_col(tx, c)];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int c = 0; c < TN; ++c) mdot[r] = fma(kernel_of_r2<double>(KIND, acc[r][c]), tv[c], mdot[r]);
  }

  // reduce the row partials over the 16 column-threads (fixed order -> deterministic)
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 8; ++r) red[tx][tile_row(ty, r)] = mdot[r];
  __syncthreads();
  if (tid < BT) {
    double v = 0.0;
    for (int q = 0; q < 16; ++q) v += red[q][tid];
    const int j = c0 + tid;
    if (j < M) {
      const double m = (double)amp2[s] * v;
      p[(long)s * ldm + j] = 0.5 * erfc(-gain[s] * m * 0.7071067811865476);
      if (m_out) m_out[(long)s * ldm + j] = m;
    }
  }
}

template <typename T>
int constraint_prob(int kind, int N, int Npad, int M, int D, int S, const T* X, const T* Cc, const T* inv_ls,
                    const T* amp2, const double* t_alpha, const double* gain, double* p, double* m_out, int ldm,
                    cudaStream_t st) {
  if (kind < 0 || kind > 3) return -1;
  if (N <= 0) return -2;
  if (Npad < N) return -3;
  if (M <= 0) return -4;
  if (D <= 0) return -5;
  if (S <= 0) return -6;
  if (!X) return -7;
  if (!Cc) return -8;
  if (!inv_ls) return -9;
  if (!amp2) return -10;
  if (!t_alpha) return -11;
  if (!gain) return -12;
  if (!p) return -13;
  if (ldm < M) return -15;
  timing_begin("constraint_prob_kernel", st);
  const dim3 grid((M + 127) / 128, S);
  if (kind <= 1)         // SE and ARDSE differ only in the length scales the caller passes
    constraint_prob_kernel<T, 0><<<grid, 256, 0, st>>>(N, Npad, M, D, X, Cc, inv_ls, amp2, t_alpha, gain, p, m_out, ldm);
  else if (kind == 2)
    constraint_prob_kernel<T, 2><<<grid, 256, 0, st>>>(N, Npad, M, D, X, Cc, inv_ls, amp2, t_alpha, gain, p, m_out, ldm);
  else
    constraint_prob_kernel<T, 3><<<grid, 256, 0, st>>>(N, Npad, M, D, X, Cc, inv_ls, amp2, t_alpha, gain, p, m_out, ldm);
  timing_end(st);
  count_launch();
  return check_launch("constraint_prob");
}

template int constraint_prob<float>(int, int, int, int, int, int, const float*, const float*, const float*, const float*,
                                    const double*, const double*, double*, double*, int, cudaStream_t);
template int constraint_prob<double>(int, int, int, int, int, int, const double*, const double*, const double*,
                                     const double*, const double*, const double*, double*, double*, int, cudaStream_t);

// ------------------------------------------------------------------------------------------------ classification GP
// Augmented row of the slice sampler's log-likelihood factorisation (solve.cu: loglik_set_rhs) with ONE right-hand side
// per batch item: the joint [amp2, ff] move of the constrained chooser (CONS:1169-1190) changes ff with every proposal.
// y: [S][ldy], no mean is subtracted (the classification GP's latent has zero mean, CONS:1179).
template <typename T>
__global__ void loglik_set_rhs_batched_kernel(int N, int Npad, const T* __restrict__ y, int ldy, T* A) {
  const int s = blockIdx.y, n = blockIdx.x * blockDim.x + threadIdx.x;
  T* row = A + (long)s * Npad * Npad + (long)N * Npad;
  if (n < N) row[n] = y[(long)s * ldy + n];
  else if (n == N) row[n] = T(1e30);            // pivot of the augmented row: c - quad must stay positive
}

template <typename T>
int loglik_set_rhs_batched(int N, int Npad, int S, const T* y, int ldy, T* A, cudaStream_t st) {
  if (N <= 0 || Npad <= N || Npad % kNpadMult) return -2;
  if (S <= 0) return -3;
  if (!y) return -4;
  if (ldy < N) return -5;
  if (!A) return -6;
  loglik_set_rhs_batched_kernel<T><<<dim3((N + 256) / 256, S), 256, 0, st>>>(N, Npad, y, ldy, A);
  count_launch();
  return check_launch("loglik_set_rhs_batched");
}
template int loglik_set_rhs_batched<float>(int, int, int, const float*, int, float*, cudaStream_t);
template int loglik_set_rhs_batched<double>(int, int, int, const double*, int, double*, cudaStream_t);

// nu = L z for a lower factor L [Npad][Npad] (one warp per row): the elliptical-slice direction (CONS:1241, nu = chol.T
// randn with the upper factor chol = L^T).  Only the lower triangle of L is read.
__global__ void __launch_bounds__(256) lower_matvec_kernel(int N, int Npad, const double* __restrict__ L,
                                                           const double* __restrict__ z, double* __restrict__ out) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= N) return;
  const double* Lr = L + (long)row * Npad;
  double acc = 0.0;
  for (int k = lane; k <= row; k += 32) acc = fma(Lr[k], z[k], acc);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) out[row] = acc;
}

int lower_matvec(int N, int Npad, const double* L, const double* z, double* out, cudaStream_t st) {
  if (N <= 0 || Npad < N) return -2;
  if (!L) return -3;
  if (!z) return -4;
  if (!out) return -5;
  lower_matvec_kernel<<<(N + 7) / 8, 256, 0, st>>>(N, Npad, L, z, out);
  count_launch();
  return check_launch("lower_matvec");
}

}  // namespace smk
