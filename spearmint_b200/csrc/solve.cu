// solve.cu -- alpha = K^-1 (y - mean) by forward + backward substitution against the blocked factor,
// plus the two scalars of the GP log marginal likelihood.
// Reference: spla.cho_solve((L, True), vals - mean) OPT:543 (vector) / OPT:603 ((N+P) x F fantasies);
// -sum(log(diag(chol))) - 0.5 * dot(vals - mean, solve)  OPT:637-640, 659-661, 690-692.
//
// One block per (sample, group of RB right-hand sides).  The right-hand sides live in shared memory;
// the factor is streamed once per direction (HBM/L2-bound: N^2/2 elements each way).  Diagonal blocks
// are applied as multiplications by the stored inverses W_II (potrf.cu).
#include "common.cuh"

namespace smk {

template <typename T> struct SolveCfg;
template <> struct SolveCfg<float>  { static constexpr int RB = 4; };
template <> struct SolveCfg<double> { static constexpr int RB = 2; };

__device__ __forceinline__ float  smk_log(float x)  { return logf(x); }
__device__ __forceinline__ double smk_log(double x) { return log(x); }

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T>
__device__ T block_sum(T v, T* red /*[8]*/) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  T t = T(0);
  for (int w = 0; w < 8; ++w) t += red[w];
  return t;
}

template <typename T>
__global__ void __launch_bounds__(256) chol_solve_kernel(int N, int Npad, int F, const T* __restrict__ L,
                                                          const T* __restrict__ winv, const T* __restrict__ y,
                                                          long long y_stride, int ldy,
                                                          const T* __restrict__ mean, T* __restrict__ alpha,
                                                          T* __restrict__ sum_log_diag, T* __restrict__ quad,
                                                          int do_backward) {
  constexpr int NB = Cfg<T>::NB, RB = SolveCfg<T>::RB, NG = 256 / NB;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* x = reinterpret_cast<T*>(smem_raw);  // [RB][Npad]
  T* tt = x + (long)RB * Npad;            // [RB][NB]
  T* red = tt + RB * NB;                  // [NG][RB][NB]
  __shared__ T red8[8];

  const int s = blockIdx.y, f0 = blockIdx.x * RB, tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const T* Ls = L + (long)s * Npad * Npad;
  const T* Ws = winv + (long)s * (Npad / NB) * NB * NB;
  // Only the block steps that hold rows < N run, and only rows < N of L and winv are read below the diagonal: under
  // n_lead (N < Npad) the rows >= N belong to a larger joint factor and may hold anything, NaN included.
  const int nblk = (N + NB - 1) / NB;
  const T mu = mean ? mean[s] : T(0);

  for (int n = tid; n < Npad; n += 256)
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      int f = f0 + r;
      x[r * Npad + n] = (n < N && f < F) ? y[(long long)s * y_stride + (long)f * ldy + n] - mu : T(0);
    }
  __syncthreads();

  // ---------------- forward: L t = r
  for (int I = 0; I < nblk; ++I) {
    const int base = I * NB;
    const T* Wb = Ws + (long)I * NB * NB;
    // phase A: tt[i] = r[base+i] - L[base+i, 0:base] . t[0:base]   (a warp owns 4 rows at a time)
    for (int i0 = warp * 4; i0 < NB; i0 += 32) {
      T p[4][RB];
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int r = 0; r < RB; ++r) p[q][r] = T(0);
      const T* Lr = Ls + (long)(base + i0) * Npad;
      for (int k = lane; k < base; k += 32) {
        T l[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) l[q] = Lr[(long)q * Npad + k];
#pragma unroll
        for (int r = 0; r < RB; ++r) {
          T xv = x[r * Npad + k];
#pragma unroll
          for (int q = 0; q < 4; ++q) p[q][r] = fma(l[q], xv, p[q][r]);
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int r = 0; r < RB; ++r) {
          T v = warp_sum(p[q][r]);
          if (lane == 0) tt[r * NB + i0 + q] = x[r * Npad + base + i0 + q] - v;
        }
    }
    __syncthreads();
    // phase B: t[base+i] = W_II[i, 0:i+1] . tt
    for (int i = warp; i < NB; i += 8) {
      T p[RB];
#pragma unroll
      for (int r = 0; r < RB; ++r) p[r] = T(0);
      for (int k = lane; k <= i; k += 32) {
        T w = Wb[(long)i * NB + k];
#pragma unroll
        for (int r = 0; r < RB; ++r) p[r] = fma(w, tt[r * NB + k], p[r]);
      }
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        T v = warp_sum(p[r]);
        if (lane == 0) x[r * Npad + base + i] = v;
      }
    }
    __syncthreads();
  }

  // Rows >= N are outside the (leading) system being solved: when L is the factor of a larger joint
  // matrix (observed + pending, OPT:574 "use the sub-Cholesky") they hold joint-factor rows, not the
  // identity, so their forward values (rows >= N of the last block step) must not leak into the quadratic
  // form or the backward pass.
  for (int n = N + tid; n < Npad; n += 256)
#pragma unroll
    for (int r = 0; r < RB; ++r) x[r * Npad + n] = T(0);
  __syncthreads();

  if (quad) {
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      T a = T(0);
      for (int n = tid; n < Npad; n += 256) a = fma(x[r * Npad + n], x[r * Npad + n], a);
      a = block_sum(a, red8);
      if (tid == 0 && f0 + r < F) quad[(long)s * F + f0 + r] = a;
    }
  }
  if (sum_log_diag && blockIdx.x == 0) {
    T a = T(0);
    for (int n = tid; n < N; n += 256) a += smk_log(Ls[(long)n * Npad + n]);
    a = block_sum(a, red8);
    if (tid == 0) sum_log_diag[s] = a;
  }
  if (!do_backward) return;

  // ---------------- backward: L^T a = t
  const int i = tid % NB, g = tid / NB;
  for (int I = nblk - 1; I >= 0; --I) {
    const int base = I * NB;
    const T* Wb = Ws + (long)I * NB * NB;
    T p[RB];
#pragma unroll
    for (int r = 0; r < RB; ++r) p[r] = T(0);
    // phase A: sum over rows base+NB <= k < N of L[k, base+i] * a[k]
    const T* Lc = Ls + base + i;
    int k = base + NB + g;
    for (; k + 3 * NG < N; k += 4 * NG) {
      T l0 = Lc[(long)k * Npad], l1 = Lc[(long)(k + NG) * Npad], l2 = Lc[(long)(k + 2 * NG) * Npad],
        l3 = Lc[(long)(k + 3 * NG) * Npad];
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        p[r] = fma(l0, x[r * Npad + k], p[r]);
        p[r] = fma(l1, x[r * Npad + k + NG], p[r]);
        p[r] = fma(l2, x[r * Npad + k + 2 * NG], p[r]);
        p[r] = fma(l3, x[r * Npad + k + 3 * NG], p[r]);
      }
    }
    for (; k < N; k += NG) {
      T l0 = Lc[(long)k * Npad];
#pragma unroll
      for (int r = 0; r < RB; ++r) p[r] = fma(l0, x[r * Npad + k], p[r]);
    }
#pragma unroll
    for (int r = 0; r < RB; ++r) red[(g * RB + r) * NB + i] = p[r];
    __syncthreads();
    if (g == 0) {
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        T v = x[r * Npad + base + i];
        for (int gg = 0; gg < NG; ++gg) v -= red[(gg * RB + r) * NB + i];
        tt[r * NB + i] = v;
      }
    }
    __syncthreads();
    // phase B: a[base+i] = sum_{i<=k, base+k<N} W_II[k, i] * tt[k]  (0 for the rows >= N of the last block step;
    // rows >= N of W_II are masked rather than cut from the loop: the constant trip bound keeps the float64 loop as fast)
#pragma unroll
    for (int r = 0; r < RB; ++r) p[r] = T(0);
    for (int kk = i + g; kk < NB; kk += NG) {
      T w = base + kk < N ? Wb[(long)kk * NB + i] : T(0);
#pragma unroll
      for (int r = 0; r < RB; ++r) p[r] = fma(w, tt[r * NB + kk], p[r]);
    }
#pragma unroll
    for (int r = 0; r < RB; ++r) red[(g * RB + r) * NB + i] = p[r];
    __syncthreads();
    if (g == 0) {
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        T v = T(0);
        for (int gg = 0; gg < NG; ++gg) v += red[(gg * RB + r) * NB + i];
        x[r * Npad + base + i] = v;
      }
    }
    __syncthreads();
  }
  for (int n = tid; n < Npad; n += 256)
#pragma unroll
    for (int r = 0; r < RB; ++r)
      if (f0 + r < F) alpha[((long)s * F + f0 + r) * Npad + n] = x[r * Npad + n];
}

// ---------------------------------------------------------------------------------------------------------------
// The same solve with the right-hand sides in global memory (alpha is the working vector), for any Npad.
// Right-looking in both directions, one launch per block step; L is read once per direction by the whole grid.
// A CTA owns (one FB-group of right-hand sides, one target tile, one sample); it forms the step's diagonal-block
// product t = W x redundantly (NB^2 per right-hand side) and applies it to its own tile:
//   forward, step J:   x_I -= L_IJ t_J,        t_J = W_JJ x_J,     every block row I > J
//   backward, step I:  x_J -= L_IJ^T a_I,      a_I = W_II^T x_I,   every block column J < I
// The CTAs of step J all read x_J, so none of them may overwrite it: CTA 0 of the NEXT launch forms the same product
// again and stores it (no other CTA of that launch touches that block).  Only rows < N are read or written: under
// n_lead < N the rows >= N of L and winv belong to a larger joint factor and may hold anything, and alpha keeps zeros
// there from the initialisation.
template <typename T>
__global__ void solve_gm_init_kernel(int N, int Npad, int F, const T* __restrict__ y, long long y_stride, int ldy,
                                     const T* __restrict__ mean, T* __restrict__ x, long long total) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
    const long long sf = e / Npad;
    const int n = (int)(e - sf * Npad);
    const long long s = sf / F;
    const int f = (int)(sf - s * F);
    x[e] = n < N ? y[s * y_stride + (long long)f * ldy + n] - (mean ? mean[s] : T(0)) : T(0);
  }
}

// xs[r][k] = x[s][f0+r][base+k] for rows < N and f < F, else 0
template <typename T, int FB>
__device__ __forceinline__ void solve_gm_load(T (*xs)[Cfg<T>::NB], const T* x, int N, int Npad, int F, int f0, int base) {
  constexpr int NB = Cfg<T>::NB;
  for (int e = threadIdx.x; e < FB * NB; e += 256) {
    const int r = e / NB, k = e % NB;
    xs[r][k] = (f0 + r < F && base + k < N) ? x[(long long)(f0 + r) * Npad + base + k] : T(0);
  }
}

template <typename T, int FB>
__device__ __forceinline__ void solve_gm_store(const T (*ts)[Cfg<T>::NB], T* x, int N, int Npad, int F, int f0, int base) {
  constexpr int NB = Cfg<T>::NB;
  for (int e = threadIdx.x; e < FB * NB; e += 256) {
    const int r = e / NB, k = e % NB;
    if (f0 + r < F && base + k < N) x[(long long)(f0 + r) * Npad + base + k] = ts[r][k];
  }
}

// Forward step J (launch J = 0 .. nbN): blockIdx.y == 0 stores t_{J-1} into x_{J-1}; blockIdx.y = b > 0 updates block
// row I = J + b with t_J.  Rows of a tile are dotted by one warp, four at a time, lanes along the contiguous columns.
template <typename T, int FB>
__global__ void __launch_bounds__(256) solve_gm_fwd_kernel(int N, int Npad, int F, int J, const T* __restrict__ L,
                                                           const T* __restrict__ winv, T* __restrict__ x) {
  constexpr int NB = Cfg<T>::NB;
  __shared__ T xs[FB][NB], ts[FB][NB];
  const bool store = blockIdx.y == 0;
  const int K = store ? J - 1 : J;
  if (K < 0) return;
  const int f0 = blockIdx.x * FB, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long s = blockIdx.z;
  const T* Ls = L + s * Npad * (long long)Npad;
  const T* Wb = winv + (s * (Npad / NB) + K) * (long long)(NB * NB);
  T* xs_g = x + s * F * (long long)Npad;
  const int base = K * NB;
  solve_gm_load<T, FB>(xs, xs_g, N, Npad, F, f0, base);
  __syncthreads();
  // t[i] = sum_{k <= i} W[i][k] x[k], rows i < N
  for (int i0 = warp * 4; i0 < NB; i0 += 32) {
    T p[4][FB];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int r = 0; r < FB; ++r) p[q][r] = T(0);
    for (int k = lane; k < NB; k += 32) {
      T w[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) w[q] = (k <= i0 + q && base + i0 + q < N) ? Wb[(i0 + q) * NB + k] : T(0);
#pragma unroll
      for (int r = 0; r < FB; ++r) {
        const T xv = xs[r][k];
#pragma unroll
        for (int q = 0; q < 4; ++q) p[q][r] = fma(w[q], xv, p[q][r]);
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int r = 0; r < FB; ++r) {
        const T v = warp_sum(p[q][r]);
        if (lane == 0) ts[r][i0 + q] = v;
      }
  }
  __syncthreads();
  if (store) {
    solve_gm_store<T, FB>(ts, xs_g, N, Npad, F, f0, base);
    return;
  }
  // x_I[i] -= sum_k L[I*NB + i][base + k] t[k], rows < N (columns base + k < I*NB are then < N too)
  const int rbase = (J + blockIdx.y) * NB;
  for (int i0 = warp * 4; i0 < NB; i0 += 32) {
    T p[4][FB];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int r = 0; r < FB; ++r) p[q][r] = T(0);
    for (int k = lane; k < NB; k += 32) {
      T l[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        l[q] = rbase + i0 + q < N ? Ls[(long long)(rbase + i0 + q) * Npad + base + k] : T(0);
#pragma unroll
      for (int r = 0; r < FB; ++r) {
        const T tv = ts[r][k];
#pragma unroll
        for (int q = 0; q < 4; ++q) p[q][r] = fma(l[q], tv, p[q][r]);
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int r = 0; r < FB; ++r) {
        const T v = warp_sum(p[q][r]);
        const int row = rbase + i0 + q;
        if (lane == ((q * FB + r) & 31) && row < N && f0 + r < F) xs_g[(long long)(f0 + r) * Npad + row] -= v;
      }
  }
}

// Backward step I (launch I = nbN-1 .. -1): blockIdx.y == 0 stores a_{I+1} into x_{I+1}; blockIdx.y = b > 0 updates
// block column J = b - 1 < I with a_I.  A thread owns one column and walks rows in NG interleaved groups (coalesced
// row reads of W and L); the groups are summed in a fixed order.
template <typename T, int FB>
__global__ void __launch_bounds__(256) solve_gm_bwd_kernel(int N, int Npad, int F, int I, int nbN,
                                                           const T* __restrict__ L, const T* __restrict__ winv,
                                                           T* __restrict__ x) {
  constexpr int NB = Cfg<T>::NB, NG = 256 / NB;
  __shared__ T xs[FB][NB], ts[FB][NB], red[NG][FB][NB];
  const bool store = blockIdx.y == 0;
  const int K = store ? I + 1 : I;
  if (K < 0 || K >= nbN) return;
  const int f0 = blockIdx.x * FB, tid = threadIdx.x, c = tid % NB, g = tid / NB;
  const long long s = blockIdx.z;
  const T* Ls = L + s * Npad * (long long)Npad;
  const T* Wb = winv + (s * (Npad / NB) + K) * (long long)(NB * NB);
  T* xs_g = x + s * F * (long long)Npad;
  const int base = K * NB;
  solve_gm_load<T, FB>(xs, xs_g, N, Npad, F, f0, base);
  __syncthreads();
  // a[c] = sum_{c <= k, base + k < N} W[k][c] x[k]
  T p[FB];
#pragma unroll
  for (int r = 0; r < FB; ++r) p[r] = T(0);
  for (int k = c + g; k < NB && base + k < N; k += NG) {
    const T w = Wb[k * NB + c];
#pragma unroll
    for (int r = 0; r < FB; ++r) p[r] = fma(w, xs[r][k], p[r]);
  }
#pragma unroll
  for (int r = 0; r < FB; ++r) red[g][r][c] = p[r];
  __syncthreads();
  for (int e = tid; e < FB * NB; e += 256) {
    const int r = e / NB, k = e % NB;
    T v = T(0);
#pragma unroll
    for (int gg = 0; gg < NG; ++gg) v += red[gg][r][k];
    ts[r][k] = v;
  }
  __syncthreads();
  if (store) {
    solve_gm_store<T, FB>(ts, xs_g, N, Npad, F, f0, base);
    return;
  }
  // x_J[c] -= sum_{i: base + i < N} L[base + i][J*NB + c] a[i]
  const int cbase = (blockIdx.y - 1) * NB;
#pragma unroll
  for (int r = 0; r < FB; ++r) p[r] = T(0);
  for (int i = g; i < NB && base + i < N; i += NG) {
    const T l = Ls[(long long)(base + i) * Npad + cbase + c];
#pragma unroll
    for (int r = 0; r < FB; ++r) p[r] = fma(l, ts[r][i], p[r]);
  }
#pragma unroll
  for (int r = 0; r < FB; ++r) red[g][r][c] = p[r];
  __syncthreads();
  for (int e = tid; e < FB * NB; e += 256) {
    const int r = e / NB, k = e % NB;
    if (f0 + r >= F) continue;
    T v = T(0);
#pragma unroll
    for (int gg = 0; gg < NG; ++gg) v += red[gg][r][k];
    xs_g[(long long)(f0 + r) * Npad + cbase + k] -= v;
  }
}

// quad[s][f] = |x[s][f]|^2 after the forward pass (rows >= N are zero);  sum_log_diag[s] from blockIdx.x == 0
template <typename T>
__global__ void __launch_bounds__(256) solve_gm_scalars_kernel(int N, int Npad, int F, const T* __restrict__ L,
                                                               const T* __restrict__ x, T* __restrict__ sum_log_diag,
                                                               T* __restrict__ quad) {
  __shared__ T red8[8];
  const long long s = blockIdx.y;
  const int f = blockIdx.x, tid = threadIdx.x;
  if (quad) {
    const T* xr = x + (s * F + f) * (long long)Npad;
    T a = T(0);
    for (int n = tid; n < N; n += 256) a = fma(xr[n], xr[n], a);
    a = block_sum(a, red8);
    if (tid == 0) quad[s * F + f] = a;
  }
  if (sum_log_diag && f == 0) {
    const T* Ls = L + s * Npad * (long long)Npad;
    T a = T(0);
    for (int n = tid; n < N; n += 256) a += smk_log(Ls[(long long)n * Npad + n]);
    a = block_sum(a, red8);
    if (tid == 0) sum_log_diag[s] = a;
  }
}

template <typename T, int FB>
static void solve_gm_forward(int N, int Npad, int S, int F, const T* L, const T* winv, T* alpha, cudaStream_t st) {
  constexpr int NB = Cfg<T>::NB;
  const int nbN = (N + NB - 1) / NB, ng = (F + FB - 1) / FB;
  for (int J = 0; J <= nbN; ++J)
    solve_gm_fwd_kernel<T, FB><<<dim3(ng, J < nbN ? nbN - J : 1, S), 256, 0, st>>>(N, Npad, F, J, L, winv, alpha);
  count_launch(nbN + 1);
}

template <typename T, int FB>
static void solve_gm_backward(int N, int Npad, int S, int F, const T* L, const T* winv, T* alpha, cudaStream_t st) {
  constexpr int NB = Cfg<T>::NB;
  const int nbN = (N + NB - 1) / NB, ng = (F + FB - 1) / FB;
  for (int I = nbN - 1; I >= -1; --I)
    solve_gm_bwd_kernel<T, FB><<<dim3(ng, I + 1 > 0 ? I + 1 : 1, S), 256, 0, st>>>(N, Npad, F, I, nbN, L, winv, alpha);
  count_launch(nbN + 1);
}

template <typename T>
int chol_solve_gm(int N, int Npad, int S, int F, const T* L, const T* winv, const T* y, long long y_stride, int ldy,
                  const T* mean, T* alpha, T* sum_log_diag, T* quad, cudaStream_t st) {
  if (N <= 0) return -1;
  if (Npad < N || Npad % kNpadMult) return -2;
  if (S <= 0 || S > 65535) return -3;
  if (F <= 0) return -4;
  if (!L) return -5;
  if (!winv) return -6;
  if (!y) return -7;
  if (ldy < N) return -9;
  if (!alpha) return -11;
  const long long total = (long long)S * F * Npad;
  const int ib = (int)(total / 256 + 1 < 132 * 16 ? total / 256 + 1 : 132 * 16);
  solve_gm_init_kernel<T><<<ib, 256, 0, st>>>(N, Npad, F, y, y_stride, ldy, mean, alpha, total);
  count_launch();
  // FB right-hand sides per CTA: one when there is one, else a group that reuses each L element 4 or 8 times
  if (F == 1) solve_gm_forward<T, 1>(N, Npad, S, F, L, winv, alpha, st);
  else if (F <= 4) solve_gm_forward<T, 4>(N, Npad, S, F, L, winv, alpha, st);
  else solve_gm_forward<T, 8>(N, Npad, S, F, L, winv, alpha, st);
  if (quad || sum_log_diag) {
    solve_gm_scalars_kernel<T><<<dim3(F, S), 256, 0, st>>>(N, Npad, F, L, alpha, sum_log_diag, quad);
    count_launch();
  }
  if (F == 1) solve_gm_backward<T, 1>(N, Npad, S, F, L, winv, alpha, st);
  else if (F <= 4) solve_gm_backward<T, 4>(N, Npad, S, F, L, winv, alpha, st);
  else solve_gm_backward<T, 8>(N, Npad, S, F, L, winv, alpha, st);
  return check_launch("chol_solve_gm");
}

template <typename T>
int chol_solve(int N, int Npad, int S, int F, const T* L, const T* winv, const T* y, long long y_stride, int ldy,
               const T* mean, T* alpha, T* sum_log_diag, T* quad, cudaStream_t st) {
  constexpr int NB = Cfg<T>::NB, RB = SolveCfg<T>::RB, NG = 256 / NB;
  if (N <= 0) return -1;
  if (Npad < N || Npad % kNpadMult) return -2;
  if (S <= 0) return -3;
  if (F <= 0) return -4;
  if (!L) return -5;
  if (!winv) return -6;
  if (!y) return -7;
  if (ldy < N) return -9;
  const size_t dsm = sizeof(T) * ((size_t)RB * Npad + RB * NB + (size_t)NG * RB * NB);
  // the right-hand sides of one CTA no longer fit in shared memory (next to the kernel's static red8[8])
  if (dsm + 8 * sizeof(T) > 227 * 1024) return chol_solve_gm<T>(N, Npad, S, F, L, winv, y, y_stride, ldy, mean, alpha, sum_log_diag,
                                                quad, st);
  static size_t attr_set = 0;
  if (dsm > attr_set) {
    cudaFuncSetAttribute(chol_solve_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsm);
    attr_set = dsm;
  }
  dim3 grid((F + RB - 1) / RB, S);
  chol_solve_kernel<T><<<grid, 256, dsm, st>>>(N, Npad, F, L, winv, y, y_stride, ldy, mean, alpha, sum_log_diag,
                                              quad, alpha != nullptr);
  count_launch();
  return check_launch("chol_solve");
}

// ---------------------------------------------------------------------------------------------------------------
// Log-likelihood by augmentation: put r = y - mean in row N of the (padded) covariance before factoring it,
//   [ K  . ]   [ L        0 ] [ L^T  L^-1 r ]
//   [ r' c ] = [ (L^-1r)' * ] [ 0    *      ]
// so the Cholesky panel/trailing kernels perform the forward substitution as part of the factorisation (one extra
// row in a block row that exists anyway) and   quad = |L[N, 0:N]|^2,   sum_log_diag = sum_{i<N} log L_ii.
// Needs Npad > N (the caller pads to ceil128(N + 1)).  Replaces the serial chol_solve on the slice-sampler path.
template <typename T>
__global__ void loglik_set_rhs_kernel(int N, int Npad, const T* __restrict__ y, const T* __restrict__ mean, T* A) {
  const int s = blockIdx.y, n = blockIdx.x * blockDim.x + threadIdx.x;
  T* row = A + (long)s * Npad * Npad + (long)N * Npad;
  if (n < N) row[n] = y[n] - mean[s];
  else if (n == N) row[n] = T(1e30);            // pivot of the augmented row: c - quad must stay positive
}

template <typename T>
__global__ void __launch_bounds__(256) loglik_finish_kernel(int N, int Npad, const T* __restrict__ L, T* __restrict__ sld,
                                                             T* __restrict__ quad) {
  __shared__ T red8[8];
  const int s = blockIdx.x, tid = threadIdx.x;
  const T* Ls = L + (long)s * Npad * Npad;
  T a = T(0), q = T(0);
  for (int n = tid; n < N; n += 256) {
    a += smk_log(Ls[(long)n * Npad + n]);
    T v = Ls[(long)N * Npad + n];
    q = fma(v, v, q);
  }
  a = block_sum(a, red8);
  q = block_sum(q, red8);
  if (tid == 0) { sld[s] = a; quad[s] = q; }
}

template <typename T>
int loglik_set_rhs(int N, int Npad, int S, const T* y, const T* mean, T* A, cudaStream_t st) {
  if (N <= 0 || Npad <= N || Npad % kNpadMult) return -2;
  if (S <= 0) return -3;
  if (!y || !mean || !A) return -4;
  loglik_set_rhs_kernel<T><<<dim3((N + 256) / 256, S), 256, 0, st>>>(N, Npad, y, mean, A);
  count_launch();
  return check_launch("loglik_set_rhs");
}
template <typename T>
int loglik_finish(int N, int Npad, int S, const T* L, T* sld, T* quad, cudaStream_t st) {
  if (N <= 0 || Npad <= N) return -2;
  if (S <= 0) return -3;
  if (!L || !sld || !quad) return -4;
  loglik_finish_kernel<T><<<S, 256, 0, st>>>(N, Npad, L, sld, quad);
  count_launch();
  return check_launch("loglik_finish");
}
template int loglik_set_rhs<float>(int, int, int, const float*, const float*, float*, cudaStream_t);
template int loglik_set_rhs<double>(int, int, int, const double*, const double*, double*, cudaStream_t);
template int loglik_finish<float>(int, int, int, const float*, float*, float*, cudaStream_t);
template int loglik_finish<double>(int, int, int, const double*, double*, double*, cudaStream_t);

template int chol_solve<float>(int, int, int, int, const float*, const float*, const float*, long long, int,
                               const float*, float*, float*, float*, cudaStream_t);
template int chol_solve<double>(int, int, int, int, const double*, const double*, const double*, long long, int,
                                const double*, double*, double*, double*, cudaStream_t);
template int chol_solve_gm<float>(int, int, int, int, const float*, const float*, const float*, long long, int,
                                  const float*, float*, float*, float*, cudaStream_t);
template int chol_solve_gm<double>(int, int, int, int, const double*, const double*, const double*, long long, int,
                                   const double*, double*, double*, double*, cudaStream_t);

}  // namespace smk
