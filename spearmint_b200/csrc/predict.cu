// predict.cu -- fused GP prediction at the candidate grid, batched over hyper-samples.
//
// Reference spans replaced (per hyper-sample, OPT = chooser/GPEIOptChooser.py):
//   cand_cross = self.cov(comp, cand)                               OPT:536  (N x M, float64)
//   beta       = spla.solve_triangular(obsv_chol, cand_cross)       OPT:544  (N x M, float64)
//   func_m     = np.dot(cand_cross.T, alpha) + self.mean            OPT:547
//   func_v     = self.amp2*(1+1e-6) - np.sum(beta**2, axis=0)       OPT:548
// The reference materialises cand_cross and beta (2 x 8 x N x M bytes per sample, 6.5 GB each at
// N=8192, M=100k).  Here a persistent block owns a tile of BN candidates and walks the row blocks
// I = 0..N/NB-1 of the factor:
//     T_I    = Kx_I - sum_{J<I} L_IJ * beta_J      (Kx_I generated on the fly from X_I and the tile)
//     beta_I = W_II * T_I                          (W_II = L_II^-1 from potrf.cu)
//     ssq   += colsum(beta_I^2);  mdot += colsum(alpha_I * Kx_I)
// beta_J tiles are parked in a per-block scratch slab (Npad x BN elements, L2-resident) because later
// row blocks need them; nothing N x M-sized is ever written.  Algorithmic work per
// (candidate, sample) pair: N^2 flops (triangular solve) + (3D + ~25) N (cross covariance).
#include "common.cuh"

namespace smk {

template <typename T>
struct PredictArgs {
  int kind, N, Npad, M, D, S, ldm, ntiles;
  const T *X, *C, *inv_ls, *amp2, *mean, *L, *winv, *alpha;
  T *mu, *var;
  T* scratch;  // [gridDim.x][Npad][BN]
};

template <typename T>
struct PredictSmem {
  using C = Cfg<T>;
  TileSmem<T> g;                    // GEMM staging; also reused as xs/cs staging of the Kx generator
  T Ts[C::BM][C::BN + kPad];        // T_I tile as the smem-resident B operand of the diagonal solve
  T colred[16][C::BN];              // cross-thread column reductions
};

constexpr int kDCp = 32;  // D chunk of the cross-covariance generator

template <typename T>
__global__ void __launch_bounds__(256, 2) predict_kernel(PredictArgs<T> p) {
  using C = Cfg<T>;
  constexpr int BM = C::BM, BN = C::BN, TM = C::TM, TN = C::TN, NB = C::NB;
  static_assert(BM == NB && BN == NB, "predict assumes square blocks equal to the factor block");
  static_assert(kDCp * (BM + kPad) <= 2 * kBK * (BM + kPad), "xs staging must fit in As");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  PredictSmem<T>& sm = *reinterpret_cast<PredictSmem<T>*>(smem_raw);
  // xs[dd][i], cs[dd][c] alias the GEMM staging buffers (never live at the same time)
  T (*xs)[BM + kPad] = reinterpret_cast<T (*)[BM + kPad]>(&sm.g.As[0][0][0]);
  T (*cs)[BN + kPad] = reinterpret_cast<T (*)[BN + kPad]>(&sm.g.Bs[0][0][0]);

  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const int nblk = p.Npad / NB;
  T* scr = p.scratch + (long)blockIdx.x * p.Npad * BN;
  const long nwork = (long)p.S * p.ntiles;

  for (long w = blockIdx.x; w < nwork; w += gridDim.x) {
    const int s = (int)(w / p.ntiles), tile = (int)(w % p.ntiles);
    const int c0 = tile * BN;
    const T* ils = p.inv_ls + (long)s * p.D;
    const T a2 = p.amp2[s];
    const T* Ls = p.L + (long)s * p.Npad * p.Npad;
    const T* Ws = p.winv + (long)s * nblk * NB * NB;
    const T* al = p.alpha + (long)s * p.Npad;

    T ssq[TN], mdot[TN];
#pragma unroll
    for (int c = 0; c < TN; ++c) { ssq[c] = T(0); mdot[c] = T(0); }

    for (int I = 0; I < nblk; ++I) {
      const int base = I * NB;
      T acc[TM][TN];
#pragma unroll
      for (int r = 0; r < TM; ++r)
#pragma unroll
        for (int c = 0; c < TN; ++c) acc[r][c] = T(0);

      // ---- 1. cross-covariance tile Kx_I (rows base.., candidates c0..) into acc
      for (int d0 = 0; d0 < p.D; d0 += kDCp) {
        __syncthreads();
        for (int e = tid; e < BM * kDCp; e += 256) {
          int row = e / kDCp, dd = e % kDCp, d = d0 + dd;
          int gi = base + row, gc = min(c0 + row, p.M - 1);
          T sc = (d < p.D) ? ils[d] : T(0);
          xs[dd][row] = (d < p.D && gi < p.N) ? p.X[(long)gi * p.D + d] * sc : T(0);
          cs[dd][row] = (d < p.D) ? p.C[(long)gc * p.D + d] * sc : T(0);
        }
        __syncthreads();
        const int dmax = min(kDCp, p.D - d0);
        for (int dd = 0; dd < dmax; ++dd) {
          T a[TM], b[TN];
#pragma unroll
          for (int g = 0; g < TM / 4; ++g) {
            V4<T> t = ld4(&xs[dd][g * 64 + ty * 4]);
#pragma unroll
            for (int e = 0; e < 4; ++e) a[g * 4 + e] = t.v[e];
          }
#pragma unroll
          for (int g = 0; g < TN / 4; ++g) {
            V4<T> t = ld4(&cs[dd][g * 64 + tx * 4]);
#pragma unroll
            for (int e = 0; e < 4; ++e) b[g * 4 + e] = t.v[e];
          }
#pragma unroll
          for (int r = 0; r < TM; ++r)
#pragma unroll
            for (int c = 0; c < TN; ++c) {
              T df = a[r] - b[c];
              acc[r][c] = fma(df, df, acc[r][c]);
            }
        }
      }
#pragma unroll
      for (int r = 0; r < TM; ++r) {
        const int gi = base + tile_row(ty, r);
        const T valid = (gi < p.N) ? a2 : T(0);      // padded rows of Kx are zero
        const T ar = al[gi];                          // alpha padding is zero
#pragma unroll
        for (int c = 0; c < TN; ++c) {
          T k = valid * kernel_of_r2<T>(p.kind, acc[r][c]);
          acc[r][c] = k;
          mdot[c] = fma(ar, k, mdot[c]);
        }
      }

      // ---- 2. acc -= L[I, 0:base] * beta[0:base]   (beta tiles from this block's scratch slab)
      TileGemm<T, Lay::KContig, Lay::MContig, true>::run(acc, Ls + (long)base * p.Npad, p.Npad, scr, BN, base,
                                                         sm.g);

      // ---- 3. T_I -> shared (as the [k][col] operand of the diagonal solve)
      __syncthreads();
#pragma unroll
      for (int r = 0; r < TM; ++r)
#pragma unroll
        for (int g = 0; g < TN / 4; ++g) {
          V4<T> v;
#pragma unroll
          for (int e = 0; e < 4; ++e) v.v[e] = acc[r][g * 4 + e];
          st4(&sm.Ts[tile_row(ty, r)][g * 64 + tx * 4], v);
        }
#pragma unroll
      for (int r = 0; r < TM; ++r)
#pragma unroll
        for (int c = 0; c < TN; ++c) acc[r][c] = T(0);

      // ---- 4. beta_I = W_II * T_I
      TileGemm<T, Lay::KContig, Lay::MContig, false>::run_bsmem(acc, Ws + (long)I * NB * NB, NB, &sm.Ts[0][0],
                                                               BN + kPad, NB, sm.g);

      // ---- 5. accumulate |beta|^2 and park beta_I for the later row blocks
#pragma unroll
      for (int r = 0; r < TM; ++r) {
#pragma unroll
        for (int c = 0; c < TN; ++c) ssq[c] = fma(acc[r][c], acc[r][c], ssq[c]);
        if (I + 1 < nblk) {
#pragma unroll
          for (int g = 0; g < TN / 4; ++g) {
            V4<T> v;
#pragma unroll
            for (int e = 0; e < 4; ++e) v.v[e] = acc[r][g * 4 + e];
            st4(scr + (long)(base + tile_row(ty, r)) * BN + g * 64 + tx * 4, v);
          }
        }
      }
    }

    // ---- epilogue: reduce the per-thread column partials over the 16 row-threads
    __syncthreads();
#pragma unroll
    for (int c = 0; c < TN; ++c) sm.colred[ty][tile_col(tx, c)] = ssq[c];
    __syncthreads();
    T tot_ssq = T(0), tot_m = T(0);
    if (tid < BN) {
      for (int q = 0; q < 16; ++q) tot_ssq += sm.colred[q][tid];
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < TN; ++c) sm.colred[ty][tile_col(tx, c)] = mdot[c];
    __syncthreads();
    if (tid < BN) {
      for (int q = 0; q < 16; ++q) tot_m += sm.colred[q][tid];
      const int gc = c0 + tid;
      if (gc < p.M) {
        p.mu[(long)s * p.ldm + gc] = tot_m + p.mean[s];
        p.var[(long)s * p.ldm + gc] = a2 * T(1.000001) - tot_ssq;
      }
    }
    __syncthreads();
  }
}

template <typename T>
size_t predict_workspace_bytes(int Npad, int grid) {
  return (size_t)grid * Npad * Cfg<T>::BN * sizeof(T);
}

static int g_num_sms = 0;
int num_sms() {
  if (!g_num_sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;   // H100 SXM
  }
  return g_num_sms;
}

template <typename T>
int predict_grid() {
  // float: ~103 KB smem/block -> 2 resident blocks per SM; double: 1-2.  Persistent grid = 2 x SMs.
  return 2 * num_sms();
}

template <typename T>
int predict(int kind, int N, int Npad, int M, int D, int S, const T* X, const T* Cc, const T* inv_ls, const T* amp2,
            const T* mean, const T* L, const T* winv, const T* alpha, T* mu, T* var, int ldm, void* workspace,
            size_t workspace_bytes, cudaStream_t st) {
  using C = Cfg<T>;
  if (kind < 0 || kind > 3) return -1;
  if (N <= 0) return -2;
  if (Npad < N || Npad % kNpadMult) return -3;
  if (M <= 0) return -4;
  if (D <= 0) return -5;
  if (S <= 0) return -6;
  if (!X || !Cc || !inv_ls || !amp2 || !mean || !L || !winv || !alpha) return -7;
  if (!mu || !var) return -15;
  if (ldm < M) return -17;
  const int ntiles = (M + C::BN - 1) / C::BN;
  long nwork = (long)S * ntiles;
  int grid = predict_grid<T>();
  if (nwork < grid) grid = (int)nwork;
  if (!workspace || workspace_bytes < predict_workspace_bytes<T>(Npad, grid)) return -18;
  const size_t dsm = sizeof(PredictSmem<T>);
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(predict_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsm);
    attr_done = true;
  }
  PredictArgs<T> a;
  a.kind = kind; a.N = N; a.Npad = Npad; a.M = M; a.D = D; a.S = S; a.ldm = ldm; a.ntiles = ntiles;
  a.X = X; a.C = Cc; a.inv_ls = inv_ls; a.amp2 = amp2; a.mean = mean; a.L = L; a.winv = winv; a.alpha = alpha;
  a.mu = mu; a.var = var; a.scratch = reinterpret_cast<T*>(workspace);
  timing_begin("predict_kernel", st);
  predict_kernel<T><<<grid, 256, dsm, st>>>(a);
  timing_end(st);
  count_launch();
  return check_launch("predict");
}

size_t predict_workspace_bytes_any(int elem_bytes, int Npad) {
  return elem_bytes == 8 ? predict_workspace_bytes<double>(Npad, 2 * num_sms())
                         : predict_workspace_bytes<float>(Npad, 2 * num_sms());
}

template int predict<float>(int, int, int, int, int, int, const float*, const float*, const float*, const float*,
                            const float*, const float*, const float*, const float*, float*, float*, int, void*,
                            size_t, cudaStream_t);
template int predict<double>(int, int, int, int, int, int, const double*, const double*, const double*,
                             const double*, const double*, const double*, const double*, const double*, double*,
                             double*, int, void*, size_t, cudaStream_t);

// ---------------------------------------------------------------------------------------------------
// cross mean only: mu[s][f][j] = sum_n alpha[s][f][n] * amp2 k(X_n, C_j) + mean[s]
// (time-GP mean PSEC:442-459; fantasy means OPT:609).  One block per (32-candidate tile, sample);
// the N x 32 cross-covariance strip is regenerated, never stored.  F right-hand sides are processed
// in register groups of FB.
// ---------------------------------------------------------------------------------------------------
constexpr int kFB = 8;

template <typename T>
__global__ void __launch_bounds__(256) cross_mean_kernel(int kind, int N, int Npad, int M, int D, int F,
                                                          const T* __restrict__ X, const T* __restrict__ Cc,
                                                          const T* __restrict__ inv_ls, const T* __restrict__ amp2,
                                                          const T* __restrict__ mean, const T* __restrict__ alpha,
                                                          T* __restrict__ mu, int ldm) {
  // block: 32 candidates (tx) x 8 row-lanes (ty); rows n strided by 8
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* cs = reinterpret_cast<T*>(smem_raw);  // [32][D+1] scaled candidates
  T* il = cs + 32 * (D + 1);               // [D]
  T* red = il + D;                         // [8][32]
  const int s = blockIdx.y, c0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int d = threadIdx.x; d < D; d += 256) il[d] = inv_ls[(long)s * D + d];
  __syncthreads();
  for (int e = threadIdx.x; e < 32 * D; e += 256) {
    int c = e / D, d = e % D;
    int gc = min(c0 + c, M - 1);
    cs[c * (D + 1) + d] = Cc[(long)gc * D + d] * il[d];
  }
  __syncthreads();
  const T a2 = amp2[s];
  const T* myc = cs + tx * (D + 1);
  for (int f0 = 0; f0 < F; f0 += kFB) {
    T acc[kFB];
#pragma unroll
    for (int f = 0; f < kFB; ++f) acc[f] = T(0);
    for (int n = ty; n < N; n += 8) {
      const T* xr = X + (long)n * D;
      T r2 = T(0);
      for (int d = 0; d < D; ++d) {
        T df = xr[d] * il[d] - myc[d];
        r2 = fma(df, df, r2);
      }
      T k = a2 * kernel_of_r2<T>(kind, r2);
#pragma unroll
      for (int f = 0; f < kFB; ++f)
        if (f0 + f < F) acc[f] = fma(alpha[((long)s * F + f0 + f) * Npad + n], k, acc[f]);
    }
#pragma unroll
    for (int f = 0; f < kFB; ++f) {
      __syncthreads();
      red[ty * 32 + tx] = acc[f];
      __syncthreads();
      if (ty == 0 && f0 + f < F && c0 + tx < M) {
        T v = T(0);
        for (int q = 0; q < 8; ++q) v += red[q * 32 + tx];
        mu[((long)s * F + f0 + f) * ldm + c0 + tx] = v + mean[s];
      }
    }
  }
}

template <typename T>
int cross_mean(int kind, int N, int Npad, int M, int D, int S, int F, const T* X, const T* Cc, const T* inv_ls,
               const T* amp2, const T* mean, const T* alpha, T* mu, int ldm, cudaStream_t st) {
  if (kind < 0 || kind > 3) return -1;
  if (N <= 0 || Npad < N) return -2;
  if (M <= 0) return -4;
  if (D <= 0) return -5;
  if (S <= 0) return -6;
  if (F <= 0) return -7;
  if (!X || !Cc || !inv_ls || !amp2 || !mean || !alpha || !mu) return -8;
  if (ldm < M) return -15;
  const size_t dsm = sizeof(T) * (32 * (size_t)(D + 1) + D + 256);
  static size_t attr_set = 48 * 1024;
  if (dsm > attr_set) {
    cudaFuncSetAttribute(cross_mean_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsm);
    attr_set = dsm;
  }
  dim3 grid((M + 31) / 32, S);
  cross_mean_kernel<T><<<grid, 256, dsm, st>>>(kind, N, Npad, M, D, F, X, Cc, inv_ls, amp2, mean, alpha, mu, ldm);
  count_launch();
  return check_launch("cross_mean");
}

template int cross_mean<float>(int, int, int, int, int, int, int, const float*, const float*, const float*,
                               const float*, const float*, const float*, float*, int, cudaStream_t);
template int cross_mean<double>(int, int, int, int, int, int, int, const double*, const double*, const double*,
                                const double*, const double*, const double*, double*, int, cudaStream_t);

}  // namespace smk
