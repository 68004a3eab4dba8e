// predict_mma.cu -- float64 fused GP prediction on the fp64 tensor cores (DMMA: mma.sync.m8n8k4.f64).
//
// Same outputs and the same dataflow as predict_kernel<double> (predict.cu), which does its N^2 work per (candidate,
// sample) pair on DFMA.  A persistent CTA owns a tile of BN = 64 candidates of one hyper-sample and walks the row blocks
// I = 0..Npad/NB-1 of the factor (NB = 64, the block of potrf<double>):
//     Kx_I   = amp2 k(X_I, C_tile)                 float64 on the CUDA cores, straight into the DMMA accumulator layout
//     T_I    = Kx_I - L_{I,<I} beta_{<I}           DMMA; L and beta tiles staged through a 3-stage cp.async ring
//     beta_I = W_II T_I                            DMMA; W_II = L_II^-1 from potrf<double>, T_I resident in shared memory
//     ssq   += colsum(beta_I^2);  mdot += colsum(alpha_I Kx_I)
// beta_I is parked in the CTA's scratch slab for the later row blocks, candidate-major ([c][k], k contiguous) so that it
// is staged exactly like the L tile.  Work items (sample, tile) go sample-major over the CTAs: a float64 factor at
// N = 4096 is 134 MB, larger than L2, so the CTAs running at the same time stream the same sample's L.
//
// 8 warps as 2 (rows) x 4 (candidates); a warp owns a 32 x 16 block of the 64 x 64 tile: 4 x 2 DMMA tiles of 8 x 8.
// Shared-memory operands use a row stride of 20 doubles (16 + 4), so that the 8-byte fragment loads hit distinct banks
// (as in potrf_ll.cu).
#include "common.cuh"

namespace smk {
int num_sms();

namespace pm {

constexpr int NB = 64;      // row block (= Cfg<double>::NB, the diagonal block of winv)
constexpr int BN = 64;      // candidates per work item
constexpr int KC = 16;      // k per ring stage
constexpr int LDS = 20;     // ring row stride (doubles)
constexpr int ST = 3;       // ring stages
constexpr int LDT = NB + 4; // row stride of T_I as [candidate][row]
constexpr int DC = 32;      // dimension chunk of the cross-covariance generator
constexpr int LDX = NB + 1; // generator staging row stride (odd: conflict-free column stores)
static_assert(NB == BN, "the generator stages rows and candidates with one loop");

struct Smem {
  union {
    struct { double A[ST][NB][LDS]; double B[ST][BN][LDS]; } ring;   // GEMM operands
    struct { double xs[DC][LDX]; double cs[DC][LDX]; } gen;          // scaled inputs / candidates of the generator
  } u;
  double Ts[BN][LDT];      // T_I, the B operand of the diagonal solve
  double colred[16][BN];   // cross-thread column reductions
};

struct Args {
  int kind, N, Npad, M, D, S, ldm, ntiles;
  const double *X, *C, *inv_ls, *amp2, *mean, *L, *winv, *alpha;
  double *mu, *var;
  double* scratch;         // [gridDim.x][BN][Npad]
};

__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// acc[mi][ni][e] += sum_{k<K} A(row, k) B(col, k), row = wm*32 + mi*8 + gq, col = wn*16 + ni*8 + 2*t4 + e.
// A(row, k) = A[row * lda + k] in global memory (NB rows).  B(col, k) = B[col * ldb + k]: global memory (staged through
// the ring) or, with BSM, shared memory read in place.  K % KC == 0.  All 256 threads call this; it starts and ends with a
// barrier, so the ring may alias the generator's staging and B may be written just before the call.
template <bool BSM>
__device__ __forceinline__ void gemm(double (&acc)[4][2][2], const double* A, long lda, const double* B, long ldb, int K,
                                     Smem& sm) {
  const int nk = K / KC;
  if (nk == 0) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = warp >> 2, wn = warp & 3, gq = lane >> 2, t4 = lane & 3;
  auto load = [&](int st, int k0) {
#pragma unroll
    for (int q = 0; q < NB * (KC / 2) / 256; ++q) {       // 16-byte chunks: row = chunk / 8, 2 doubles each
      const int ch = tid + q * 256, row = ch >> 3, pc = ch & 7;
      cp_async16(&sm.u.ring.A[st][row][pc * 2], A + (long)row * lda + k0 + pc * 2);
      if (!BSM) cp_async16(&sm.u.ring.B[st][row][pc * 2], B + (long)row * ldb + k0 + pc * 2);
    }
  };
  __syncthreads();
#pragma unroll
  for (int s = 0; s < ST - 1; ++s) {
    if (s < nk) load(s, s * KC);
    cp_async_commit();
  }
  for (int kt = 0; kt < nk; ++kt) {
    cp_async_wait<ST - 2>();
    __syncthreads();
    if (kt + ST - 1 < nk) load((kt + ST - 1) % ST, (kt + ST - 1) * KC);
    cp_async_commit();
    const double* as = &sm.u.ring.A[kt % ST][wm * 32 + gq][t4];
    const double* bs = BSM ? B + (long)(wn * 16 + gq) * ldb + kt * KC + t4 : &sm.u.ring.B[kt % ST][wn * 16 + gq][t4];
    const long ldbs = BSM ? ldb : LDS;
#pragma unroll
    for (int kk = 0; kk < KC; kk += 4) {
      double af[4], bf[2];
#pragma unroll
      for (int mi = 0; mi < 4; ++mi) af[mi] = as[mi * 8 * LDS + kk];
#pragma unroll
      for (int ni = 0; ni < 2; ++ni) bf[ni] = bs[ni * 8 * ldbs + kk];
#pragma unroll
      for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 2; ++ni) dmma(acc[mi][ni], af[mi], bf[ni]);
    }
  }
  cp_async_wait<0>();
  __syncthreads();
}

__global__ void __launch_bounds__(256, 2) predict_mma_kernel(Args p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = warp >> 2, wn = warp & 3, gq = lane >> 2, t4 = lane & 3;
  const int nblk = p.Npad / NB;
  double* scr = p.scratch + (long)blockIdx.x * BN * p.Npad;
  const long nwork = (long)p.S * p.ntiles;

  for (long w = blockIdx.x; w < nwork; w += gridDim.x) {
    const int s = (int)(w / p.ntiles), tile = (int)(w % p.ntiles);
    const int c0 = tile * BN;
    const double* ils = p.inv_ls + (long)s * p.D;
    const double a2 = p.amp2[s];
    const double* Ls = p.L + (long)s * p.Npad * p.Npad;
    const double* Ws = p.winv + (long)s * nblk * NB * NB;
    const double* al = p.alpha + (long)s * p.Npad;

    double ssq[4], mdot[4];          // per candidate column (ni, e) of this thread
#pragma unroll
    for (int c = 0; c < 4; ++c) { ssq[c] = 0.0; mdot[c] = 0.0; }

    for (int I = 0; I < nblk; ++I) {
      const int base = I * NB;
      double acc[4][2][2];
#pragma unroll
      for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 2; ++ni) { acc[mi][ni][0] = 0.0; acc[mi][ni][1] = 0.0; }

      // ---- 1. squared scaled distances of the tile, in the accumulator layout
      for (int d0 = 0; d0 < p.D; d0 += DC) {
        __syncthreads();
        for (int e = tid; e < NB * DC; e += 256) {
          const int row = e / DC, dd = e % DC, d = d0 + dd;
          const int gi = base + row, gc = min(c0 + row, p.M - 1);
          const double sc = (d < p.D) ? ils[d] : 0.0;
          sm.u.gen.xs[dd][row] = (d < p.D && gi < p.N) ? p.X[(long)gi * p.D + d] * sc : 0.0;
          sm.u.gen.cs[dd][row] = (d < p.D) ? p.C[(long)gc * p.D + d] * sc : 0.0;
        }
        __syncthreads();
        const int dmax = min(DC, p.D - d0);
        for (int dd = 0; dd < dmax; ++dd) {
          double a[4], b[4];
#pragma unroll
          for (int mi = 0; mi < 4; ++mi) a[mi] = sm.u.gen.xs[dd][wm * 32 + mi * 8 + gq];
#pragma unroll
          for (int c = 0; c < 4; ++c) b[c] = sm.u.gen.cs[dd][wn * 16 + (c >> 1) * 8 + 2 * t4 + (c & 1)];
#pragma unroll
          for (int mi = 0; mi < 4; ++mi)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const double df = a[mi] - b[c];
              acc[mi][c >> 1][c & 1] = fma(df, df, acc[mi][c >> 1][c & 1]);
            }
        }
      }
      // Kx (padded rows are zero; alpha's padding is zero) -> mdot; the accumulator starts at -Kx
#pragma unroll
      for (int mi = 0; mi < 4; ++mi) {
        const int gi = base + wm * 32 + mi * 8 + gq;
        const double valid = (gi < p.N) ? a2 : 0.0;
        const double ar = al[gi];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const double k = valid * kernel_of_r2<double>(p.kind, acc[mi][c >> 1][c & 1]);
          acc[mi][c >> 1][c & 1] = -k;
          mdot[c] = fma(ar, k, mdot[c]);
        }
      }

      // ---- 2. -T_I = -Kx_I + L[I, 0:base] beta[0:base]
      gemm<false>(acc, Ls + (long)base * p.Npad, p.Npad, scr, p.Npad, base, sm);

      // ---- 3. T_I -> shared as [candidate][row]  (the last reader of Ts, step 4 of the previous block, ended on a barrier)
#pragma unroll
      for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          sm.Ts[wn * 16 + (c >> 1) * 8 + 2 * t4 + (c & 1)][wm * 32 + mi * 8 + gq] = -acc[mi][c >> 1][c & 1];
          acc[mi][c >> 1][c & 1] = 0.0;
        }

      // ---- 4. beta_I = W_II T_I
      gemm<true>(acc, Ws + (long)I * NB * NB, NB, &sm.Ts[0][0], LDT, NB, sm);

      // ---- 5. |beta|^2, and beta_I parked for the later row blocks
#pragma unroll
      for (int mi = 0; mi < 4; ++mi) {
        const int r = base + wm * 32 + mi * 8 + gq;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const double b = acc[mi][c >> 1][c & 1];
          ssq[c] = fma(b, b, ssq[c]);
          if (I + 1 < nblk) scr[(long)(wn * 16 + (c >> 1) * 8 + 2 * t4 + (c & 1)) * p.Npad + r] = b;
        }
      }
    }

    // ---- epilogue: reduce the per-thread column partials over the 16 row-threads of each column
#pragma unroll
    for (int c = 0; c < 4; ++c) sm.colred[wm * 8 + gq][wn * 16 + (c >> 1) * 8 + 2 * t4 + (c & 1)] = ssq[c];
    __syncthreads();
    double tot_ssq = 0.0, tot_m = 0.0;
    if (tid < BN)
      for (int q = 0; q < 16; ++q) tot_ssq += sm.colred[q][tid];
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 4; ++c) sm.colred[wm * 8 + gq][wn * 16 + (c >> 1) * 8 + 2 * t4 + (c & 1)] = mdot[c];
    __syncthreads();
    if (tid < BN) {
      for (int q = 0; q < 16; ++q) tot_m += sm.colred[q][tid];
      const int gc = c0 + tid;
      if (gc < p.M) {
        p.mu[(long)s * p.ldm + gc] = tot_m + p.mean[s];
        p.var[(long)s * p.ldm + gc] = a2 * 1.000001 - tot_ssq;
      }
    }
    __syncthreads();
  }
}

}  // namespace pm

// Same arguments, codes and workspace as predict<double> (predict.cu); the scratch slab of a CTA is BN x Npad doubles, the
// size of predict<double>'s, so smk_predict_workspace_bytes(8, Npad) covers both.
int predict_mma_f64(int kind, int N, int Npad, int M, int D, int S, const double* X, const double* Cc,
                    const double* inv_ls, const double* amp2, const double* mean, const double* L, const double* winv,
                    const double* alpha, double* mu, double* var, int ldm, void* workspace, size_t workspace_bytes,
                    cudaStream_t st) {
  if (kind < 0 || kind > 3) return -1;
  if (N <= 0) return -2;
  if (Npad < N || Npad % kNpadMult) return -3;
  if (M <= 0) return -4;
  if (D <= 0) return -5;
  if (S <= 0) return -6;
  if (!X || !Cc || !inv_ls || !amp2 || !mean || !L || !winv || !alpha) return -7;
  if (!mu || !var) return -15;
  if (ldm < M) return -17;
  const int ntiles = (M + pm::BN - 1) / pm::BN;
  const long nwork = (long)S * ntiles;
  int grid = 2 * num_sms();
  if (nwork < grid) grid = (int)nwork;
  if (!workspace || workspace_bytes < (size_t)grid * pm::BN * Npad * sizeof(double)) return -18;
  const size_t dsm = sizeof(pm::Smem);
  static bool attr_done = false;
  if (!attr_done) {
    cudaFuncSetAttribute(pm::predict_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsm);
    attr_done = true;
  }
  pm::Args a;
  a.kind = kind; a.N = N; a.Npad = Npad; a.M = M; a.D = D; a.S = S; a.ldm = ldm; a.ntiles = ntiles;
  a.X = X; a.C = Cc; a.inv_ls = inv_ls; a.amp2 = amp2; a.mean = mean; a.L = L; a.winv = winv; a.alpha = alpha;
  a.mu = mu; a.var = var; a.scratch = reinterpret_cast<double*>(workspace);
  timing_begin("predict_mma_kernel", st);
  pm::predict_mma_kernel<<<grid, 256, dsm, st>>>(a);
  timing_end(st);
  count_launch();
  return check_launch("predict_mma");
}

}  // namespace smk
