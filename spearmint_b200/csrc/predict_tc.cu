// predict_tc.cu -- tensor-core (wgmma / TMA) version of the fused predict stage, and the tensor-core variants
// of the two N^3 factor steps that share its kernel.
//
// Same contract as predict.cu (reference spans OPT:536, 544, 547-548), different dataflow:
//   1. trtri   : Linv = L^-1 explicitly (row-block recurrence on wgmma, mode 3; SIMT version for small N) -- removes the
//                row-block dependency chain of the triangular solve: beta = Linv * Kx is one dense (lower-trapezoidal)
//                contraction.  Kept as a tf32 (hi, lo) pair of float arrays (hi = tf32 round-to-nearest of x, lo = x - hi, exact).
//   2. pack    : GEMM-operand copy of Linv: per-sample power-of-two scale 2^eb (largest |entry| -> [2^14, 2^15)) and the
//                round-to-nearest fp16 (hi, lo) pair (linv_pack_f16).
//   3. kxt     : Kxt[s][c][n] = amp2 k(X_n, C_c) * 2^ea for a chunk of candidates, candidate-major (n contiguous, i.e.
//                K-major for the MMA) as an fp16 (hi, lo) pair; fused mu[c] = sum_n alpha[n] Kx[c][n] + mean.
//                (kxt_kernel below: SIMT, the default; kxt_tc.cu: opt-in tensor-core generator.)
//   4. mma     : per (sample, 128-candidate tile, row-group pair):  D[c][i] = sum_n Kxt[c][n] * Linv[i][n]
//                as 3 x FP16 (lo*hi + hi*lo + hi*hi) with wgmma m64n256k16, fp32 accumulation, operands staged by
//                TMA (64-byte swizzle, 4 stages) by a producer warpgroup, two consumer warpgroups with the 128 x 256
//                accumulator in registers; epilogue = un-scale by 2^-(ea+eb), sum of squares per candidate row (over
//                the 4 lanes that share a row), partial sums per row-group pair.
//   5. finish  : var = amp2 (1 + 1e-6) - sum_p partial[p]
// Why a split at all: a single TF32/FP16 pass (11-bit significand) cannot resolve var = amp2 - |beta|^2 (it goes negative
// on the reference's own test problems).  Why fp16 rather than tf32 halves: same significand, twice the tensor rate; the
// missing exponent range is supplied by the exact scaling (DESIGN.md section 6).  3 MMAs per product => 1/3 of the dense
// bf16 tensor peak is the ceiling of this formulation; the kernel runs the tensor pipe 98.8 % active.
// Modes 2 (Cholesky update) and 3 (triangular inverse) of the same kernel keep tf32 (hi, lo) operands: they are produced
// block by block, before a global scale is known.
#include <cuda_fp16.h>
#include <cuda.h>

#include <algorithm>
#include <vector>
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "tc_common.cuh"

namespace smk {

// ================================================================================================= trtri (SIMT)
// X = L^-1, right-looking by block rows (the critical path is nblk small steps, so it scales down to a handful of
// matrices per GPU):   for K = 0..nblk-1:
//   finalize : X_KJ = W_KK * acc_KJ (J < K),  X_KK = W_KK          acc_KJ holds  -sum_{K'<K} L_KK' X_K'J
//   update   : acc_IJ -= L_IK * X_KJ  for I > K, J <= K
__global__ void __launch_bounds__(256, 2) trtri_finalize_kernel(int Npad, int ldx, int K, const float* __restrict__ winv,
                                                                 float* X) {
  using C = Cfg<float>;
  constexpr int NB = C::NB, TM = C::TM, TN = C::TN;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TileSmem<float>& sm = *reinterpret_cast<TileSmem<float>*>(smem_raw);
  float (*Ts)[NB + kPad] = reinterpret_cast<float (*)[NB + kPad]>(smem_raw + sizeof(TileSmem<float>));
  const int nblk = Npad / NB, J = blockIdx.x, s = blockIdx.y;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const float* W = winv + ((long)s * nblk + K) * NB * NB;
  float* Xt = X + (long)s * ldx * ldx + (long)K * NB * ldx + (long)J * NB;
  float acc[TM][TN];
  if (J == K) {
#pragma unroll
    for (int r = 0; r < TM; ++r)
#pragma unroll
      for (int g = 0; g < TN / 4; ++g) {
        V4<float> v = ld4(W + (long)tile_row(ty, r) * NB + g * 64 + tx * 4);
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[r][g * 4 + e] = v.v[e];
      }
  } else {
    // stage the accumulated tile in shared memory (it is overwritten in place), then multiply by W_KK
#pragma unroll
    for (int r = 0; r < TM; ++r)
#pragma unroll
      for (int g = 0; g < TN / 4; ++g) {
        V4<float> v = ld4(Xt + (long)tile_row(ty, r) * ldx + g * 64 + tx * 4);
        st4(&Ts[tile_row(ty, r)][g * 64 + tx * 4], v);
      }
#pragma unroll
    for (int r = 0; r < TM; ++r)
#pragma unroll
      for (int c = 0; c < TN; ++c) acc[r][c] = 0.f;
    TileGemm<float, Lay::KContig, Lay::MContig, false>::run_bsmem(acc, W, NB, &Ts[0][0], NB + kPad, NB, sm);
  }
#pragma unroll
  for (int r = 0; r < TM; ++r)
#pragma unroll
    for (int g = 0; g < TN / 4; ++g) {
      V4<float> v;
#pragma unroll
      for (int e = 0; e < 4; ++e) v.v[e] = acc[r][g * 4 + e];
      st4(Xt + (long)tile_row(ty, r) * ldx + g * 64 + tx * 4, v);
    }
}

// grid = (nblk-K-1, K+1, S):  X_IJ -= L_IK * X_KJ
__global__ void __launch_bounds__(256, 2) trtri_update_kernel(int Npad, int ldx, int K, const float* __restrict__ L,
                                                               float* X) {
  using C = Cfg<float>;
  constexpr int NB = C::NB, TM = C::TM, TN = C::TN;
  __shared__ TileSmem<float> sm;
  const int I = K + 1 + blockIdx.x, J = blockIdx.y, s = blockIdx.z;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const float* Lik = L + (long)s * Npad * Npad + (long)I * NB * Npad + (long)K * NB;
  float* Xs = X + (long)s * ldx * ldx;
  float* Xij = Xs + (long)I * NB * ldx + (long)J * NB;
  const float* Xkj = Xs + (long)K * NB * ldx + (long)J * NB;
  float acc[TM][TN];
  if (K == J) {            // first contribution to this tile: start from zero (the buffer is not pre-cleared)
#pragma unroll
    for (int r = 0; r < TM; ++r)
#pragma unroll
      for (int c = 0; c < TN; ++c) acc[r][c] = 0.f;
  } else {
#pragma unroll
    for (int r = 0; r < TM; ++r)
#pragma unroll
      for (int g = 0; g < TN / 4; ++g) {
        V4<float> v = ld4(Xij + (long)tile_row(ty, r) * ldx + g * 64 + tx * 4);
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[r][g * 4 + e] = v.v[e];
      }
  }
  TileGemm<float, Lay::KContig, Lay::MContig, true>::run(acc, Lik, Npad, Xkj, ldx, NB, sm);
#pragma unroll
  for (int r = 0; r < TM; ++r)
#pragma unroll
    for (int g = 0; g < TN / 4; ++g) {
      V4<float> v;
#pragma unroll
      for (int e = 0; e < 4; ++e) v.v[e] = acc[r][g * 4 + e];
      st4(Xij + (long)tile_row(ty, r) * ldx + g * 64 + tx * 4, v);
    }
}

__device__ __forceinline__ float tf32_hi(float x) { return tf32_rn(x); }   // round-to-nearest split (common.cuh)

// hi/lo split of the lower triangle (upper triangle and padding are written as zeros)
__global__ void split_lower_kernel(int Npad, int ld, long total, const float* __restrict__ X, float* __restrict__ hi,
                                   float* __restrict__ lo) {
  long e = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  long per = (long)ld * ld;
  int r = (int)((e % per) / ld), c = (int)(e % ld);
  float x = (c <= r && r < Npad) ? X[e] : 0.f;
  float h = tf32_hi(x);
  hi[e] = h;
  lo[e] = x - h;
}

// ================================================================================================= alpha via Linv
// alpha = K^-1 (y - mean) = Linv^T (Linv (y - mean)): two fully parallel matrix-vector products with the explicit
// inverse (hi + lo is the exact float32 value) instead of the serial block substitution of solve.cu.
__global__ void __launch_bounds__(256) linv_mv_kernel(int N, int Np, const float* __restrict__ hi,
                                                      const float* __restrict__ lo, const float* __restrict__ y,
                                                      const float* __restrict__ mean, float* __restrict__ t) {
  const int s = blockIdx.y, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  if (row >= Np) return;
  const long base = ((long)s * Np + row) * Np;
  const float mu = mean[s];
  float acc = 0.f;
  for (int k = lane; k <= row && k < N; k += 32) acc = fmaf(hi[base + k] + lo[base + k], y[k] - mu, acc);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) t[(long)s * Np + row] = (row < N) ? acc : 0.f;
}
// alpha[c] = sum_{r >= c} Linv[r][c] t[r]; block = 64 columns x 4 row-phases
__global__ void __launch_bounds__(256) linv_mtv_kernel(int N, int Np, int ld_alpha, const float* __restrict__ hi,
                                                       const float* __restrict__ lo, const float* __restrict__ t,
                                                       float* __restrict__ alpha) {
  __shared__ float red[4][64];
  const int s = blockIdx.y, cl = threadIdx.x & 63, ph = threadIdx.x >> 6;
  const int c = blockIdx.x * 64 + cl;
  const float* th = t + (long)s * Np;
  const long base = (long)s * Np * Np + c;
  float acc = 0.f;
  if (c < N)
    for (int r = (c & ~3) + ph; r < N; r += 4)
      if (r >= c) acc = fmaf(hi[base + (long)r * Np] + lo[base + (long)r * Np], th[r], acc);
  red[ph][cl] = acc;
  __syncthreads();
  if (ph == 0 && c < ld_alpha) alpha[(long)s * ld_alpha + c] = (c < N) ? red[0][cl] + red[1][cl] + red[2][cl] + red[3][cl] : 0.f;
}

// max |hi + lo| per sample (bits of a non-negative float order like unsigned integers)
__global__ void __launch_bounds__(256) linv_absmax_kernel(long per4, const float4* __restrict__ hi,
                                                          const float4* __restrict__ lo, unsigned* __restrict__ maxbits) {
  const int s = blockIdx.y;
  const float4* h = hi + (long)s * per4;
  const float4* l = lo + (long)s * per4;
  float m = 0.f;
  for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < per4; e += (long)gridDim.x * blockDim.x) {
    float4 a = h[e], b = l[e];
    m = fmaxf(m, fmaxf(fmaxf(fabsf(a.x + b.x), fabsf(a.y + b.y)), fmaxf(fabsf(a.z + b.z), fabsf(a.w + b.w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(&maxbits[s], __float_as_uint(m));
}

__global__ void __launch_bounds__(256) linv_pack_f16_kernel(long per4, const float4* __restrict__ hi,
                                                            const float4* __restrict__ lo,
                                                            const unsigned* __restrict__ maxbits, uint2* __restrict__ oh,
                                                            uint2* __restrict__ ol, int* __restrict__ exps) {
  const int s = blockIdx.y;
  const int eb = scale_exp(__uint_as_float(maxbits[s]));
  const float sc = ldexpf(1.f, eb);
  if (blockIdx.x == 0 && threadIdx.x == 0) exps[s] = eb;
  const long base = (long)s * per4;
  for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < per4; e += (long)gridDim.x * blockDim.x) {
    float4 a = hi[base + e], b = lo[base + e];
    __half hh[4], ll[4];
    split16((a.x + b.x) * sc, hh[0], ll[0]);
    split16((a.y + b.y) * sc, hh[1], ll[1]);
    split16((a.z + b.z) * sc, hh[2], ll[2]);
    split16((a.w + b.w) * sc, hh[3], ll[3]);
    oh[base + e] = pack4(hh);
    ol[base + e] = pack4(ll);
  }
}

// alpha^T for the rectangular fantasy-mean GEMM, fp16 (hi, lo): out[s][f][n], f padded to Fp rows, n padded to Np
// (zeros), scaled per sample by 2^fexp[s].  One block per sample finds the scale, then the elementwise pack.
__global__ void __launch_bounds__(256) alpha_absmax_kernel(int N, int F, int Npad_alpha, const float* __restrict__ alpha,
                                                           int* __restrict__ fexp) {
  __shared__ float red[8];
  const int s = blockIdx.x;
  float m = 0.f;
  for (long e = threadIdx.x; e < (long)F * N; e += blockDim.x) {
    int f = (int)(e / N), n = (int)(e % N);
    m = fmaxf(m, fabsf(alpha[((long)s * F + f) * Npad_alpha + n]));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
    fexp[s] = scale_exp(m);
  }
}
__global__ void alpha_pack_f16_kernel(int N, int Np, int F, int Fp, int Npad_alpha, long total,
                                      const float* __restrict__ alpha, const int* __restrict__ fexp,
                                      __half* __restrict__ hi, __half* __restrict__ lo) {
  long e = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  int n = (int)(e % Np);
  long sf = e / Np;
  int f = (int)(sf % Fp), s = (int)(sf / Fp);
  float x = (f < F && n < N) ? alpha[((long)s * F + f) * Npad_alpha + n] * ldexpf(1.f, fexp[s]) : 0.f;
  split16(x, hi[e], lo[e]);
}

// ================================================================================================= kxt (SIMT)
// One block = 128 candidates x all n in tiles of 128, 8x8 register micro-tiles (rows = candidates, cols = n):
// Kxt[s][c][n] * 2^ea as an fp16 (hi, lo) pair (two 8-byte stores per 4 values, 128 B contiguous per 16 threads),
// ea = scale_exp(amp2[s] (1 + 1e-6));  mu[s][c] = sum_n alpha[n] Kx[c][n] + mean.   grid = (Mc/128, S).
// 4 B written per (3D + 25) flops.
constexpr int kKD = 16;   // D chunk staged in shared memory (25 KB total)

__global__ void __launch_bounds__(256, 2) kxt_kernel(int kind, int N, int Np, int M, int c_begin, int Mc, int D,
                                                     const float* __restrict__ X, const float* __restrict__ Cc,
                                                     const float* __restrict__ inv_ls, const float* __restrict__ amp2,
                                                     const float* __restrict__ mean, const float* __restrict__ alpha,
                                                     int Npad_alpha, __half* __restrict__ khi,
                                                     __half* __restrict__ klo, float* __restrict__ mu, int ldm) {
  constexpr int T = 128, LDC = T + kPad, LDX = T + kPad;
  // scaled candidates [d][c] and MINUS the scaled observations [d][n].  The kernel is shared-memory-bandwidth bound (per
  // dimension and warp: LDS.128 wavefronts vs 64 packed math instructions), so the candidate values are stored once and
  // duplicated into the (v, v) operand of the packed instructions in registers -- 4 instead of 6 LDS.128 per dimension.
  __shared__ __align__(16) float cs[kKD][LDC];
  __shared__ __align__(16) float xs[kKD][LDX];
  __shared__ __align__(16) float red[16][T];      // epilogue scratch of the fused mean
  static_assert((LDC * sizeof(float)) % 16 == 0 && (LDX * sizeof(float)) % 16 == 0, "128-bit shared loads");
  const int s = blockIdx.y, c0 = blockIdx.x * T;  // c0 relative to the chunk
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const float* ils = inv_ls + (long)s * D;
  const float a2 = amp2[s];
  const float2 a2s = dup2(a2 * ldexpf(1.f, kx_exp(a2)));     // amp2 * 2^ea: largest entry lands in [2^14, 2^15)
  const float* al = alpha ? alpha + (long)s * Npad_alpha : nullptr;   // NULL: no mean here (predict_tc forms it from beta)
  float2 mdot[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) mdot[r] = make_float2(0.f, 0.f);

  for (int n0 = 0; n0 < Np; n0 += T) {
    float2 acc[8][4];          // rows: 8 candidates (tile_row), columns: 4 pairs of n (pair cp = n-offsets 2cp, 2cp+1)
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] = make_float2(0.f, 0.f);
    for (int d0 = 0; d0 < D; d0 += kKD) {
      __syncthreads();
      for (int e = tid; e < T * kKD; e += 256) {
        int row = e / kKD, dd = e % kKD, d = d0 + dd;
        int gc = min(c_begin + c0 + row, M - 1), n = n0 + row;
        float sc = (d < D) ? ils[d] : 0.f;
        cs[dd][row] = (d < D) ? Cc[(long)gc * D + d] * sc : 0.f;
        xs[dd][row] = (d < D && n < N) ? -X[(long)n * D + d] * sc : 0.f;
      }
      __syncthreads();
      const int dmax = min(kKD, D - d0);
      for (int dd = 0; dd < dmax; ++dd) {
        float2 b[4];
#pragma unroll
        for (int g = 0; g < 2; ++g) {
          const V4<float> u = ld4(&xs[dd][g * 64 + tx * 4]);
          b[2 * g] = make_float2(u.v[0], u.v[1]);
          b[2 * g + 1] = make_float2(u.v[2], u.v[3]);
        }
#pragma unroll
        for (int g = 0; g < 2; ++g) {
          const float4 p0 = *reinterpret_cast<const float4*>(&cs[dd][g * 64 + ty * 4]);
          const float2 a[4] = {dup2(p0.x), dup2(p0.y), dup2(p0.z), dup2(p0.w)};
#pragma unroll
          for (int rr = 0; rr < 4; ++rr)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              const float2 df = fadd2(a[rr], b[c]);
              acc[g * 4 + rr][c] = ffma2(df, df, acc[g * 4 + rr][c]);
            }
        }
      }
    }
    const bool edge = (n0 + T > N);
    float2 av[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int n = n0 + (c >> 1) * 64 + tx * 4 + (c & 1) * 2;
      av[c] = al ? make_float2((n < N) ? al[n] : 0.f, (n + 1 < N) ? al[n + 1] : 0.f) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const long ok = ((long)s * Mc + c0 + tile_row(ty, r)) * Np + n0;
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        __half2 hh[2], ll[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int c = 2 * g + q;
          float2 kk = kernel_pair_fast(kind, acc[r][c]);
          if (edge) {                                   // padded observations carry no covariance (Linv pad rows are identity)
            const int n = n0 + g * 64 + tx * 4 + q * 2;
            if (n >= N) kk.x = 0.f;
            if (n + 1 >= N) kk.y = 0.f;
          }
          mdot[r] = ffma2(av[c], kk, mdot[r]);
          const float2 v = fmul2(kk, a2s);
          hh[q] = __floats2half2_rn(v.x, v.y);
          const float2 hf = __half22float2(hh[q]);
          ll[q] = __floats2half2_rn(v.x - hf.x, v.y - hf.y);
        }
        uint2 ph, pl;
        ph.x = *reinterpret_cast<unsigned*>(&hh[0]); ph.y = *reinterpret_cast<unsigned*>(&hh[1]);
        pl.x = *reinterpret_cast<unsigned*>(&ll[0]); pl.y = *reinterpret_cast<unsigned*>(&ll[1]);
        *reinterpret_cast<uint2*>(khi + ok + g * 64 + tx * 4) = ph;
        *reinterpret_cast<uint2*>(klo + ok + g * 64 + tx * 4) = pl;
      }
    }
  }
  // mean: reduce the per-thread row partials over the 16 column-threads (fixed order -> deterministic)
  if (!al) return;
  __syncthreads();
#pragma unroll
  for (int r = 0; r < 8; ++r) red[tx][tile_row(ty, r)] = mdot[r].x + mdot[r].y;
  __syncthreads();
  if (tid < T) {
    float v = 0.f;
    for (int q = 0; q < 16; ++q) v += red[q][tid];
    int gc = c_begin + c0 + tid;
    if (gc < M) mu[(long)s * ldm + gc] = fmaf(a2, v, mean[s]);
  }
}

// ================================================================================================= wgmma kernel
namespace tc {
constexpr int BM = 128;        // candidates per tile (MMA M: two consumer warpgroups of 64 rows)
constexpr int BN = 256;        // rows of Linv per group (MMA N: 64 x 256 fp32 accumulator per warpgroup, in registers)
// Operand rows in shared memory are one 64-byte swizzle span: 16 tf32 (modes 2, 3: Cholesky update, triangular inverse)
// or 32 fp16 (modes 0, 1: predict) -- identical tile bytes, descriptors and TMA box bytes for both element types; one
// wgmma consumes 32 bytes of k (8 tf32 / 16 fp16), i.e. two MMAs per product per stage.
constexpr int BK = 16;         // k per stage, tf32 elements
constexpr int BK16 = 32;       // k per stage, fp16 elements
constexpr int STAGES = 4;      // 4 x 48 KB: a TMA refill from HBM hides behind 3 stages of MMA
constexpr int ROW_BYTES = BK * 4;                  // swizzle span = operand row in shared memory
static_assert(ROW_BYTES == 64 && BK16 * 2 == ROW_BYTES, "operand rows must be one 64B swizzle span in both element types");
constexpr int UK_BYTES = 32;                       // k bytes per wgmma (tf32: 8 x 4 B, f16: 16 x 2 B)
constexpr int A_BYTES = BM * ROW_BYTES;   // 8 KB
constexpr int B_BYTES = BN * ROW_BYTES;   // 16 KB
constexpr int STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;   // hi + lo of both operands: 48 KB
constexpr int CONSUMERS = 2;   // warpgroups 1 and 2: MMA + epilogue, rows 64 wg .. 64 wg + 63 of the tile
constexpr int THREADS = (CONSUMERS + 1) * 128;     // warpgroup 0: TMA (one thread issues, the rest give up registers)
// Register split (setmaxnreg): 384 threads leave 168 registers per thread by default, which spills the consumers'
// 128-float accumulator; the producer warpgroup drops to 40 and the consumers take 232 (128 x 40 + 256 x 232 <= 64 K).
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
static_assert(128 * PRODUCER_REGS + CONSUMERS * 128 * CONSUMER_REGS <= 65536, "register file");
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;

struct Args {
  int S, Np, Mc, ntiles, npairs, ngroups, ldp;   // Mc = candidates per chunk (multiple of 128); ldp = partial stride
  float* partial;                                 // [npairs][S][ldp]
  const float* z;                                 // optional [S][Np]: z = Linv (y - mean); then mu = mean + z . beta is reduced here
  float* mpartial;                                // [npairs][S][ldp] partial sums of z . beta
  float* dbg;                                     // optional [S][Mc][Np] dump of beta^T (tests only)
  // rectangular mode (fantasy means, OPT:609): B = alpha^T [S][ngroups*256][Np], full k range, one group per item,
  // the epilogue stores  D[c][f] + mean[s]  to mu_f[s][f][c_begin + c]  instead of reducing squares
  int F, M, c_begin, ldm;
  const float* mean;
  float* mu_f;
  // modes 0, 1: fp16 operands scaled by 2^ea (A: cross-covariance, ea = kx_exp(amp2[s])) and 2^bexp[s] (B: Linv or alpha^T)
  int f16;
  int a_evict_first;   // experiment switch (SMK_TC_A_EVICT_FIRST=1): stream the mode-0 A operand with EVICT_FIRST
  const float* amp2;
  const int* bexp;
  // mode 2 (left-looking Cholesky update, potrf_tc): C[(jb+m)-th block row][block cols jb, jb+1] -= L[.., 0:jb] L[jb.., 0:jb]^T
  // mode 3 (triangular inverse, row block K): X[K, 0:K*128] = -Lt * X[0:K*128, 0:K*128], stored as X and X^T, hi/lo
  int mode;            // 0 tri (predict), 1 rect (fantasy means), 2 Cholesky update, 3 trtri row block
  int Npad, jb, ncols; // mode 2: factor leading dimension, first block column of the pair, valid columns (128 | 256)
  float* Cmat;         // mode 2: [S][Npad][Npad] matrix being factored
  int K;               // mode 3: row block
  float *xhi, *xlo, *xthi, *xtlo;   // mode 3 outputs, each [S][Np][Np]
};

// One unit of MMA work: A rows / B rows / k range (in elements) of a single accumulator pass.
struct Item { int valid, rowA, rowB, k0, nk, s, tile, g, pr; };

__device__ __forceinline__ Item get_item(const Args& p, long w, int h) {
  Item it;
  it.valid = 0; it.rowA = it.rowB = it.k0 = it.nk = it.s = it.tile = it.g = it.pr = 0;
  const int bk = p.f16 ? BK16 : BK;
  if (p.mode <= 1) {
    it.pr = (int)(w % p.npairs);
    const long st = w / p.npairs;
    it.tile = (int)(st % p.ntiles);
    it.s = (int)(st / p.ntiles);
    it.g = (h == 0) ? it.pr : p.ngroups - 1 - it.pr;
    if (h == 1 && (p.mode == 1 || it.g == it.pr)) return it;   // rect: one group per item; middle group of an odd count
    it.nk = (p.mode == 1) ? p.Np / bk : (it.g + 1) * (BN / bk);
    it.rowA = it.s * p.Mc + it.tile * BM;
    it.rowB = (it.s * p.ngroups + it.g) * BN;
    it.valid = 1;
  } else if (p.mode == 2) {
    if (h == 1) return it;
    it.tile = (int)(w % p.ntiles);                 // block row jb + tile
    it.s = (int)(w / p.ntiles);
    it.rowA = it.s * p.Npad + (p.jb + it.tile) * BM;
    it.rowB = it.s * p.Npad + p.jb * BM;            // block rows jb and jb+1 (256 rows)
    it.nk = p.jb * BM / bk;
    it.valid = 1;
  } else {
    if (h == 1) return it;
    it.tile = (int)(w % p.ntiles);                 // column tile t of X (256 columns)
    it.s = (int)(w / p.ntiles);
    it.rowA = it.s * BM;                            // Lt: [S][128][ld]
    it.rowB = it.s * p.Np + it.tile * BN;           // X^T rows j
    it.k0 = it.tile * BN;
    it.nk = (p.K * BM - it.tile * BN) / bk;
    it.valid = 1;
  }
  return it;
}

__global__ void __launch_bounds__(THREADS, 1)
predict_tc_kernel(const __grid_constant__ CUtensorMap mAhi, const __grid_constant__ CUtensorMap mAlo,
                  const __grid_constant__ CUtensorMap mBhi, const __grid_constant__ CUtensorMap mBlo, Args p) {
  extern __shared__ unsigned char smem_raw[];
  // 1 KB alignment of the operand tiles (swizzle atoms), by offset so the pointer keeps its shared address space
  unsigned char* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(base + STAGES * STAGE_BYTES);
  uint64_t* full = bars;                 // [STAGES]  TMA bytes landed: operands ready for the MMA
  uint64_t* empty = bars + STAGES;       // [STAGES]  stage consumed by every consumer warp

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], CONSUMERS * 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const long nitems = (long)p.S * p.ntiles * (p.mode <= 1 ? p.npairs : 1);
  const int bk = p.f16 ? BK16 : BK;
  // mode 0 item order (s, tile, pair): consecutive items share (s, tile) so the pair-blocks of one candidate tile run
  // concurrently on neighbouring SMs and hit L2 for the Kxt slab.
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PRODUCER_REGS));
    if (warp == 0 && lane == 0) {
      // A (cross-covariance slab of one candidate tile) is read by the row-group-pair CTAs of that tile at different
      // times, so mode 0 keeps it under the normal policy (EVICT_FIRST sends most of those reads to HBM).  Modes 2/3
      // stream A once.  (SMK_TC_A_EVICT_FIRST=1 selects EVICT_FIRST for A/B measurements.)
      const uint64_t hintA = (p.mode == 0 && !p.a_evict_first) ? 0x1000000000000000ull : 0x12F0000000000000ull;   // EVICT_NORMAL : EVICT_FIRST
      const uint64_t hintB = 0x14F0000000000000ull;   // EVICT_LAST : the B operand is re-read by many items
      int stage = 0;
      uint32_t phase = 0;
      for (long w = blockIdx.x; w < nitems; w += gridDim.x) {
        for (int h = 0; h < 2; ++h) {
          const Item it = get_item(p, w, h);
          if (!it.valid) break;
          for (int kc = 0; kc < it.nk; ++kc) {
            mbar_wait_relaxed(&empty[stage], phase ^ 1, 64);
            unsigned char* sb = base + stage * STAGE_BYTES;
            const int kk = it.k0 + kc * bk;
            mbar_expect_tx(&full[stage], STAGE_BYTES);
            tma_load_2d(&mAhi, &full[stage], sb, kk, it.rowA, hintA);
            tma_load_2d(&mAlo, &full[stage], sb + A_BYTES, kk, it.rowA, hintA);
            tma_load_2d(&mBhi, &full[stage], sb + 2 * A_BYTES, kk, it.rowB, hintB);
            tma_load_2d(&mBlo, &full[stage], sb + 2 * A_BYTES + B_BYTES, kk, it.rowB, hintB);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ---- consumers: warpgroup 1 + wg owns accumulator rows 64 wg .. 64 wg + 63; this thread rows r0 and r0 + 8, and in
  // every 8-column block the columns cq, cq + 1 (fragment layout: tc_common.cuh)
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(CONSUMER_REGS));
  const int wg = (warp >> 2) - 1;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const uint32_t a_off = (uint32_t)wg * 64 * ROW_BYTES;
  float d[BN / 2];
  int stage = 0;
  uint32_t phase = 0;
  for (long w = blockIdx.x; w < nitems; w += gridDim.x) {
    float acc[2] = {0.f, 0.f}, accm[2] = {0.f, 0.f};
    const Item it0 = get_item(p, w, 0);
    for (int h = 0; h < 2; ++h) {
      const Item it = get_item(p, w, h);
      if (!it.valid) break;
      int prev = -1;
      for (int kc = 0; kc < it.nk; ++kc) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(base + stage * STAGE_BYTES);
        const uint64_t ahi = wgmma_desc_sw64(sa + a_off), alo = wgmma_desc_sw64(sa + A_BYTES + a_off);
        const uint64_t bhi = wgmma_desc_sw64(sa + 2 * A_BYTES), blo = wgmma_desc_sw64(sa + 2 * A_BYTES + B_BYTES);
        wgmma_fence();
        if (p.f16) {
#pragma unroll
          for (int k = 0; k < ROW_BYTES / UK_BYTES; ++k) {
            const uint64_t ko = (uint64_t)((k * UK_BYTES) >> 4);   // advance inside the swizzle atom (16 B units)
            wgmma_f16_n256(d, alo + ko, bhi + ko, (kc | k) ? 1u : 0u);   // small terms first
            wgmma_f16_n256(d, ahi + ko, blo + ko, 1u);
            wgmma_f16_n256(d, ahi + ko, bhi + ko, 1u);
          }
        } else {
#pragma unroll
          for (int k = 0; k < ROW_BYTES / UK_BYTES; ++k) {
            const uint64_t ko = (uint64_t)((k * UK_BYTES) >> 4);
            wgmma_tf32_n256(d, alo + ko, bhi + ko, (kc | k) ? 1u : 0u);
            wgmma_tf32_n256(d, ahi + ko, blo + ko, 1u);
            wgmma_tf32_n256(d, ahi + ko, bhi + ko, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<1>();                                   // the previous stage's MMAs are done: hand it back to TMA
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_hold(d);
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
      // undo the exact power-of-two operand scaling of the fp16 path
      const float scl = p.f16 ? ldexpf(1.f, -(kx_exp(p.amp2[it.s]) + p.bexp[it.s])) : 1.f;
      if (p.mode == 0) {
        // predictive mean from the same accumulator when z is given: mu - mean = alpha . kx = z . beta
        const float* zrow = p.z ? p.z + (long)it.s * p.Np + it.g * BN : nullptr;
#pragma unroll
        for (int nb = 0; nb < BN / 8; ++nb) {
          const int c = nb * 8 + cq;
          const float2 z2 = zrow ? __ldg(reinterpret_cast<const float2*>(zrow + c)) : make_float2(0.f, 0.f);
#pragma unroll
          for (int rh = 0; rh < 2; ++rh) {
            const float v0 = d[nb * 4 + rh * 2] * scl, v1 = d[nb * 4 + rh * 2 + 1] * scl;
            acc[rh] = fmaf(v0, v0, acc[rh]);
            acc[rh] = fmaf(v1, v1, acc[rh]);
            accm[rh] = fmaf(v0, z2.x, accm[rh]);
            accm[rh] = fmaf(v1, z2.y, accm[rh]);
            if (p.dbg) {
              float* o = p.dbg + ((long)it.s * p.Mc + it.tile * BM + r0 + 8 * rh) * p.Np + it.g * BN + c;
              o[0] = v0;
              o[1] = v1;
            }
          }
        }
      } else if (p.mode == 1) {
        const float mu0 = p.mean[it.s];
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
          const int gc = p.c_begin + it.tile * BM + r0 + 8 * rh;
          if (gc >= p.M) continue;
#pragma unroll
          for (int nb = 0; nb < BN / 8; ++nb)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int f = it.g * BN + nb * 8 + cq + e;
              if (f < p.F) p.mu_f[((long)it.s * p.F + f) * p.ldm + gc] = fmaf(d[nb * 4 + rh * 2 + e], scl, mu0);
            }
        }
      } else if (p.mode == 2) {
#pragma unroll
        for (int nb = 0; nb < BN / 8; ++nb) {
          const int c = nb * 8 + cq;
          if (c >= p.ncols) continue;
#pragma unroll
          for (int rh = 0; rh < 2; ++rh) {
            float2* cp = reinterpret_cast<float2*>(
                p.Cmat + ((long)it.s * p.Npad + (long)(p.jb + it.tile) * BM + r0 + 8 * rh) * p.Npad + (long)p.jb * BM + c);
            float2 v = *cp;
            v.x -= d[nb * 4 + rh * 2];
            v.y -= d[nb * 4 + rh * 2 + 1];
            *cp = v;
          }
        }
      } else {
#pragma unroll
        for (int nb = 0; nb < BN / 8; ++nb) {
          const int jcol = it.tile * BN + nb * 8 + cq;      // first of this thread's two columns of X
          if (jcol >= p.K * BM) continue;
#pragma unroll
          for (int rh = 0; rh < 2; ++rh) {
            const int row = p.K * BM + r0 + 8 * rh;
            const long xr = ((long)it.s * p.Np + row) * p.Np + jcol;
            float hh[2], ll[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float v = -d[nb * 4 + rh * 2 + e];
              hh[e] = tf32_rn(v);
              ll[e] = v - hh[e];
              const long xt = ((long)it.s * p.Np + jcol + e) * p.Np + row;   // transposed copy
              p.xthi[xt] = hh[e];
              p.xtlo[xt] = tf32_lo(v, hh[e]);
            }
            *reinterpret_cast<float2*>(p.xhi + xr) = make_float2(hh[0], hh[1]);
            *reinterpret_cast<float2*>(p.xlo + xr) = make_float2(ll[0], ll[1]);
          }
        }
      }
    }
    if (p.mode == 0) {             // row sums over the 4 lanes that share a row, fixed order
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        float a = acc[rh], m = accm[rh];
        a += __shfl_xor_sync(0xffffffffu, a, 1);
        a += __shfl_xor_sync(0xffffffffu, a, 2);
        m += __shfl_xor_sync(0xffffffffu, m, 1);
        m += __shfl_xor_sync(0xffffffffu, m, 2);
        if ((lane & 3) == 0) {
          const long o = ((long)it0.pr * p.S + it0.s) * p.ldp + it0.tile * BM + r0 + 8 * rh;
          p.partial[o] = a;
          if (p.z) p.mpartial[o] = m;
        }
      }
    }
  }
}

// var = amp2 (1 + 1e-6) - sum_p partial[p]; with the tensor-core generator also mu = amp2 * sum_j mu_partial[j] + mean
__global__ void finish_var_kernel(int M, int c_begin, int Mc, int S, int npairs, int ldp, const float* __restrict__ partial,
                                  const float* __restrict__ amp2, float* __restrict__ var, int ldm, int nmp,
                                  const float* __restrict__ mu_partial, const float* __restrict__ mean,
                                  float* __restrict__ mu, const float* __restrict__ mpartial) {
  int c = blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y;
  if (c >= Mc || c_begin + c >= M) return;
  float t = 0.f;
  for (int pr = 0; pr < npairs; ++pr) t += partial[((long)pr * S + s) * ldp + c];
  var[(long)s * ldm + c_begin + c] = amp2[s] * 1.000001f - t;
  if (mpartial) {                               // mean reduced by the GEMM epilogue: mu = mean + z . beta
    float m = 0.f;
    for (int pr = 0; pr < npairs; ++pr) m += mpartial[((long)pr * S + s) * ldp + c];
    mu[(long)s * ldm + c_begin + c] = mean[s] + m;
    return;
  }
  if (nmp > 0) {
    float m = 0.f;
    for (int j = 0; j < nmp; ++j) m += mu_partial[((long)j * S + s) * ldp + c];
    mu[(long)s * ldm + c_begin + c] = fmaf(amp2[s], m, mean[s]);
  }
}

}  // namespace tc
__global__ void kxt_mu_finish_kernel(int M, int Mc, int S, int nmp, const float* __restrict__ mu_partial,
                                     const float* __restrict__ amp2, const float* __restrict__ mean,
                                     float* __restrict__ mu, int ldm) {
  int c = blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y;
  if (c >= M) return;
  float m = 0.f;
  for (int j = 0; j < nmp; ++j) m += mu_partial[((long)j * S + s) * Mc + c];
  mu[(long)s * ldm + c] = fmaf(amp2[s], m, mean[s]);
}
namespace tc {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess) fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 2-D row-major float matrix [rows][cols] (cols contiguous), box = (BK cols) x (box_rows rows), swizzle = row bytes
static int make_map(CUtensorMap* m, const float* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  EncodeTiledFn f = encode_fn();
  if (!f) return 1;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * sizeof(float)};
  cuuint32_t box[2] = {(cuuint32_t)BK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = f(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : 2;
}
// same for an fp16 matrix: box = (BK16 cols) x (box_rows rows) -- the same 64-byte rows
static int make_map_h(CUtensorMap* m, const __half* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  EncodeTiledFn f = encode_fn();
  if (!f) return 1;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * sizeof(__half)};
  cuuint32_t box[2] = {(cuuint32_t)BK16, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = f(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(ptr), dims, strides, box, estr,
                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : 2;
}
}  // namespace tc

int num_sms();
// tensor-core cross-covariance generator (kxt_tc.cu)
bool kxt_tc_supported(int D, int S);
bool kxt_tc_preferred(int D, int S);
int kxt_tc_ngroups(int Np);
size_t kxt_tc_workspace_bytes(int Np, int Mc, int S, int M, int D);
int kxt_tc_prepare(void* ws, int N, int Np, int M, int Mc, int D, int S, const float* X, const float* Cc, cudaStream_t st);
int kxt_tc(void* ws, int kind, int N, int Np, int M, int c_begin, int Mc, int mc_used, int D, int S, const float* inv_ls,
           const float* amp2, const float* alpha, int Npad_alpha, __half* khi, __half* klo, cudaStream_t st);
float* kxt_tc_mu_partial(void* ws, int Np, int Mc, int S, int M, int D);
static const int kKxtWsD = 32;     // the generator workspace is sized for its largest supported dimension

// ---------------------------------------------------------------------------------------------------- host side
int tc_np(int N) { return ((N + tc::BN - 1) / tc::BN) * tc::BN; }

size_t trtri_workspace_bytes(int Np, int S) { return (size_t)S * Np * Np * sizeof(float); }

int trtri_split(int Npad, int Np, int S, const float* L, const float* winv, float* linv_hi, float* linv_lo,
                void* workspace, size_t workspace_bytes, cudaStream_t st) {
  if (Npad <= 0 || Npad % kNpadMult) return -1;
  if (Np < Npad || Np % tc::BN) return -2;
  if (S <= 0) return -3;
  if (!L || !winv || !linv_hi || !linv_lo) return -4;
  if (!workspace || workspace_bytes < trtri_workspace_bytes(Np, S)) return -8;
  float* X = reinterpret_cast<float*>(workspace);
  const size_t dsm = sizeof(TileSmem<float>) + sizeof(float) * 128 * (128 + kPad);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(trtri_finalize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsm);
    attr = true;
  }
  const int nblk = Npad / 128;
  timing_begin("trtri_kernel", st);
  for (int K = 0; K < nblk; ++K) {
    trtri_finalize_kernel<<<dim3(K + 1, S), 256, dsm, st>>>(Npad, Np, K, winv, X);
    if (K + 1 < nblk) trtri_update_kernel<<<dim3(nblk - K - 1, K + 1, S), 256, 0, st>>>(Npad, Np, K, L, X);
  }
  timing_end(st);
  count_launch(2 * nblk - 1);
  const long total = (long)S * Np * Np;
  split_lower_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(Npad, Np, total, X, linv_hi, linv_lo);
  count_launch(1);
  return check_launch("trtri_split");
}

// ---------------------------------------------------------------------------------- tensor-core Cholesky update
static void tc_args_init(tc::Args& a) {
  memset(&a, 0, sizeof(a));
}

int tc_chol_update(int Npad, int S, int jb, int ncols, float* A, const float* lhi, const float* llo, cudaStream_t st) {
  CUtensorMap mAhi, mAlo, mBhi, mBlo;
  if (tc::make_map(&mAhi, lhi, (uint64_t)S * Npad, Npad, tc::BM) || tc::make_map(&mAlo, llo, (uint64_t)S * Npad, Npad, tc::BM) ||
      tc::make_map(&mBhi, lhi, (uint64_t)S * Npad, Npad, tc::BN) || tc::make_map(&mBlo, llo, (uint64_t)S * Npad, Npad, tc::BN))
    return 1999;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(tc::predict_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_BYTES);
    attr = true;
  }
  tc::Args a;
  tc_args_init(a);
  a.mode = 2; a.S = S; a.Npad = Npad; a.jb = jb; a.ncols = ncols; a.Cmat = A;
  a.ntiles = Npad / tc::BM - jb; a.npairs = 1; a.ngroups = 1;
  long nitems = (long)S * a.ntiles;
  int grid = (int)std::min<long>(nitems, num_sms());
  timing_begin("tc_chol_update", st);
  tc::predict_tc_kernel<<<grid, tc::THREADS, tc::SMEM_BYTES, st>>>(mAhi, mAlo, mBhi, mBlo, a);
  timing_end(st);
  count_launch();
  return check_launch("tc_chol_update");
}

// ---------------------------------------------------------------------------------- tensor-core triangular inverse
// Row block K of X = L^-1:  X_KK = W_KK;  X[K, 0:K*128] = -(W_KK L[K, 0:K*128]) X[0:K*128, 0:K*128].
// Lt = W_KK * L[K, 0:K*128] (SIMT, 128 x K*128), written as tf32 hi/lo [S][128][ld]
__global__ void __launch_bounds__(256, 2) trtri_lt_kernel(int Npad, int K, const float* __restrict__ L,
                                                           const float* __restrict__ winv, float* __restrict__ lthi,
                                                           float* __restrict__ ltlo) {
  using C = Cfg<float>;
  constexpr int NB = C::NB, TM = C::TM, TN = C::TN;
  __shared__ TileSmem<float> sm;
  const int nblk = Npad / NB, J = blockIdx.x, s = blockIdx.y;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  const float* W = winv + ((long)s * nblk + K) * NB * NB;
  const float* Lk = L + (long)s * Npad * Npad + (long)K * NB * Npad + (long)J * NB;   // B(col c, k) = Lk[k*Npad + c]
  float acc[TM][TN];
#pragma unroll
  for (int r = 0; r < TM; ++r)
#pragma unroll
    for (int c = 0; c < TN; ++c) acc[r][c] = 0.f;
  TileGemm<float, Lay::KContig, Lay::MContig, false>::run(acc, W, NB, Lk, Npad, NB, sm);
  const long off = (long)s * NB * Npad + (long)J * NB;
#pragma unroll
  for (int r = 0; r < TM; ++r)
#pragma unroll
    for (int g = 0; g < TN / 4; ++g) {
      V4<float> h, l;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float x = acc[r][g * 4 + e];
        h.v[e] = tf32_hi(x);
        l.v[e] = tf32_lo(x, h.v[e]);
      }
      const long o = off + (long)tile_row(ty, r) * Npad + g * 64 + tx * 4;
      st4(lthi + o, h);
      st4(ltlo + o, l);
    }
}

// X_KK = W_KK and its transpose into X / X^T (hi, lo)
__global__ void trtri_diag_store_kernel(int Npad, int Np, int K, const float* __restrict__ winv, float* __restrict__ xhi,
                                        float* __restrict__ xlo, float* __restrict__ xthi, float* __restrict__ xtlo) {
  constexpr int NB = 128;
  const int s = blockIdx.y, nblk = Npad / NB;
  const float* W = winv + ((long)s * nblk + K) * NB * NB;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < NB * NB; e += gridDim.x * blockDim.x) {
    int i = e / NB, k = e % NB;
    float x = W[e], h = tf32_hi(x), l = x - h;
    long o = ((long)s * Np + (long)K * NB + i) * Np + (long)K * NB + k;
    long ot = ((long)s * Np + (long)K * NB + k) * Np + (long)K * NB + i;
    xhi[o] = h; xlo[o] = l; xthi[ot] = h; xtlo[ot] = tf32_lo(x, h);
  }
}

size_t trtri_tc_workspace_bytes(int Npad, int Np, int S) {
  return (2 * (size_t)S * Np * Np + 2 * (size_t)S * 128 * Npad) * sizeof(float);     // X^T hi|lo, Lt hi|lo
}

int potrf_lower_batched_tc(int, int, float*, float*, int*, float*, float*, cudaStream_t, cudaEvent_t*);
void potrf_winv_block(int, int, int, const float*, float*, cudaStream_t);

// blk_done == NULL: everything on st, winv complete on entry (the two-call sequence).  Otherwise row block K starts when
// blk_done[K] has fired on the factorisation's stream, and forms W_KK itself.
static int trtri_tc_run(int Npad, int Np, int S, const float* L, float* winv, float* linv_hi, float* linv_lo,
                        void* workspace, size_t workspace_bytes, cudaStream_t st, cudaEvent_t* blk_done) {
  if (Npad <= 0 || Npad % kNpadMult) return -1;
  if (Np < Npad || Np % tc::BN) return -2;
  if (S <= 0) return -3;
  if (!L || !winv || !linv_hi || !linv_lo) return -4;
  if (!workspace || workspace_bytes < trtri_tc_workspace_bytes(Npad, Np, S)) return -8;
  float* xthi = reinterpret_cast<float*>(workspace);
  float* xtlo = xthi + (size_t)S * Np * Np;
  float* lthi = xtlo + (size_t)S * Np * Np;
  float* ltlo = lthi + (size_t)S * 128 * Npad;
  const size_t xb = (size_t)S * Np * Np * sizeof(float);
  cudaMemsetAsync(linv_hi, 0, xb, st);
  cudaMemsetAsync(linv_lo, 0, xb, st);
  cudaMemsetAsync(xthi, 0, 2 * xb, st);
  CUtensorMap mAhi, mAlo, mBhi, mBlo;
  if (tc::make_map(&mAhi, lthi, (uint64_t)S * 128, Npad, tc::BM) || tc::make_map(&mAlo, ltlo, (uint64_t)S * 128, Npad, tc::BM) ||
      tc::make_map(&mBhi, xthi, (uint64_t)S * Np, Np, tc::BN) || tc::make_map(&mBlo, xtlo, (uint64_t)S * Np, Np, tc::BN))
    return 1999;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(tc::predict_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_BYTES);
    attr = true;
  }
  const int nblk = Npad / 128;
  timing_begin("trtri_kernel", st);
  for (int K = 0; K < nblk; ++K) {
    if (blk_done) {
      cudaStreamWaitEvent(st, blk_done[K], 0);
      potrf_winv_block(Npad, S, K, L, winv, st);
    }
    trtri_diag_store_kernel<<<dim3(8, S), 256, 0, st>>>(Npad, Np, K, winv, linv_hi, linv_lo, xthi, xtlo);
    count_launch();
    if (K == 0) continue;
    trtri_lt_kernel<<<dim3(K, S), 256, 0, st>>>(Npad, K, L, winv, lthi, ltlo);
    tc::Args a;
    tc_args_init(a);
    a.mode = 3; a.S = S; a.Np = Np; a.Npad = Npad; a.K = K;
    a.ntiles = (K * 128 + tc::BN - 1) / tc::BN; a.npairs = 1; a.ngroups = 1;
    a.xhi = linv_hi; a.xlo = linv_lo; a.xthi = xthi; a.xtlo = xtlo;
    long nitems = (long)S * a.ntiles;
    int grid = (int)std::min<long>(nitems, num_sms());
    tc::predict_tc_kernel<<<grid, tc::THREADS, tc::SMEM_BYTES, st>>>(mAhi, mAlo, mBhi, mBlo, a);
    count_launch(2);
  }
  timing_end(st);
  return check_launch("trtri_split_tc");
}

int trtri_split_tc(int Npad, int Np, int S, const float* L, const float* winv, float* linv_hi, float* linv_lo,
                   void* workspace, size_t workspace_bytes, cudaStream_t st) {
  return trtri_tc_run(Npad, Np, S, L, const_cast<float*>(winv), linv_hi, linv_lo, workspace, workspace_bytes, st, nullptr);
}

// Factor and invert in one call, pipelined: row block K of the inverse needs W_KK, row block K of L and the rows of the
// inverse above it -- all final as soon as block column K of the factorisation is.  So the inversion runs ONE STEP BEHIND
// the factorisation on a second stream instead of after it.  Both are chains of small dependent launches (32 block steps at
// N = 4096); with few hyper-samples per GPU (the 8-GPU shape: 5) neither fills the machine and the two chains simply
// overlap.  With a full batch (40) each is throughput-bound and the overlap fills the bubbles of the other's spine.
int potrf_trtri_tc(int Npad, int Np, int S, float* A, float* winv, int* info, float* lhi, float* llo, float* linv_hi,
                   float* linv_lo, void* tws, size_t tws_bytes, cudaStream_t st) {
  if (Npad <= 0 || Npad % kNpadMult) return -1;
  static cudaStream_t aux = nullptr;
  static cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  static std::vector<cudaEvent_t> blk;
  if (!aux) {
    cudaStreamCreateWithFlags(&aux, cudaStreamNonBlocking);
    cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ev_out, cudaEventDisableTiming);
  }
  const int nblk = Npad / 128;
  while ((int)blk.size() < nblk) {
    cudaEvent_t e;
    cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    blk.push_back(e);
  }
  cudaEventRecord(ev_in, st);                      // the buffers are free / the covariance is built
  cudaStreamWaitEvent(aux, ev_in, 0);
  int rc = potrf_lower_batched_tc(Npad, S, A, winv, info, lhi, llo, st, blk.data());
  if (rc) return rc;
  rc = trtri_tc_run(Npad, Np, S, A, winv, linv_hi, linv_lo, tws, tws_bytes, aux, blk.data());
  cudaEventRecord(ev_out, aux);
  cudaStreamWaitEvent(st, ev_out, 0);
  return rc;
}

// fp16 operand copy of the explicit inverse for the predict GEMM: per-sample power-of-two scale + (hi, lo) split.
// exps: [2*S] ints -- [0, S) receives the scale exponents, [S, 2S) is scratch (max |entry| bits).
int linv_pack_f16(int Np, int S, const float* linv_hi, const float* linv_lo, __half* out_hi, __half* out_lo, int* exps,
                  cudaStream_t st) {
  if (Np <= 0 || Np % tc::BN) return -1;
  if (S <= 0) return -2;
  if (!linv_hi || !linv_lo || !out_hi || !out_lo || !exps) return -3;
  unsigned* maxbits = reinterpret_cast<unsigned*>(exps + S);
  cudaMemsetAsync(maxbits, 0, sizeof(unsigned) * S, st);
  const long per4 = (long)Np * Np / 4;
  const int gx = (int)std::min<long>((per4 + 255) / 256, 4L * num_sms());
  timing_begin("linv_pack_f16", st);
  linv_absmax_kernel<<<dim3(gx, S), 256, 0, st>>>(per4, reinterpret_cast<const float4*>(linv_hi),
                                                  reinterpret_cast<const float4*>(linv_lo), maxbits);
  linv_pack_f16_kernel<<<dim3(gx, S), 256, 0, st>>>(per4, reinterpret_cast<const float4*>(linv_hi),
                                                    reinterpret_cast<const float4*>(linv_lo), maxbits,
                                                    reinterpret_cast<uint2*>(out_hi), reinterpret_cast<uint2*>(out_lo), exps);
  timing_end(st);
  count_launch(2);
  return check_launch("linv_pack_f16");
}

int linv_alpha(int N, int Np, int S, const float* linv_hi, const float* linv_lo, const float* y, const float* mean,
               float* alpha, int ld_alpha, float* tmp, cudaStream_t st) {
  if (N <= 0 || Np < N) return -1;
  if (S <= 0) return -3;
  if (!linv_hi || !linv_lo || !y || !mean || !alpha || !tmp) return -4;
  if (ld_alpha < N) return -9;
  linv_mv_kernel<<<dim3((Np + 7) / 8, S), 256, 0, st>>>(N, Np, linv_hi, linv_lo, y, mean, tmp);
  linv_mtv_kernel<<<dim3((ld_alpha + 63) / 64, S), 256, 0, st>>>(N, Np, ld_alpha, linv_hi, linv_lo, tmp, alpha);
  count_launch(2);
  return check_launch("linv_alpha");
}

// kxt(i+1) / MMA(i) overlap on two streams: both kernels share the card's power budget, so running them together lowers
// the clock for both and saves nothing on a power-capped card; opt-in (SMK_TC_OVERLAP=1), not measured on H100.
static bool tc_overlap_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("SMK_TC_OVERLAP"); v = (e && e[0] == '1') ? 1 : 0; }
  return v == 1;
}
// workspace: Kxt hi (fp16) | Kxt lo (fp16) | partial | alpha^T hi | alpha^T lo | fantasy scale exponents
static size_t tc_chunk_cands(int Np, int M, int S, size_t budget) {
  size_t per_cand = (size_t)S * Np * 2 * sizeof(__half);
  size_t mpad = ((size_t)M + 127) / 128 * 128;
  size_t mc = budget / per_cand;
  if (mc >= mpad) return mpad;                  // everything in one chunk: single buffer
  if (tc_overlap_enabled()) mc = (budget / 2) / per_cand;   // two half-size buffers (kxt of chunk i+1 overlaps MMA of i)
  mc = mc / 128 * 128;
  if (mc < 128) mc = 128;
  return mc;
}
static int tc_nbuf(int Np, int M, int S, size_t budget) {
  size_t mpad = ((size_t)M + 127) / 128 * 128;
  if (!tc_overlap_enabled()) return 1;
  return tc_chunk_cands(Np, M, S, budget) >= mpad ? 1 : 2;
}
// Operand-chunk budget: 20 GB of cross-covariance per candidate chunk.  SMK_TC_BUDGET_MB overrides it (tests use a
// small value to push a few thousand candidates through the multi-chunk + ragged-tail path of the headline shape).
static size_t tc_budget() {
  const char* e = getenv("SMK_TC_BUDGET_MB");
  if (e && e[0]) { long mb = atol(e); if (mb > 0) return (size_t)mb << 20; }
  return (size_t)20 << 30;
}
#define kTcBudget (tc_budget())

static int fant_rows(int F) { return F > 1 ? ((F + tc::BN - 1) / tc::BN) * tc::BN : 0; }

size_t predict_tc_workspace_bytes(int Np, int M, int S, int F) {
  size_t mc = tc_chunk_cands(Np, M, S, kTcBudget);
  int ngroups = Np / tc::BN, npairs = (ngroups + 1) / 2, nbuf = tc_nbuf(Np, M, S, kTcBudget);
  return (size_t)nbuf * S * mc * Np * 2 * sizeof(__half) + 2 * (size_t)npairs * S * mc * sizeof(float) +
         2 * (size_t)S * fant_rows(F) * Np * sizeof(__half) + (size_t)S * sizeof(int) + 1024 +
         kxt_tc_workspace_bytes(Np, (int)mc, S, M, kKxtWsD);
}

// Generator only (one chunk, Mc = ceil128(M)): khi/klo [S][Mc][Np] halves, mu [S][ldm].  impl: 0 = packed SIMT kernel,
// 1 = tensor-core kernel.  Used by the tests to compare the two implementations element by element.
size_t kxt_pack_workspace_bytes(int Np, int M, int S) {
  return kxt_tc_workspace_bytes(Np, ((M + 127) / 128) * 128, S, M, kKxtWsD) + 256;
}
int kxt_pack(int impl, int kind, int N, int Np, int M, int D, int S, const float* X, const float* Cc, const float* inv_ls,
             const float* amp2, const float* mean, const float* alpha, int Npad_alpha, __half* khi, __half* klo,
             float* mu, int ldm, void* workspace, size_t workspace_bytes, cudaStream_t st) {
  if (kind < 0 || kind > 3) return -2;
  if (N <= 0 || Np < N || Np % tc::BN) return -4;
  if (M <= 0 || D <= 0 || S <= 0) return -5;
  if (!X || !Cc || !inv_ls || !amp2 || !mean || !alpha || !khi || !klo || !mu) return -8;
  if (ldm < M) return -18;
  const int Mc = ((M + 127) / 128) * 128;
  if (impl == 0) {
    kxt_kernel<<<dim3(Mc / 128, S), 256, 0, st>>>(kind, N, Np, M, 0, Mc, D, X, Cc, inv_ls, amp2, mean, alpha, Npad_alpha,
                                                  khi, klo, mu, ldm);
    count_launch();
    return check_launch("kxt_pack");
  }
  if (!kxt_tc_supported(D, S)) return -1;
  if (!workspace || workspace_bytes < kxt_pack_workspace_bytes(Np, M, S)) return -20;
  const int nmp = kxt_tc_ngroups(Np);
  int rc = kxt_tc_prepare(workspace, N, Np, M, Mc, D, S, X, Cc, st);
  if (rc) return rc;
  rc = kxt_tc(workspace, kind, N, Np, M, 0, Mc, Mc, D, S, inv_ls, amp2, alpha, Npad_alpha, khi, klo, st);
  if (rc) return rc;
  float* mu_partial = kxt_tc_mu_partial(workspace, Np, Mc, S, M, D);
  kxt_mu_finish_kernel<<<dim3((Mc + 255) / 256, S), 256, 0, st>>>(M, Mc, S, nmp, mu_partial, amp2, mean, mu, ldm);
  count_launch();
  return check_launch("kxt_pack");
}

// Chunk 0 of the cross-covariance generated AHEAD of the GEMM, on an internal stream forked from `st`: the generator needs
// the observations, the candidates and the kernel hyper-parameters only (the mean comes out of the GEMM epilogue as z . beta),
// so it runs while the caller's stream factors and inverts K.  predict_tc(..., pregenerated = 1) with the same workspace
// picks the chunk up.  One outstanding pre-generation per process.
struct PregenState {
  bool valid = false;
  void* ws = nullptr;
  int M = 0, S = 0, Np = 0, N = 0;
  cudaEvent_t done = nullptr, fork = nullptr;
  cudaStream_t stream = nullptr;
};
static PregenState g_pregen;

int predict_tc_pregen(int kind, int N, int Np, int M, int D, int S, const float* X, const float* Cc, const float* inv_ls,
                      const float* amp2, void* workspace, size_t workspace_bytes, int F, cudaStream_t st) {
  if (kind < 0 || kind > 3) return -1;
  if (N <= 0 || Np < N || Np % tc::BN) return -3;
  if (M <= 0 || D <= 0 || S <= 0) return -4;
  if (!X || !Cc || !inv_ls || !amp2) return -7;
  const bool fant = F > 1;
  if (!workspace || workspace_bytes < predict_tc_workspace_bytes(Np, M, S, fant ? F : 1)) return -20;
  if (tc_nbuf(Np, M, S, kTcBudget) != 1) return -22;
  const int Mc = (int)tc_chunk_cands(Np, M, S, kTcBudget);
  const int ngroups = Np / tc::BN, npairs = (ngroups + 1) / 2;
  const size_t kelems = (size_t)S * Mc * Np;
  __half* kbase = reinterpret_cast<__half*>(workspace);
  float* partial = reinterpret_cast<float*>(kbase + 2 * kelems);
  const int Fp = fant ? fant_rows(F) : 0;
  __half* ahi = reinterpret_cast<__half*>(partial + 2 * (size_t)npairs * S * Mc);
  int* fexp = reinterpret_cast<int*>(ahi + 2 * (size_t)S * Fp * Np);
  void* kws = reinterpret_cast<void*>(fexp + S);
  static int gen_env = -1;
  if (gen_env < 0) { const char* e = getenv("SMK_KXT_IMPL"); gen_env = (e && !strcmp(e, "tc")) ? 1 : 0; }
  const bool gen_tc = gen_env == 1 && kxt_tc_preferred(D, S);
  PregenState& g = g_pregen;
  if (!g.stream) {
    cudaStreamCreateWithFlags(&g.stream, cudaStreamNonBlocking);
    cudaEventCreateWithFlags(&g.done, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&g.fork, cudaEventDisableTiming);
  }
  cudaEventRecord(g.fork, st);                       // inputs uploaded, the workspace's previous users done
  cudaStreamWaitEvent(g.stream, g.fork, 0);
  const int mc_used = min(Mc, (M + 127) / 128 * 128);
  timing_begin("kxt_kernel", g.stream);
  if (gen_tc) {
    int rc = kxt_tc_prepare(kws, N, Np, M, Mc, D, S, X, Cc, g.stream);
    if (rc) return rc;
    rc = kxt_tc(kws, kind, N, Np, M, 0, Mc, mc_used, D, S, inv_ls, amp2, nullptr, 0, kbase, kbase + kelems, g.stream);
    if (rc) return rc;
  } else {
    kxt_kernel<<<dim3(mc_used / 128, S), 256, 0, g.stream>>>(kind, N, Np, M, 0, Mc, D, X, Cc, inv_ls, amp2, nullptr, nullptr, 0,
                                                             kbase, kbase + kelems, nullptr, 0);
    count_launch();
  }
  timing_end(g.stream);
  cudaEventRecord(g.done, g.stream);
  g.valid = true; g.ws = workspace; g.M = M; g.S = S; g.Np = Np; g.N = N;
  return check_launch("predict_tc_pregen");
}

int predict_tc(int kind, int N, int Np, int M, int D, int S, const float* X, const float* Cc, const float* inv_ls,
               const float* amp2, const float* mean, const __half* linv_hi, const __half* linv_lo, const int* linv_exp,
               const float* alpha, int Npad_alpha, float* mu, float* var, int ldm, void* workspace,
               size_t workspace_bytes, float* dbg, int F, const float* alpha_f, float* mu_f, const float* z,
               int pregenerated, cudaStream_t st) {
  if (kind < 0 || kind > 3) return -1;
  if (N <= 0) return -2;
  if (Np < N || Np % tc::BN) return -3;
  if (M <= 0) return -4;
  if (D <= 0) return -5;
  if (S <= 0) return -6;
  if (!X || !Cc || !inv_ls || !amp2 || !mean || !linv_hi || !linv_lo || !linv_exp || !alpha || !mu || !var) return -7;
  if (ldm < M) return -19;
  const bool fant = (F > 1 && alpha_f && mu_f);
  if (!workspace || workspace_bytes < predict_tc_workspace_bytes(Np, M, S, fant ? F : 1)) return -20;
  const int Mc = (int)tc_chunk_cands(Np, M, S, kTcBudget);
  const int nbuf = tc_nbuf(Np, M, S, kTcBudget);
  const int ngroups = Np / tc::BN, npairs = (ngroups + 1) / 2;
  const size_t kelems = (size_t)S * Mc * Np;                               // one Kxt buffer, elements per half-array
  __half* kbase = reinterpret_cast<__half*>(workspace);                    // [nbuf]{hi [S][Mc][Np] | lo [S][Mc][Np]}
  float* partial = reinterpret_cast<float*>(kbase + (size_t)nbuf * 2 * kelems);
  float* mpartial = partial + (size_t)npairs * S * Mc;                           // z . beta partial sums (when z is given)
  const int Fp = fant ? fant_rows(F) : 0;
  __half* ahi = reinterpret_cast<__half*>(mpartial + (size_t)npairs * S * Mc);  // alpha^T hi | lo  [S][Fp][Np]
  __half* alo = ahi + (size_t)S * Fp * Np;
  int* fexp = reinterpret_cast<int*>(alo + (size_t)S * Fp * Np);
  // generator: the SIMT kernel above; SMK_KXT_IMPL=tc selects the tensor-core kernel of kxt_tc.cu (contraction over
  // dimensions on wgmma) where it applies.  On an H100 SXM the SIMT kernel is the faster of the two at the headline
  // (80 against 95 ms per step, S = 40), and the tensor-core one only loses ground with fewer samples.
  static int gen_env = -1;
  if (gen_env < 0) { const char* e = getenv("SMK_KXT_IMPL"); gen_env = (e && !strcmp(e, "tc")) ? 1 : 0; }
  const bool gen_tc = gen_env == 1 && kxt_tc_preferred(D, S) && nbuf == 1;
  const int nmp = (gen_tc && !z) ? kxt_tc_ngroups(Np) : 0;
  void* kws = reinterpret_cast<void*>(fexp + S);
  float* mu_partial = gen_tc ? kxt_tc_mu_partial(kws, Np, Mc, S, M, D) : nullptr;
  const float* gen_alpha = z ? nullptr : alpha;     // with z the mean comes out of the GEMM epilogue: the generator needs no alpha
  // chunk 0 may have been generated ahead of time (predict_tc_pregen: while the factorisation was running)
  const bool pre = pregenerated && z && nbuf == 1 && g_pregen.valid && g_pregen.ws == workspace && g_pregen.M == M &&
                   g_pregen.S == S && g_pregen.Np == Np && g_pregen.N == N;
  if (pregenerated && !pre) return -21;
  if (g_pregen.valid && g_pregen.ws == workspace) {   // picked up below -- or abandoned by the caller: either way ordered behind it
    cudaStreamWaitEvent(st, g_pregen.done, 0);
    g_pregen.valid = false;
  }
  if (!pre && gen_tc) {
    int rc = kxt_tc_prepare(kws, N, Np, M, Mc, D, S, X, Cc, st);
    if (rc) return rc;
  }
  CUtensorMap mFhi, mFlo;
  if (fant) {
    const long total = (long)S * Fp * Np;
    alpha_absmax_kernel<<<S, 256, 0, st>>>(N, F, Npad_alpha, alpha_f, fexp);
    alpha_pack_f16_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(N, Np, F, Fp, Npad_alpha, total, alpha_f, fexp,
                                                                           ahi, alo);
    count_launch(2);
    if (tc::make_map_h(&mFhi, ahi, (uint64_t)S * Fp, Np, tc::BN) || tc::make_map_h(&mFlo, alo, (uint64_t)S * Fp, Np, tc::BN))
      return 1999;
  }

  CUtensorMap mAhi[2], mAlo[2], mBhi, mBlo;
  for (int b = 0; b < nbuf; ++b) {
    __half* kh = kbase + (size_t)b * 2 * kelems;
    if (tc::make_map_h(&mAhi[b], kh, (uint64_t)S * Mc, Np, tc::BM) ||
        tc::make_map_h(&mAlo[b], kh + kelems, (uint64_t)S * Mc, Np, tc::BM))
      return 1999;                                                              // cuTensorMapEncodeTiled failed
  }
  if (tc::make_map_h(&mBhi, linv_hi, (uint64_t)S * Np, Np, tc::BN) || tc::make_map_h(&mBlo, linv_lo, (uint64_t)S * Np, Np, tc::BN))
    return 1999;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(tc::predict_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, tc::SMEM_BYTES);
    attr = true;
  }
  // The cross-covariance of chunk i+1 is generated on an auxiliary stream while the MMA kernel consumes chunk i
  // (two Kxt buffers; event fork/join keeps everything ordered with respect to the caller's stream).
  static cudaStream_t aux = nullptr;
  static cudaEvent_t ev_fork = nullptr, ev_kxt[2] = {nullptr, nullptr}, ev_mma[2] = {nullptr, nullptr};
  if (!aux) {
    cudaStreamCreateWithFlags(&aux, cudaStreamNonBlocking);
    cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming);
    for (int i = 0; i < 2; ++i) {
      cudaEventCreateWithFlags(&ev_kxt[i], cudaEventDisableTiming);
      cudaEventCreateWithFlags(&ev_mma[i], cudaEventDisableTiming);
    }
  }
  const bool overlap = (nbuf == 2);
  cudaStream_t kst = overlap ? aux : st;
  if (overlap) {
    cudaEventRecord(ev_fork, st);
    cudaStreamWaitEvent(aux, ev_fork, 0);
  }
  int ci = 0;
  for (int c_begin = 0; c_begin < M; c_begin += Mc, ++ci) {
    const int b = overlap ? (ci & 1) : 0;
    __half* kh = kbase + (size_t)b * 2 * kelems;
    const int mc_used = min(Mc, ((M - c_begin) + 127) / 128 * 128);
    if (overlap && ci >= 2) cudaStreamWaitEvent(aux, ev_mma[b], 0);      // buffer b is free again
    if (!(pre && ci == 0)) {
      timing_begin("kxt_kernel", kst);
      if (gen_tc) {
        int rc = kxt_tc(kws, kind, N, Np, M, c_begin, Mc, mc_used, D, S, inv_ls, amp2, gen_alpha, Npad_alpha, kh, kh + kelems, kst);
        if (rc) return rc;
      } else {
        kxt_kernel<<<dim3(mc_used / 128, S), 256, 0, kst>>>(kind, N, Np, M, c_begin, Mc, D, X, Cc, inv_ls, amp2, mean,
                                                            gen_alpha, Npad_alpha, kh, kh + kelems, mu, ldm);
      }
      timing_end(kst);
    }
    if (overlap) {
      cudaEventRecord(ev_kxt[b], aux);
      cudaStreamWaitEvent(st, ev_kxt[b], 0);
    }
    tc::Args a;
    tc_args_init(a);
    a.S = S; a.Np = Np; a.Mc = Mc; a.ntiles = mc_used / tc::BM; a.npairs = npairs; a.ngroups = ngroups; a.ldp = Mc;
    a.partial = partial; a.dbg = dbg; a.z = z; a.mpartial = mpartial;
    a.M = M; a.c_begin = c_begin; a.ldm = ldm; a.mean = mean;
    a.mode = 0; a.f16 = 1; a.amp2 = amp2; a.bexp = linv_exp;
    { const char* e = getenv("SMK_TC_A_EVICT_FIRST"); a.a_evict_first = (e && e[0] == '1') ? 1 : 0; }
    long nitems = (long)S * a.ntiles * npairs;
    int grid = (int)std::min<long>(nitems, num_sms());
    timing_begin("predict_tc_kernel", st);
    tc::predict_tc_kernel<<<grid, tc::THREADS, tc::SMEM_BYTES, st>>>(mAhi[b], mAlo[b], mBhi, mBlo, a);
    timing_end(st);
    tc::finish_var_kernel<<<dim3((mc_used + 255) / 256, S), 256, 0, st>>>(M, c_begin, mc_used, S, npairs, Mc, partial,
                                                                        amp2, var, ldm, nmp, mu_partial, mean, mu,
                                                                        z ? mpartial : nullptr);
    count_launch(3);
    if (fant) {      // fantasy means: same Kxt chunk against alpha^T, rectangular k range (OPT:609)
      tc::Args r = a;
      r.mode = 1; r.F = F; r.mu_f = mu_f; r.bexp = fexp; r.z = nullptr; r.ngroups = Fp / tc::BN; r.npairs = r.ngroups;
      long nit = (long)S * r.ntiles * r.npairs;
      int gr = (int)std::min<long>(nit, num_sms());
      timing_begin("predict_tc_kernel_rect", st);
      tc::predict_tc_kernel<<<gr, tc::THREADS, tc::SMEM_BYTES, st>>>(mAhi[b], mAlo[b], mFhi, mFlo, r);
      timing_end(st);
      count_launch();
    }
    if (overlap) cudaEventRecord(ev_mma[b], st);
  }
  return check_launch("predict_tc");
}

}  // namespace smk
