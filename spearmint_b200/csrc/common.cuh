// common.cuh -- shared device machinery for libspearmint_b200 (sm_90a).
//
// The SIMT data path is one register-tiled block GEMM (TileGemm) reused by the Cholesky
// panel/trailing updates, the multi-RHS triangular solves and the fused predict kernel.
// Everything is templated on the element type: float is the production path, double is used
// for the slice-sampler log-likelihood (where accept/reject comparisons must track the
// reference's float64 chain) and for bit-tight logic tests.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace smk {

constexpr int kThreads = 256;  // every tiled kernel runs 16x16 threads
constexpr int kBK = 16;        // k-chunk staged through shared memory
constexpr int kPad = 4;        // row padding of the staged tiles (keeps 16B alignment)
constexpr int kNpadMult = 128; // factor storage is padded to a multiple of this

template <typename T> struct Cfg;
template <> struct Cfg<float> {
  static constexpr int BM = 128, BN = 128, TM = 8, TN = 8, NB = 128;
};
template <> struct Cfg<double> {
  static constexpr int BM = 64, BN = 64, TM = 4, TN = 4, NB = 64;
};

// ---- 4-element vector access (16B for float, 2x16B for double) -------------------------------
template <typename T> struct V4 { T v[4]; };

__device__ __forceinline__ V4<float> ld4(const float* p) {
  float4 t = *reinterpret_cast<const float4*>(p);
  V4<float> r; r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w; return r;
}
__device__ __forceinline__ V4<double> ld4(const double* p) {
  double2 a = *reinterpret_cast<const double2*>(p);
  double2 b = *reinterpret_cast<const double2*>(p + 2);
  V4<double> r; r.v[0] = a.x; r.v[1] = a.y; r.v[2] = b.x; r.v[3] = b.y; return r;
}
__device__ __forceinline__ void st4(float* p, const V4<float>& r) {
  *reinterpret_cast<float4*>(p) = make_float4(r.v[0], r.v[1], r.v[2], r.v[3]);
}
__device__ __forceinline__ void st4(double* p, const V4<double>& r) {
  *reinterpret_cast<double2*>(p) = make_double2(r.v[0], r.v[1]);
  *reinterpret_cast<double2*>(p + 2) = make_double2(r.v[2], r.v[3]);
}

// ---- thread <-> micro-tile mapping ------------------------------------------------------------
// 256 threads as ty = tid/16, tx = tid%16.  A thread owns TM rows and TN columns in groups of 4
// contiguous elements, groups 64 apart: row(r) = (r/4)*64 + ty*4 + r%4 (same for columns with tx).
__device__ __forceinline__ int tile_row(int ty, int r) { return (r >> 2) * 64 + ty * 4 + (r & 3); }
__device__ __forceinline__ int tile_col(int tx, int c) { return (c >> 2) * 64 + tx * 4 + (c & 3); }

template <typename T>
struct TileSmem {
  using C = Cfg<T>;
  T As[2][kBK][C::BM + kPad];
  T Bs[2][kBK][C::BN + kPad];
};

// Operand sources for TileGemm::run.
//   KContig : element (row, k) at p[row*ld + k]   (k contiguous)  -> transposed on staging
//   MContig : element (row, k) at p[k*ld + row]   (row contiguous) -> staged directly
enum class Lay { KContig, MContig };

template <typename T, Lay LA, Lay LB, bool SUB>
struct TileGemm {
  using C = Cfg<T>;
  static constexpr int BM = C::BM, BN = C::BN, TM = C::TM, TN = C::TN;
  static constexpr int VA = BM * kBK / 4 / kThreads;  // vec4 loads per thread for the A chunk
  static constexpr int VB = BN * kBK / 4 / kThreads;
  static_assert(VA >= 1 && VB >= 1, "tile too small");

  // ---- global -> registers
  template <Lay L, int ROWS, int NV>
  static __device__ __forceinline__ void gload(V4<T> (&reg)[NV], const T* p, long ld,
                                               int k0, int tid) {
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      int v = tid + j * kThreads;
      if (L == Lay::KContig) {
        int row = v / (kBK / 4), kq = v % (kBK / 4);
        reg[j] = ld4(p + (long)row * ld + k0 + kq * 4);
      } else {
        int kr = v / (ROWS / 4), rq = v % (ROWS / 4);
        reg[j] = ld4(p + (long)(k0 + kr) * ld + rq * 4);
      }
    }
  }
  // ---- registers -> shared ([k][row] layout)
  template <Lay L, int ROWS, int NV>
  static __device__ __forceinline__ void sstore(T (*S)[ROWS + kPad], const V4<T> (&reg)[NV], int tid) {
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      int v = tid + j * kThreads;
      if (L == Lay::KContig) {
        int row = v / (kBK / 4), kq = v % (kBK / 4);
#pragma unroll
        for (int e = 0; e < 4; ++e) S[kq * 4 + e][row] = reg[j].v[e];
      } else {
        int kr = v / (ROWS / 4), rq = v % (ROWS / 4);
        st4(&S[kr][rq * 4], reg[j]);
      }
    }
  }

  static __device__ __forceinline__ void fma_chunk(T (&acc)[TM][TN], const T (*As)[BM + kPad],
                                                   const T (*Bs)[BN + kPad], int ty, int tx) {
#pragma unroll
    for (int kk = 0; kk < kBK; ++kk) {
      T a[TM], b[TN];
#pragma unroll
      for (int g = 0; g < TM / 4; ++g) {
        V4<T> t = ld4(&As[kk][g * 64 + ty * 4]);
#pragma unroll
        for (int e = 0; e < 4; ++e) a[g * 4 + e] = t.v[e];
      }
#pragma unroll
      for (int g = 0; g < TN / 4; ++g) {
        V4<T> t = ld4(&Bs[kk][g * 64 + tx * 4]);
#pragma unroll
        for (int e = 0; e < 4; ++e) b[g * 4 + e] = t.v[e];
      }
#pragma unroll
      for (int r = 0; r < TM; ++r)
#pragma unroll
        for (int c = 0; c < TN; ++c) acc[r][c] = SUB ? fma(-a[r], b[c], acc[r][c]) : fma(a[r], b[c], acc[r][c]);
    }
  }

  // acc (+/-)= sum_{k<K} A(row,k) * B(col,k).   A: BM rows, B: BN rows ("rows" of B are output columns).
  // K must be a multiple of kBK.  All 256 threads of the block must call this.
  // NOTE: no __restrict__ on A/B -- predict's scratch operand is written earlier by the same block and
  // must be read through the coherent path (never ld.global.nc).
  static __device__ __forceinline__ void run(T (&acc)[TM][TN], const T* A, long lda,
                                             const T* B, long ldb, int K, TileSmem<T>& sm) {
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    V4<T> ra[VA], rb[VB];
    const int nk = K / kBK;
    if (nk == 0) return;
    __syncthreads();  // staging buffers may still be read by a previous phase
    gload<LA, BM, VA>(ra, A, lda, 0, tid);
    gload<LB, BN, VB>(rb, B, ldb, 0, tid);
    sstore<LA, BM, VA>(sm.As[0], ra, tid);
    sstore<LB, BN, VB>(sm.Bs[0], rb, tid);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
      const int cur = kt & 1;
      if (kt + 1 < nk) {
        gload<LA, BM, VA>(ra, A, lda, (kt + 1) * kBK, tid);
        gload<LB, BN, VB>(rb, B, ldb, (kt + 1) * kBK, tid);
      }
      fma_chunk(acc, sm.As[cur], sm.Bs[cur], ty, tx);
      if (kt + 1 < nk) {
        sstore<LA, BM, VA>(sm.As[cur ^ 1], ra, tid);
        sstore<LB, BN, VB>(sm.Bs[cur ^ 1], rb, tid);
      }
      __syncthreads();
    }
  }

  // Same, but B is already resident in shared memory as Bsm[k][col] (row stride ldbs, K rows).
  static __device__ __forceinline__ void run_bsmem(T (&acc)[TM][TN], const T* A, long lda,
                                                   const T* Bsm, int ldbs, int K, TileSmem<T>& sm) {
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    V4<T> ra[VA];
    const int nk = K / kBK;
    if (nk == 0) return;
    __syncthreads();
    gload<LA, BM, VA>(ra, A, lda, 0, tid);
    sstore<LA, BM, VA>(sm.As[0], ra, tid);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
      const int cur = kt & 1;
      if (kt + 1 < nk) gload<LA, BM, VA>(ra, A, lda, (kt + 1) * kBK, tid);
#pragma unroll
      for (int kk = 0; kk < kBK; ++kk) {
        T a[TM], b[TN];
        const T* brow = Bsm + (long)(kt * kBK + kk) * ldbs;
#pragma unroll
        for (int g = 0; g < TM / 4; ++g) {
          V4<T> t = ld4(&sm.As[cur][kk][g * 64 + ty * 4]);
#pragma unroll
          for (int e = 0; e < 4; ++e) a[g * 4 + e] = t.v[e];
        }
#pragma unroll
        for (int g = 0; g < TN / 4; ++g) {
          V4<T> t = ld4(brow + g * 64 + tx * 4);
#pragma unroll
          for (int e = 0; e < 4; ++e) b[g * 4 + e] = t.v[e];
        }
#pragma unroll
        for (int r = 0; r < TM; ++r)
#pragma unroll
          for (int c = 0; c < TN; ++c) acc[r][c] = SUB ? fma(-a[r], b[c], acc[r][c]) : fma(a[r], b[c], acc[r][c]);
      }
      if (kt + 1 < nk) sstore<LA, BM, VA>(sm.As[cur ^ 1], ra, tid);
      __syncthreads();
    }
  }
};

// ---- stationary kernels on the scaled squared distance (GP:87-127) ----------------------------
__device__ __forceinline__ float  smk_sqrt(float x)  { return sqrtf(x); }
__device__ __forceinline__ double smk_sqrt(double x) { return sqrt(x); }
__device__ __forceinline__ float  smk_exp(float x)   { return expf(x); }
__device__ __forceinline__ double smk_exp(double x)  { return exp(x); }

template <typename T>
__device__ __forceinline__ T kernel_of_r2(int kind, T r2) {
  if (kind <= 1) return smk_exp(T(-0.5) * r2);                       // SE / ARDSE
  T r = smk_sqrt(r2);
  if (kind == 2) { T a = T(1.7320508075688772) * r; return (T(1) + a) * smk_exp(-a); }   // Matern32
  T a = T(2.23606797749979) * r;                                      // Matern52
  return (T(1) + a + T(5.0 / 3.0) * r2) * smk_exp(-a);
}

// round-to-nearest tf32 (10 explicit mantissa bits); x - tf32_rn(x) is exact in float32 and symmetric around zero, unlike the
// truncating split (x & 0xffffe000) whose dropped lo*lo products are all of one sign
__device__ __forceinline__ float tf32_rn(float x) {
  unsigned u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
// lo part of a split whose ONLY use is as a tf32 tensor-core operand: rounded to tf32 as well.  The MMA reads just the
// top 10 mantissa bits of an operand, so the unrounded x - tf32_rn(x) would be truncated toward zero -- a bias that
// accumulates along k through the Cholesky update and the triangular inverse.  (A split that is also read as a float32
// value, hi + lo, keeps the exact lo.)
__device__ __forceinline__ float tf32_lo(float x, float hi) { return tf32_rn(x - hi); }

// launch bookkeeping (api.cu)
void count_launch(int n = 1);
long long launch_count();
int check_launch(const char* what);
// optional per-kernel CUDA-event timing on the launch stream (bench.py's roofline leg): no-ops unless enabled
void timing_begin(const char* name, cudaStream_t st);
void timing_end(cudaStream_t st);

}  // namespace smk
