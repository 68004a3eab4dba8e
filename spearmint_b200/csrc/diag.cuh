// diag.cuh -- the serial spine of every blocked Cholesky in the library, taken off the critical path as far as it goes.
//
// Reference: spla.cholesky at OPT:540, 567, 585 and inside every slice-sampler log-probability OPT:637, 659, 690.  A
// blocked factorisation runs Npad / NB diagonal-block steps strictly one after the other, so the latency of one step --
// not its flops -- bounds the factorisation of a single matrix.  A first version did everything a step needs in one
// kernel with block-wide barriers around every column of every 32 x 32 piece; a clock64() timeline of it
// (tools/microbench/diag_bench.cu) showed most of a step going to assembling the off-diagonal tiles of W = L^-1 and to a
// latency-bound load loop rather than to the 32 x 32 factorisations and rank-32 updates -- hence this split:
//
//   diag_factor_block   (one CTA per matrix, ON the spine)  load (8 loads in flight per thread) -> for each 32-piece:
//                       warp-synchronous Cholesky of the piece (lane = row, row in registers), substitution for the rows
//                       below (thread = row), rank-32 update of the rest (float64: mma.sync.m8n8k4.f64 tiles, float32:
//                       4 x 4 register tiles) -> the four 32 x 32 diagonal inverses (one warp each).  Writes L and the
//                       compact  wd[4][32][32].
//   panel_sub_block     (many CTAs, 32 rows each)  L_Ij = A_Ij L_jj^-T by BLOCK substitution with the diagonal inverses:
//                       X_p = (A_p - sum_{q<p} X_q L_pq^T) W_pp^T  -- the full inverse is not needed for the panel.
//   winv_assemble_block (one CTA per block, OFF the spine, after the factorisation, all blocks at once)  full W_jj from
//                       L_jj and wd for the consumers that multiply by it (triangular inverse, multi-RHS solves, SIMT
//                       predict).
// Shared-memory tiles are 32 x 32 with row stride LDT = 36 (float64: conflict-free 8-byte DMMA fragment loads in both
// orientations) or 33 (float32: conflict-free by row and by column).
#pragma once
#include "common.cuh"

namespace smk {

// optional phase timeline (tools/microbench/diag_bench.cu defines SMK_DIAG_TIMELINE): clock64() stamps of thread 0
#ifdef SMK_DIAG_TIMELINE
__device__ long long g_diag_tl[64];
#define DIAG_STAMP(i) do { if (threadIdx.x == 0 && blockIdx.x == 0) g_diag_tl[i] = clock64(); } while (0)
#else
#define DIAG_STAMP(i) do { } while (0)
#endif

template <typename T> struct TileLd { static constexpr int v = 33; };
template <> struct TileLd<double> { static constexpr int v = 36; };

template <typename T, int NB>
struct DiagSmem {
  static constexpr int SB = 32, LDT = TileLd<T>::v, NP = NB / SB, NT = NP * (NP + 1) / 2;
  static constexpr int TILE = SB * LDT;
  // a tiles (lower block triangle) | NP diagonal inverse tiles | broadcast columns [2][32] (16-byte aligned) | inverse pivots [NB]
  static constexpr size_t bytes = sizeof(T) * ((size_t)(NT + NP) * TILE + 64 + NB);
  static __host__ __device__ __forceinline__ int tile(int bi, int bj) { return (bi * (bi + 1) / 2 + bj) * TILE; }
};

__device__ __forceinline__ void dmma_884(double (&c)[2], double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}

// ------------------------------------------------------------------------------------------------ 32 x 32 block product
// acc (+)= A * B^T for one 32 x 32 output block, K = 32, all 256 threads.  A(r, k) at A[r * sar + k * sak], B(c, k) at
// B[c * sbc + k * sbk] (shared memory).  The accumulator fragment stays in registers across calls:
//   double: warp w owns the 8 x 8 tiles 2w and 2w+1 (tile t: rows (t / 4) * 8.., columns (t % 4) * 8..), DMMA layout;
//   float : thread (ty = tid / 16, tx = tid % 16) owns rows 2ty, 2ty+1 x columns 2tx, 2tx+1.
template <typename T> struct BlkAcc;
template <> struct BlkAcc<double> { double c[2][2]; };
template <> struct BlkAcc<float> { float c[2][2]; };

template <typename T> __device__ __forceinline__ void blk_zero(BlkAcc<T>& a) {
  a.c[0][0] = a.c[0][1] = a.c[1][0] = a.c[1][1] = T(0);
}
__device__ __forceinline__ void blk_mma(BlkAcc<double>& acc, const double* A, int sar, int sak, const double* B, int sbc,
                                        int sbk) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t4 = lane & 3;
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int t = 2 * warp + u, r0 = (t >> 2) * 8, c0 = (t & 3) * 8;
    const double* ap = A + (r0 + gq) * sar + t4 * sak;
    const double* bp = B + (c0 + gq) * sbc + t4 * sbk;
#pragma unroll
    for (int k = 0; k < 32; k += 4) dmma_884(acc.c[u], ap[k * sak], bp[k * sbk]);
  }
}
__device__ __forceinline__ void blk_mma(BlkAcc<float>& acc, const float* A, int sar, int sak, const float* B, int sbc,
                                        int sbk) {
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  const float* a0 = A + (2 * ty) * sar;
  const float* b0 = B + (2 * tx) * sbc;
#pragma unroll 8
  for (int k = 0; k < 32; ++k) {
    const float x0 = a0[k * sak], x1 = a0[sar + k * sak], y0 = b0[k * sbk], y1 = b0[sbc + k * sbk];
    acc.c[0][0] = fmaf(x0, y0, acc.c[0][0]); acc.c[0][1] = fmaf(x0, y1, acc.c[0][1]);
    acc.c[1][0] = fmaf(x1, y0, acc.c[1][0]); acc.c[1][1] = fmaf(x1, y1, acc.c[1][1]);
  }
}
// element (i, j) of the calling thread's fragment -> (row, column) inside the 32 x 32 block
__device__ __forceinline__ void blk_coord(const BlkAcc<double>&, int i, int j, int& r, int& c) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t = 2 * warp + i;
  r = (t >> 2) * 8 + (lane >> 2);
  c = (t & 3) * 8 + (lane & 3) * 2 + j;
}
__device__ __forceinline__ void blk_coord(const BlkAcc<float>&, int i, int j, int& r, int& c) {
  r = 2 * (threadIdx.x >> 4) + i;
  c = 2 * (threadIdx.x & 15) + j;
}

// ------------------------------------------------------------------------------------------------ 32 x 32 pieces
// 1 / sqrt(x) without a branch: hardware seed (MUFU, ~2^-22) and one third-order step  y = y0 + y0 e (1/2 + 3/8 e),
// e = 1 - x y0^2  (remainder 5/16 e^3 ~ 2^-65; ~1 ulp).  The library rsqrt(double) / 1.0f / sqrtf() carry a slow-path branch
// and 7-8 DEPENDENT operations; on the pivot chain of a Cholesky step that latency is paid once per column.
template <typename T> __device__ __forceinline__ T fast_rsqrt(T x);
template <> __device__ __forceinline__ double fast_rsqrt<double>(double x) {
  double y0;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y0) : "d"(x));
  const double t = x * y0, e = fma(-t, y0, 1.0);
  return fma(y0 * e, fma(0.375, e, 0.5), y0);
}
template <> __device__ __forceinline__ float fast_rsqrt<float>(float x) {
  const float y0 = rsqrtf(x);
  const float t = x * y0, e = fmaf(-t, y0, 1.f);
  return fmaf(y0 * e, fmaf(0.375f, e, 0.5f), y0);
}
template <typename T> struct Vec16;
template <> struct Vec16<double> { typedef double2 type; static constexpr int n = 2; };
template <> struct Vec16<float> { typedef float4 type; static constexpr int n = 4; };
__device__ __forceinline__ double vget(const double2& v, int i) { return i ? v.y : v.x; }
__device__ __forceinline__ float vget(const float4& v, int i) { return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w; }

// Lower Cholesky of the 32 x 32 piece at `a` (tile, row stride LDT) by the calling warp; lane = row, the row lives in
// registers.  `col`: 64-entry, 16-byte aligned broadcast buffer; ipv receives 1 / L_jj; st ([32][32], 16-byte aligned)
// receives the scaled transpose  st[m][k] = L[k][m] / L[k][k]  (k > m) that fwd_subst32 reads.  `bad`: first non-positive
// pivot (or -1).
//
// What bounds it is the chain  pivot -> rsqrt -> scale -> (column to the other lanes) -> update -> next pivot, once per
// column, and -- the whole piece being straight-line code that runs once -- the instruction stream itself
// (tools/microbench/chol32_bench.cu measures it):
//   * the next pivot  r[j+1] - l^2  needs no other lane's data: lane j+1 forms it from its own l, so the broadcast of the
//     column is off the chain;
//   * the column is broadcast through shared memory with 16-byte loads instead of one shuffle per element: 3.5 k
//     instructions per piece instead of 9.7 k (float64), and the function is NOT inlined -- one copy for all call sites,
//     because the first execution of every further copy cost ~10 k cycles of instruction fetch.
template <typename T>
__device__ __noinline__ void warp_chol32(T* a, T* col, T* ipv, T* st, int lane, int& bad) {
  constexpr int LDT = TileLd<T>::v, NV = Vec16<T>::n;
  typedef typename Vec16<T>::type V;
  T r[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) r[k] = (k <= lane) ? a[lane * LDT + k] : T(0);
  T piv = r[0];                                  // this lane's candidate for the pivot of the next column (valid at lane j)
  T myip = T(0);
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    T d = __shfl_sync(0xffffffffu, piv, j);
    if (!(d > T(0))) { if (bad < 0) bad = j; d = T(1); }
    const T ip = fast_rsqrt<T>(d);
    const T l = r[j] * ip;                       // lane j: d / sqrt(d) = sqrt(d)
    if (lane >= j) r[j] = l;
    if (lane == j) { ipv[j] = ip; myip = ip; }
    if (j < 31) piv = fma(-l, l, r[j + 1]);      // bitwise what the update below leaves in r[j+1] of lane j+1
    T* cb = col + (j & 1) * 32;                  // two buffers: one warp barrier per column
    cb[lane] = l;
    __syncwarp();
    const V* cv = reinterpret_cast<const V*>(cb);
#pragma unroll
    for (int q = (j + 1) / NV; q < 32 / NV; ++q) {
      const V v = cv[q];                         // same address in every lane: broadcast
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int k = q * NV + i;
        if (k > j) r[k] = fma(-l, vget(v, i), r[k]);      // meaningful for j < k <= lane
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    if (k <= lane) a[lane * LDT + k] = r[k];
    st[k * 32 + lane] = r[k] * myip;             // row k of st = column k of L, every row scaled by its inverse pivot
  }
}

// Forward substitution  L y = b  for one right-hand side per thread, in place (x: b in, y out); L as the scaled transpose
// st written by warp_chol32, ipv = 1 / L_kk.  Right-looking with pre-scaled multipliers:
//     x_k <- b_k / L_kk;   for m = 0..31:  x_k -= (L_km / L_kk) x_m  for all k > m
// so the step from x_m to x_m+1 is ONE fused multiply-add (the left-looking form  x_k = (b_k - sum_m L_km x_m) / L_kk  puts
// a multiply-add, the reduction of its partial sums and the scaling on that chain: 2.5 - 3.7 k cycles per 32 x 32 piece in
// the timeline against ~1 k), and every read is a 16-byte broadcast load of a row of st.
template <typename T>
__device__ __forceinline__ void fwd_subst32(const T* st, const T* ipv, T (&x)[32]) {
  constexpr int NV = Vec16<T>::n;
  typedef typename Vec16<T>::type V;
#pragma unroll
  for (int q = 0; q < 32 / NV; ++q) {
    const V v = reinterpret_cast<const V*>(ipv)[q];
#pragma unroll
    for (int i = 0; i < NV; ++i) x[q * NV + i] *= vget(v, i);
  }
#pragma unroll
  for (int m = 0; m < 31; ++m) {
    const V* row = reinterpret_cast<const V*>(st + m * 32);
#pragma unroll
    for (int q = (m + 1) / NV; q < 32 / NV; ++q) {
      const V v = row[q];
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int k = q * NV + i;
        if (k > m) x[k] = fma(-vget(v, i), x[m], x[k]);
      }
    }
  }
}

// W = L^-1 of a 32 x 32 lower-triangular tile by the calling warp: lane = column c solves L w = e_c.  st / ipv as above;
// w (tile, row stride LDT) may be the memory st lives in (every lane has read all it needs before the first write).
template <typename T>
__device__ __forceinline__ void warp_trinv32(const T* st, const T* ipv, T* w, int lane) {
  constexpr int LDT = TileLd<T>::v;
  T x[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) x[i] = (i == lane) ? T(1) : T(0);
  fwd_subst32<T>(st, ipv, x);                    // x[i] stays exactly 0 for i < lane
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 32; ++i) w[i * LDT + lane] = x[i];
}

// rank-32 update of the lower triangle left of piece p:  C[r][c] -= X[r] . X[c]  for r >= c (rows relative to the first
// remaining row; X = tiles (bi, p), C = tiles (bi, bj)).  Two parts, so that the NEXT diagonal piece can be factored while
// the bulk of the update is still running (look-ahead inside the block):
//   part 0: the tile (p+1, p+1) only, all 8 warps;   part 1: everything else, warps 1..7 (warp 0 is factoring).
template <int NB>
__device__ __forceinline__ void diag_update(double* a, int p, int part) {
  using DS = DiagSmem<double, NB>;
  constexpr int LDT = DS::LDT;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, t4 = lane & 3;
  const int nt8 = (NB - (p + 1) * 32) / 8;                // 8 x 8 tiles per side
  // lower tile triangle in row-major order: entries 0..9 are exactly the tile rows 0..3 = the 32 x 32 tile (p+1, p+1)
  const int e0 = part ? 10 + warp - 1 : warp, e1 = part ? nt8 * (nt8 + 1) / 2 : 10, step = part ? 7 : 8;
  if (part && warp == 0) return;
  for (int e = e0; e < e1; e += step) {                   // one DMMA tile per warp and round
    int tr = (int)((sqrtf(8.f * (float)e + 1.f) - 1.f) * 0.5f);
    while (tr * (tr + 1) / 2 > e) --tr;
    while ((tr + 1) * (tr + 2) / 2 <= e) ++tr;
    const int tc = e - tr * (tr + 1) / 2;
    const int r0 = tr * 8, c0 = tc * 8;
    const double* xr = a + DS::tile(p + 1 + (r0 >> 5), p) + ((r0 & 31) + gq) * LDT + t4;
    const double* xc = a + DS::tile(p + 1 + (c0 >> 5), p) + ((c0 & 31) + gq) * LDT + t4;
    double c[2] = {0.0, 0.0};
#pragma unroll
    for (int k = 0; k < 32; k += 4) dmma_884(c, xr[k], xc[k]);
    double* ct = a + DS::tile(p + 1 + (r0 >> 5), p + 1 + (c0 >> 5)) + ((r0 & 31) + gq) * LDT + (c0 & 31) + t4 * 2;
    ct[0] -= c[0];
    ct[1] -= c[1];                                        // entries above the diagonal of a diagonal tile are never read
  }
}
template <int NB>
__device__ __forceinline__ void diag_update(float* a, int p, int part) {
  using DS = DiagSmem<float, NB>;
  constexpr int LDT = DS::LDT, SB = 32;
  if (part == 0) {
    // tile (p+1, p+1): thread (ty, tx) owns rows 2ty, 2ty+1 x columns 2tx, 2tx+1 (tx <= ty: the lower half)
    const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
    if (tx > ty) return;
    const float* x = a + DS::tile(p + 1, p);
    const float *a0 = x + (2 * ty) * LDT, *b0 = x + (2 * tx) * LDT;
    float c00 = 0.f, c01 = 0.f, c10 = 0.f, c11 = 0.f;
#pragma unroll 8
    for (int k = 0; k < SB; ++k) {
      const float x0 = a0[k], x1 = a0[LDT + k], y0 = b0[k], y1 = b0[LDT + k];
      c00 = fmaf(x0, y0, c00); c01 = fmaf(x0, y1, c01); c10 = fmaf(x1, y0, c10); c11 = fmaf(x1, y1, c11);
    }
    float* ct = a + DS::tile(p + 1, p + 1) + (2 * ty) * LDT + 2 * tx;
    ct[0] -= c00; ct[1] -= c01; ct[LDT] -= c10; ct[LDT + 1] -= c11;      // (2ty, 2tx+1) with tx == ty is above the diagonal: never read
    return;
  }
  // everything else, threads 32..255.  A thread owns the 4 x 4 elements (gr + i nt, gc + j nt): consecutive lanes read
  // consecutive rows of X (conflict-free, stride 33) and share the other operand (broadcast).  i > j is always below the
  // diagonal, i == j iff gr >= gc.
  if (threadIdx.x < 32) return;
  const int rows = NB - (p + 1) * SB, nt = rows / 4;
  for (int e = threadIdx.x - 32; e < nt * nt; e += 224) {
    const int gr = e / nt, gc = e % nt;
    const bool dg = gr >= gc;
    const float* xr[4];
    const float* xc[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int r = gr + i * nt, c = gc + i * nt;
      xr[i] = a + DS::tile(p + 1 + (r >> 5), p) + (r & 31) * LDT;
      xc[i] = a + DS::tile(p + 1 + (c >> 5), p) + (c & 31) * LDT;
    }
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 8
    for (int k = 0; k < SB; ++k) {
      float xa[4], xb[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { xa[i] = xr[i][k]; xb[i] = xc[i][k]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j <= i; ++j) acc[i][j] = fmaf(xa[i], xb[j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j <= i; ++j) {
        if (i == j && !dg) continue;
        const int r = gr + i * nt, c = gc + j * nt;
        if (r < SB && c < SB) continue;                     // tile (p+1, p+1): part 0
        a[DS::tile(p + 1 + (r >> 5), p + 1 + (c >> 5)) + (r & 31) * LDT + (c & 31)] -= acc[i][j];
      }
  }
}

// ------------------------------------------------------------------------------------------------ the spine kernel body
// Ab: block (jb, jb) of this sample's matrix (row stride ld), factored in place (lower triangle; the strict upper triangle
// is left untouched).  wd: [NB/32][32][32] receives the inverses of the 32 x 32 diagonal pieces of L_jj.
// info (may be NULL): 1-based index of the first non-positive pivot, written once.
template <typename T, int NB>
__device__ void diag_factor_block(T* __restrict__ Ab, int ld, T* __restrict__ wd, int* info, int info_base, T* sm,
                                  bool trigger = false) {
  using DS = DiagSmem<T, NB>;
  constexpr int SB = 32, LDT = DS::LDT, NP = DS::NP, TILE = DS::TILE;
  T* a = sm;
  T* w = a + DS::NT * TILE;                 // NP tiles: scaled transposes of the diagonal pieces, then their inverses
  T* col = w + NP * TILE;
  T* ipv = col + 64;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  DIAG_STAMP(0);
  // ---- load the lower block triangle tile by tile: a warp reads 32 contiguous elements of a row, 4 loads in flight
  for (int bi = 0; bi < NP; ++bi)
    for (int bj = 0; bj <= bi; ++bj) {
      T v[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int e = tid + q * 256, i = e >> 5, k = e & 31;
        v[q] = (bj < bi || k <= i) ? Ab[(long)(bi * SB + i) * ld + bj * SB + k] : T(0);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int e = tid + q * 256;
        a[DS::tile(bi, bj) + (e >> 5) * LDT + (e & 31)] = v[q];
      }
    }
  __syncthreads();
  DIAG_STAMP(1);

  // Look-ahead inside the block: after the substitution of piece p the tile (p+1, p+1) is updated first (all warps, a few
  // hundred cycles); then warp 0 factors piece p+1 while warps 1..7 finish the rank-32 update and store the finished block
  // column p.  The critical path is  chol32 -> substitution -> one tile update -> chol32 ...; the bulk of the updates and
  // of the stores hides behind the factorisations.
  auto chol_piece = [&](int p) {
    int bad = -1;
    warp_chol32<T>(a + DS::tile(p, p), col, ipv + p * SB, w + p * TILE, lane, bad);
    if (bad >= 0 && lane == 0 && info && *info == 0) *info = info_base + p * SB + bad + 1;
  };
  auto store_column = [&](int p) {                          // tiles (p..NP-1, p) are final; threads 32..255
    for (int bi = p; bi < NP; ++bi)
      for (int e = tid - 32; e < SB * SB; e += 224) {
        const int i = e >> 5, k = e & 31;
        if (p < bi || k <= i) Ab[(long)(bi * SB + i) * ld + p * SB + k] = a[DS::tile(bi, p) + i * LDT + k];
      }
  };
  if (warp == 0) chol_piece(0);
  __syncthreads();
  DIAG_STAMP(2);
  for (int p = 0; p + 1 < NP; ++p) {
    const int rows = NB - (p + 1) * SB;
    // (b) rows below: X L_pp^T = A_sub by substitution, one thread per row
    if (tid < rows) {
      const int bi = p + 1 + (tid >> 5);
      T* ar = a + DS::tile(bi, p) + (tid & 31) * LDT;
      T x[32];
#pragma unroll
      for (int k = 0; k < 32; ++k) x[k] = ar[k];
      fwd_subst32<T>(w + p * TILE, ipv + p * SB, x);
#pragma unroll
      for (int k = 0; k < 32; ++k) ar[k] = x[k];
    }
    __syncthreads();
    DIAG_STAMP(3 + 4 * p);
    // (c) rank-32 update: the next diagonal tile first ...
    diag_update<NB>(a, p, 0);
    __syncthreads();
    DIAG_STAMP(4 + 4 * p);
    // ... then the next piece's factorisation (warp 0) next to the rest of the update and the stores of column p
    if (warp == 0) { chol_piece(p + 1); DIAG_STAMP(5 + 4 * p); }
    else { diag_update<NB>(a, p, 1); store_column(p); }
    __syncthreads();
    DIAG_STAMP(6 + 4 * p);
  }
  DIAG_STAMP(20);
  // programmatic dependent launch (potrf_ll): let the panel's CTAs come up while the inverses are formed and stored;
  // they wait (griddepcontrol.wait) for this grid to finish before they read anything
  if (trigger) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  // ---- inverses of the diagonal pieces, one warp each
  if (warp < NP) warp_trinv32<T>(w + warp * TILE, ipv + warp * SB, w + warp * TILE, lane);
  __syncthreads();
  DIAG_STAMP(21);

  // ---- store what is left of L (the last diagonal tile; the block columns before it went out during the look-ahead) and
  // the compact diagonal inverses
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int e = tid + q * 256, i = e >> 5, k = e & 31;
    if (k <= i) Ab[(long)((NP - 1) * SB + i) * ld + (NP - 1) * SB + k] = a[DS::tile(NP - 1, NP - 1) + i * LDT + k];
  }
  for (int e = tid; e < NP * SB * SB; e += 256) {
    const int pp = e >> 10, i = (e >> 5) & 31, k = e & 31;
    wd[e] = (k <= i) ? w[pp * TILE + i * LDT + k] : T(0);
  }
  DIAG_STAMP(22);
}

// ------------------------------------------------------------------------------------------------ panel by block substitution
// 32 rows of the panel below block (jb, jb):  X = A L_jj^-T  as  X_p = (A_p - sum_{q<p} X_q L_pq^T) W_pp^T, p = 0..NP-1.
// Ap: first of the 32 rows (row stride ld), columns of block column jb;  Ljj: the factored diagonal block (row stride ld);
// wd: its diagonal inverses.  Result overwrites Ap; optional tf32 (hi, lo) copies for the tensor-core update (float only).
template <typename T, int NB>
struct PanelSmem {
  static constexpr int SB = 32, LDT = TileLd<T>::v, NP = NB / SB, TILE = SB * LDT;
  // L off-diagonal tiles (NP (NP-1) / 2) | NP diagonal inverses | NP row tiles of the panel | 1 scratch tile
  static constexpr int NL = NP * (NP - 1) / 2;
  static constexpr size_t bytes = sizeof(T) * (size_t)(NL + NP + NP + 1) * TILE;
};

template <typename T, int NB>
__device__ void panel_sub_block(T* __restrict__ Ap, int ld, const T* __restrict__ Ljj, const T* __restrict__ wd,
                                T* __restrict__ hi, T* __restrict__ lo, T* sm, bool trigger = false) {
  using PS = PanelSmem<T, NB>;
  constexpr int SB = 32, LDT = PS::LDT, NP = PS::NP, TILE = PS::TILE;
  T* lt = sm;                               // off-diagonal tile (pi, pj), pj < pi, at index pi (pi - 1) / 2 + pj
  T* wt = lt + PS::NL * TILE;
  T* xt = wt + NP * TILE;                   // panel rows: tile q = columns 32 q .. 32 q + 31
  T* tt = xt + NP * TILE;                   // scratch: A_p - sum
  const int tid = threadIdx.x;
  // ---- loads: every thread issues all of its global reads before the first shared-memory store (this kernel sits on the
  //      spine: a load loop with one request in flight per thread is latency-bound)
  {
    constexpr int NLV = PS::NL * 4, NWV = NP * 4, NXV = NB / 8;       // values per thread: L tiles, W tiles, panel rows
    T lv[NLV > 0 ? NLV : 1], wv[NWV], xv[NXV];
#pragma unroll
    for (int t = 0; t < PS::NL; ++t) {
      int bi = 1;
      while (bi * (bi + 1) / 2 <= t) ++bi;                              // tile t = (bi, bk), bk < bi
      const int bk = t - bi * (bi - 1) / 2;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int e = tid + q * 256;
        lv[t * 4 + q] = Ljj[(long)(bi * SB + (e >> 5)) * ld + bk * SB + (e & 31)];
      }
    }
#pragma unroll
    for (int q = 0; q < NWV; ++q) wv[q] = wd[tid + q * 256];
#pragma unroll
    for (int q = 0; q < NXV; ++q) {
      const int e = tid + q * 256;
      xv[q] = Ap[(long)(e / NB) * ld + (e % NB)];
    }
#pragma unroll
    for (int t = 0; t < PS::NL; ++t)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int e = tid + q * 256;
        lt[t * TILE + (e >> 5) * LDT + (e & 31)] = lv[t * 4 + q];
      }
#pragma unroll
    for (int q = 0; q < NWV; ++q) {
      const int e = tid + q * 256;
      wt[(e >> 10) * TILE + ((e >> 5) & 31) * LDT + (e & 31)] = wv[q];
    }
#pragma unroll
    for (int q = 0; q < NXV; ++q) {
      const int e = tid + q * 256, i = e / NB, k = e % NB;
      xt[(k >> 5) * TILE + i * LDT + (k & 31)] = xv[q];
    }
  }
  __syncthreads();
  BlkAcc<T> acc;
  for (int p = 0; p < NP; ++p) {
    blk_zero(acc);
    for (int q = 0; q < p; ++q)               // sum_q X_q L_pq^T : A(r, k) = X_q[r][k], B(c, k) = L_pq[c][k]
      blk_mma(acc, xt + q * TILE, LDT, 1, lt + (p * (p - 1) / 2 + q) * TILE, LDT, 1);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        int r, c;
        blk_coord(acc, i, j, r, c);
        tt[r * LDT + c] = xt[p * TILE + r * LDT + c] - acc.c[i][j];
      }
    __syncthreads();
    blk_zero(acc);
    blk_mma(acc, tt, LDT, 1, wt + p * TILE, LDT, 1);      // X_p = T W_pp^T : B(c, k) = W_pp[c][k]
    __syncthreads();                                       // everybody is done reading tt (and X_p's old values)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        int r, c;
        blk_coord(acc, i, j, r, c);
        xt[p * TILE + r * LDT + c] = acc.c[i][j];
      }
    __syncthreads();
  }
  if (trigger) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  for (int e = tid; e < SB * NB; e += 256) {
    const int i = e / NB, k = e % NB;
    const T x = xt[(k >> 5) * TILE + i * LDT + (k & 31)];
    Ap[(long)i * ld + k] = x;
    if constexpr (sizeof(T) == 4) {
      if (hi != nullptr) {                   // tf32 (hi, lo) copy of the finished panel: round-to-nearest split
        const float h = tf32_rn(x);
        hi[(long)i * ld + k] = h;
        lo[(long)i * ld + k] = tf32_lo(x, h);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ full inverse, off the spine
// W_jj = L_jj^-1 (NB x NB row-major, zeros above the diagonal) from L_jj and the diagonal inverses:
//   W_ij = -W_ii (sum_{k=j}^{i-1} L_ik W_kj)   by block distance d = i - j = 1, 2, ...
template <typename T, int NB>
struct WinvSmem {
  static constexpr int SB = 32, LDT = TileLd<T>::v, NP = NB / SB, NT = NP * (NP + 1) / 2, TILE = SB * LDT;
  static constexpr size_t bytes = sizeof(T) * (size_t)(2 * NT + 1) * TILE;     // L tiles | W tiles | scratch
};
template <typename T, int NB>
__device__ void winv_assemble_block(const T* __restrict__ Ljj, int ld, const T* wd, T* Wb, T* sm) {   // wd may alias Wb
  using WS = WinvSmem<T, NB>;
  using DS = DiagSmem<T, NB>;
  constexpr int SB = 32, LDT = WS::LDT, NP = WS::NP, TILE = WS::TILE;
  T* a = sm;
  T* w = a + WS::NT * TILE;
  T* tt = w + WS::NT * TILE;
  const int tid = threadIdx.x;
  for (int e = tid; e < NB * NB; e += 256) {
    const int i = e / NB, k = e % NB;
    if ((k >> 5) < (i >> 5)) a[DS::tile(i >> 5, k >> 5) + (i & 31) * LDT + (k & 31)] = Ljj[(long)i * ld + k];
  }
  for (int e = tid; e < NP * SB * SB; e += 256) {
    const int pp = e / (SB * SB);
    w[DS::tile(pp, pp) + ((e / SB) % SB) * LDT + (e % SB)] = wd[e];
  }
  __syncthreads();
  BlkAcc<T> acc;
  for (int d = 1; d < NP; ++d)
    for (int j = 0; j + d < NP; ++j) {
      const int i = j + d;
      blk_zero(acc);
      for (int kb = j; kb < i; ++kb)          // T = sum L_ik W_kj : A(r, m) = L_ik[r][m], B(c, m) = W_kj[m][c]
        blk_mma(acc, a + DS::tile(i, kb), LDT, 1, w + DS::tile(kb, j), 1, LDT);
#pragma unroll
      for (int x = 0; x < 2; ++x)
#pragma unroll
        for (int y = 0; y < 2; ++y) {
          int r, c;
          blk_coord(acc, x, y, r, c);
          tt[r * LDT + c] = acc.c[x][y];
        }
      __syncthreads();
      blk_zero(acc);
      blk_mma(acc, w + DS::tile(i, i), LDT, 1, tt, 1, LDT);      // W_ii T : B(c, m) = T[m][c]
#pragma unroll
      for (int x = 0; x < 2; ++x)
#pragma unroll
        for (int y = 0; y < 2; ++y) {
          int r, c;
          blk_coord(acc, x, y, r, c);
          w[DS::tile(i, j) + r * LDT + c] = -acc.c[x][y];
        }
      __syncthreads();
    }
  for (int e = tid; e < NB * NB; e += 256) {
    const int i = e / NB, k = e % NB;
    Wb[e] = (k <= i) ? w[DS::tile(i >> 5, k >> 5) + (i & 31) * LDT + (k & 31)] : T(0);
  }
}

}  // namespace smk
