// potrf_ll.cu -- float64 batched Cholesky for the slice-sampler log-likelihood (f2; reference: the spla.cholesky inside
// every logprob closure, OPT:637, 659, 690, ~50 D/8 calls per hyper-sample, thousands per next() at N = 4096).
//
// The generic SIMT factorisation (NB = 64, 4 x 4 register tiles) is far from the fp64 tensor rate here, and a single
// matrix is bound by its chain of diagonal steps.  This file is the dedicated path:
//   * NB = 128 block columns in pairs, right-looking, look-ahead on three streams: while the rank-256 update of the
//     trailing matrix (pair j) runs in the background, the next pair's diagonal blocks and panels are already being
//     factored, and of the look-ahead updates only the one 128 x 128 block the next diagonal kernel reads stays on
//     the serial spine  diag -> panel -> block update -> diag ...;
//   * diagonal blocks by the warp-synchronous single-SM kernel of diag.cuh, panels by its block substitution;
//   * the trailing updates (A_IK -= L_Ij L_Kj^T) as one tiled GEMM kernel on the fp64 tensor
//     path: mma.sync.m8n8k4.f64 (DMMA), operands staged by cp.async through a 3-stage shared-memory ring
//     (row stride 20 doubles: conflict-free 8-byte fragment loads), 128 x 128 output tiles (32 x 64 per warp) for the
//     update and 32-row tiles for the thin panel / look-ahead column so that even one matrix spreads over the SMs;
//   * the whole launch sequence of one batch is captured once into a CUDA graph per (pointer, shape) and replayed.
// Only L (lower triangle) is produced; W_jj (inverse diagonal blocks) is internal workspace.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <map>
#include <tuple>

#include "common.cuh"
#include "diag.cuh"

namespace smk {
int num_sms();
namespace ll {

constexpr int NB = 128;
constexpr int KC = 16;         // k per stage
constexpr int LDS = 20;        // shared row stride in doubles (16 + 4): fragment loads hit 16 distinct 8-byte banks
constexpr int STAGES = 3;

constexpr int WD = NB * 32;     // compact diagonal inverses of one block: [4][32][32]

// Programmatic dependent launch along the spine (diag -> panel -> block update -> diag ...): a kernel launched with the
// attribute may start while its predecessor in the stream is still running (after the predecessor's launch_dependents);
// nothing of the predecessor's output is touched before this wait.  Without the attribute the wait returns at once.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__global__ void __launch_bounds__(256) diag_kernel(int ld, int jb, double* __restrict__ A, long a_stride,
                                                    double* __restrict__ W, long w_stride, int* __restrict__ info) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int s = blockIdx.x;
  double* Ab = A + (long)s * a_stride + (long)jb * NB * ld + (long)jb * NB;
  pdl_wait();
  diag_factor_block<double, NB>(Ab, ld, W + (long)s * w_stride + (long)jb * WD, info ? info + s : nullptr, jb * NB,
                                reinterpret_cast<double*>(smem_raw), true);
}

// L_Ij = A_Ij L_jj^-T by block substitution, 32 rows per CTA, block rows row_blk0, row_blk0 + 1, ...; grid = (rows / 32, 1, S)
__global__ void __launch_bounds__(256) panel_kernel(int ld, int jb, int row_blk0, double* __restrict__ A, long a_stride,
                                                     const double* __restrict__ W, long w_stride) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int s = blockIdx.z;
  double* As = A + (long)s * a_stride;
  pdl_wait();
  panel_sub_block<double, NB>(As + ((long)row_blk0 * NB + (long)blockIdx.x * 32) * ld + (long)jb * NB, ld,
                              As + (long)jb * NB * ld + (long)jb * NB, W + (long)s * w_stride + (long)jb * WD, nullptr,
                              nullptr, reinterpret_cast<double*>(smem_raw), true);
}

__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) { dmma_884(c, a, b); }

// C[r0 + 0..BM)[c0 + 0..128) (op)= A[r0 + ..][0..K) * B[c0 + ..][0..K)^T, all row-major (k contiguous).
//   sub = 1 : C -= A B^T (trailing / column update);  sub = 0 : C = A B^T (panel; C may alias A: each CTA reads its
//   whole A tile before it writes).  tri = 1: tiles strictly above the block diagonal are skipped (BM == 128 only).
struct GemmArgs {
  const double* A; const double* B; double* C;
  long a_stride, b_stride, c_stride;     // per matrix (blockIdx.z)
  int lda, ldb, ldc, K;
  int row0, col0;                        // first output row / column (elements) of tile (0, 0)
  int brow0;                             // first row of B for column tile 0
  int sub, tri;
  int persist, nt, batch;                // persist = 1: grid-stride loop over the batch x lower-triangle tiles (nt per side)
};

template <int BM, int ST>
__global__ void __launch_bounds__(256) dgemm_nt_kernel(GemmArgs g) {
  constexpr int WM = BM / 32, WN = 8 / WM;          // warp grid
  constexpr int WTN = 128 / WN;                     // columns per warp: 64 / 32 / 16
  constexpr int NT = WTN / 8;                       // 8-column DMMA tiles per warp
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* As = reinterpret_cast<double*>(smem_raw);           // [ST][BM][LDS]
  double* Bs = As + ST * BM * LDS;                             // [ST][128][LDS]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wm = warp / WN, wn = warp % WN, gq = lane >> 2, t4 = lane & 3;
  const int ntri = g.nt * (g.nt + 1) / 2;
  const long items = g.persist ? (long)g.batch * ntri : 1;
  for (long item = g.persist ? blockIdx.x : 0; item < items; item += gridDim.x) {
    int bx = blockIdx.x, by = blockIdx.y, bz = blockIdx.z;
    if (g.persist) {                                  // item -> (matrix, tile row >= tile column)
      bz = (int)(item / ntri);
      const int e = (int)(item - (long)bz * ntri);
      bx = (int)((sqrtf(8.f * (float)e + 1.f) - 1.f) * 0.5f);
      while (bx * (bx + 1) / 2 > e) --bx;
      while ((bx + 1) * (bx + 2) / 2 <= e) ++bx;
      by = e - bx * (bx + 1) / 2;
    }
    const int r0 = g.row0 + bx * BM, c0 = g.col0 + by * 128;
    if (g.tri && c0 > r0 + BM - 1) continue;          // the whole tile lies above the diagonal
    const double* A = g.A + (long)bz * g.a_stride + (long)r0 * g.lda;
    const double* B = g.B + (long)bz * g.b_stride + (long)(g.brow0 + by * 128) * g.ldb;
    double* C = g.C + (long)bz * g.c_stride + (long)r0 * g.ldc + c0;

    auto load_stage = [&](int st, int k0) {
      // 16-byte chunks: row = chunk / 8, piece = chunk % 8 (2 doubles each)
#pragma unroll
      for (int q = 0; q < BM * 8 / 256; ++q) {
        const int ch = tid + q * 256, row = ch >> 3, pc = ch & 7;
        cp_async16(As + ((size_t)st * BM + row) * LDS + pc * 2, A + (long)row * g.lda + k0 + pc * 2);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int ch = tid + q * 256, row = ch >> 3, pc = ch & 7;
        cp_async16(Bs + ((size_t)st * 128 + row) * LDS + pc * 2, B + (long)row * g.ldb + k0 + pc * 2);
      }
    };

    double acc[4][NT][2];
#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) { acc[mi][ni][0] = 0.0; acc[mi][ni][1] = 0.0; }

    const int nk = g.K / KC;
#pragma unroll
    for (int s = 0; s < ST - 1; ++s) {
      if (s < nk) load_stage(s, s * KC);
      cp_async_commit();
    }
    for (int kt = 0; kt < nk; ++kt) {
      cp_async_wait<ST - 2>();
      __syncthreads();
      if (kt + ST - 1 < nk) load_stage((kt + ST - 1) % ST, (kt + ST - 1) * KC);
      cp_async_commit();
      const double* as = As + ((size_t)(kt % ST) * BM + wm * 32 + gq) * LDS + t4;
      const double* bs = Bs + ((size_t)(kt % ST) * 128 + wn * WTN + gq) * LDS + t4;
#pragma unroll
      for (int kk = 0; kk < KC; kk += 4) {
        double af[4], bf[NT];
#pragma unroll
        for (int mi = 0; mi < 4; ++mi) af[mi] = as[mi * 8 * LDS + kk];
#pragma unroll
        for (int ni = 0; ni < NT; ++ni) bf[ni] = bs[ni * 8 * LDS + kk];
#pragma unroll
        for (int mi = 0; mi < 4; ++mi)
#pragma unroll
          for (int ni = 0; ni < NT; ++ni) dmma(acc[mi][ni], af[mi], bf[ni]);
      }
    }
    cp_async_wait<0>();
    __syncthreads();          // panel mode writes over its own A tile: every warp is done reading (and the ring is free)

#pragma unroll
    for (int mi = 0; mi < 4; ++mi)
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        double2* cp = reinterpret_cast<double2*>(C + (long)(wm * 32 + mi * 8 + gq) * g.ldc + wn * WTN + ni * 8 + t4 * 2);
        double2 v;
        if (g.sub) { v = *cp; v.x -= acc[mi][ni][0]; v.y -= acc[mi][ni][1]; }
        else { v.x = acc[mi][ni][0]; v.y = acc[mi][ni][1]; }
        *cp = v;
      }
  }
}

// The one update the NEXT diagonal kernel waits for: block (b, b) -= P P^T with P = rows of block b, columns [k0, k0 + K) of
// the factor (K = 128 after one panel, 256 for the look-ahead of a pair).  On the 32-row GEMM above (4 CTAs, 256 - 512
// dependent DMMAs per warp) this is a long serial chain on every spine step.  Here: one CTA per 32 x 32 tile
// of the lower triangle (10 CTAs per matrix), both operand strips loaded in one burst of cp.async (every load in flight at
// once), then K / 4 DMMAs per 8 x 8 tile in two independent chains -- 64 - 128 DMMAs per warp.
constexpr int DBU_MAXK = 256;
__global__ void __launch_bounds__(256) diag_block_update_kernel(int ld, int b, int k0, int K, double* __restrict__ A, long a_stride) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int LD = K + 4;                              // row stride: 8-byte fragment loads hit distinct banks
  double* Ar = reinterpret_cast<double*>(smem_raw);  // [32][LD] rows of the tile's row strip
  double* Br = Ar + 32 * LD;                         // [32][LD] rows of its column strip
  int ti = 0, e = blockIdx.x;                        // tile (ti, tj), ti >= tj, row-major over the lower triangle
  while ((ti + 1) * (ti + 2) / 2 <= e) ++ti;
  const int tj = e - ti * (ti + 1) / 2;
  double* As = A + (long)blockIdx.y * a_stride;
  const double* pa = As + ((long)b * NB + ti * 32) * ld + k0;
  const double* pb = As + ((long)b * NB + tj * 32) * ld + k0;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, t4 = lane & 3;
  pdl_wait();
  pdl_trigger();                                     // the diagonal kernel behind this one is a single CTA per matrix
  const int cpr = K / 2;                             // 16-byte chunks per row
  for (int ch = tid; ch < 32 * cpr; ch += 256) {
    const int row = ch / cpr, pc = ch - row * cpr;
    cp_async16(Ar + row * LD + pc * 2, pa + (long)row * ld + pc * 2);
    cp_async16(Br + row * LD + pc * 2, pb + (long)row * ld + pc * 2);
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  double* Ct = As + ((long)b * NB + ti * 32) * ld + (long)b * NB + tj * 32;
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int t = 2 * warp + u, r0 = (t >> 2) * 8, c0 = (t & 3) * 8;
    const double* ap = Ar + (r0 + gq) * LD + t4;
    const double* bp = Br + (c0 + gq) * LD + t4;
    double c[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
#pragma unroll 8
    for (int k = 0; k < K; k += 8) {
      dmma(c[0], ap[k], bp[k]);
      dmma(c[1], ap[k + 4], bp[k + 4]);
    }
    double2* cp = reinterpret_cast<double2*>(Ct + (long)(r0 + gq) * ld + c0 + t4 * 2);
    double2 v = *cp;
    v.x -= c[0][0] + c[1][0];
    v.y -= c[0][1] + c[1][1];
    *cp = v;
  }
}

template <int BM>
static void launch_gemm(const GemmArgs& g, int tiles_m, int tiles_n, int S, cudaStream_t st) {
  constexpr int ST = STAGES;
  const size_t smem = sizeof(double) * ST * (BM + 128) * LDS;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(dgemm_nt_kernel<BM, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr = true;
  }
  dgemm_nt_kernel<BM, ST><<<dim3(tiles_m, tiles_n, S), 256, smem, st>>>(g);
}

// The background update: 128 x 128 tiles of the lower triangle (nt per side) of S matrices as a grid-stride loop over at
// most `ctas` CTAs.  Two things make room for the spine next to it (its register use allows one CTA per SM):
//   * ctas < number of SMs: the diagonal kernel cannot share an SM with this kernel (registers), and a tile of it runs
//     long -- launched over all SMs it would make every diagonal block wait for a tile to drain;
//   * a 2-stage ring (82 KB): the panel kernel (138 KB) and the 32-row GEMMs (77 KB) fit beside it on the same SM.
template <int ST>
static void launch_gemm_background_st(GemmArgs g, int nt, int S, int ctas, cudaStream_t st) {
  const size_t smem = sizeof(double) * ST * (128 + 128) * LDS;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(dgemm_nt_kernel<128, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    attr = true;
  }
  g.persist = 1; g.nt = nt; g.batch = S;
  const long items = (long)S * nt * (nt + 1) / 2;
  dgemm_nt_kernel<128, ST><<<(unsigned)std::min<long>(items, ctas), 256, smem, st>>>(g);
}
static void launch_gemm_background(const GemmArgs& g, int nt, int S, int ctas, cudaStream_t st) {
  static int stages = -1;
  if (stages < 0) { const char* e = getenv("SMK_LL_BG_STAGES"); stages = (e && e[0] == '3') ? 3 : 2; }
  if (stages == 3) launch_gemm_background_st<3>(g, nt, S, ctas, st);
  else launch_gemm_background_st<2>(g, nt, S, ctas, st);
}

// kernel launch on the spine: programmatic stream serialization unless SMK_LL_PDL=0
template <typename... KArgs, typename... Args>
static void launch_spine(void (*kern)(KArgs...), dim3 grid, size_t smem, cudaStream_t st, Args... args) {
  static int pdl = -1;
  if (pdl < 0) { const char* e = getenv("SMK_LL_PDL"); pdl = (e && e[0] == '0') ? 0 : 1; }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = pdl ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

struct Streams {
  cudaStream_t main = nullptr, near = nullptr, side = nullptr;
  cudaEvent_t diag0 = nullptr, diag1 = nullptr, head0 = nullptr, col = nullptr, la = nullptr, larest = nullptr, larest2 = nullptr, panel = nullptr, rest = nullptr,
              join_near = nullptr, join_side = nullptr;
};
static Streams& streams() {
  static Streams s;
  if (!s.main) {
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);              // hi = numerically lowest = most urgent
    cudaStreamCreateWithPriority(&s.main, cudaStreamNonBlocking, hi);
    cudaStreamCreateWithPriority(&s.near, cudaStreamNonBlocking, hi < lo ? hi + 1 : hi);   // the diagonal kernel needs an EMPTY SM: it goes first
    cudaStreamCreateWithPriority(&s.side, cudaStreamNonBlocking, lo);
    for (cudaEvent_t* e : {&s.diag0, &s.diag1, &s.head0, &s.col, &s.la, &s.larest, &s.larest2, &s.panel, &s.rest, &s.join_near, &s.join_side})
      cudaEventCreateWithFlags(e, cudaEventDisableTiming);
  }
  return s;
}

// The launch sequence on (main, near, side); called directly or under stream capture.
static int enqueue(int Npad, int S, double* A, double* W, int* info, Streams& ss) {
  const int nblk = Npad / NB;
  const long as = (long)Npad * Npad, ws = (long)nblk * WD;
  const size_t dsm = DiagSmem<double, NB>::bytes, psm = PanelSmem<double, NB>::bytes;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(diag_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dsm);
    cudaFuncSetAttribute(panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)psm);
    cudaFuncSetAttribute(diag_block_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)(sizeof(double) * 2 * 32 * (DBU_MAXK + 4)));
    attr = true;
  }
  const size_t dbu_smem = sizeof(double) * 2 * 32 * (DBU_MAXK + 4);
  cudaStream_t m = ss.main, nr = ss.near, sd = ss.side;
  // Block columns in PAIRS (j, j+1), three streams.  Only what the NEXT diagonal block needs stays on the spine, and the
  // spine's kernels are small enough (1, 4 and 10 CTAs per matrix) to run on the SMs the background update leaves free --
  // next to a background CTA they share the SM's float64 pipe and take twice as long:
  //   main (urgent): diag j, panel HEAD j (the 128 rows of block row j+1), update of block (j+1, j+1), diag j+1, panel head
  //                  j+1 (block row j+2), rank-256 update of block (j+2, j+2) -- then straight on to diag j+2;
  //   near (urgent): everything else of the two block columns while the diagonal kernels run: panel rest j, rest of column
  //                  j+1, panel rest j+1, then the look-ahead columns j+2 (panel head j+2 waits for it) and j+3;
  //   side (background): the rank-256 update of everything to the right of the next pair.
  // A single matrix is bound by this spine, not by flops (22.9 Gflop at N = 4096 is 0.34 ms at the H100 SXM data-sheet fp64 tensor rate of 67 TFLOP/s).
  auto gemm_args = [&](int jcol, int K, int row_blk, int col_blk, int tri) {
    GemmArgs g{};
    g.A = A + (long)jcol * NB; g.lda = Npad; g.a_stride = as;
    g.B = A + (long)jcol * NB; g.ldb = Npad; g.b_stride = as; g.brow0 = col_blk * NB;
    g.C = A; g.ldc = Npad; g.c_stride = as;
    g.K = K; g.row0 = row_blk * NB; g.col0 = col_blk * NB; g.sub = 1; g.tri = tri;
    return g;
  };
  bool pend_col = false, pend_la = false, pend_la2 = false, side_used = false, near_used = false;
  const int reserve = std::min(24, std::max(8, 10 * S + 2));          // the widest spine kernel: 10 CTAs per matrix
  const int bg_ctas = std::max(num_sms() - reserve, 1);
  const double* Wc = W;
  for (int j = 0; j < nblk; j += 2) {
    launch_spine(diag_kernel, dim3(S), dsm, m, Npad, j, A, as, W, ws, info);
    count_launch();
    const int rem = nblk - j - 1;                // block rows below block j
    if (rem <= 0) break;
    if (pend_la) { cudaStreamWaitEvent(m, ss.larest, 0); pend_la = false; }     // column j below the diagonal is up to date
    if (rem > 1) {                               // panel rest j next to the head: rows from block j+2 on
      cudaEventRecord(ss.diag0, m);
      cudaStreamWaitEvent(nr, ss.diag0, 0);
      panel_kernel<<<dim3((rem - 1) * 4, 1, S), 256, psm, nr>>>(Npad, j, j + 2, A, as, Wc, ws);
      count_launch();
      near_used = true;
    }
    launch_spine(panel_kernel, dim3(4, 1, S), psm, m, Npad, j, j + 1, A, as, Wc, ws);          // head: L_(j+1)j
    if (pend_la2) { cudaStreamWaitEvent(m, ss.larest2, 0); pend_la2 = false; }   // block (j+1, j+1) carries the look-ahead
    launch_spine(diag_block_update_kernel, dim3(10, S), dbu_smem, m, Npad, j + 1, j * NB, NB, A, as);   // block (j+1, j+1) -= L L^T
    count_launch(2);
    if (rem > 1) {                               // rest of column j+1 (needs L_(j+1)j and panel rest j), next to diag j+1
      cudaEventRecord(ss.head0, m);
      cudaStreamWaitEvent(nr, ss.head0, 0);
      launch_gemm<32>(gemm_args(j, NB, j + 2, j + 1, 0), (rem - 1) * 4, 1, S, nr);
      cudaEventRecord(ss.col, nr);
      count_launch();
      pend_col = true;
    }
    launch_spine(diag_kernel, dim3(S), dsm, m, Npad, j + 1, A, as, W, ws, info);
    count_launch();
    const int rem2 = nblk - j - 2;               // block rows below block j+1
    if (rem2 <= 0) break;
    if (rem2 > 1) {                              // panel rest j+1: rows from block j+3 on (column j+1 there: ss.col, same stream)
      cudaEventRecord(ss.diag1, m);
      cudaStreamWaitEvent(nr, ss.diag1, 0);
      panel_kernel<<<dim3((rem2 - 1) * 4, 1, S), 256, psm, nr>>>(Npad, j + 1, j + 3, A, as, Wc, ws);
      cudaEventRecord(ss.panel, nr);
      count_launch();
    }
    if (pend_col) { cudaStreamWaitEvent(m, ss.col, 0); pend_col = false; }       // column j+1 (and panel rest j) complete
    launch_spine(panel_kernel, dim3(4, 1, S), psm, m, Npad, j + 1, j + 2, A, as, Wc, ws);      // head: L_(j+2)(j+1)
    count_launch();
    // look-ahead: the next pair's columns (j+2, j+3) with respect to panels j and j+1; the side stream's update for the
    // previous pair also wrote those columns, so wait for it first
    if (side_used) cudaStreamWaitEvent(m, ss.rest, 0);
    launch_spine(diag_block_update_kernel, dim3(10, S), dbu_smem, m, Npad, j + 2, j * NB, 2 * NB, A, as);   // block (j+2, j+2)
    count_launch();
    if (rem2 > 1) {                              // columns j+2, j+3 below block j+2: column j+2 first -- panel j+2 waits for it
      cudaEventRecord(ss.la, m);                 // (orders them behind the previous pair's background update as well)
      cudaStreamWaitEvent(nr, ss.la, 0);
      launch_gemm<32>(gemm_args(j, 2 * NB, j + 3, j + 2, 0), (rem2 - 1) * 4, 1, S, nr);
      cudaEventRecord(ss.larest, nr);
      launch_gemm<32>(gemm_args(j, 2 * NB, j + 3, j + 3, 1), (rem2 - 1) * 4, 1, S, nr);
      cudaEventRecord(ss.larest2, nr);
      count_launch(2);
      pend_la = pend_la2 = true;
    }
    if (rem2 > 2) {                              // everything to the right of the next pair, in the background
      cudaStreamWaitEvent(sd, ss.panel, 0);      // both panels down to the last row
      launch_gemm_background(gemm_args(j, 2 * NB, j + 4, j + 4, 1), rem2 - 2, S, bg_ctas, sd);
      cudaEventRecord(ss.rest, sd);
      count_launch();
      side_used = true;
    }
  }
  if (near_used) {
    cudaEventRecord(ss.join_near, nr);
    cudaStreamWaitEvent(m, ss.join_near, 0);
  }
  if (side_used) {
    cudaEventRecord(ss.join_side, sd);
    cudaStreamWaitEvent(m, ss.join_side, 0);
  }
  return 0;
}

}  // namespace ll

static std::map<cudaGraphExec_t, int>& launches_per_graph() {
  static std::map<cudaGraphExec_t, int> m;
  return m;
}

size_t potrf_ll_workspace_bytes(int Npad, int S) { return (size_t)S * (Npad / ll::NB) * ll::WD * sizeof(double); }

// A: [S][Npad][Npad] (lower triangle in/out), W: workspace, info[S].  Npad % 128 == 0.
// use_graph: capture the sequence once per (A, W, info, Npad, S) on internal streams and replay it behind `st`.
int potrf_ll_f64(int Npad, int S, double* A, double* W, int* info, int use_graph, cudaStream_t st) {
  if (Npad <= 0 || Npad % ll::NB) return -1;
  if (S <= 0) return -2;
  if (!A || !W || !info) return -3;
  ll::Streams& ss = ll::streams();
  static cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  if (!ev_in) {
    cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ev_out, cudaEventDisableTiming);
  }
  cudaMemsetAsync(info, 0, sizeof(int) * S, st);
  if (!use_graph) {
    cudaEventRecord(ev_in, st);
    cudaStreamWaitEvent(ss.main, ev_in, 0);
    ll::enqueue(Npad, S, A, W, info, ss);
    cudaEventRecord(ev_out, ss.main);
    cudaStreamWaitEvent(st, ev_out, 0);
    return check_launch("potrf_ll");
  }
  typedef std::tuple<double*, double*, int*, int, int> Key;
  static std::map<Key, cudaGraphExec_t> cache;
  const Key key(A, W, info, Npad, S);
  auto it = cache.find(key);
  if (it == cache.end()) {
    // first use: run it once un-captured (sets the kernel attributes outside capture), then capture
    cudaEventRecord(ev_in, st);
    cudaStreamWaitEvent(ss.main, ev_in, 0);
    const long long before = launch_count();
    ll::enqueue(Npad, S, A, W, info, ss);
    const int per_run = (int)(launch_count() - before);
    cudaEventRecord(ev_out, ss.main);
    cudaStreamWaitEvent(st, ev_out, 0);
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    if (cudaStreamBeginCapture(ss.main, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
      ll::enqueue(Npad, S, A, W, info, ss);
      count_launch(-per_run);                     // the captured enqueue launched nothing
      if (cudaStreamEndCapture(ss.main, &graph) == cudaSuccess && graph &&
          cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess) {
        if (cache.size() > 64) { for (auto& kv : cache) cudaGraphExecDestroy(kv.second); cache.clear(); }
        cache[key] = exec;
        launches_per_graph()[exec] = per_run;
      }
      if (graph) cudaGraphDestroy(graph);
    }
    cudaGetLastError();
    return check_launch("potrf_ll");
  }
  cudaGraphLaunch(it->second, st);
  count_launch(launches_per_graph()[it->second]);
  return check_launch("potrf_ll(graph)");
}

}  // namespace smk
