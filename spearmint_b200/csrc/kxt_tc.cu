// kxt_tc.cu -- cross-covariance generator on the tensor cores.
//
// The generator writes Kxt[s][c][n] = amp2_s k(r2_s(X_n, C_c)) for every hyper-sample s (reference: gp.dist2 + the kernel
// functions + chooser.cov, gp.py:34-127, GPEIOptChooser.py:536), as the scaled fp16 (hi, lo) operand of the predict GEMM,
// and the predictive mean  mu[s][c] = sum_n alpha_s[n] Kxt[s][c][n] + mean_s  (GPEIOptChooser.py:544).
//
// The SIMT generator (predict_tc.cu: kxt_kernel) spends 2 float32 operations per (candidate, observation, dimension,
// SAMPLE) on  r2_s = sum_d ((x_d - c_d) / ls_sd)^2  and is bound by the float32 pipe.  But
//     r2_s(c, n) = sum_d  w_sd * q_d(c, n),      q_d = (x_nd - c_cd)^2   (sample independent),  w_sd = 1 / ls_sd^2
// is a GEMM over d:  q is formed ONCE per (pair, dimension) on the CUDA cores -- in the difference form, so nothing
// cancels, and every term of the sum is non-negative -- and the contraction for all S samples runs on wgmma as
// 3 x FP16 products with exact power-of-two operand scaling (the scheme of the predict GEMM; DESIGN.md 6).
//
// Mapping (chosen for the epilogue, which is where the time goes):  accumulator row = (candidate slot j, sample s),
// column = observation n.  J = min(128 / S, 96 / Dp) candidates share the 128 rows through a block-diagonal A operand:
// row (j, s) holds w_s in k-block j and zeros elsewhere; the B operand row of observation n is [q(c_0, n) | ... |
// q(c_J-1, n)].  The per-row constants (sample scale, amplitude) are fixed per thread, and the predictive mean is a
// running sum per row.
//
// A CTA is two warpgroups; warpgroup g owns accumulator rows 64 g .. 64 g + 63 (wgmma m64n128k16, 3 x FP16 products per
// k step, accumulator in registers).  Work item = J candidates x all observations, in tiles of 128 observations.  All 256
// threads build the q operand of tile t + 1 (fp16 hi, lo in the 64-byte-swizzled K-major layout, one [128 x 64 B] block
// per candidate slot) while the MMAs of tile t run, then turn the accumulator of tile t into kernel values.  Each warp
// transposes its 16 rows x 128 columns of output through shared memory, so that every store instruction writes one
// 256-byte row of hi and one of lo.  Opt-in (SMK_KXT_IMPL=tc): on an H100 SXM it is slower than the SIMT generator at the
// headline shape (95 against 80 ms per step); predict_tc() uses the SIMT generator otherwise, and always for D > 32 or
// where kxt_tc_preferred() says few samples would leave most accumulator rows empty.
#include <cuda_fp16.h>
#include <cuda.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "tc_common.cuh"

namespace smk {

int num_sms();

namespace ktc {
using namespace tc;

constexpr int TN = 128;            // observations per tile (MMA N)
constexpr int MAXD = 32;           // padded dimension limit
constexpr int MAXK = 96;           // J * Dp limit: one q buffer = 128 x 96 halves x (hi, lo) = 48 KB
constexpr int MAXS = 64;           // samples per launch (one sample per accumulator row: <= 128)
constexpr int THREADS = 256;       // two warpgroups
constexpr int NGRP = 1;            // mean partial planes per chunk
constexpr int OLDH = TN + 8;       // halves per row of the output staging: 272-byte stride, conflict-free fragment stores
constexpr int WARP_STG = 2 * 16 * OLDH;           // halves of one warp's staging: hi rows 0-15, then lo rows 0-15

struct Args {
  int kind, N, Np, M, c_begin, Mc, D, Dp, S, J, K, Npad_alpha;
  int nitems;                      // ceil(candidates of the chunk / J)
  int mc_used;                     // candidates of this chunk (multiple of 128; rows beyond M are clamped copies)
  const float *Xp, *Cp;            // scaled, zero-padded coordinates: observations dimension-major [Dp][Np], candidates [..][Dp]
  const float *inv_ls, *amp2, *alpha;
  const unsigned* qmax;            // [2] float bits of max|X|, max|C|
  __half *khi, *klo;               // [S][Mc][Np]
  float* mu_partial;               // [NGRP][S][Mc]
  long long* tl;                   // optional timeline (SMK_KXT_TIMELINE=1): [tile < 64][8] clock64() stamps of CTA 0 (slots 0-3 used)
};
constexpr int TL_TILES = 64;
__device__ long long g_timeline[TL_TILES * 8];

__host__ __device__ inline int slots(int S, int Dp) { int j = 128 / S, k = MAXK / Dp; return j < k ? j : k; }

__host__ __device__ inline size_t smem_bytes(int K, int /*S*/) {
  return (size_t)2 * 128 * K * 2 /*A hi, lo*/ + (size_t)2 * 2 * TN * K * 2 /*two q buffers*/ +
         (size_t)(THREADS / 32) * WARP_STG * 2 /*output staging*/ + 1024 /*align*/;
}

// Operand tiles are K-major with the 64-byte swizzle (one candidate slot = 32 halves = one 64-byte row), stored as
// J blocks of [128 rows x 64 B]; the 16-byte chunk c of row r sits at chunk (c ^ ((r >> 1) & 3)) -- the pattern TMA
// produces for CU_TENSOR_MAP_SWIZZLE_64B and wgmma expects for a 64-byte-swizzle descriptor.
constexpr uint32_t SLOT_BYTES = 128 * 64;
__device__ __forceinline__ uint32_t core_off(int r, int jbg) {
  return (uint32_t)(jbg >> 2) * SLOT_BYTES + (uint32_t)r * 64u + (uint32_t)(((jbg & 3) ^ ((r >> 1) & 3)) << 4);
}

__device__ __forceinline__ unsigned h2_bits(__half2 h) { return *reinterpret_cast<unsigned*>(&h); }

template <int KIND, bool MU>
__global__ void __launch_bounds__(THREADS, 1) kxt_tc_kernel(Args p) {
  extern __shared__ unsigned char smem_raw[];
  // 1 KB alignment by OFFSET, not by integer arithmetic on the pointer: a pointer rebuilt from a uintptr_t loses its
  // address space, and every shared-memory access would become a generic one.
  unsigned char* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int Dp = p.Dp, K = p.K, C = K >> 3, CD = Dp >> 3;   // 16-byte k blocks per operand row / per candidate slot (4)
  const uint32_t BH = (uint32_t)TN * K * 2;          // bytes of one B half (hi or lo)
  const uint32_t WH = (uint32_t)128 * K * 2;
  unsigned char* sW = base;
  unsigned char* sB = sW + 2 * WH;                   // [2 buffers][hi | lo]
  __half* stg = reinterpret_cast<__half*>(sB + 4 * BH);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // operand scale of q = (x - c)^2: even exponent, half of it is already applied to the coordinates (kxt_prep_kernel)
  const float xmax = __uint_as_float(p.qmax[0]) + __uint_as_float(p.qmax[1]);
  const int eq = scale_exp(xmax * xmax) & ~1;

  // A operand: row (j, s) = w_s * 2^ew_s in k-block j, zero elsewhere (and zero rows beyond J * S); fp16 (hi, lo)
  for (int e = tid; e < 128 * C; e += THREADS) {     // one 16-byte block (8 dimensions) per iteration
    const int r = e / C, jb = e % C;
    const int j = r / p.S, s = r - j * p.S;
    __half2 hh[4], ll[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) { hh[k] = __floats2half2_rn(0.f, 0.f); ll[k] = hh[k]; }
    if (j < p.J && jb / CD == j) {
      float wmax = 0.f;
      for (int d = 0; d < p.D; ++d) { const float il = p.inv_ls[(long)s * p.D + d]; wmax = fmaxf(wmax, il * il); }
      const float sc = ldexpf(1.f, scale_exp(wmax));
      const int d0 = (jb % CD) * 8;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float w[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int d = d0 + 2 * k + u;
          const float il = (d < p.D) ? p.inv_ls[(long)s * p.D + d] : 0.f;
          w[u] = il * il * sc;
        }
        hh[k] = __floats2half2_rn(w[0], w[1]);
        const float2 hf = __half22float2(hh[k]);
        ll[k] = __floats2half2_rn(w[0] - hf.x, w[1] - hf.y);
      }
    }
    const uint32_t off = core_off(r, jb);
    *reinterpret_cast<uint4*>(sW + off) = make_uint4(h2_bits(hh[0]), h2_bits(hh[1]), h2_bits(hh[2]), h2_bits(hh[3]));
    *reinterpret_cast<uint4*>(sW + WH + off) = make_uint4(h2_bits(ll[0]), h2_bits(ll[1]), h2_bits(ll[2]), h2_bits(ll[3]));
  }

  const int nblocks = p.Np / TN;
  // q operand of tile t (item blockIdx.x + (t / nblocks) * gridDim.x, observations of block t % nblocks) into buffer buf.
  // Thread = observation row (tid % 128) and every other 8-dimension block of the item's candidate slots; Xp is stored
  // dimension-major ([Dp][Np]), so a warp reads 128 contiguous bytes per dimension.
  auto build = [&](long t, int buf) {
    const long item = blockIdx.x + (t / nblocks) * gridDim.x;
    const int nb = (int)(t % nblocks);
    const int c0 = p.c_begin + (int)item * p.J;     // first candidate of the item (rows of Cp beyond M are clamped copies)
    const int r = tid & 127;
    unsigned char* bh = sB + (size_t)buf * 2 * BH;
    unsigned char* bl = bh + BH;
    const float* xcol = p.Xp + (size_t)nb * TN + r;
    for (int jbg = tid >> 7; jbg < p.J * CD; jbg += 2) {
      const int j = jbg / CD, jb = jbg - j * CD;
      const float4* crow = reinterpret_cast<const float4*>(p.Cp + (size_t)(c0 + j) * Dp + 8 * jb);
      const float4 c0v = __ldg(crow), c1v = __ldg(crow + 1);
      const float cc[8] = {c0v.x, c0v.y, c0v.z, c0v.w, c1v.x, c1v.y, c1v.z, c1v.w};
      __half2 hh[4], ll[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 xx = make_float2(__ldg(xcol + (size_t)(8 * jb + 2 * k) * p.Np), __ldg(xcol + (size_t)(8 * jb + 2 * k + 1) * p.Np));
        const float2 df = fadd2(xx, make_float2(-cc[2 * k], -cc[2 * k + 1]));
        const float2 q = fmul2(df, df);
        hh[k] = __floats2half2_rn(q.x, q.y);
        const float2 hf = __half22float2(hh[k]);
        ll[k] = __floats2half2_rn(q.x - hf.x, q.y - hf.y);
      }
      const uint32_t off = core_off(r, jbg);
      *reinterpret_cast<uint4*>(bh + off) = make_uint4(h2_bits(hh[0]), h2_bits(hh[1]), h2_bits(hh[2]), h2_bits(hh[3]));
      *reinterpret_cast<uint4*>(bl + off) = make_uint4(h2_bits(ll[0]), h2_bits(ll[1]), h2_bits(ll[2]), h2_bits(ll[3]));
    }
  };

  // this thread's accumulator rows r0 and r0 + 8 (fragment layout: tc_common.cuh) and their per-row constants
  const int wg = warp >> 2;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int cq = 2 * (lane & 3);
  int rj[2], rs[2];
  float2 scl2[2], a2s[2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh) {
    const int L = r0 + 8 * rh;
    rj[rh] = L / p.S;
    rs[rh] = L - rj[rh] * p.S;
    float scl = 0.f, a2 = 0.f;
    if (rj[rh] < p.J) {
      float wmax = 0.f;
      for (int d = 0; d < p.D; ++d) { const float il = p.inv_ls[(long)rs[rh] * p.D + d]; wmax = fmaxf(wmax, il * il); }
      scl = ldexpf(1.f, -(eq + scale_exp(wmax)));
      a2 = p.amp2[rs[rh]];
    }
    scl2[rh] = dup2(scl);
    a2s[rh] = dup2(a2 * ldexpf(1.f, kx_exp(a2)));
  }
  __half* wst = stg + (size_t)warp * WARP_STG;
  const uint32_t a_off = (uint32_t)wg * 64 * 64;      // first row of this warpgroup inside every slot block
  const int ksteps = K / 16;

  const long my_items = (p.nitems - blockIdx.x + gridDim.x - 1) / gridDim.x;
  const long T = my_items * nblocks;
  build(0, 0);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
  __syncthreads();
  float d[TN / 2];
  float2 v[2] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
  for (long t = 0; t < T; ++t) {
    const int buf = (int)(t & 1);
    const bool stamp = p.tl && blockIdx.x == 0 && t < TL_TILES && tid == 0;
    if (stamp) p.tl[t * 8 + 0] = clock64();
    const uint32_t sa = smem_u32(sW), sb = smem_u32(sB + (size_t)buf * 2 * BH);
    wgmma_fence();
#pragma unroll 1
    for (int q = 0; q < ksteps; ++q) {
      const uint32_t ko = (uint32_t)(q >> 1) * SLOT_BYTES + (uint32_t)(q & 1) * 32;   // slot block, then 32 B inside the row
      const uint64_t ahi = wgmma_desc_sw64(sa + a_off + ko), alo = wgmma_desc_sw64(sa + WH + a_off + ko);
      const uint64_t bhi = wgmma_desc_sw64(sb + ko), blo = wgmma_desc_sw64(sb + BH + ko);
      wgmma_f16_n128(d, alo, bhi, q ? 1u : 0u);                 // small terms first
      wgmma_f16_n128(d, ahi, blo, 1u);
      wgmma_f16_n128(d, ahi, bhi, 1u);
    }
    wgmma_commit();
    if (t + 1 < T) {
      build(t + 1, buf ^ 1);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    if (stamp) p.tl[t * 8 + 1] = clock64();
    wgmma_wait<0>();
    wgmma_hold(d);
    if (stamp) p.tl[t * 8 + 2] = clock64();

    const long item = blockIdx.x + (t / nblocks) * gridDim.x;
    const int nb = (int)(t % nblocks), n0 = nb * TN;
    const bool edge = n0 + TN > p.N;
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      const float* al = MU ? p.alpha + (size_t)rs[rh] * p.Npad_alpha : nullptr;
      __half* shi = wst + (size_t)((lane >> 2) + 8 * rh) * OLDH;
#pragma unroll
      for (int blk = 0; blk < TN / 8; ++blk) {
        const int col = blk * 8 + cq, n = n0 + col;
        float2 r2 = fmul2(make_float2(d[blk * 4 + rh * 2], d[blk * 4 + rh * 2 + 1]), scl2[rh]);
        r2.x = fmaxf(r2.x, 0.f);               // the (hi, lo) products can leave -1 ulp at coincident points
        r2.y = fmaxf(r2.y, 0.f);
        float2 kk = kernel_pair_fast_t<KIND>(r2);
        if (edge) {                            // padded observations carry no covariance
          if (n >= p.N) kk.x = 0.f;
          if (n + 1 >= p.N) kk.y = 0.f;
        }
        if (MU) {
          const float2 a = make_float2(n < p.N ? __ldg(al + n) : 0.f, n + 1 < p.N ? __ldg(al + n + 1) : 0.f);
          v[rh] = ffma2(kk, a, v[rh]);
        }
        const float2 val = fmul2(kk, a2s[rh]);
        const __half2 h2 = __floats2half2_rn(val.x, val.y);
        const float2 hf = __half22float2(h2);
        *reinterpret_cast<__half2*>(shi + col) = h2;
        *reinterpret_cast<__half2*>(shi + 16 * OLDH + col) = __floats2half2_rn(val.x - hf.x, val.y - hf.y);
      }
    }
    __syncwarp();
    // coalesced write-out: row i of the warp's 16; lanes 0-15 store its hi, lanes 16-31 its lo, 16 bytes each
#pragma unroll 4
    for (int i = 0; i < 16; ++i) {
      const int L = wg * 64 + (warp & 3) * 16 + i;
      const int j = L / p.S, s = L - j * p.S;
      const int crow = (int)item * p.J + j;               // candidate row inside the chunk
      if (j < p.J && crow < p.mc_used) {
        const int seg = lane >> 4, piece = lane & 15;
        const uint4 dv = *reinterpret_cast<const uint4*>(wst + (size_t)(seg * 16 + i) * OLDH + piece * 8);
        __half* dst = (seg ? p.klo : p.khi) + ((size_t)s * p.Mc + crow) * p.Np + n0 + piece * 8;
        *reinterpret_cast<uint4*>(dst) = dv;
      }
    }
    __syncwarp();
    if (MU && nb == nblocks - 1) {                       // the item's last tile: mean partials of its rows
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        float m = v[rh].x + v[rh].y;
        m += __shfl_xor_sync(0xffffffffu, m, 1);
        m += __shfl_xor_sync(0xffffffffu, m, 2);
        const int crow = (int)item * p.J + rj[rh];
        if ((lane & 3) == 0 && rj[rh] < p.J && crow < p.mc_used) p.mu_partial[(size_t)rs[rh] * p.Mc + crow] = m;
        v[rh] = make_float2(0.f, 0.f);
      }
    }
    if (stamp) p.tl[t * 8 + 3] = clock64();
    __syncthreads();   // buffer buf is free for tile t + 2, and tile t + 1's operand is complete
  }
}

// max |v| as float bits (non-negative floats order like unsigned integers)
__global__ void __launch_bounds__(256) absmax_kernel(long n, const float* __restrict__ v, unsigned* __restrict__ out) {
  float m = 0.f;
  for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(v[e]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}

// out[r][d] = in[min(r, rows - 1)][d] * 2^(eq / 2) for d < D (zero for the padded dimensions; zero rows if zero_tail)
__global__ void __launch_bounds__(256) kxt_prep_kernel(long rows_out, int rows, int D, int Dp, int zero_tail, int transpose,
                                                       const float* __restrict__ in, const unsigned* __restrict__ qmax,
                                                       float* __restrict__ out) {
  const float xmax = __uint_as_float(qmax[0]) + __uint_as_float(qmax[1]);
  const float hs = ldexpf(1.f, (scale_exp(xmax * xmax) & ~1) / 2);
  for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < rows_out * Dp; e += (long)gridDim.x * blockDim.x) {
    const long r = e / Dp;
    const int d = (int)(e % Dp);
    float x = 0.f;
    if (d < D && !(zero_tail && r >= rows)) x = in[(r < rows ? r : rows - 1) * D + d] * hs;
    if (transpose) out[(long)d * rows_out + r] = x;      // dimension-major (observations: coalesced per-dimension reads)
    else out[e] = x;
  }
}

}  // namespace ktc

// ---------------------------------------------------------------------------------------------------- host side
bool kxt_tc_supported(int D, int S) {
  if (D > ktc::MAXD || S > ktc::MAXS) return false;
  const int Dp = ktc::MAXD;
  return ktc::smem_bytes(ktc::slots(S, Dp) * Dp, S) <= (size_t)227 * 1024;
}
// Worth it?  An accumulator row is one (candidate slot, sample) pair and at most 3 slots fit the operand stage, so with few
// samples most of the 128 accumulator rows are empty (S = 5 uses 15) while the epilogue still walks all of them; the
// tensor-core generator is chosen from half the rows on (SMK_KXT_TC_MIN_LANES overrides the threshold).
bool kxt_tc_preferred(int D, int S) {
  static int min_lanes = -1;
  if (min_lanes < 0) { const char* e = getenv("SMK_KXT_TC_MIN_LANES"); min_lanes = e ? atoi(e) : 64; }
  return kxt_tc_supported(D, S) && ktc::slots(S, ktc::MAXD) * S >= min_lanes;
}

int kxt_tc_ngroups(int) { return ktc::NGRP; }       // mean partial planes per chunk

static int kxt_dp(int) { return ktc::MAXD; }         // one candidate slot = one 64-byte swizzle row (32 halves)
static size_t kxt_cp_rows(int M) { return (size_t)((M + 127) / 128) * 128 + 128; }   // chunk tail + J slack, clamped copies

// workspace: mean partials of one chunk | padded scaled coordinates of X and of all candidates | range words
size_t kxt_tc_workspace_bytes(int Np, int Mc, int S, int M, int D) {
  const int Dp = kxt_dp(D);
  return (size_t)ktc::NGRP * S * Mc * sizeof(float) + ((size_t)Np + kxt_cp_rows(M)) * Dp * sizeof(float) + 512;
}

struct KxtPlan {
  float* mu_partial; float* Xp; float* Cp; unsigned* qmax;
};
static KxtPlan kxt_plan(void* ws, int Np, int Mc, int S, int M, int D) {
  KxtPlan pl;
  const int Dp = kxt_dp(D);
  pl.mu_partial = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~uintptr_t(255));
  pl.Xp = pl.mu_partial + (((size_t)ktc::NGRP * S * Mc + 63) / 64) * 64;
  pl.Cp = pl.Xp + (size_t)Np * Dp;
  pl.qmax = reinterpret_cast<unsigned*>(pl.Cp + kxt_cp_rows(M) * Dp);
  return pl;
}

// Once per candidate set: coordinate ranges -> operand scale, then the padded / scaled copies the producers read.
int kxt_tc_prepare(void* ws, int N, int Np, int M, int Mc, int D, int S, const float* X, const float* Cc, cudaStream_t st) {
  const KxtPlan pl = kxt_plan(ws, Np, Mc, S, M, D);
  const int Dp = kxt_dp(D);
  cudaMemsetAsync(pl.qmax, 0, 2 * sizeof(unsigned), st);
  const long nx = (long)N * D, nc = (long)M * D;
  ktc::absmax_kernel<<<(unsigned)std::min<long>((nx + 255) / 256, 1024), 256, 0, st>>>(nx, X, pl.qmax);
  ktc::absmax_kernel<<<(unsigned)std::min<long>((nc + 255) / 256, 1024), 256, 0, st>>>(nc, Cc, pl.qmax + 1);
  const long rx = Np, rc = (long)kxt_cp_rows(M);
  ktc::kxt_prep_kernel<<<(unsigned)std::min<long>((rx * Dp + 255) / 256, 4096), 256, 0, st>>>(rx, N, D, Dp, 1, 1, X, pl.qmax, pl.Xp);
  ktc::kxt_prep_kernel<<<(unsigned)std::min<long>((rc * Dp + 255) / 256, 4096), 256, 0, st>>>(rc, M, D, Dp, 0, 0, Cc, pl.qmax, pl.Cp);
  count_launch(4);
  return check_launch("kxt_tc_prepare");
}

int kxt_tc(void* ws, int kind, int N, int Np, int M, int c_begin, int Mc, int mc_used, int D, int S,
           const float* inv_ls, const float* amp2, const float* alpha, int Npad_alpha, __half* khi, __half* klo,
           cudaStream_t st) {
  if (!kxt_tc_supported(D, S)) return -1;
  const KxtPlan pl = kxt_plan(ws, Np, Mc, S, M, D);
  ktc::Args a;
  memset(&a, 0, sizeof(a));
  a.kind = kind; a.N = N; a.Np = Np; a.M = M; a.c_begin = c_begin; a.Mc = Mc; a.D = D; a.S = S;
  a.Dp = kxt_dp(D);
  a.J = ktc::slots(S, a.Dp);
  a.K = a.J * a.Dp;
  a.Npad_alpha = Npad_alpha;
  a.mc_used = mc_used;
  a.nitems = (mc_used + a.J - 1) / a.J;
  a.Xp = pl.Xp; a.Cp = pl.Cp; a.inv_ls = inv_ls; a.amp2 = amp2; a.alpha = alpha; a.qmax = pl.qmax;
  a.khi = khi; a.klo = klo; a.mu_partial = pl.mu_partial;
  { const char* e = getenv("SMK_KXT_TIMELINE");
    if (e && e[0] == '1') { void* sym = nullptr; cudaGetSymbolAddress(&sym, ktc::g_timeline); a.tl = reinterpret_cast<long long*>(sym); } }
  const size_t smem = ktc::smem_bytes(a.K, S);
  const int grid = (int)std::min<long>(a.nitems, num_sms());
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(ktc::kxt_tc_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(ktc::kxt_tc_kernel<2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(ktc::kxt_tc_kernel<3, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(ktc::kxt_tc_kernel<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(ktc::kxt_tc_kernel<2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(ktc::kxt_tc_kernel<3, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    attr = true;
  }
  // alpha == NULL: covariance operand only (no predictive-mean partials; predict_tc reduces the mean in its GEMM epilogue)
  if (alpha) {
    switch (kind) {
      case 0: case 1: ktc::kxt_tc_kernel<1, true><<<grid, ktc::THREADS, smem, st>>>(a); break;
      case 2: ktc::kxt_tc_kernel<2, true><<<grid, ktc::THREADS, smem, st>>>(a); break;
      default: ktc::kxt_tc_kernel<3, true><<<grid, ktc::THREADS, smem, st>>>(a); break;
    }
  } else {
    switch (kind) {
      case 0: case 1: ktc::kxt_tc_kernel<1, false><<<grid, ktc::THREADS, smem, st>>>(a); break;
      case 2: ktc::kxt_tc_kernel<2, false><<<grid, ktc::THREADS, smem, st>>>(a); break;
      default: ktc::kxt_tc_kernel<3, false><<<grid, ktc::THREADS, smem, st>>>(a); break;
    }
  }
  count_launch();
  return check_launch("kxt_tc");
}

// debug: copies the timeline of the last launch made with SMK_KXT_TIMELINE=1 (64 tiles x 8 stamps) to the host
int kxt_tc_timeline(long long* out, int n) {
  if (n > ktc::TL_TILES * 8) n = ktc::TL_TILES * 8;
  return cudaMemcpyFromSymbol(out, ktc::g_timeline, sizeof(long long) * n) == cudaSuccess ? 0 : 1;
}

float* kxt_tc_mu_partial(void* ws, int Np, int Mc, int S, int M, int D) { return kxt_plan(ws, Np, Mc, S, M, D).mu_partial; }

}  // namespace smk
