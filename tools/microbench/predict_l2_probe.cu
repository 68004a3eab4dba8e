// predict_l2_probe.cu -- is the mode-0 predict GEMM (tc::predict_tc_kernel, csrc/predict_tc.cu) held back by the
// operand bytes it pulls from L2, or by its MMA issue, and what does sharing the B operand in a cluster buy?  The
// kernel's main loop on synthetic fp16 operands, at the headline chunk (S = 40, N = 4096: 16 row groups in 8 pairs,
// 136 stages per item; 256 candidate tiles of 128), with the same 4 x 48 KB TMA ring, 64-byte swizzle,
// 6 wgmma.m64n256k16 per stage, item order and persistent grid, in six variants:
//   (a) one CTA per item, each loading its whole 48 KB per stage;
//   (b) MMA only: the ring is filled once, then the same four stages are reused (no TMA after the first four);
//   (c) TMA only: every stage is loaded and released without MMAs;
//   (d) as in production: 2-CTA clusters, each CTA loads its own A tile and half of the B box, multicast to both;
//   (e) (a) launched in 2-CTA clusters, but each CTA loads its whole B box itself (no multicast, no shared barriers);
//   (f) (e) with the barriers of (d): a stage is refilled only when the consumers of both CTAs have released it.
// Times per launch (CUDA events, after a warm-up), and the card, power limit and SM clock read while the launches run.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o predict_l2_probe predict_l2_probe.cu
//   ./predict_l2_probe [launches]
#include <cuda_fp16.h>
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "../../spearmint_b200/csrc/tc_common.cuh"

using namespace smk::tc;

#define CK(x)                                                                                  \
  do {                                                                                         \
    cudaError_t e_ = (x);                                                                      \
    if (e_ != cudaSuccess) {                                                                   \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_));       \
      exit(1);                                                                                 \
    }                                                                                          \
  } while (0)

constexpr int BM = 128, BN = 256, BK16 = 32, STAGES = 4, ROW_BYTES = 64;
constexpr int A_BYTES = BM * ROW_BYTES, B_BYTES = BN * ROW_BYTES, STAGE_BYTES = 2 * A_BYTES + 2 * B_BYTES;
constexpr int CONSUMERS = 2, THREADS = (CONSUMERS + 1) * 128;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 + 256;
enum { kFull = 0, kMmaOnly = 1, kTmaOnly = 2, kNoMulticast = 3, kCoupled = 4 };

struct Shape { int S, ntiles, ngroups, npairs, Np, Mc; };

template <int VAR, int CL>
__global__ void __launch_bounds__(THREADS, 1)
probe_kernel(const __grid_constant__ CUtensorMap mAhi, const __grid_constant__ CUtensorMap mAlo,
             const __grid_constant__ CUtensorMap mBhi, const __grid_constant__ CUtensorMap mBlo, Shape p, float* sink) {
  extern __shared__ unsigned char smem_raw[];
  unsigned char* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full = reinterpret_cast<uint64_t*>(base + STAGES * STAGE_BYTES);
  uint64_t* empty = full + STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = CL > 1 ? cluster_ctarank() : 0;
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], (VAR == kNoMulticast ? 1 : CL) * CONSUMERS * 4); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (CL > 1) cluster_sync(); else __syncthreads();
  const int ntp = (p.ntiles + CL - 1) / CL;
  const long nitems = (long)p.S * ntp * p.npairs;
  const long w0 = blockIdx.x / CL, dw = gridDim.x / CL;
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(40));
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      long count = 0;
      for (long w = w0; w < nitems; w += dw)
        for (int h = 0; h < 2; ++h) {
          const int pr = (int)(w % p.npairs);
          const long st = w / p.npairs;
          const int tile = min((int)(st % ntp) * CL + (int)rank, p.ntiles - 1), s = (int)(st / ntp);
          const int g = h == 0 ? pr : p.ngroups - 1 - pr;
          if (h == 1 && g == pr) break;
          const int rowA = s * p.Mc + tile * BM, rowB = (s * p.ngroups + g) * BN;
          for (int kc = 0; kc < (g + 1) * (BN / BK16); ++kc, ++count) {
            if (VAR == kMmaOnly && count >= STAGES) continue;
            mbar_wait_relaxed(&empty[stage], phase ^ 1, 64);
            unsigned char* sb = base + stage * STAGE_BYTES;
            const int kk = kc * BK16;
            mbar_expect_tx(&full[stage], STAGE_BYTES);
            tma_load_2d(&mAhi, &full[stage], sb, kk, rowA, 0x1000000000000000ull);
            tma_load_2d(&mAlo, &full[stage], sb + A_BYTES, kk, rowA, 0x1000000000000000ull);
            if (CL == 1 || VAR == kNoMulticast || VAR == kCoupled) {
              tma_load_2d(&mBhi, &full[stage], sb + 2 * A_BYTES, kk, rowB, 0x14F0000000000000ull);
              tma_load_2d(&mBlo, &full[stage], sb + 2 * A_BYTES + B_BYTES, kk, rowB, 0x14F0000000000000ull);
            } else {
              const int hb = (BN / CL) * rank;
              tma_load_2d_multicast(&mBhi, &full[stage], sb + 2 * A_BYTES + hb * ROW_BYTES, kk, rowB + hb, 3,
                                    0x14F0000000000000ull);
              tma_load_2d_multicast(&mBlo, &full[stage], sb + 2 * A_BYTES + B_BYTES + hb * ROW_BYTES, kk, rowB + hb, 3,
                                    0x14F0000000000000ull);
            }
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(232));
    const int wg = (warp >> 2) - 1;
    const uint32_t a_off = (uint32_t)wg * 64 * ROW_BYTES;
    auto release = [&](int st) {            // production: this CTA's barrier; clusters: both CTAs' barriers
      if (CL == 1 || VAR == kNoMulticast) mbar_arrive(&empty[st]);
      else
        for (int r = 0; r < CL; ++r) mbar_arrive_cluster(&empty[st], r);
    };
    float d[BN / 2];
    float sum = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    long count = 0;
    for (long w = w0; w < nitems; w += dw)
      for (int h = 0; h < 2; ++h) {
        const int pr = (int)(w % p.npairs);
        const int g = h == 0 ? pr : p.ngroups - 1 - pr;
        if (h == 1 && g == pr) break;
        int prev = -1;
        for (int kc = 0; kc < (g + 1) * (BN / BK16); ++kc, ++count) {
          if (!(VAR == kMmaOnly && count >= STAGES)) mbar_wait(&full[stage], phase);
          if (VAR == kTmaOnly) {
            if (lane == 0) release(stage);
          } else {
            const uint32_t sa = smem_u32(base + stage * STAGE_BYTES);
            const uint64_t ahi = wgmma_desc_sw64(sa + a_off), alo = wgmma_desc_sw64(sa + A_BYTES + a_off);
            const uint64_t bhi = wgmma_desc_sw64(sa + 2 * A_BYTES), blo = wgmma_desc_sw64(sa + 2 * A_BYTES + B_BYTES);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 2; ++k) {
              const uint64_t ko = (uint64_t)((k * 32) >> 4);
              wgmma_f16_n256(d, alo + ko, bhi + ko, (kc | k) ? 1u : 0u);
              wgmma_f16_n256(d, ahi + ko, blo + ko, 1u);
              wgmma_f16_n256(d, ahi + ko, bhi + ko, 1u);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (prev >= 0 && lane == 0) release(prev);
            prev = stage;
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        if (VAR != kTmaOnly) {
          wgmma_wait<0>();
          wgmma_hold(d);
          if (prev >= 0 && lane == 0) release(prev);
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) sum += d[i];
        }
      }
    sink[blockIdx.x * THREADS + threadIdx.x] = sum;
  }
  if (CL > 1) cluster_sync();   // no remote arrive or multicast may target a CTA that has exited
}

__global__ void fill_kernel(__half* x, long n, unsigned seed) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    unsigned h = (unsigned)i * 2654435761u ^ seed;
    h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
    x[i] = __float2half((float)(h & 0xFFFF) / 65536.f - 0.5f);
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static CUtensorMap make_map(const __half* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q));
    fn = (EncodeTiledFn)f;
  }
  CUtensorMap m;
  cuuint64_t dims[2] = {cols, rows}, strides[1] = {cols * sizeof(__half)};
  cuuint32_t box[2] = {(cuuint32_t)BK16, box_rows}, estr[2] = {1, 1};
  if (fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(ptr), dims, strides, box, estr,
         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
    fprintf(stderr, "cuTensorMapEncodeTiled failed\n");
    exit(1);
  }
  return m;
}

static void smi(const char* when) {
  FILE* f = popen("nvidia-smi --query-gpu=name,power.limit,power.draw,clocks.sm,clocks.max.sm --format=csv,noheader", "r");
  char line[512];
  if (!f) return;
  while (fgets(line, sizeof line, f)) printf("  nvidia-smi %s: %s", when, line);
  pclose(f);
}

template <int VAR, int CL>
static void run(const char* name, const CUtensorMap* m, const CUtensorMap* mh, Shape p, float* sink, int launches) {
  auto k = probe_kernel<VAR, CL>;
  CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.blockDim = dim3(THREADS);
  cfg.dynamicSmemBytes = SMEM_BYTES;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int dev, sms, clusters = 0;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  cfg.gridDim = dim3(sms);
  CK(cudaOccupancyMaxActiveClusters(&clusters, k, &cfg));
  const long nitems = (long)p.S * ((p.ntiles + CL - 1) / CL) * p.npairs;
  cfg.gridDim = dim3((unsigned)(std::min<long>(nitems, CL == 1 ? sms : clusters) * CL));
  const CUtensorMap* b = (CL == 1 || VAR == kNoMulticast || VAR == kCoupled) ? m : mh;
  CK(cudaLaunchKernelEx(&cfg, k, m[0], m[1], b[2], b[3], p, sink));      // warm-up
  CK(cudaDeviceSynchronize());
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  CK(cudaEventRecord(e0));
  for (int i = 0; i < launches; ++i) CK(cudaLaunchKernelEx(&cfg, k, m[0], m[1], b[2], b[3], p, sink));
  CK(cudaEventRecord(e1));
  smi("during");                      // the launches are still running: the clock under this load
  CK(cudaEventSynchronize(e1));
  float ms;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  const double stages = (double)p.S * p.ntiles * p.npairs * (p.ngroups + 1) * (BN / BK16);
  const double l2_bytes = stages * (VAR == kMmaOnly ? 0.0 : ((CL == 1 || VAR == kNoMulticast || VAR == kCoupled) ? STAGE_BYTES : 2 * A_BYTES + 2 * B_BYTES / CL));
  printf("%-34s grid %4u  %8.2f ms/launch  %6.2f TB/s L2->SM  %7.1f TFLOP/s fp16\n", name, cfg.gridDim.x, ms / launches,
         l2_bytes / (ms / launches * 1e-3) / 1e12, VAR == kTmaOnly ? 0.0 : stages * 6 * 2.0 * 64 * 256 * 16 * 2 / (ms / launches * 1e-3) / 1e12);
  fflush(stdout);
}

int main(int argc, char** argv) {
  const int launches = argc > 1 ? atoi(argv[1]) : 5;
  Shape p;
  p.S = 40; p.Np = 4096; p.ntiles = 256; p.Mc = p.ntiles * BM; p.ngroups = p.Np / BN; p.npairs = (p.ngroups + 1) / 2;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  printf("%s, %d SMs; S = %d, N = %d, %d candidate tiles of %d (one headline chunk)\n", prop.name,
         prop.multiProcessorCount, p.S, p.Np, p.ntiles, BM);
  smi("idle");
  const long na = (long)p.S * p.Mc * p.Np, nb = (long)p.S * p.Np * p.Np;
  __half *ahi, *alo, *bhi, *blo;
  float* sink;
  CK(cudaMalloc(&ahi, na * sizeof(__half)));
  CK(cudaMalloc(&alo, na * sizeof(__half)));
  CK(cudaMalloc(&bhi, nb * sizeof(__half)));
  CK(cudaMalloc(&blo, nb * sizeof(__half)));
  CK(cudaMalloc(&sink, (size_t)prop.multiProcessorCount * THREADS * sizeof(float)));
  fill_kernel<<<1024, 256>>>(ahi, na, 1u);
  fill_kernel<<<1024, 256>>>(alo, na, 2u);
  fill_kernel<<<1024, 256>>>(bhi, nb, 3u);
  fill_kernel<<<1024, 256>>>(blo, nb, 4u);
  CK(cudaDeviceSynchronize());
  CUtensorMap m[4] = {make_map(ahi, (uint64_t)p.S * p.Mc, p.Np, BM), make_map(alo, (uint64_t)p.S * p.Mc, p.Np, BM),
                      make_map(bhi, (uint64_t)p.S * p.Np, p.Np, BN), make_map(blo, (uint64_t)p.S * p.Np, p.Np, BN)};
  CUtensorMap mh[4] = {m[0], m[1], make_map(bhi, (uint64_t)p.S * p.Np, p.Np, BN / 2),
                       make_map(blo, (uint64_t)p.S * p.Np, p.Np, BN / 2)};
  run<kFull, 1>("(a) single CTA", m, mh, p, sink, launches);
  run<kMmaOnly, 1>("(b) MMA only (ring filled once)", m, mh, p, sink, launches);
  run<kTmaOnly, 1>("(c) TMA only (no MMA)", m, mh, p, sink, launches);
  run<kFull, 2>("(d) 2-CTA clusters, B multicast", m, mh, p, sink, launches);
  run<kNoMulticast, 2>("(e) 2-CTA clusters, no multicast", m, mh, p, sink, launches);
  run<kCoupled, 2>("(f) (e) with cluster-wide release", m, mh, p, sink, launches);
  run<kFull, 1>("(a) single CTA, again", m, mh, p, sink, launches);
  CK(cudaFree(ahi)); CK(cudaFree(alo)); CK(cudaFree(bhi)); CK(cudaFree(blo)); CK(cudaFree(sink));
  return 0;
}
