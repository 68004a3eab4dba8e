// diag_bench.cu -- phase timeline (clock64) and a standalone correctness check of the spine kernels of csrc/diag.cuh:
// diag_factor_block (L, diagonal inverses), winv_assemble_block (W L = I), panel_sub_block (X L^T = A).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -DSMK_DIAG_TIMELINE -I../../spearmint_b200/csrc -o diag_bench diag_bench.cu
#include <cmath>
#include <cstdio>
#include <vector>
#include "diag.cuh"

namespace smk { void count_launch(int) {} long long launch_count() { return 0; } int check_launch(const char*) { return 0; }
void timing_begin(const char*, cudaStream_t) {} void timing_end(cudaStream_t) {} }
using namespace smk;

template <typename T, int NB>
__global__ void __launch_bounds__(256) k_diag(T* A, T* wd, int* info) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  diag_factor_block<T, NB>(A, NB, wd, info, 0, reinterpret_cast<T*>(smem_raw));
}
template <typename T, int NB>
__global__ void __launch_bounds__(256) k_winv(const T* A, const T* wd, T* W) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  winv_assemble_block<T, NB>(A, NB, wd, W, reinterpret_cast<T*>(smem_raw));
}
template <typename T, int NB>
__global__ void __launch_bounds__(256) k_panel(T* P, const T* A, const T* wd) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  panel_sub_block<T, NB>(P + (long)blockIdx.x * 32 * NB, NB, A, wd, nullptr, nullptr, reinterpret_cast<T*>(smem_raw));
}

template <typename T, int NB>
void run(const char* name) {
  std::vector<double> B(NB * NB), A(NB * NB), L(NB * NB, 0.0), P(64 * NB);
  srand(1);
  for (auto& v : B) v = (rand() / (double)RAND_MAX - 0.5);
  for (auto& v : P) v = (rand() / (double)RAND_MAX - 0.5);
  for (int i = 0; i < NB; ++i)
    for (int j = 0; j < NB; ++j) {
      double s = 0; for (int k = 0; k < NB; ++k) s += B[i * NB + k] * B[j * NB + k];
      A[i * NB + j] = s / NB + (i == j ? 0.05 : 0.0);
    }
  for (int j = 0; j < NB; ++j) {           // host reference Cholesky
    double d = A[j * NB + j]; for (int k = 0; k < j; ++k) d -= L[j * NB + k] * L[j * NB + k];
    L[j * NB + j] = sqrt(d);
    for (int i = j + 1; i < NB; ++i) {
      double s = A[i * NB + j]; for (int k = 0; k < j; ++k) s -= L[i * NB + k] * L[j * NB + k];
      L[i * NB + j] = s / L[j * NB + j];
    }
  }
  std::vector<T> hA(NB * NB), hP(64 * NB);
  for (int e = 0; e < NB * NB; ++e) hA[e] = (T)A[e];
  for (int e = 0; e < 64 * NB; ++e) hP[e] = (T)P[e];
  T *dA, *dW, *dwd, *dP; int* dinfo;
  cudaMalloc(&dA, sizeof(T) * NB * NB); cudaMalloc(&dW, sizeof(T) * NB * NB); cudaMalloc(&dwd, sizeof(T) * NB * 32);
  cudaMalloc(&dP, sizeof(T) * 64 * NB); cudaMalloc(&dinfo, sizeof(int));
  cudaFuncSetAttribute(k_diag<T, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DiagSmem<T, NB>::bytes);
  cudaFuncSetAttribute(k_winv<T, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WinvSmem<T, NB>::bytes);
  cudaFuncSetAttribute(k_panel<T, NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PanelSmem<T, NB>::bytes);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float best = 1e9, bw = 1e9, bp = 1e9;
  for (int it = 0; it < 5; ++it) {
    cudaMemcpy(dA, hA.data(), sizeof(T) * NB * NB, cudaMemcpyHostToDevice);
    cudaMemcpy(dP, hP.data(), sizeof(T) * 64 * NB, cudaMemcpyHostToDevice);
    cudaMemset(dinfo, 0, sizeof(int));
    float ms;
    cudaEventRecord(e0); k_diag<T, NB><<<1, 256, DiagSmem<T, NB>::bytes>>>(dA, dwd, dinfo); cudaEventRecord(e1);
    cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
    cudaEventRecord(e0); k_winv<T, NB><<<1, 256, WinvSmem<T, NB>::bytes>>>(dA, dwd, dW); cudaEventRecord(e1);
    cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1); if (ms < bw) bw = ms;
    cudaEventRecord(e0); k_panel<T, NB><<<2, 256, PanelSmem<T, NB>::bytes>>>(dP, dA, dwd); cudaEventRecord(e1);
    cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1); if (ms < bp) bp = ms;
  }
  cudaError_t err = cudaGetLastError();
  std::vector<T> gL(NB * NB), gW(NB * NB), gX(64 * NB);
  cudaMemcpy(gL.data(), dA, sizeof(T) * NB * NB, cudaMemcpyDeviceToHost);
  cudaMemcpy(gW.data(), dW, sizeof(T) * NB * NB, cudaMemcpyDeviceToHost);
  cudaMemcpy(gX.data(), dP, sizeof(T) * 64 * NB, cudaMemcpyDeviceToHost);
  double eL = 0, eW = 0, eX = 0;
  for (int i = 0; i < NB; ++i)
    for (int j = 0; j < NB; ++j) {
      if (j <= i) eL = fmax(eL, fabs((double)gL[i * NB + j] - L[i * NB + j]));
      double s = 0; for (int kk = 0; kk < NB; ++kk) s += (double)gW[i * NB + kk] * (kk >= j ? L[kk * NB + j] : 0.0);   // (W L)_ij
      eW = fmax(eW, fabs(s - (i == j ? 1.0 : 0.0)));
    }
  for (int r = 0; r < 64; ++r)
    for (int c = 0; c < NB; ++c) {
      double s = 0; for (int kk = 0; kk <= c; ++kk) s += (double)gX[r * NB + kk] * L[c * NB + kk];                   // (X L^T)_rc
      eX = fmax(eX, fabs(s - P[r * NB + c]));
    }
  long long tl[64];
  cudaMemcpyFromSymbol(tl, g_diag_tl, sizeof(tl));
  printf("%s NB=%d: diag %.1f us, winv %.1f us, panel(2 CTAs) %.1f us (%s)  max|dL| %.2e  max|WL - I| %.2e  max|X L^T - A| %.2e\n",
         name, NB, best * 1e3, bw * 1e3, bp * 1e3, cudaGetErrorString(err), eL, eW, eX);
  printf("   load %lld | chol0 %lld", tl[1] - tl[0], tl[2] - tl[1]);
  for (int p = 0; p + 1 < NB / 32; ++p) {
    long long t0 = p ? tl[6 + 4 * (p - 1)] : tl[2];
    printf(" | p%d subst %lld tile %lld chol%d %lld (+wait %lld)", p, tl[3 + 4 * p] - t0, tl[4 + 4 * p] - tl[3 + 4 * p], p + 1,
           tl[5 + 4 * p] - tl[4 + 4 * p], tl[6 + 4 * p] - tl[5 + 4 * p]);
  }
  printf(" | Wdiag %lld store %lld | total %lld cycles\n", tl[21] - tl[20], tl[22] - tl[21], tl[22] - tl[0]);
}

int main() {
  run<double, 128>("double");
  run<double, 64>("double");
  run<float, 128>("float");
  return 0;
}
