// fp64_rates.cu -- measured fp64 issue rates on the device: DFMA (SIMT) vs DMMA (mma.sync.m8n8k4.f64 and the sm_90
// shape mma.sync.m16n8k16.f64).  Decides how the float64 Cholesky trailing update (slice-sampler log-likelihood, f2) and
// the float64 predict (csrc/predict_mma.cu) are written.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_rates fp64_rates.cu
#include <cstdio>
#include <cuda_runtime.h>

__global__ void dfma_kernel(double* out, int iters) {
  double a[16];
  for (int i = 0; i < 16; ++i) a[i] = threadIdx.x * 1e-3 + i;
  const double b = 1.0000001, c = 1e-9;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = fma(a[i], b, c);
  }
  double s = 0;
  for (int i = 0; i < 16; ++i) s += a[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int NACC>
__global__ void dmma_kernel(double* out, int iters) {
  double c0[NACC], c1[NACC];
  for (int i = 0; i < NACC; ++i) { c0[i] = 0; c1[i] = 0; }
  double a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-6;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < NACC; ++i)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
                   : "+d"(c0[i]), "+d"(c1[i]) : "d"(a), "d"(b));
  }
  double s = 0;
  for (int i = 0; i < NACC; ++i) s += c0[i] + c1[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <int NACC>
__global__ void dmma16_kernel(double* out, int iters) {
  double c[NACC][4];
  for (int i = 0; i < NACC; ++i) c[i][0] = c[i][1] = c[i][2] = c[i][3] = 0;
  double a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-6;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < NACC; ++i)
      asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
                   "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
                   : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3])
                   : "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(b), "d"(b), "d"(b), "d"(b));
  }
  double s = 0;
  for (int i = 0; i < NACC; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

template <typename F>
float time_ms(F f) {
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  f();
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  f();
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  return ms;
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  const int sms = p.multiProcessorCount;
  double* out; cudaMalloc(&out, sizeof(double) * sms * 8 * 1024);
  const int iters = 20000;
  for (int wps = 4; wps <= 32; wps *= 2) {          // warps per SM
    const int threads = 256, blocks = sms * wps * 32 / threads;
    float ms = time_ms([&] { dfma_kernel<<<blocks, threads>>>(out, iters); });
    double fl = 2.0 * 16 * iters * (double)blocks * threads;
    printf("DFMA  warps/SM=%2d  %.2f ms  %.2f TFLOP/s\n", wps, ms, fl / ms / 1e9);
    ms = time_ms([&] { dmma_kernel<8><<<blocks, threads>>>(out, iters); });
    fl = 2.0 * 8 * 8 * 4 * 8 * iters * (double)blocks * threads / 32;
    printf("DMMA8 warps/SM=%2d  %.2f ms  %.2f TFLOP/s\n", wps, ms, fl / ms / 1e9);
    ms = time_ms([&] { dmma_kernel<32><<<blocks, threads>>>(out, iters / 4); });
    fl = 2.0 * 8 * 8 * 4 * 32 * (iters / 4) * (double)blocks * threads / 32;
    printf("DMMA32 warps/SM=%2d  %.2f ms  %.2f TFLOP/s\n", wps, ms, fl / ms / 1e9);
    ms = time_ms([&] { dmma16_kernel<8><<<blocks, threads>>>(out, iters / 8); });
    fl = 2.0 * 16 * 8 * 16 * 8 * (iters / 8) * (double)blocks * threads / 32;
    printf("DMMA16x8x16 x8 warps/SM=%2d  %.2f ms  %.2f TFLOP/s\n", wps, ms, fl / ms / 1e9);
  }
  printf("clock %d kHz, SMs %d\n", p.clockRate, sms);
  return 0;
}
