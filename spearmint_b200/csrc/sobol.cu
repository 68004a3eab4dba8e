// sobol.cu -- the candidate grid generator on the device (row f4; reference: sobol_lib.i4_sobol_generate,
// spearmint/spearmint/sobol_lib.py:125-156, called by ExperimentGrid GRID:192-196 and spearmint-lite LITE:171-173).
//
// The reference walks the Gray-code recurrence point by point in Python (20000 x 2 points: 0.1 s; 100k x 32: minutes).
// Unrolled, point `seed` is  2^-30 * XOR_{b in bits(seed ^ (seed >> 1))} V[d][b], so every (point, dimension) is independent:
// one thread per element, V (D x 30 words) staged in shared memory, the output written row-major [n][D] (the layout
// the chooser consumes: ExperimentGrid transposes the reference's (D, n) result) with fully coalesced stores.
// HBM-bound by construction: 8 bytes written per ~log2(n) / 2 XORs.
#include "common.cuh"

namespace smk {

int num_sms();

template <typename T>
__global__ void __launch_bounds__(256) sobol_kernel(int D, long n, long skip, const uint32_t* __restrict__ V,
                                                     T* __restrict__ out) {
  extern __shared__ uint32_t vs[];                      // [D][30]
  for (int e = threadIdx.x; e < D * 30; e += blockDim.x) vs[e] = V[e];
  __syncthreads();
  const long total = n * D;
  for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
    const long j = e / D;
    const int d = (int)(e - j * D);
    long seed = skip + j - 1;                           // sobol_lib.py:153: seed = skip + j - 2 with j counted from 1
    if (seed < 0) seed = 0;
    unsigned long long g = (unsigned long long)seed ^ ((unsigned long long)seed >> 1);
    uint32_t q = 0;
    const uint32_t* vd = vs + d * 30;
    while (g) {
      const int b = __ffsll((long long)g) - 1;
      q ^= vd[b];
      g &= g - 1;
    }
    out[e] = (T)((double)q * 9.313225746154785e-10);    // 2^-30 (recipd, sobol_lib.py: 1 / (2 l))
  }
}

template <typename T>
int sobol_generate(int D, long n, long skip, const uint32_t* V, T* out, cudaStream_t st) {
  if (D <= 0 || D > 1111) return -1;
  if (n <= 0) return -2;
  if (skip + n - 1 >= (1L << 30)) return -3;           // the reference's MAXCOL = 30 limit ("Too many calls!")
  if (!V || !out) return -4;
  const long total = n * D;
  const long cap = 16L * num_sms();
  const int blocks = (int)((total + 255) / 256 < cap ? (total + 255) / 256 : cap);
  const size_t smem = sizeof(uint32_t) * D * 30;
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(sobol_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(sizeof(uint32_t) * 1111 * 30));
    attr = true;
  }
  sobol_kernel<T><<<blocks, 256, smem, st>>>(D, n, skip, V, out);
  count_launch();
  return check_launch("sobol_generate");
}

template int sobol_generate<float>(int, long, long, const uint32_t*, float*, cudaStream_t);
template int sobol_generate<double>(int, long, long, const uint32_t*, double*, cudaStream_t);

}  // namespace smk
